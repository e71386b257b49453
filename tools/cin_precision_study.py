"""CPU study: which operand splits keep the CIN feature-map GEMMs inside the 1e-3 parity bar?

Emulates split-operand tensor-core GEMMs (each fp32 operand rounded to one or two 16-bit terms, exact products,
fp32-or-better accumulation) for the xDeepFM CIN (26 fields x 16, 128x128x128, half-split) on random rows and
compares the pooled feature maps with a float64 evaluation.  Schemes: bf16 x1 / x3 (the product path), fp16 x1,
fp16 x2 with the on-the-fly operand Z split (Z_hi W + Z_lo W) or the weights split (Z W_hi + Z W_lo), all with
power-of-two scaling into the fp16 range (per GEMM row for Z, per layer for W).
    python tools/cin_precision_study.py [rows]"""
import sys

import torch

torch.manual_seed(0)
B = int(sys.argv[1]) if len(sys.argv) > 1 else 192
F, D, SIZES = 26, 16, (128, 128, 128)


def rnd(x, fmt):
    return x.to(fmt).to(torch.float64)


def split(x, fmt, n):
    """n-term split of x into `fmt` values (hi, lo, ...)."""
    parts, r = [], x.clone()
    for _ in range(n):
        p = rnd(r, fmt)
        parts.append(p)
        r = r - p
    return parts


def pow2_scale(x, target, dim=None):
    m = x.abs().amax(dim=dim, keepdim=True) if dim is not None else x.abs().max()
    m = torch.clamp(m, min=1e-30)
    return torch.exp2(torch.floor(torch.log2(target / m)))


def gemm(z, w, scheme):
    """z [M,K] float64 (exact products of fp32 operands), w [K,L] float64 -> emulated tensor-core result."""
    if scheme == 'exact':
        return z @ w
    fmt = torch.bfloat16 if scheme.startswith('bf16') else torch.float16
    sz = sw = 1.0
    if fmt is torch.float16:                      # bring both operands into the fp16 normal range (exact scaling)
        sz = pow2_scale(z, 1024.0, dim=1)
        sw = pow2_scale(w, 1024.0)
    zs, ws = z * sz, w * sw
    zf32 = zs.to(torch.float32).to(torch.float64)     # the producer computes the product in fp32 first
    if scheme in ('bf16x1', 'fp16x1'):
        acc = rnd(zf32, fmt) @ rnd(ws, fmt)
    elif scheme == 'bf16x3':
        zh, zl = split(zf32, fmt, 2)
        wh, wl = split(ws, fmt, 2)
        acc = zh @ wh + zl @ wh + zh @ wl
    elif scheme == 'fp16x2_splitZ':
        zh, zl = split(zf32, fmt, 2)
        acc = (zh + zl) @ rnd(ws, fmt)
    elif scheme == 'fp16x2_splitW':
        wh, wl = split(ws, fmt, 2)
        acc = rnd(zf32, fmt) @ (wh + wl)
    else:
        raise ValueError(scheme)
    return (acc / (sz * sw)).to(torch.float32).to(torch.float64)      # accumulator is fp32


def cin(x0, weights, scheme):
    """x0 [B,F,D] -> pooled [B, 64+64+128]; the chained layers see the emulated activations."""
    b = x0.shape[0]
    h = x0
    pooled = []
    for k, size in enumerate(SIZES):
        z = (x0.unsqueeze(2) * h.unsqueeze(1)).permute(0, 3, 1, 2).reshape(b * D, -1)      # [(b,d), (i,j)]
        c = torch.relu(gemm(z, weights[k], scheme)).reshape(b, D, size)
        if k + 1 < len(SIZES):
            h = c[:, :, :size // 2].permute(0, 2, 1)
            pooled.append(c[:, :, size // 2:].sum(dim=1))
        else:
            pooled.append(c.sum(dim=1))
    return torch.cat(pooled, dim=1)


def main():
    x0 = ((torch.rand(B, F, D, dtype=torch.float64) - 0.5) * 0.1).to(torch.float32).to(torch.float64)   # U(-0.05, 0.05)
    hs = [F, SIZES[0] // 2, SIZES[1] // 2]
    weights = []
    for k, size in enumerate(SIZES):
        fan_in = F * hs[k]
        lim = (6.0 / fan_in) ** 0.5                                     # he_uniform
        weights.append(((torch.rand(fan_in, size, dtype=torch.float64) * 2 - 1) * lim).to(torch.float32).to(torch.float64))
    ref = cin(x0, weights, 'exact')
    scale = float(ref.abs().max())
    print(f'{B} rows, pooled scale {scale:.3e}; tolerance of the parity tests: |err| <= 1e-3*|ref| + 1e-4*scale')
    for scheme in ('bf16x1', 'fp16x1', 'fp16x2_splitW', 'fp16x2_splitZ', 'bf16x3'):
        got = cin(x0, weights, scheme)
        err = (got - ref).abs()
        viol = float((err > 1e-3 * ref.abs() + 1e-4 * scale).double().mean())
        print(f'{scheme:15s} max|err|/scale {float(err.max()) / scale:.2e}   rms/scale {float(err.pow(2).mean().sqrt()) / scale:.2e}'
              f'   entries outside rtol 1e-3 / atol 1e-4*scale: {100 * viol:.3f} %')




# ---------------------------------------------------------------------------------------------------------------
# backward: dgrad  dZ = dC . W^T  (A = dC row, per-row scale)   and   wgrad  dW = Z^T . dC  (reduction over the batch
# rows: ONE scale per operand and layer)
# ---------------------------------------------------------------------------------------------------------------
def gemm_bwd(a, b, scheme, row_scale):
    """a [M,K] @ b [K,N] with both operands rounded per `scheme`; row_scale: per-row (True) or global scale for a."""
    if scheme == 'exact':
        return a @ b
    fmt = torch.bfloat16 if scheme.startswith('bf16') else torch.float16
    sa = sb = 1.0
    if fmt is torch.float16:
        sa = pow2_scale(a, 1024.0, dim=1) if row_scale else pow2_scale(a, 1024.0)
        sb = pow2_scale(b, 1024.0)
    a32, b32 = (a * sa).to(torch.float32).to(torch.float64), (b * sb).to(torch.float32).to(torch.float64)
    if scheme.endswith('x1'):
        acc = rnd(a32, fmt) @ rnd(b32, fmt)
    else:                                                   # bf16x3
        ah, al = split(a32, fmt, 2)
        bh, bl = split(b32, fmt, 2)
        acc = ah @ bh + al @ bh + ah @ bl
    return (acc / (sa * sb)).to(torch.float32).to(torch.float64)


def cin_backward(x0, weights, d_pooled, scheme):
    b = x0.shape[0]
    hs, cs = [x0], []
    h = x0
    for k, size in enumerate(SIZES):                        # exact forward: isolates the backward arithmetic
        z = (x0.unsqueeze(2) * h.unsqueeze(1)).permute(0, 3, 1, 2).reshape(b * D, -1)
        c = torch.relu(z @ weights[k]).reshape(b, D, size)
        cs.append(c)
        if k + 1 < len(SIZES):
            h = c[:, :, :size // 2].permute(0, 2, 1)
            hs.append(h)
    dx0 = torch.zeros_like(x0)
    dws = [None] * len(SIZES)
    dh_next = None
    col = sum(s // 2 for s in SIZES[:-1]) + SIZES[-1]
    for k in range(len(SIZES) - 1, -1, -1):
        size = SIZES[k]
        npool = size if k == len(SIZES) - 1 else size // 2
        col -= npool
        dc = torch.zeros(b, D, size, dtype=torch.float64)
        dc[:, :, size - npool:] = d_pooled[:, col:col + npool].unsqueeze(1)
        if dh_next is not None:
            dc[:, :, :size // 2] += dh_next.permute(0, 2, 1)
        dc = (dc * (cs[k] > 0)).reshape(b * D, size)
        h = hs[k]
        hk = h.shape[1]
        z = (x0.unsqueeze(2) * h.unsqueeze(1)).permute(0, 3, 1, 2).reshape(b * D, -1)
        dws[k] = gemm_bwd(z.t().contiguous(), dc, scheme, row_scale=False)                    # wgrad
        dz = gemm_bwd(dc, weights[k].t().contiguous(), scheme, row_scale=True).reshape(b, D, F, hk)   # dgrad
        dx0 += (dz * h.permute(0, 2, 1).unsqueeze(2)).sum(dim=3).permute(0, 2, 1)
        dh = (dz * x0.permute(0, 2, 1).unsqueeze(3)).sum(dim=2).permute(0, 2, 1)              # [b, hk, D]
        if k == 0:
            dx0 += dh
        dh_next = dh
    return dx0, dws


def main_backward():
    torch.manual_seed(2)
    b = max(32, B // 2)
    x0 = ((torch.rand(b, F, D, dtype=torch.float64) - 0.5) * 0.1).to(torch.float32).to(torch.float64)
    hs = [F, SIZES[0] // 2, SIZES[1] // 2]
    weights = [(((torch.rand(F * hs[k], s, dtype=torch.float64) * 2 - 1) * (6.0 / (F * hs[k])) ** 0.5)
                .to(torch.float32).to(torch.float64)) for k, s in enumerate(SIZES)]
    d_pooled = torch.randn(b, sum(s // 2 for s in SIZES[:-1]) + SIZES[-1], dtype=torch.float64) * 1e-3
    ref_dx, ref_dw = cin_backward(x0, weights, d_pooled, 'exact')
    print(f'backward, {b} rows (forward exact, so only the backward GEMM arithmetic differs):')
    for scheme in ('bf16x1', 'fp16x1', 'bf16x3'):
        dx, dw = cin_backward(x0, weights, d_pooled, scheme)
        ex = float((dx - ref_dx).abs().max() / ref_dx.abs().max())
        ew = max(float((a - r).abs().max() / r.abs().max()) for a, r in zip(dw, ref_dw))
        print(f'{scheme:8s} embedding grad max|err|/max {ex:.2e}   filter grad max|err|/max {ew:.2e}')


if __name__ == '__main__':
    main()
    main_backward()
