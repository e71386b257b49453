"""Kernel times of the fused CIN forward and backward at the headline shape (26 fields, D = 16, CIN 128x128x128,
65 536 rows): cin_wg_fwd_kernel in training (activations saved) and in inference, cin_wg_dgrad_kernel and each of the
three cin_wg_wgrad_kernel launches, read from torch.profiler over repeated dtb_cin_fwd and dtb_cin_bwd_phase calls
with L2 flushed before each call, as bench.py does.

    python tools/bench_cin_bwd.py [--batch 65536] [--iters 10] [--precision 2]

--precision is the forward's precision code (2 = bf16x3, 3 = one bf16 pass, 4 = one scaled fp16 pass); the backward
runs bf16x3 for every code.  Prints ms per kernel and TFLOP/s per kernel: executed (what the tensor cores run: padded
tiles, bf16x3 = 3 passes) and algorithmic (the FMAs of the math alone), both counted from the shape below, plus the
card name and power limit.  For the forward and the data gradient it also prints the bytes of weight chunks copied
into shared memory and their rate; for each weight-gradient layer, the microseconds per 64-row block of its busiest
CTA and the bytes bulk-copied per block.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

F, D, SIZES = 26, 16, (128, 128, 128)


def _shape(b):
    from oracle import layers_ref as L
    bd = b * D
    n_blocks = (bd + 63) // 64
    H = L.cin_field_nums(F, SIZES, False)[:len(SIZES)]
    npj = 16
    while npj < max((h + 15) // 16 * 16 for h in H):
        npj *= 2
    return bd, n_blocks, H, npj


def fwd_chunks(b, precision):
    """Bytes of weight chunks cin_wg_fwd_kernel copies per call: one chunk per layer and x0 field (NP x Hp_k; bf16 hi +
    lo for bf16x3, one 2-byte image otherwise) for each pair of 64-row tiles, which share every copy."""
    bd, n_blocks, H, _ = _shape(b)
    np_ = 16
    while np_ < max(SIZES):
        np_ *= 2
    per_pair = sum(F * np_ * ((h + 15) // 16 * 16) * 2 * (2 if precision == 2 else 1) for h in H)
    return per_pair * ((n_blocks + 1) // 2)


def dgrad_chunks(b):
    """(weight chunks per layer, their bytes) one 64-row tile of cin_wg_dgrad_kernel multiplies, and the tile count.
    A chunk is the W_k^T image of one x0 field, or of two where 2 H_k <= NPJ: NPJ x LP, bf16 hi + lo."""
    bd, n_blocks, H, npj = _shape(b)
    nch = [(F + 1) // 2 if 2 * h <= npj else F for h in H]
    nbytes = sum(c * npj * ((s + 15) // 16 * 16) * 4 for c, s in zip(nch, SIZES))
    return nch, nbytes, n_blocks


def wgrad_plan(b, sms, f=F, d=D, sizes=SIZES):
    """Per layer, the launch of cin_wg_wgrad_kernel as csrc/cin_wgmma.cu plans it: field groups of four m64 A tiles,
    the h copy, the ring depth, the row splits and the bytes bulk-copied per 64-row block."""
    from oracle import layers_ref as L
    bd = b * d
    n_blocks = (bd + 63) // 64
    H = L.cin_field_nums(f, sizes, False)[:len(sizes)]
    np_ = 16
    while np_ < max(sizes):
        np_ *= 2
    r128 = lambda x: (x + 127) // 128 * 128

    def fit(splits):
        splits = min(max(splits, 1), n_blocks)
        bps = -(-n_blocks // splits)
        return -(-n_blocks // bps), bps

    plans = []
    for k, h in enumerate(H):
        ldh = f if k == 0 else sizes[k - 1]
        fpt = 2 if h <= 32 else 1
        htensor = k > 0 and ldh % 4 == 0
        if htensor:
            h4 = (h + 3) // 4 * 4
            hpitch = h4 + (20 - h4 % 16) % 16
        else:
            hpitch = ldh if k > 0 else 0
        stage = r128(np_ * 64 * 4 + r128(64 * f * 4)) if hpitch == 0 else np_ * 64 * 4 + r128(64 * f * 4) + r128(64 * hpitch * 4)
        stages = 4
        while stages > 2 and stages * stage + 16 * stages > 227 * 1024:
            stages -= 1
        a_tiles = -(-f // fpt)
        groups = -(-a_tiles // 4)
        pair = a_tiles - 4 * (groups - 1) <= 2 and stages >= 3
        if not pair:
            sf, bps = fit(sms // groups)
            sl, bpsl = sf, bps
        elif groups == 1:
            sf, bps = 0, 0
            sl, bpsl = fit(sms)
        else:
            best = None
            for s in range(1, sms):
                if s * (groups - 1) >= sms:
                    break
                a, ab = fit(s)
                c, cb = fit(sms - s * (groups - 1))
                cost = max(ab, (cb + 1) // 2)
                if best is None or cost < best[0]:
                    best = (cost, a, ab, c, cb)
            _, sf, bps, sl, bpsl = best
        copied = np_ * 64 * 4 + 64 * f * 4 + (0 if k == 0 else 64 * hpitch * 4 if htensor else 64 * ldh * 4)
        # blocks the busiest CTA multiplies with each warpgroup (a paired last group splits its blocks in two)
        crit = max(bps, (bpsl + 1) // 2 if pair else bpsl)
        plans.append(dict(fields_per_tile=fpt, a_tiles=a_tiles, groups=groups, htensor=htensor, hpitch=hpitch,
                          stages=stages, last_pair=pair, splits=sf, blocks_per_split=bps, last_splits=sl,
                          last_blocks_per_split=bpsl, ctas=(groups - 1) * sf + sl, bytes_per_block=copied,
                          critical_blocks=crit))
    return plans


def flop_counts(b):
    """FMA counts per kernel: {name: (executed, algorithmic)}; mirrors the tiling of csrc/cin_wgmma.cu."""
    bd, n_blocks, H, npj = _shape(b)
    np_ = 16
    while np_ < max(SIZES):
        np_ *= 2
    out = {}
    fwd = (n_blocks * 64 * F * sum(np_ * ((h + 15) // 16 * 16) for h in H), bd * F * sum(h * s for h, s in zip(H, SIZES)))
    out['cin_wg_fwd_kernel training'] = out['cin_wg_fwd_kernel inference'] = fwd
    nch, _, _ = dgrad_chunks(b)
    exe = sum(n_blocks * 64 * c * npj * ((s + 15) // 16 * 16) * 3 for c, s in zip(nch, SIZES))
    out['cin_wg_dgrad_kernel'] = (exe, sum(bd * F * h * s for h, s in zip(H, SIZES)))
    for k, (h, s) in enumerate(zip(H, SIZES)):
        fpt = 2 if h <= 32 else 1
        a_tiles = (F + fpt - 1) // fpt
        groups = (a_tiles + 3) // 4
        # each block is multiplied by all four tiles of a full field group, and by the two tiles of a last group that
        # has tiles for one warpgroup only (whether one warpgroup runs them or both do, on alternate blocks); an
        # absent tile past the last field runs on zero rows
        tiles = 4 * (groups - 1) + (4 if a_tiles - 4 * (groups - 1) > 2 else 2)
        out[f'cin_wg_wgrad_kernel layer {k}'] = (tiles * 64 * np_ * n_blocks * 64 * 3, bd * F * h * s)
    return out


def gpu_info():
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else f'nvidia-smi failed: {r.stderr.strip()}'
    except (OSError, subprocess.SubprocessError) as e:
        return f'nvidia-smi unavailable: {e}'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=65536)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--precision', type=int, default=2, choices=(2, 3, 4))
    args = ap.parse_args()
    import numpy as np
    import torch
    from torch.profiler import profile, ProfilerActivity
    from deeptables_b200 import _native as N
    from oracle import layers_ref as L

    if not torch.cuda.is_available():
        sys.exit('bench_cin_bwd: no CUDA device')
    b, n = args.batch, len(SIZES)
    sizes_c = N.int_array(SIZES)
    g = np.random.default_rng(0)
    vocab = [10000] * F
    dev = 'cuda'
    table = torch.tensor(g.uniform(-0.05, 0.05, size=(sum(vocab), D)).astype(np.float32), device=dev)
    offs = torch.tensor(np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64), device=dev)
    idx = torch.tensor(np.stack([g.integers(0, v, size=b) for v in vocab], axis=1).astype(np.int32), device=dev)
    fns = L.cin_field_nums(F, SIZES, False)
    w = torch.tensor(np.concatenate([(g.normal(size=(F * fns[k], s)) / np.sqrt(F * fns[k])).astype(np.float32).reshape(-1)
                                     for k, s in enumerate(SIZES)]), device=dev)
    pw = L.cin_pooled_width(F, dict(cross_layer_size=SIZES, direct=False))
    pooled = torch.empty(b, pw, device=dev)
    d_pooled = torch.randn(b, pw, device=dev) * 1e-3
    ws_bytes = N.lib.dtb_cin_workspace_bytes(b, F, D, sizes_c, n, 0, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    saved = torch.empty(N.lib.dtb_cin_saved_bytes(b, F, D, sizes_c, n, 0), dtype=torch.uint8, device=dev)
    gt = torch.zeros_like(table)
    dw = torch.zeros_like(w)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    flush = torch.zeros(512 << 20, dtype=torch.uint8, device=dev)

    def fwd(sv, precision):
        N.check(N.lib.dtb_cin_fwd(P(idx), P(table), P(offs), P(w), None, P(pooled), sv, P(ws), ws_bytes, b, F, D,
                                  sizes_c, n, 0, 1, precision, None, N.stream_ptr()), 'cin_fwd')

    for _ in range(3):
        fwd(P(saved), args.precision)
        fwd(None, args.precision)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            for sv in (P(saved), None):
                flush.sum()
                fwd(sv, args.precision)
        torch.cuda.synchronize()
    fwd_kern = sorted((e for e in prof.events() if 'cin_wg_fwd_kernel' in e.name), key=lambda e: e.time_range.start)
    times = {}
    for j, e in enumerate(fwd_kern):      # training and inference calls alternate
        times.setdefault('cin_wg_fwd_kernel ' + ('training' if j % 2 == 0 else 'inference'), []).append(
            e.time_range.elapsed_us() * 1e-3)
    fwd(P(saved), 2)      # the backward reads the activations of a bf16x3 forward

    def bwd():
        for phase in (1, 2):
            N.check(N.lib.dtb_cin_bwd_phase(P(idx), P(table), P(offs), P(w), P(d_pooled), P(saved), P(gt), P(dw), None,
                                            P(ws), ws_bytes, b, F, D, sizes_c, n, 0, 1, 2, phase, N.stream_ptr()),
                    'cin_bwd_phase')

    for _ in range(3):
        bwd()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.iters):
            flush.sum()
            bwd()
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if 'cin_wg_' in e.name),
                  key=lambda e: e.time_range.start)
    wg_seen = 0
    for e in kern:
        if 'cin_wg_dgrad_kernel' in e.name:
            key = 'cin_wg_dgrad_kernel'
        elif 'cin_wg_wgrad_kernel' in e.name:
            key = f'cin_wg_wgrad_kernel layer {wg_seen % n}'
            wg_seen += 1
        else:
            continue
        times.setdefault(key, []).append(e.time_range.elapsed_us() * 1e-3)
    flops = flop_counts(b)
    plans = wgrad_plan(b, torch.cuda.get_device_properties(0).multi_processor_count)
    res = {'gpu': gpu_info(), 'batch': b, 'gemm_rows': b * D, 'iters': args.iters, 'fwd_precision': args.precision,
           'kernels': {}}
    wg_total = 0.0
    for key, (exe, alg) in flops.items():
        ts = sorted(times.get(key, []))
        if len(ts) != args.iters:
            sys.exit(f'bench_cin_bwd: expected {args.iters} records of {key}, got {len(ts)}')
        ms = ts[len(ts) // 2]
        if key.startswith('cin_wg_wgrad'):
            wg_total += ms
            # time per 64-row block of the busiest CTA, and what one block brings into shared memory
            pl = plans[int(key.rsplit(' ', 1)[1])]
            res['kernels'].setdefault(key, {}).update(
                us_per_block_per_cta=round(ms * 1e3 / pl['critical_blocks'], 3), bytes_per_block=pl['bytes_per_block'],
                ctas=pl['ctas'], h_copy='tensor' if pl['htensor'] else ('rows' if pl['hpitch'] else 'none'))
        if key.startswith('cin_wg_fwd') and args.precision == 2:
            exe *= 3      # hi*hi, lo*hi, hi*lo
        res['kernels'].setdefault(key, {}).update(ms=round(ms, 4), executed_tflops=round(2 * exe / ms * 1e-9, 1),
                                                  algorithmic_tflops=round(2 * alg / ms * 1e-9, 1))
        if key == 'cin_wg_dgrad_kernel':
            # weight chunks bulk-copied from L2 into shared memory, one copy per tile and chunk
            _, tile_bytes, n_tiles = dgrad_chunks(b)
            gb = tile_bytes * n_tiles * 1e-9
            res['kernels'][key].update(weight_chunk_gb=round(gb, 2), weight_chunk_gbps=round(gb / ms * 1e3, 1))
        if key.startswith('cin_wg_fwd'):
            gb = fwd_chunks(b, args.precision) * 1e-9
            res['kernels'][key].update(weight_chunk_gb=round(gb, 2), weight_chunk_gbps=round(gb / ms * 1e3, 1))
    res['wgrad_ms_total'] = round(wg_total, 4)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
