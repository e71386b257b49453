"""Kernel times of the fused CIN backward at the headline shape (26 fields, D = 16, CIN 128x128x128, 65 536 rows):
cin_wg_dgrad_kernel and each of the three cin_wg_wgrad_kernel launches, read from torch.profiler over repeated
dtb_cin_bwd_phase calls with L2 flushed before each backward, as bench.py does.

    python tools/bench_cin_bwd.py [--batch 65536] [--iters 10]

Prints ms per kernel and TFLOP/s per kernel: executed (what the tensor cores run: padded tiles, bf16x3 = 3 passes) and
algorithmic (the FMAs of the math alone), both counted from the shape below, plus the card name and power limit.
For the data gradient it also prints the bytes of weight chunks copied into shared memory and their rate.
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


def dgrad_chunks(b):
    """(weight chunks per layer, their bytes) one 64-row tile of cin_wg_dgrad_kernel multiplies, and the tile count.
    A chunk is the W_k^T image of one x0 field, or of two where 2 H_k <= NPJ: NPJ x LP, bf16 hi + lo."""
    bd, n_blocks, H, npj = _shape(b)
    nch = [(F + 1) // 2 if 2 * h <= npj else F for h in H]
    nbytes = sum(c * npj * ((s + 15) // 16 * 16) * 4 for c, s in zip(nch, SIZES))
    return nch, nbytes, n_blocks


def flop_counts(b):
    """FMA counts per kernel: {name: (executed, algorithmic)}; mirrors the tiling of csrc/cin_wgmma.cu."""
    bd, n_blocks, H, npj = _shape(b)
    np_ = 16
    while np_ < max(SIZES):
        np_ *= 2
    out = {}
    nch, _, _ = dgrad_chunks(b)
    exe = sum(n_blocks * 64 * c * npj * ((s + 15) // 16 * 16) * 3 for c, s in zip(nch, SIZES))
    out['cin_wg_dgrad_kernel'] = (exe, sum(bd * F * h * s for h, s in zip(H, SIZES)))
    for k, (h, s) in enumerate(zip(H, SIZES)):
        fpt = 2 if h <= 32 else 1
        a_tiles = (F + fpt - 1) // fpt
        groups = (a_tiles + 3) // 4
        # every working warpgroup runs both of its tiles (an absent one on zero rows)
        tiles = sum(2 for g in range(groups) for w in range(2) if (4 * g + 2 * w) * fpt < F)
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
    N.check(N.lib.dtb_cin_fwd(P(idx), P(table), P(offs), P(w), None, P(pooled), P(saved), P(ws), ws_bytes, b, F, D,
                              sizes_c, n, 0, 1, 2, None, N.stream_ptr()), 'cin_fwd')
    flush = torch.zeros(512 << 20, dtype=torch.uint8, device=dev)

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
    times = {}
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
    res = {'gpu': gpu_info(), 'batch': b, 'gemm_rows': b * D, 'iters': args.iters, 'kernels': {}}
    wg_total = 0.0
    for key, (exe, alg) in flops.items():
        ts = sorted(times.get(key, []))
        if len(ts) != args.iters:
            sys.exit(f'bench_cin_bwd: expected {args.iters} records of {key}, got {len(ts)}')
        ms = ts[len(ts) // 2]
        if key.startswith('cin_wg_wgrad'):
            wg_total += ms
        res['kernels'][key] = {'ms': round(ms, 4), 'executed_tflops': round(2 * exe / ms * 1e-9, 1),
                               'algorithmic_tflops': round(2 * alg / ms * 1e-9, 1)}
        if key == 'cin_wg_dgrad_kernel':
            # weight chunks bulk-copied from L2 into shared memory, one copy per tile and chunk
            _, tile_bytes, n_tiles = dgrad_chunks(b)
            gb = tile_bytes * n_tiles * 1e-9
            res['kernels'][key].update(weight_chunk_gb=round(gb, 2), weight_chunk_gbps=round(gb / ms * 1e3, 1))
    res['wgrad_ms_total'] = round(wg_total, 4)
    print(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
