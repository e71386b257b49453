"""Columns of different embedding widths (fixed_embedding_dim=False) on one GPU, in one call:

    python tools/bench_widths.py [--rows 65536] [--iters 50] [--steps 20]

* the card's name and power limit;
* the ragged flatten / concat kernels (dtb_ragged_concat_emb_dense_fwd / _bwd) at 65 536 rows, 26 fields with the
  reference's formula widths min(4 * int(V ** 0.25), 20) over the Criteo Kaggle vocabulary sizes and 13 continuous
  columns, with achieved GB/s from the algorithmic bytes (forward: ids + gathered rows + dense + X written; backward: ids
  + dX read + the rows added into the gradient);
* the same for the uniform concat kernels at the nearest uniform width with the same total;
* dnn_nets train-step rows/s with the formula widths and with a uniform D = 20 (no dropout, CUDA-graph replay).

Prints one JSON object."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

CRITEO_VOCAB = [1460, 583, 10131227, 2202608, 305, 24, 12517, 633, 3, 93145, 5683, 8351593, 3194, 27, 14992, 5461306, 10,
                5652, 2173, 4, 7046547, 18, 15, 286181, 105, 142572]
N_CONT = 13


def formula_width(v):
    return min(4 * int(v ** 0.25), 20)


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        power = out[torch.cuda.current_device()] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        power = 'unknown'
    return {'name': name, 'power_limit_and_max_sm_clock': power}


def time_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernels(rows, iters):
    from deeptables_b200 import _native as N
    p, f = N.ptr, len(CRITEO_VOCAB)
    dims = [formula_width(v) for v in CRITEO_VOCAB]
    sd, dmax = sum(dims), max(dims)
    g = torch.Generator(device='cuda').manual_seed(0)
    offs = torch.tensor(np.cumsum([0] + CRITEO_VOCAB), dtype=torch.int64, device='cuda')
    ids = torch.stack([torch.randint(0, v, (rows,), device='cuda', generator=g, dtype=torch.int32) for v in CRITEO_VOCAB], 1)
    ids = ids.contiguous()
    dense = torch.randn(rows, N_CONT, device='cuda')
    out = {}
    d_uni = max(1, round(sd / f))
    for kind, width, dcols in (('ragged', dmax, dims), ('uniform', d_uni, [d_uni] * f)):
        sdk = sum(dcols)
        table = torch.rand(sum(CRITEO_VOCAB), width, device='cuda', generator=g)
        grad = torch.zeros_like(table)
        x = torch.empty(rows, sdk + N_CONT, device='cuda')
        dx = torch.randn_like(x)
        if kind == 'ragged':
            dims_c = N.int_array(dcols)
            fwd = lambda: N.check(N.lib.dtb_ragged_concat_emb_dense_fwd(p(ids), p(table), p(offs), dims_c, p(dense), p(x),
                                                                        rows, f, width, N_CONT, None, N.stream_ptr()))
            bwd = lambda: N.check(N.lib.dtb_ragged_concat_emb_dense_bwd(p(ids), p(offs), dims_c, p(dx), p(grad), rows, f,
                                                                        width, N_CONT, N.stream_ptr()))
        else:
            fwd = lambda: N.check(N.lib.dtb_concat_emb_dense_fwd(p(ids), p(table), p(offs), p(dense), p(x), rows, f, width,
                                                                 N_CONT, None, N.stream_ptr()))
            bwd = lambda: N.check(N.lib.dtb_concat_emb_dense_bwd(p(ids), p(offs), p(dx), p(grad), rows, f, width, N_CONT,
                                                                 N.stream_ptr()))
        ms_f, ms_b = time_ms(fwd, iters), time_ms(bwd, iters)
        bytes_f = 4 * rows * (f + sdk + N_CONT + sdk + N_CONT)
        bytes_b = 4 * rows * (f + sdk + sdk)
        out[kind] = {'row_width': width, 'sum_widths': sdk, 'fwd_ms': ms_f, 'fwd_GBps': bytes_f / ms_f / 1e6,
                     'bwd_ms': ms_b, 'bwd_GBps': bytes_b / ms_b / 1e6}
        del table, grad
    out['formula_widths'] = dims
    return out


def train_rows_per_s(rows, steps, dims):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    conf = deeptable.ModelConfig(nets=['dnn_nets'], embedding_dropout=0, fixed_embedding_dim=len(set(dims)) == 1)
    cats = [CategoricalColumn(f'C{i + 1}', v, d) for i, (v, d) in enumerate(zip(CRITEO_VOCAB, dims))]
    conts = [ContinuousColumn('input_continuous_all', [f'I{i + 1}' for i in range(N_CONT)])]
    model = DeepModel('binary', 2, conf, cats, conts, seed=0)
    model._build_model()
    g = torch.Generator(device='cuda').manual_seed(1)
    cat = torch.stack([torch.randint(0, v, (rows,), device='cuda', generator=g, dtype=torch.int32) for v in CRITEO_VOCAB],
                      1).contiguous()
    cont = torch.randn(rows, N_CONT, device='cuda', generator=g)
    y = (torch.rand(rows, 1, device='cuda', generator=g) < 0.25).float()
    for _ in range(5):
        model.train_step(cat, cont, y)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        model.train_step(cat, cont, y)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / steps
    res = {'ms_per_step': ms, 'rows_per_s': rows / ms * 1e3, 'graphed': bool(model._graphs),
           'table_update': 'row-wise' if model.table.lazy_active else 'dense sweep', 'stored_width': model.table.dim,
           'padding_share': model.table.padding_share()}
    model.release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=65536)
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_widths needs a CUDA device')
    out = {'card': card(), 'rows': args.rows, 'fields': len(CRITEO_VOCAB), 'continuous': N_CONT,
           'kernels': kernels(args.rows, args.iters)}
    formula = [formula_width(v) for v in CRITEO_VOCAB]
    out['dnn_train'] = {'formula_widths': train_rows_per_s(args.rows, args.steps, formula),
                        'uniform_20': train_rows_per_s(args.rows, args.steps, [20] * len(CRITEO_VOCAB))}
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
