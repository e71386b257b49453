"""Cost of Keras weight regularization on one GPU: the fused Adam table sweep with the L2 term at the Criteo table size,
and the xDeepFM headline train step (bench.py's 'xdeepfm' config) with ``embeddings_regularizer=L2(1e-5)``.

    python tools/bench_reg.py [--steps 20] [--warmup 5] [--sweeps 10]

Sweep: dtb_adam_dense (no regularization), dtb_adam_dense_reg (fused, loss term included) and dtb_reg_grad followed by
dtb_adam_dense (unfused).  The bytes per element are those the fused algorithm must move: p, m, v, g read and written,
32 B; the data-sheet bound is that over 3.35 TB/s.
Train step: without a regularizer (exact-lazy table), without a regularizer with the table forced to the dense sweep,
with L2(1e-5) on the table (fused sweep) and with L2(1e-5) through dtb_reg_grad + dtb_adam_dense (unfused).

Prints one JSON line per measurement and a final summary line; the card name and power limit come first, read in the
same run."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'tools')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from bench_optim import TABLE_DIM, TABLE_ROWS, card, events_time  # noqa: E402

HBM_TBPS = 3.35           # H100 SXM data sheet
L2_FACTOR = 1e-5


def sweeps(reps):
    import torch
    from deeptables_b200 import _native as N, engine as E
    from deeptables_b200._native import ptr, check
    n = TABLE_ROWS * TABLE_DIM
    p, m, v, g = [torch.zeros(n, dtype=torch.float32, device='cuda') for _ in range(4)]
    p.uniform_(-0.05, 0.05)
    acc = torch.zeros(1, dtype=torch.float64, device='cuda')
    alpha = E.adam_alpha(10)
    adam = lambda: check(N.lib.dtb_adam_dense(ptr(p), ptr(m), ptr(v), ptr(g), n, alpha, E.ADAM_B1, E.ADAM_B2,
                                              E.ADAM_EPS, 1, None), 'adam_dense')
    fused = lambda: check(N.lib.dtb_adam_dense_reg(ptr(p), ptr(m), ptr(v), ptr(g), n, alpha, E.ADAM_B1, E.ADAM_B2,
                                                   E.ADAM_EPS, 1, 0.0, L2_FACTOR, ptr(acc), 1.0, None), 'adam_dense_reg')

    def unfused():
        check(N.lib.dtb_reg_grad(ptr(p), ptr(g), n, 0.0, L2_FACTOR, ptr(acc), 1.0, None), 'reg_grad')
        adam()

    results = []
    bytes_min = n * 32
    for name, fn in (('adam_dense', adam), ('adam_dense_reg (fused)', fused), ('reg_grad + adam_dense', unfused)):
        secs = events_time(fn, reps)
        results.append({'what': 'table_sweep', 'kernel': name, 'elements': n, 'ms': round(secs * 1e3, 3),
                        'GBps_at_32B_per_element': round(bytes_min / secs / 1e9, 1),
                        'share_of_datasheet_hbm': round(bytes_min / secs / (HBM_TBPS * 1e12), 3),
                        'datasheet_bound_ms': round(bytes_min / (HBM_TBPS * 1e12) * 1e3, 3)})
        print(json.dumps(results[-1]), flush=True)
    del p, m, v, g
    torch.cuda.empty_cache()
    return results


class _Unfused:
    """Stands in for the library inside DeepModel: the table's fused sweep becomes dtb_reg_grad + dtb_adam_dense."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def dtb_adam_dense_reg(self, p, m, v, g, n, alpha, b1, b2, eps, zero_grad, l1, l2, loss_acc, scale, stream):
        rc = self._lib.dtb_reg_grad(p, g, n, l1, l2, loss_acc, scale, stream)
        return rc or self._lib.dtb_adam_dense(p, m, v, g, n, alpha, b1, b2, eps, zero_grad, stream)

    def dtb_adam_dense_reg_dev(self, p, m, v, g, n, table, step_dev, b1, b2, eps, zero_grad, l1, l2, loss_acc, scale,
                               stream):
        rc = self._lib.dtb_reg_grad(p, g, n, l1, l2, loss_acc, scale, stream)
        return rc or self._lib.dtb_adam_dense_dev(p, m, v, g, n, table, step_dev, b1, b2, eps, zero_grad, stream)


def train_steps(steps, warmup):
    import torch
    import bench
    from deeptables_b200 import _native as N, regularizers as R
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    spec = bench.CONFIGS['xdeepfm']
    batch, vocab = spec['batch'], 1_000_000
    host = bench.synth_batches(warmup + steps, batch, vocab, 1234)
    devb = [tuple(t.cuda(non_blocking=True) for t in hb) for hb in host]
    results = []
    lib = N.lib
    for name, reg, mode, unfused in (('none', None, None, False), ('none, dense table', None, 'dense', False),
                                     ('L2(1e-5) fused', R.L2(L2_FACTOR), None, False),
                                     ('L2(1e-5) unfused', R.L2(L2_FACTOR), None, True)):
        conf = bench.make_config('xdeepfm')._replace(embeddings_regularizer=reg)
        cats = [CategoricalColumn(f'C{i + 1}', vocab, spec['dim']) for i in range(bench.F_FIELDS)]
        conts = [ContinuousColumn('input_continuous_all', [f'I{i + 1}' for i in range(bench.N_DENSE)])]
        model = DeepModel('binary', 2, conf, cats, conts, seed=1234)
        model._build_model()
        model._table_mode_override = mode
        N.lib = _Unfused(lib) if unfused else lib
        try:
            for s in range(warmup):
                model.train_step(*devb[s])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for s in range(steps):
                model.train_step(*devb[warmup + s])
            e1.record()
            torch.cuda.synchronize()
        finally:
            N.lib = lib
        secs = e0.elapsed_time(e1) * 1e-3
        loss = float(model._loss_acc.item()) / ((warmup + steps) * batch)
        results.append({'what': 'train_step', 'config': 'xdeepfm', 'regularizer': name, 'batch': batch, 'steps': steps,
                        'ms_per_step': round(secs * 1e3 / steps, 2), 'rows_per_s': round(steps * batch / secs),
                        'table_mode': 'lazy' if model.table.lazy_active else 'dense',
                        'graphed': bool(model._graphs), 'mean_loss': round(loss, 5)})
        print(json.dumps(results[-1]), flush=True)
        model.release()
        del model
        torch.cuda.empty_cache()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--sweeps', type=int, default=10, help='timed repetitions of each table sweep')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_reg needs a CUDA device')
    info = card()
    print(json.dumps(info), flush=True)
    out = {'card': info, 'table_sweeps': sweeps(args.sweeps), 'train_steps': train_steps(args.steps, args.warmup)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
