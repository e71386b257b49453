"""Optimiser cost on one GPU: the dense sweep of every optimiser at the Criteo table size, and the xDeepFM headline
train step (bench.py's 'xdeepfm' config) with each optimiser.

    python tools/bench_optim.py [--steps 20] [--warmup 5] [--sweeps 10]

Prints one JSON line per measurement and a final summary line; the card name and power limit come first, read in the
same run.  The sweep's bytes per element are those the algorithm must move: p, g and the state slots read and written
(Adam: p, m, v, g -> 32 B)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TABLE_ROWS, TABLE_DIM = 26_000_000, 16          # 26 fields x 1 M ids, embed_dim 16


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(',')]
        return {'gpu': name, 'power_limit': power, 'max_sm_clock': clock}
    except Exception as exc:                       # informational only
        return {'gpu': 'unknown', 'error': str(exc)}


def events_time(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / reps


def sweeps(reps):
    import torch
    from deeptables_b200 import _native as N, engine as E, optimizers as O
    from deeptables_b200.deepmodel import _native_optim_params
    from deeptables_b200._native import ptr, check
    n = TABLE_ROWS * TABLE_DIM
    bufs = [torch.zeros(n, dtype=torch.float32, device='cuda') for _ in range(5)]     # p, g, s0, s1, s2 (Adam: p, m, v, g)
    p, g = bufs[0], bufs[1]
    results = []
    adam = lambda: check(N.lib.dtb_adam_dense(ptr(p), ptr(bufs[2]), ptr(bufs[3]), ptr(g), n, E.adam_alpha(10), E.ADAM_B1,
                                              E.ADAM_B2, E.ADAM_EPS, 1, None), 'adam_dense')
    cases = [('adam', None, adam, 2)]
    for name, opt in (('sgd', 'sgd'), ('sgd_momentum', O.SGD(momentum=0.9)), ('rmsprop', 'rmsprop'),
                      ('rmsprop_centered_momentum', O.RMSprop(momentum=0.9, centered=True)), ('adagrad', 'adagrad')):
        spec = O.resolve(opt)
        hp = _native_optim_params(spec)
        slots = [None if s is None else bufs[2 + k] for k, s in enumerate(O.slot_inits(spec))]
        fn = (lambda hp=hp, slots=slots: check(N.lib.dtb_optim_dense(ptr(p), ptr(g), *[ptr(s) for s in slots], n, hp, 1,
                                                                       None), 'optim_dense'))
        cases.append((name, spec, fn, sum(s is not None for s in slots)))
    for name, spec, fn, n_slots in cases:
        secs = events_time(fn, reps)
        bytes_per_elem = 2 * 4 * (2 + n_slots)             # p, g and the slots: read once, written once
        results.append({'what': 'dense_sweep', 'optimizer': name, 'elements': n, 'slots': n_slots,
                        'bytes_per_element': bytes_per_elem, 'ms': round(secs * 1e3, 3),
                        'hbm_GBps': round(n * bytes_per_elem / secs / 1e9, 1)})
        print(json.dumps(results[-1]), flush=True)
    del bufs, p, g
    torch.cuda.empty_cache()
    return results


def train_steps(steps, warmup):
    import torch
    import bench
    from deeptables_b200 import optimizers as O
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    spec = bench.CONFIGS['xdeepfm']
    batch, vocab = spec['batch'], 1_000_000
    host = bench.synth_batches(warmup + steps, batch, vocab, 1234)
    devb = [tuple(t.cuda(non_blocking=True) for t in hb) for hb in host]
    results = []
    for name, opt in (('auto', 'auto'), ('sgd', 'sgd'), ('sgd_momentum', O.SGD(momentum=0.9)), ('rmsprop', 'rmsprop'),
                      ('adagrad', 'adagrad')):
        conf = bench.make_config('xdeepfm')._replace(optimizer=opt)
        cats = [CategoricalColumn(f'C{i + 1}', vocab, spec['dim']) for i in range(bench.F_FIELDS)]
        conts = [ContinuousColumn('input_continuous_all', [f'I{i + 1}' for i in range(bench.N_DENSE)])]
        model = DeepModel('binary', 2, conf, cats, conts, seed=1234)
        model._build_model()
        for s in range(warmup):
            model.train_step(*devb[s])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in range(steps):
            model.train_step(*devb[warmup + s])
        e1.record()
        torch.cuda.synchronize()
        secs = e0.elapsed_time(e1) * 1e-3
        loss = float(model._loss_acc.item()) / ((warmup + steps) * batch)
        results.append({'what': 'train_step', 'config': 'xdeepfm', 'optimizer': name, 'batch': batch, 'steps': steps,
                        'ms_per_step': round(secs * 1e3 / steps, 2), 'rows_per_s': round(steps * batch / secs),
                        'table_mode': 'lazy' if model.table.lazy_active else 'dense', 'mean_loss': round(loss, 5)})
        print(json.dumps(results[-1]), flush=True)
        model.release()
        del model
        torch.cuda.empty_cache()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--sweeps', type=int, default=10, help='timed repetitions of each dense sweep')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_optim needs a CUDA device')
    info = card()
    print(json.dumps(info), flush=True)
    out = {'card': info, 'dense_sweeps': sweeps(args.sweeps), 'train_steps': train_steps(args.steps, args.warmup)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
