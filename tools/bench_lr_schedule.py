"""Cost of learning-rate schedules on one GPU: the xDeepFM headline train step (bench.py's 'xdeepfm' config, 65 536
rows) with Adam and RMSprop at a constant rate, ExponentialDecay and CosineDecay with warmup, and the dense sweep over
the 26 x 1 M x 16 table with the constant-rate kernel and the rate-table kernel (host step and device step).

    python tools/bench_lr_schedule.py [--steps 20] [--warmup 5] [--rounds 3] [--sweeps 10]

The variants of each group are timed alternately, round by round, so that clock and thermal drift fall on all of them
alike; each reports the median over rounds.  Prints one JSON line per measurement, the card name and power limit first,
read in the same run, and a final summary line."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_optim import TABLE_DIM, TABLE_ROWS, card, events_time  # noqa: E402


def sweeps(reps, rounds):
    import torch
    from deeptables_b200 import _native as N, optimizers as O
    from deeptables_b200._native import check, ptr
    from deeptables_b200.deepmodel import _native_optim_params
    n = TABLE_ROWS * TABLE_DIM
    spec = O.resolve(O.RMSprop(momentum=0.9))
    hp = _native_optim_params(spec)
    p, g, s0, s2 = (torch.zeros(n, dtype=torch.float32, device='cuda') for _ in range(4))
    table = torch.full((4096,), 1e-3, dtype=torch.float32, device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    cases = {
        'constant': lambda: check(N.lib.dtb_optim_dense(ptr(p), ptr(g), ptr(s0), None, ptr(s2), n, hp, 1, None)),
        'table_host_step': lambda: check(N.lib.dtb_optim_dense_lr(ptr(p), ptr(g), ptr(s0), None, ptr(s2), n, hp,
                                                                  ptr(table), 7, None, 1, None)),
        'table_device_step': lambda: check(N.lib.dtb_optim_dense_lr(ptr(p), ptr(g), ptr(s0), None, ptr(s2), n, hp,
                                                                    ptr(table), 0, ptr(step_dev), 1, None)),
    }
    times = {k: [] for k in cases}
    for _ in range(rounds):
        for k, fn in cases.items():
            times[k].append(events_time(fn, reps))
    results = []
    for k, ts in times.items():
        ms = statistics.median(ts) * 1e3
        results.append({'what': 'dense_sweep', 'optimizer': 'rmsprop_momentum', 'kernel': k, 'elements': n,
                        'ms': round(ms, 3), 'hbm_GBps': round(n * 2 * 4 * 4 / (ms * 1e-3) / 1e9, 1),
                        'ms_rounds': [round(t * 1e3, 3) for t in ts]})
        print(json.dumps(results[-1]), flush=True)
    del p, g, s0, s2
    torch.cuda.empty_cache()
    return results


def train_steps(steps, warmup, rounds):
    import torch
    import bench
    from deeptables_b200 import optimizers as O, schedules as S
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    spec = bench.CONFIGS['xdeepfm']
    batch, vocab = spec['batch'], 1_000_000
    host = bench.synth_batches(warmup + steps, batch, vocab, 1234)
    devb = [tuple(t.cuda(non_blocking=True) for t in hb) for hb in host]
    rates = {'constant': lambda lr: lr,
             'exponential': lambda lr: S.ExponentialDecay(lr, decay_steps=1000, decay_rate=0.9),
             'cosine_warmup': lambda lr: S.CosineDecay(lr / 10, decay_steps=10000, warmup_target=lr, warmup_steps=1000)}
    results = []
    for opt_name, make in (('adam', lambda lr: O.Adam(learning_rate=lr)),
                           ('rmsprop', lambda lr: O.RMSprop(learning_rate=lr))):
        models = {}
        for rate_name, rate in rates.items():
            conf = bench.make_config('xdeepfm')._replace(optimizer=make(rate(1e-3)))
            cats = [CategoricalColumn(f'C{i + 1}', vocab, spec['dim']) for i in range(bench.F_FIELDS)]
            conts = [ContinuousColumn('input_continuous_all', [f'I{i + 1}' for i in range(bench.N_DENSE)])]
            model = DeepModel('binary', 2, conf, cats, conts, seed=1234)
            model._build_model()
            for s in range(warmup):
                model.train_step(*devb[s])
            models[rate_name] = model
        torch.cuda.synchronize()
        times = {k: [] for k in models}
        for _ in range(rounds):
            for rate_name, model in models.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for s in range(steps):
                    model.train_step(*devb[warmup + s])
                e1.record()
                torch.cuda.synchronize()
                times[rate_name].append(e0.elapsed_time(e1) / steps)
        for rate_name, model in models.items():
            ts = times[rate_name]
            results.append({'what': 'train_step', 'config': 'xdeepfm', 'optimizer': opt_name, 'rate': rate_name,
                            'batch': batch, 'steps_per_round': steps, 'ms_per_step': round(statistics.median(ts), 3),
                            'ms_rounds': [round(t, 3) for t in ts], 'cuda_graph': bool(model._graphs),
                            'table_mode': 'lazy' if model.table.lazy_active else 'dense',
                            'next_learning_rate': model.optimizer.learning_rate})
            print(json.dumps(results[-1]), flush=True)
            model.release()
        del models
        torch.cuda.empty_cache()
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--sweeps', type=int, default=10, help='timed repetitions of each dense sweep per round')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_lr_schedule needs a CUDA device')
    info = card()
    print(json.dumps(info), flush=True)
    out = {'card': info, 'dense_sweeps': sweeps(args.sweeps, args.rounds),
           'train_steps': train_steps(args.steps, args.warmup, args.rounds)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
