"""Cost of the streaming metrics (deeptables_b200/metrics.py) on one GPU.

1. ``dtb_metrics_update`` alone, binary predictions at 65 536 and 8 192 rows: a 2-bucket plan (Precision / Recall at 0.5)
   a 201-bucket plan (AUC(num_thresholds=200)) and a plan of float64 sums only (R2Score + MeanSquaredError, on the same
   arrays), on uniform random predictions and on predictions that are all 0.5
   (every thread of a block counts into one bucket, what an untrained model produces).  100 launches are captured in
   one CUDA graph so that the kernels run back to back, and CUDA events time its replays; reported against the 8 bytes
   per row the kernel must read and NVIDIA's H100 SXM data-sheet 3.35 TB/s of HBM3.  At these sizes the inputs stay in
   L2 between launches, so this is the kernel's own time, not an HBM rate.
2. Train steps: DeepFM at 8 192 rows and xDeepFM at 65 536 rows (bench.py's 'deepfm_bs8192' and 'xdeepfm' configs) with
   metrics=[], ['AUC'] (an epoch function: nothing runs per step) and [AUC(), Precision(), Recall()] (one more kernel
   per step), each replayed as a CUDA graph and with eager launches (DTB_CUDA_GRAPH=0).
3. Epoch end at 10 M predictions: the rank-sum 'AUC' function on the collected predictions against one
   dtb_metrics_update over them plus reading and finishing the streaming state.

    python tools/bench_metrics.py [--steps 20] [--warmup 5] [--rounds 3]

The arms of a group are timed alternately, round by round, in one process; each reports the median over rounds.  Prints
one JSON line per measurement, the card name and power limit first, read in the same run, and a final summary line.
There is no fallback: without a CUDA device it exits with an error."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_optim import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # NVIDIA's H100 SXM data sheet
LAUNCHES_PER_GRAPH = 100


def update_kernel(rounds):
    import torch
    from deeptables_b200 import engine as E, metrics as M
    plans = {'2_buckets': ('binary', [M.Precision(), M.Recall()]), '201_buckets': ('binary', [M.AUC()]),
             'r2_mse_sums': ('regression', [M.R2Score(), M.MeanSquaredError()])}
    cases = {}
    for rows in (65536, 8192):
        g = torch.Generator(device='cuda').manual_seed(rows)
        y = (torch.rand(rows, 1, device='cuda', generator=g) < 0.25).float()
        preds = {'uniform': torch.rand(rows, 1, device='cuda', generator=g), 'all_0.5': torch.full((rows, 1), 0.5, device='cuda')}
        for plan_name, (task, entries) in plans.items():
            st = E.MetricsState(M.Plan([M.resolve(e, task, 2) for e in entries], 1), torch.device('cuda'))
            for pred_name, p in preds.items():
                st.update(p, y)
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    for _ in range(LAUNCHES_PER_GRAPH):
                        st.update(p, y)
                cases[(rows, plan_name, pred_name)] = (graph, st, p, y)
    times = {k: [] for k in cases}
    for _ in range(rounds):
        for k, (graph, *_) in cases.items():
            graph.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e-3 / (20 * LAUNCHES_PER_GRAPH))
    results = []
    for (rows, plan_name, pred_name), ts in times.items():
        sec = statistics.median(ts)
        nbytes = 8 * rows
        results.append({'what': 'metrics_update', 'rows': rows, 'plan': plan_name, 'predictions': pred_name,
                        'us': round(sec * 1e6, 3), 'bytes_read': nbytes, 'GBps': round(nbytes / sec / 1e9, 1),
                        'data_sheet_hbm_us': round(nbytes / HBM_BYTES_PER_S * 1e6, 3),
                        'us_rounds': [round(t * 1e6, 3) for t in ts]})
        print(json.dumps(results[-1]), flush=True)
    return results


def train_steps(steps, warmup, rounds):
    import torch
    import bench
    from deeptables_b200 import _native as N, metrics as M
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    results = []
    vocab = 1_000_000
    metric_arms = {'none': [], "'AUC'": ['AUC'], 'AUC()+Precision()+Recall()': [M.AUC(name='auc_200'), M.Precision(), M.Recall()]}
    for name in ('deepfm_bs8192', 'xdeepfm'):
        spec = bench.CONFIGS[name]
        batch = spec['batch']
        host = bench.synth_batches(warmup + steps, batch, vocab, 1234)
        devb = [tuple(t.cuda(non_blocking=True) for t in hb) for hb in host]
        arms = {}
        for arm, metrics in metric_arms.items():
            for graph in ('1', '0'):
                os.environ['DTB_CUDA_GRAPH'] = graph
                conf = bench.make_config(name)._replace(metrics=metrics)
                cats = [CategoricalColumn(f'C{i + 1}', vocab, spec['dim']) for i in range(bench.F_FIELDS)]
                conts = [ContinuousColumn('input_continuous_all', [f'I{i + 1}' for i in range(bench.N_DENSE)])]
                model = DeepModel('binary', 2, conf, cats, conts, seed=1234)
                model._build_model()
                for s in range(warmup):
                    model.train_step(*devb[s])
                arms[(arm, graph)] = model
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        launches = {}
        for _ in range(rounds):
            for (arm, graph), model in arms.items():
                os.environ['DTB_CUDA_GRAPH'] = graph
                l0 = N.lib.dtb_launch_count()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for s in range(steps):
                    model.train_step(*devb[warmup + s])
                e1.record()
                torch.cuda.synchronize()
                times[(arm, graph)].append(e0.elapsed_time(e1) / steps)
                launches[(arm, graph)] = (N.lib.dtb_launch_count() - l0) / steps
        for (arm, graph), model in arms.items():
            ts = times[(arm, graph)]
            ms = statistics.median(ts)
            assert bool(model._graphs) == (graph == '1'), 'the arm did not run in the mode it is labelled with'
            results.append({'what': 'train_step', 'config': name, 'batch': batch, 'metrics': arm,
                            'cuda_graph': graph == '1', 'ms_per_step': round(ms, 4),
                            'rows_per_s': round(batch / (ms * 1e-3)), 'launches_per_step': launches[(arm, graph)],
                            'steps_per_round': steps, 'ms_rounds': [round(t, 4) for t in ts]})
            print(json.dumps(results[-1]), flush=True)
            model.release()
        del arms, devb
        torch.cuda.empty_cache()
    os.environ.pop('DTB_CUDA_GRAPH', None)
    return results


def epoch_end(rounds, n=10_000_000):
    import torch
    from deeptables_b200 import deepmodel, engine as E, metrics as M
    g = torch.Generator(device='cuda').manual_seed(1)
    y = (torch.rand(n, 1, device='cuda', generator=g) < 0.25).float()
    p = torch.sigmoid(torch.randn(n, 1, device='cuda', generator=g) + y)
    plan = M.Plan([M.resolve(M.AUC(), 'binary', 2)], 1)
    st = E.MetricsState(plan, torch.device('cuda'))

    def exact():
        return deepmodel._auc(y, p)

    def read_only():                 # what an epoch pays when every batch was added during its train step
        return plan.finish(st.read())['auc']

    def update_and_read():
        st.reset()
        st.update(p, y)
        return read_only()

    arms = {"'AUC' (rank sum over the epoch's predictions)": exact,
            'AUC(): one update over all rows, read, finish': update_and_read, 'AUC(): read and finish the state': read_only}
    values, times = {}, {k: [] for k in arms}
    for k, fn in arms.items():
        values[k] = fn()
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    results = []
    for k, ts in times.items():
        results.append({'what': 'epoch_end', 'predictions': n, 'arm': k, 'ms': round(statistics.median(ts) * 1e3, 3),
                        'value': values[k], 'ms_rounds': [round(t * 1e3, 3) for t in ts]})
        print(json.dumps(results[-1]), flush=True)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_metrics needs a CUDA device')
    info = card()
    print(json.dumps(info), flush=True)
    out = {'card': info, 'update_kernel': update_kernel(args.rounds), 'epoch_end': epoch_end(args.rounds),
           'train_steps': train_steps(args.steps, args.warmup, args.rounds)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
