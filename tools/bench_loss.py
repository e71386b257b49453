"""Cost of the Keras losses (deeptables_b200/losses.py) on one GPU.

1. ``dtb_keras_loss_fwd_bwd`` alone at 65 536 rows x C in {1, 10, 100}, for every loss code, against the kernel 'auto'
   runs (``dtb_loss_fwd_bwd``): C = 1 on a sigmoid output with 0 / 1 labels, C = 10 and 100 on a softmax output with
   one-hot labels, dz written.  100 launches are captured in one CUDA graph so that the kernels run back to back, and
   CUDA events time its replays; reported against the 16 bytes per element the kernel must move (z and y read, prob
   and dz written) and NVIDIA's H100 SXM data-sheet 3.35 TB/s of HBM3.  At these sizes the arrays stay in L2 between
   launches, so this is the kernel's own time, not an HBM rate.
2. Train steps: DeepFM at 8 192 rows and xDeepFM at 65 536 rows (bench.py's 'deepfm_bs8192' and 'xdeepfm' configs) with
   loss='auto', Huber() and BinaryCrossentropy(label_smoothing=0.1), each replayed as a CUDA graph and with eager
   launches (DTB_CUDA_GRAPH=0).

    python tools/bench_loss.py [--steps 20] [--warmup 5] [--rounds 3]

The arms of a group are timed alternately, round by round, in one process; each reports the median over rounds.  Prints
one JSON line per measurement, the card name and power limit first, read in the same run, and a final summary line.
There is no fallback: without a CUDA device it exits with an error."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_optim import card  # noqa: E402

HBM_BYTES_PER_S = 3.35e12       # NVIDIA's H100 SXM data sheet
LAUNCHES_PER_GRAPH = 100
ROWS = 65536


def loss_kernel(rounds):
    import torch
    from deeptables_b200 import _native as N, losses as LS
    cases = {}
    keep = []
    for cols in (1, 10, 100):
        task = 0 if cols == 1 else 2
        g = torch.Generator(device='cuda').manual_seed(cols)
        z = torch.randn(ROWS, cols, device='cuda', generator=g) * 2
        if cols == 1:
            y = (torch.rand(ROWS, 1, device='cuda', generator=g) < 0.3).float()
        else:
            y = torch.nn.functional.one_hot(torch.randint(0, cols, (ROWS,), device='cuda', generator=g), cols).float()
        prob, dz = torch.empty_like(z), torch.empty_like(z)
        acc = torch.zeros(1, dtype=torch.float64, device='cuda')
        scratch = torch.empty(1, dtype=torch.int32, device='cuda')
        keep += [z, y, prob, dz, acc, scratch]
        arms = {'auto kernel (dtb_loss_fwd_bwd)': None}
        arms.update({kind: LS.LossSpec(kind) for kind in LS.CODES})
        for arm, spec in arms.items():
            if spec is None:
                def launch(z=z, y=y, prob=prob, dz=dz, acc=acc, cols=cols, task=task):
                    N.check(N.lib.dtb_loss_fwd_bwd(N.ptr(z), N.ptr(y), None, N.ptr(prob), N.ptr(dz), N.ptr(acc), ROWS,
                                                   cols, task, N.stream_ptr()))
            else:
                lp = N.LossParams(loss=spec.code, delta=spec.delta, label_smoothing=spec.label_smoothing,
                                  scratch=scratch.data_ptr())
                keep.append(lp)

                def launch(z=z, y=y, prob=prob, dz=dz, acc=acc, cols=cols, task=task, lp=lp):
                    N.check(N.lib.dtb_keras_loss_fwd_bwd(N.ptr(z), N.ptr(y), None, N.ptr(prob), N.ptr(dz), N.ptr(acc),
                                                         ROWS, cols, task, lp, N.stream_ptr()))
            launch()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(LAUNCHES_PER_GRAPH):
                    launch()
            cases[(cols, arm)] = graph
    times = {k: [] for k in cases}
    for _ in range(rounds):
        for k, graph in cases.items():
            graph.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                graph.replay()
            e1.record()
            torch.cuda.synchronize()
            times[k].append(e0.elapsed_time(e1) * 1e-3 / (20 * LAUNCHES_PER_GRAPH))
    results = []
    for (cols, arm), ts in times.items():
        sec = statistics.median(ts)
        nbytes = 16 * ROWS * cols
        results.append({'what': 'loss_kernel', 'rows': ROWS, 'cols': cols, 'output': 'sigmoid' if cols == 1 else 'softmax',
                        'loss': arm, 'us': round(sec * 1e6, 3), 'bytes_moved': nbytes,
                        'GBps': round(nbytes / sec / 1e9, 1), 'data_sheet_hbm_us': round(nbytes / HBM_BYTES_PER_S * 1e6, 3),
                        'us_rounds': [round(t * 1e6, 3) for t in ts]})
        print(json.dumps(results[-1]), flush=True)
    return results


def train_steps(steps, warmup, rounds):
    import torch
    import bench
    from deeptables_b200 import _native as N, losses as LS
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    results = []
    vocab = 1_000_000
    loss_arms = {"'auto'": 'auto', 'Huber()': LS.Huber(), 'BinaryCrossentropy(label_smoothing=0.1)':
                 LS.BinaryCrossentropy(label_smoothing=0.1)}
    for name in ('deepfm_bs8192', 'xdeepfm'):
        spec = bench.CONFIGS[name]
        batch = spec['batch']
        host = bench.synth_batches(warmup + steps, batch, vocab, 1234)
        devb = [tuple(t.cuda(non_blocking=True) for t in hb) for hb in host]
        arms = {}
        for arm, loss in loss_arms.items():
            for graph in ('1', '0'):
                os.environ['DTB_CUDA_GRAPH'] = graph
                conf = bench.make_config(name)._replace(loss=loss)
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
            results.append({'what': 'train_step', 'config': name, 'batch': batch, 'loss': arm,
                            'model_desc_loss': model.model_desc.loss, 'cuda_graph': graph == '1',
                            'ms_per_step': round(ms, 4), 'rows_per_s': round(batch / (ms * 1e-3)),
                            'launches_per_step': launches[(arm, graph)], 'steps_per_round': steps,
                            'ms_rounds': [round(t, 4) for t in ts]})
            print(json.dumps(results[-1]), flush=True)
            model.release()
        del arms, devb
        torch.cuda.empty_cache()
    os.environ.pop('DTB_CUDA_GRAPH', None)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_loss needs a CUDA device')
    info = card()
    print(json.dumps(info), flush=True)
    out = {'card': info, 'loss_kernel': loss_kernel(args.rounds), 'train_steps': train_steps(args.steps, args.warmup,
                                                                                             args.rounds)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
