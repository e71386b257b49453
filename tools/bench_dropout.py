"""Cost of dropout on one GPU.

1. Train steps: DeepFM at 8 192 rows and xDeepFM at 65 536 rows (bench.py's 'deepfm_bs8192' and 'xdeepfm' configs) with
   embedding_dropout 0 and 0.3 (the reference's default), each replayed as a CUDA graph and with eager launches
   (DTB_CUDA_GRAPH=0): time per step, rows/s and the library's kernel launches per step.
2. The AutoInt attention kernels (embeddings_output_dim 32, 4 heads, 26 fields, 65 536 rows: one of the three layers
   of bench.py's 'dcn6_autoint4x32'): forward and backward at dropout_rate 0 and 0.1, with the bytes and operations
   the algorithm needs over the measured time.  These are CUDA-core kernels; the H100 SXM data-sheet rates they are
   compared with are 3.35 TB/s of HBM3 and 67 TFLOP/s in FP32, and the bound named is the larger of the two times.

    python tools/bench_dropout.py [--steps 20] [--warmup 5] [--rounds 3] [--reps 20]

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

from bench_optim import card, events_time  # noqa: E402

HBM_BYTES_PER_S, FP32_FLOP_PER_S = 3.35e12, 67e12      # NVIDIA's H100 SXM data sheet


def train_steps(steps, warmup, rounds):
    import torch
    import bench
    from deeptables_b200 import _native as N
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    results = []
    vocab = 1_000_000
    for name in ('deepfm_bs8192', 'xdeepfm'):
        spec = bench.CONFIGS[name]
        batch = spec['batch']
        host = bench.synth_batches(warmup + steps, batch, vocab, 1234)
        devb = [tuple(t.cuda(non_blocking=True) for t in hb) for hb in host]
        arms = {}
        for rate in (0.0, 0.3):
            for graph in ('1', '0'):
                os.environ['DTB_CUDA_GRAPH'] = graph
                conf = bench.make_config(name)._replace(embedding_dropout=rate)
                cats = [CategoricalColumn(f'C{i + 1}', vocab, spec['dim']) for i in range(bench.F_FIELDS)]
                conts = [ContinuousColumn('input_continuous_all', [f'I{i + 1}' for i in range(bench.N_DENSE)])]
                model = DeepModel('binary', 2, conf, cats, conts, seed=1234)
                model._build_model()
                for s in range(warmup):
                    model.train_step(*devb[s])
                arms[(rate, graph)] = model
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        launches = {}
        for _ in range(rounds):
            for (rate, graph), model in arms.items():
                os.environ['DTB_CUDA_GRAPH'] = graph
                l0 = N.lib.dtb_launch_count()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for s in range(steps):
                    model.train_step(*devb[warmup + s])
                e1.record()
                torch.cuda.synchronize()
                times[(rate, graph)].append(e0.elapsed_time(e1) / steps)
                launches[(rate, graph)] = (N.lib.dtb_launch_count() - l0) / steps
        for (rate, graph), model in arms.items():
            ts = times[(rate, graph)]
            ms = statistics.median(ts)
            assert bool(model._graphs) == (graph == '1'), 'the arm did not run in the mode it is labelled with'
            results.append({'what': 'train_step', 'config': name, 'batch': batch, 'embedding_dropout': rate,
                            'cuda_graph': graph == '1', 'ms_per_step': round(ms, 3),
                            'rows_per_s': round(batch / (ms * 1e-3)), 'launches_per_step': launches[(rate, graph)],
                            'steps_per_round': steps, 'ms_rounds': [round(t, 3) for t in ts]})
            print(json.dumps(results[-1]), flush=True)
            model.release()
        del arms, devb
        torch.cuda.empty_cache()
    os.environ.pop('DTB_CUDA_GRAPH', None)
    return results


def attention_kernels(reps, rounds):
    import torch
    from deeptables_b200 import _native as N
    from deeptables_b200._native import check, ptr
    b, f, d, heads = 65536, 26, 32, 4
    g = torch.Generator(device='cuda').manual_seed(7)
    x = torch.relu(torch.randn(b, f, 4 * d, device='cuda', generator=g))
    dy = torch.randn(b, f, d, device='cuda', generator=g)
    y, dq = torch.empty(b, f, d, device='cuda'), torch.empty_like(x)
    # what the algorithm has to move and compute: [Q|K|V|R] in, Y out; backward reads Y and dY too and writes d[Q|K|V|R];
    # per (row, head, query, key) two Q.K products (max, then weights) and the weight times V; backward three sweeps
    # of Q.K and dout.V plus the dQ / dK / dV accumulations
    pairs = b * heads * f * f * (d // heads)
    work = {'fwd': (4 * b * f * 5 * d, 2 * 3 * pairs), 'bwd': (4 * b * f * 10 * d, 2 * 9 * pairs)}

    def fwd(rate):
        return lambda: check(N.lib.dtb_attention_core_dropout_fwd(ptr(x), ptr(y), b, f, d, heads, 1, rate, 12345, None, 0,
                                                                  None))

    def bwd(rate):
        return lambda: check(N.lib.dtb_attention_core_dropout_bwd(ptr(x), ptr(y), ptr(dy), ptr(dq), b, f, d, heads, 1, 1,
                                                                  rate, 12345, None, 0, None))

    fwd(0.0)()
    cases = {('fwd', 0.0): fwd(0.0), ('fwd', 0.1): fwd(0.1), ('bwd', 0.0): bwd(0.0), ('bwd', 0.1): bwd(0.1)}
    times = {k: [] for k in cases}
    for _ in range(rounds):
        for k, fn in cases.items():
            times[k].append(events_time(fn, reps))
    results = []
    for (kind, rate), ts in times.items():
        sec = statistics.median(ts)
        nbytes, flop = work[kind]
        t_hbm, t_fp32 = nbytes / HBM_BYTES_PER_S, flop / FP32_FLOP_PER_S
        results.append({'what': 'attention_core_' + kind, 'rows': b, 'fields': f, 'dim': d, 'heads': heads,
                        'dropout_rate': rate, 'ms': round(sec * 1e3, 4), 'algorithmic_GB': round(nbytes / 1e9, 3),
                        'GBps': round(nbytes / sec / 1e9, 1), 'algorithmic_GFLOP': round(flop / 1e9, 2),
                        'TFLOPps': round(flop / sec / 1e12, 2), 'bound': 'HBM' if t_hbm >= t_fp32 else 'FP32',
                        'share_of_data_sheet_bound': round(max(t_hbm, t_fp32) / sec, 3),
                        'ms_rounds': [round(t * 1e3, 4) for t in ts]})
        print(json.dumps(results[-1]), flush=True)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--reps', type=int, default=20, help='timed launches of each attention kernel per round')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_dropout needs a CUDA device')
    info = card()
    print(json.dumps(info), flush=True)
    out = {'card': info, 'attention_kernels': attention_kernels(args.reps, args.rounds),
           'train_steps': train_steps(args.steps, args.warmup, args.rounds)}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
