"""Throughput of linear probes (deeptables_b200/probe.py) on one GPU, against the host path.

1. ``dtb_probe_loss_grad`` alone, event-timed over ``--reps`` launches, at N = 1 000 000 rows, d in {64, 429, 1079}
   and K in {1, 10}: seconds, bytes/s of the 4 N d bytes of X it must read against the data sheet's 3.35 TB/s, and
   FP64 operations/s (2 K DFMA, 4 K flops, per element) against the data sheet's 34 TFLOP/s of vector FP64.
2. ``probe_evaluate`` on a Criteo-shaped frame (13 continuous, 26 categorical columns; tools/bench_importance.py) of
   ``--rows`` rows, split 80 / 20, with DeepFM and xDeepFM fitted for one epoch, over the layers of the reference's
   test: seconds per call and the encode / forward / fit / score split, with the L-BFGS iteration and objective
   evaluation counts.
3. The reference's path on the same machine: ``dt.apply`` to numpy, then scikit-learn's
   ``LogisticRegression(random_state=0)`` per layer, with the CPU cores it may use.

    python tools/bench_probe.py [--rows 1000000] [--reps 100] [--no-host]

Prints one JSON line per measurement, the card name and power limit first, read in the same run.  There is no
fallback: without a CUDA device it exits with an error."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from bench_optim import card, events_time  # noqa: E402
from bench_importance import N_CAT, frame  # noqa: E402

LAYERS = ['flatten_embeddings', 'dnn_dense_1', 'dnn_dense_2']
HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
FP64_FLOPS = 34e12                 # H100 SXM data sheet, FP64 without tensor cores


def kernel_rows(n, reps):
    import numpy as np
    import torch
    from deeptables_b200 import probe
    out = []
    g = torch.Generator(device='cuda').manual_seed(0)
    for d in (64, 429, 1079):
        X = torch.randn(n, d, device='cuda', generator=g)
        for K in (1, 10):
            codes = torch.randint(0, 2 if K == 1 else K, (n,), device='cuda', generator=g, dtype=torch.int32)
            obj = probe.DeviceObjective(X, codes, K, True)
            obj.W.copy_(torch.from_numpy(np.random.default_rng(1).normal(scale=0.05, size=K * (d + 1))))
            launch = lambda: probe.check(probe.N.lib.dtb_probe_loss_grad(
                probe.ptr(X), X.stride(0), probe.ptr(codes), probe.ptr(obj.W), n, d, K, 1, 0, probe.ptr(obj.partials),
                probe.stream_ptr()), 'probe_loss_grad')
            s = events_time(launch, reps)
            bytes_s, flops_s = 4.0 * n * d / s, 4.0 * K * n * d / s
            out.append({'what': 'dtb_probe_loss_grad', 'N': n, 'd': d, 'K': K, 'seconds': s,
                        'hbm_bytes_per_s': bytes_s, 'hbm_share_of_datasheet': bytes_s / HBM_BYTES_PER_S,
                        'fp64_flops_per_s': flops_s, 'fp64_share_of_datasheet': flops_s / FP64_FLOPS,
                        'bound': 'hbm' if 4.0 * d / HBM_BYTES_PER_S > 4.0 * K * d / FP64_FLOPS else 'fp64'})
            del obj, codes
        del X
    return out


def fitted(nets, X, y):
    from deeptables_b200 import deepnets, deeptable
    conf = deeptable.ModelConfig(nets=getattr(deepnets, nets), metrics=['AUC'], embeddings_output_dim=16,
                                 categorical_columns=[f'C{i}' for i in range(N_CAT)], earlystopping_patience=1)
    dt = deeptable.DeepTable(config=conf)
    dt.fit(X, y, epochs=1, batch_size=8192, verbose=0)
    return dt


def host_path(dt, X, y, Xt, yt):
    """The reference's probe_evaluate with score_fn={}: apply to numpy, scikit-learn per layer."""
    from sklearn.linear_model import LogisticRegression
    t0 = time.perf_counter()
    f_train = dt.apply(X, output_layers=LAYERS, batch_size=8192)
    f_test = dt.apply(Xt, output_layers=LAYERS, batch_size=8192)
    yc, ytc = dt.preprocessor.transform_y(y), dt.preprocessor.transform_y(yt)
    t_apply = time.perf_counter() - t0
    fits, scores = {}, {}
    for name, a, b in zip(LAYERS, f_train, f_test):
        t1 = time.perf_counter()
        clf = LogisticRegression(random_state=0).fit(a.reshape(len(a), -1), yc)
        fits[name] = {'seconds': time.perf_counter() - t1, 'n_iter': int(clf.n_iter_[0]), 'width': int(a[0].size)}
        scores[name] = float(clf.score(b.reshape(len(b), -1), ytc))
    return {'seconds': time.perf_counter() - t0, 'apply_seconds': t_apply, 'fits': fits, 'accuracy': scores}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=1_000_000)
    ap.add_argument('--reps', type=int, default=100)
    ap.add_argument('--no-host', action='store_true')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_probe: no CUDA device')
    from deeptables_b200 import probe
    print(json.dumps(card()), flush=True)
    for row in kernel_rows(1_000_000, args.reps):
        print(json.dumps(row), flush=True)
    X, y = frame(args.rows, 0)
    cut = args.rows * 4 // 5
    Xtr, ytr, Xte, yte = X.iloc[:cut], y[:cut], X.iloc[cut:], y[cut:]
    try:
        from threadpoolctl import threadpool_info
        blas = [(i.get('internal_api'), i.get('num_threads')) for i in threadpool_info()]
    except ImportError:
        blas = None
    for nets in ('DeepFM', 'xDeepFM'):
        dt = fitted(nets, Xtr, ytr)
        probe.probe_evaluate(dt, Xtr.iloc[:20_000], ytr[:20_000], Xte.iloc[:5_000], yte[:5_000], LAYERS)   # warm-up
        stages = {}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = probe.probe_evaluate(dt, Xtr, ytr, Xte, yte, LAYERS, stages=stages)
        sec = time.perf_counter() - t0
        widths = [int(a[0].numel()) for a in
                  dt.get_model().captured_outputs(*dt.get_model()._to_device_inputs(dt.preprocessor.transform_X(
                      Xte.iloc[:8])), 8, 8, LAYERS)]
        print(json.dumps({'what': 'probe_evaluate', 'nets': nets, 'train_rows': cut, 'test_rows': args.rows - cut,
                          'layers': dict(zip(LAYERS, widths)), 'seconds': sec, 'stages': stages,
                          'accuracy': {k: v['accuracy'] for k, v in res.items()}}), flush=True)
        if not args.no_host:
            host = host_path(dt, Xtr, ytr, Xte, yte)
            host.update({'what': 'host apply + scikit-learn', 'nets': nets, 'cpu_count': os.cpu_count(),
                         'cpu_affinity': len(os.sched_getaffinity(0)), 'blas_threads': blas})
            print(json.dumps(host), flush=True)
        del dt
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
