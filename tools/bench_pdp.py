"""Throughput of partial dependence (deeptables_b200/utils/partial_dependence.py) on one GPU.

A Criteo-shaped frame (13 continuous, 26 categorical columns of 1 000 values each; C1 has 20 levels) with a synthetic
binary label; the model is fitted for one epoch on 100 000 rows.  Then three curves over 1 000 000 rows: I0 on 100
points, the 20-level C1, and a 10 x 10 grid of (I1, I2), for DeepFM at 8 192-row batches and xDeepFM at 65 536.  For
each: seconds per call (encoding included), composed rows per second, and the compose / forward / reduce split from
CUDA events, with the host time spent encoding X and the grid rows.  Then ``dtb_pdp_block_sums`` alone over 100 grid
points x 1 000 000 rows, in GB/s of algorithmic bytes (probabilities and weights read once, sums written).  For comparison, scikit-learn's ``partial_dependence`` over the
adapter of tests/pdp_ref.py (``predict_proba`` per grid point) on 100 000 rows with ``grid_resolution=20``, against the
device path at that size.

    python tools/bench_pdp.py [--rounds 2] [--rows 1000000]

Prints one JSON line per measurement, the card name and power limit first, read in the same run.  Each figure is the
median over rounds.  There is no fallback: without a CUDA device it exits with an error."""
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

from bench_optim import card, events_time  # noqa: E402
from bench_importance import N_CAT, frame  # noqa: E402

CURVES = [('I0, 100 points', 'I0', {}), ('C1, 20 levels', 'C1', {'categorical_features': ['C1']}),
          ('I1 x I2, 10 x 10', ['I1', 'I2'], {'grid_resolution': 10})]


def criteo(rows, seed):
    import numpy as np
    X, y = frame(rows, seed)
    X['C1'] = np.random.default_rng(seed + 1).integers(0, 20, rows)
    return X, y


def fitted(nets, X, y):
    from deeptables_b200 import deepnets, deeptable
    conf = deeptable.ModelConfig(nets=getattr(deepnets, nets), metrics=['AUC'], embeddings_output_dim=16,
                                 categorical_columns=[f'C{i}' for i in range(N_CAT)], earlystopping_patience=1)
    dt = deeptable.DeepTable(config=conf)
    dt.fit(X.iloc[:100_000], y[:100_000], epochs=1, batch_size=8192, verbose=0, validation_split=0.1)
    return dt


def call(dt, X, features, kw, bs, stages=None):
    from deeptables_b200.utils import partial_dependence as P
    args = dict(sample_weight=None, categorical_features=None, feature_names=None, response_method='auto',
                percentiles=(0.05, 0.95), grid_resolution=100, custom_values=None, method='auto', kind='average',
                batch_size=bs)
    args.update(kw)
    return P._partial_dependence(dt, X, features, stages=stages, **args)


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--rows', type=int, default=1_000_000)
    a = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit('bench_pdp needs a CUDA device')
    print(json.dumps(card()), flush=True)
    X, y = criteo(a.rows, 0)
    for nets, bs in (('DeepFM', 8192), ('xDeepFM', 65536)):
        dt = fitted(nets, X, y)
        for name, features, kw in CURVES:
            call(dt, X.iloc[:20_000], features, kw, bs)                   # warm-up
            totals, splits = [], []
            for _ in range(a.rounds):
                t, out = timed(lambda: call(dt, X, features, kw, bs))
                totals.append(t)
                st = {}
                call(dt, X, features, kw, bs, stages=st)
                splits.append(st)
            points = out.average[0].size
            total = statistics.median(totals)
            split = {k: round(statistics.median(s[k] for s in splits), 4) for k in splits[0]}
            print(json.dumps({'what': 'device', 'nets': nets, 'batch': bs, 'curve': name, 'rows': a.rows,
                              'grid_points': points, 'call_s': round(total, 3),
                              'composed_rows_per_s': round(points * a.rows / total), 'split_s': split,
                              'rounds': a.rounds}), flush=True)

        if nets == 'DeepFM':
            # scikit-learn's brute method over the adapter: one predict_proba (with its transform_X) per grid point
            sys.path.insert(0, os.path.join(ROOT, 'tests'))
            import pdp_ref
            from sklearn.inspection import partial_dependence as sk_pd
            # float64: pandas refuses to set a float64 grid value into a float32 column in place
            Xs = X.iloc[:100_000].reset_index(drop=True).astype({'I0': 'float64'})
            t_host, theirs = timed(lambda: sk_pd(pdp_ref.adapter(dt), Xs, 'I0', grid_resolution=20, method='brute'))
            call(dt, Xs, 'I0', {'grid_resolution': 20}, bs)
            t_dev, ours = timed(lambda: call(dt, Xs, 'I0', {'grid_resolution': 20}, bs))
            print(json.dumps({'what': 'host sklearn brute vs device', 'nets': nets, 'rows': len(Xs), 'grid_points': 20,
                              'host_s': round(t_host, 3), 'device_s': round(t_dev, 3),
                              'speedup': round(t_host / t_dev, 1),
                              'max_abs_diff': float(np.abs(ours.average - theirs.average).max())}), flush=True)

    # the reduction kernel alone
    from deeptables_b200 import _native as N
    from deeptables_b200.utils.partial_dependence import _BLOCK_ROWS
    groups, rows = 100, a.rows
    prob = torch.rand(groups * rows, 1, device='cuda')
    w = torch.rand(rows, dtype=torch.float64, device='cuda')
    nb = (rows + _BLOCK_ROWS - 1) // _BLOCK_ROWS
    out = torch.empty(groups * nb, dtype=torch.float64, device='cuda')
    for weight in (None, w):
        def run():
            N.check(N.lib.dtb_pdp_block_sums(N.ptr(prob), N.ptr(weight), groups, rows, 1, _BLOCK_ROWS, N.ptr(out),
                                             N.stream_ptr()), 'pdp_block_sums')
        t = events_time(run, 20)
        nbytes = prob.numel() * 4 + out.numel() * 8 + (rows * 8 if weight is not None else 0)
        print(json.dumps({'what': 'dtb_pdp_block_sums', 'groups': groups, 'rows': rows, 'cols': 1,
                          'weighted': weight is not None, 'kernel_ms': round(t * 1e3, 3),
                          'GB_per_s': round(nbytes / t / 1e9, 1),
                          'share_of_3.35TB_per_s': round(nbytes / t / 3.35e12, 3)}), flush=True)


if __name__ == '__main__':
    main()
