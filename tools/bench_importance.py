"""Throughput of permutation feature importance (deeptables_b200/utils/feature_importance.py) on one GPU.

A Criteo-shaped frame (13 continuous, 26 categorical columns of 1 000 values each) with a synthetic binary label; the
model is fitted for one epoch on 100 000 rows.  Then ``get_score_importances(metric='auc', n_iter=1)`` on 1 000 000 rows:
DeepFM at 8 192-row batches and xDeepFM at 65 536 (bench.py's two workloads), 39 shuffled passes plus the base pass.
The call's time includes encoding the frame with the preprocessor, which is timed on its own and subtracted for the
pass rate.  For comparison, the naive host loop (shuffle the DataFrame column with numpy, ``predict_proba``,
scikit-learn's ``roc_auc_score``) is timed on 100 000 rows for a few columns, against the device path at that size.

    python tools/bench_importance.py [--rounds 2] [--rows 1000000]

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

from bench_optim import card  # noqa: E402

N_CONT, N_CAT, VOCAB = 13, 26, 1000


def frame(rows, seed):
    import numpy as np
    import pandas as pd
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'I{i}': g.normal(size=rows).astype(np.float32) for i in range(N_CONT)})
    for i in range(N_CAT):
        X[f'C{i}'] = g.integers(0, VOCAB, rows)
    logit = X['I0'].values + (X['C0'].values % 7 == 0) * 2.0 - 0.5
    y = (logit + g.normal(size=rows) > 0).astype(np.int64)
    return X, y


def fitted(nets, X, y):
    from deeptables_b200 import deepnets, deeptable
    conf = deeptable.ModelConfig(nets=getattr(deepnets, nets), metrics=['AUC'], embeddings_output_dim=16,
                                 categorical_columns=[f'C{i}' for i in range(N_CAT)], earlystopping_patience=1)
    dt = deeptable.DeepTable(config=conf)
    dt.fit(X.iloc[:100_000], y[:100_000], epochs=1, batch_size=8192, verbose=0, validation_split=0.1)
    return dt


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
    ap.add_argument('--host-rows', type=int, default=100_000)
    ap.add_argument('--host-columns', type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    from sklearn.metrics import roc_auc_score
    from deeptables_b200 import importance
    from deeptables_b200.utils.feature_importance import get_score_importances
    if not torch.cuda.is_available():
        sys.exit('bench_importance needs a CUDA device')
    print(json.dumps(card()), flush=True)
    X, y = frame(a.rows, 0)
    n_cols = X.shape[1]
    for nets, bs in (('DeepFM', 8192), ('xDeepFM', 65536)):
        dt = fitted(nets, X, y)
        get_score_importances(dt, X.iloc[:20_000], y[:20_000], 'auc', 1, mode='max', random_state=0, batch_size=bs)
        enc = statistics.median(timed(lambda: dt.preprocessor.transform_X(X))[0] for _ in range(a.rounds))
        totals = []
        for r in range(a.rounds):
            t, res = timed(lambda: importance.score_decreases(dt, X, y, 'auc', n_iter=1, mode='max', random_state=r,
                                                              batch_size=bs))
            totals.append(t)
        total = statistics.median(totals)
        passes = res.passes + 1
        print(json.dumps({'what': 'device', 'nets': nets, 'batch_size': bs, 'rows': a.rows, 'columns': n_cols,
                          'passes': passes, 'call_s': round(total, 3), 'encode_s': round(enc, 3),
                          'passes_per_s': round(passes / (total - enc), 2),
                          'rows_per_s': round(passes * a.rows / (total - enc), 0), 'rounds': a.rounds}), flush=True)
        if nets != 'DeepFM':
            continue
        Xh, yh = X.iloc[:a.host_rows], y[:a.host_rows]
        t_dev = statistics.median(timed(lambda: importance.score_decreases(
            dt, Xh, yh, 'auc', n_iter=1, mode='max', random_state=r, batch_size=bs))[0] for r in range(a.rounds))
        rng = np.random.default_rng(0)

        def host_pass(c):
            Xs = Xh.copy()
            Xs[c] = rng.permutation(Xh[c].values)
            return roc_auc_score(yh, dt.predict_proba(Xs, batch_size=bs)[:, 1])
        host_pass(X.columns[0])
        per_pass = statistics.median(timed(lambda c=c: host_pass(c))[0] for c in X.columns[:a.host_columns])
        print(json.dumps({'what': 'host loop vs device', 'nets': nets, 'batch_size': bs, 'rows': a.host_rows,
                          'host_s_per_pass': round(per_pass, 3), 'host_call_s_projected': round(per_pass * (n_cols + 1), 2),
                          'device_call_s': round(t_dev, 3), 'host_passes_timed': a.host_columns,
                          'rounds': a.rounds}), flush=True)


if __name__ == '__main__':
    main()
