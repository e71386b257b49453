"""Throughput of Kernel SHAP (deeptables_b200/utils/shap.py) on one GPU.

Two cases, nsamples='auto':
- DeepFM on a 16-column bank-shaped frame (7 numeric, 9 categorical columns) with 100 background rows: the reference
  notebook's case.
- xDeepFM on the 39-column Criteo-shaped frame (13 continuous, 26 categorical columns) with 50 background rows.
Each model is fitted for one epoch on 20 000 rows.  For each case: explained rows per second, and the time split into
host sampling, dtb_shap_compose, forward, dtb_shap_means and solve (device stages timed with CUDA events).  For
comparison, the reference's host loop on one row: the synthetic rows composed with pandas for the same coalitions, then
``model_fn`` (``predict``).

    python tools/bench_shap.py [--rows 64] [--rounds 2]

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


def bank_frame(rows, seed):
    import numpy as np
    import pandas as pd
    g = np.random.default_rng(seed)
    cats = {'job': 12, 'marital': 3, 'education': 4, 'default': 2, 'housing': 2, 'loan': 2, 'contact': 3,
            'month': 12, 'poutcome': 4}
    X = pd.DataFrame({'age': g.integers(18, 95, rows), 'balance': g.normal(1400, 3000, rows).round(),
                      'day': g.integers(1, 32, rows), 'duration': g.exponential(260, rows).round(),
                      'campaign': g.integers(1, 20, rows), 'pdays': g.integers(-1, 400, rows),
                      'previous': g.integers(0, 10, rows)})
    for c, v in cats.items():
        X[c] = np.array([f'{c}_{i}' for i in range(v)])[g.integers(0, v, rows)]
    logit = X['duration'].values / 300 - 1.5 + (X['poutcome'] == 'poutcome_0') * 1.5
    y = np.where(logit + g.normal(size=rows) > 0, 'yes', 'no')
    return X[['age', 'job', 'marital', 'education', 'default', 'balance', 'housing', 'loan', 'contact', 'day', 'month',
              'duration', 'campaign', 'pdays', 'previous', 'poutcome']], y


def criteo_frame(rows, seed):
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    from bench_importance import frame
    return frame(rows, seed)


def fitted(nets, X, y, **conf):
    from deeptables_b200 import deepnets, deeptable
    dt = deeptable.DeepTable(config=deeptable.ModelConfig(nets=getattr(deepnets, nets), metrics=['AUC'],
                                                          earlystopping_patience=1, **conf))
    dt.fit(X, y, epochs=1, batch_size=1024, verbose=0)
    return dt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=64, help='explained rows per call')
    ap.add_argument('--rounds', type=int, default=2)
    a = ap.parse_args()
    import numpy as np
    import pandas as pd
    import torch
    from deeptables_b200 import explain
    from deeptables_b200.utils.shap import DeepTablesExplainer
    if not torch.cuda.is_available():
        sys.exit('bench_shap needs a CUDA device')
    print(json.dumps(card()), flush=True)
    cases = [('DeepFM', 'bank', bank_frame, 100, 65536, {'embeddings_output_dim': 4}),
             ('xDeepFM', 'criteo', criteo_frame, 50, 65536,
              {'embeddings_output_dim': 16, 'categorical_columns': [f'C{i}' for i in range(26)]})]
    for nets, name, make, n_bg, bs, conf in cases:
        X, y = make(20_000 + 1000, 0)
        dt = fitted(nets, X.iloc[:20_000], y[:20_000], **conf)
        Xe = X.iloc[20_000:].reset_index(drop=True)
        ex = DeepTablesExplainer(dt, Xe.iloc[a.rows:], num_samples=n_bg, random_state=0, batch_size=bs)
        ex.get_shap_values(Xe.iloc[:2])                                   # warm-up
        totals, splits = [], []
        for r in range(a.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            explain.shap_values(ex._background, Xe.iloc[:a.rows], 'auto', r, bs)
            torch.cuda.synchronize()
            totals.append(time.perf_counter() - t0)
            st = {}
            explain.shap_values(ex._background, Xe.iloc[:a.rows], 'auto', r, bs, stages=st)
            splits.append(st)
        total = statistics.median(totals)
        split = {k: round(statistics.median(s[k] for s in splits), 4) for k in splits[0]}
        trace = {}
        explain.shap_values(ex._background, Xe.iloc[:1], 'auto', 0, bs, trace=trace)
        print(json.dumps({'what': 'device', 'nets': nets, 'frame': name, 'columns': X.shape[1], 'background': n_bg,
                          'explained_rows': a.rows, 'coalitions_row0': len(trace[0].masks), 'call_s': round(total, 3),
                          'rows_per_s': round(a.rows / total, 2), 'split_s': split, 'rounds': a.rounds}), flush=True)

        # the reference's host path on one row: pandas composition of the same coalitions, then model_fn (predict)
        r0 = trace[0]
        bg = pd.DataFrame({c: v for c, v in zip(ex._background.columns, ex._background.values)})
        x = Xe.iloc[0]

        def host_row():
            parts = []
            for m in r0.masks:
                f = bg.copy()
                for j in r0.varying[m]:
                    f[X.columns[j]] = x.iloc[j]
                parts.append(f)
            t1 = time.perf_counter()
            big = pd.concat(parts, ignore_index=True).to_numpy(dtype=object)
            t2 = time.perf_counter()
            ex.model_fn(big)
            return t2 - t1, time.perf_counter() - t2
        t0 = time.perf_counter()
        _, t_pred = host_row()
        t_host = time.perf_counter() - t0
        print(json.dumps({'what': 'host model_fn loop, one row', 'nets': nets, 'frame': name,
                          'synthetic_rows': len(r0.masks) * n_bg, 'compose_s': round(t_host - t_pred, 3),
                          'model_fn_s': round(t_pred, 3), 'total_s': round(t_host, 3),
                          'device_s_per_row': round(total / a.rows, 4)}), flush=True)


if __name__ == '__main__':
    main()
