"""Time target encoding on the GPU against scikit-learn's TargetEncoder on the CPU.

    python tools/bench_target_encoding.py [--rows 1000000] [--big-rows 10000000] [--rounds 3] [--skip-sklearn]

Frames: `rows` x 26 int64 Zipf(1.2) columns with a binary target, the same at `big-rows`, and 4 string columns of the
first frame.  Each frame is timed for `fit_transform` (5 stratified folds, smooth='auto') and `transform`, end to end
(host clock around work that ends in a device synchronise) and split per stage with CUDA events by a staged copy of
the pipeline: host coding, sorts, statistics kernels, encodings, gather and the device-to-host copy of the output.
Each kernel's algorithmic bytes over its time are set against the data sheet's 3.35 TB/s of HBM3.  One JSON line per
frame; the card's name and power limit go with it.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deeptables_b200 import target_encoding as T  # noqa: E402
from deeptables_b200 import _native as N  # noqa: E402
from deeptables_b200._native import check, ptr, stream_ptr  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name()
    return q


def frame(rows, cols, seed=0, strings=False):
    g = np.random.default_rng(seed)
    data = {f'c{i}': np.minimum(g.zipf(1.2, rows), 10 ** 6).astype(np.int64) for i in range(cols)}
    X = pd.DataFrame(data)
    if strings:
        X = pd.DataFrame({k: pd.Series(v).map('v{}'.format) for k, v in list(data.items())[:4]})
    y = (g.random(rows) < 0.25).astype(np.int64)
    return X, y


class Stages:
    def __init__(self):
        self.t = {}
        self.bytes = {}

    def add(self, name, ms, nbytes=0):
        self.t[name] = self.t.get(name, 0.0) + ms
        self.bytes[name] = self.bytes.get(name, 0) + nbytes


def ev():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def staged_fit_transform(X, y, st):
    """The steps of TargetEncoder.fit_transform (binary target, smooth='auto', one column group), timed per stage."""
    from sklearn.model_selection import StratifiedKFold
    n = len(X)
    h0 = time.perf_counter()
    fold, folds = T.fold_ids(StratifiedKFold(5, shuffle=True, random_state=0).split(X, y), n)
    st.add('host folds', 1e3 * (time.perf_counter() - h0))
    target = T._Target(y, 2, None, fold, folds, T.TE_AUTO, 0.0, T._TILE_ROWS, True)
    G, n_out = target.groups, target.n_out
    dev, s = torch.device('cuda'), stream_ptr()
    prior = torch.empty(G, dtype=torch.float64, device=dev)
    out = torch.empty((n, X.shape[1]), dtype=torch.float64, device=dev)
    codes_l, tabs, cats_l = [], [], []
    for i in range(X.shape[1]):
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        codes, cats = T.code_column(X.iloc[:, i])
        torch.cuda.synchronize()
        st.add('coding', 1e3 * (time.perf_counter() - h0))
        V = len(cats)
        slots = V * folds * 2
        keys = torch.empty(n, dtype=torch.int64, device=dev)
        e0 = ev()
        check(N.lib.dtb_te_keys(ptr(codes), ptr(target.fold), ptr(target.cls), n, folds, 2, 0, ptr(keys), s),
              'keys')
        e1 = ev()
        keys, _ = torch.sort(keys, stable=True)
        e2 = ev()
        starts = torch.empty(slots + 1, dtype=torch.int64, device=dev)
        check(N.lib.dtb_te_segment_starts(ptr(keys), n, slots, ptr(starts), s), 'starts')
        e3 = ev()
        table = torch.empty(G * V, dtype=torch.float64, device=dev)
        ps, psum, pm2 = target.whole
        check(N.lib.dtb_te_encodings(ptr(starts), None, None, ptr(ps), None, None, V, folds, 2, T.TE_AUTO, 0.0,
                                     ptr(table), ptr(prior), s), 'encodings')
        e4 = ev()
        torch.cuda.synchronize()
        st.add('dtb_te_keys', e0.elapsed_time(e1), n * (4 + 1 + 4 + 8))
        st.add('sort', e1.elapsed_time(e2))
        st.add('dtb_te_segment_starts', e2.elapsed_time(e3), 8 * n + 8 * (slots + 1))
        st.add('dtb_te_encodings', e3.elapsed_time(e4), 8 * (G * (2 * V * folds) + G * V))
        codes_l.append(codes)
        tabs.append(table)
        cats_l.append(V)
    e0 = ev()
    T.gather(out, 0, codes_l, tabs, cats_l, prior, target.fold, n_out, folds)
    e1 = ev()
    host = out.cpu().numpy()
    e2 = ev()
    torch.cuda.synchronize()
    st.add('dtb_te_gather', e0.elapsed_time(e1), n * X.shape[1] * (4 + 8) + n)
    st.add('copy to host', e1.elapsed_time(e2), host.nbytes)
    return host


def timed(fn, rounds):
    ts = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return res, ts


def run(name, X, y, rounds, sklearn_too):
    from sklearn.model_selection import StratifiedKFold
    enc = T.TargetEncoder(cv=StratifiedKFold(5, shuffle=True, random_state=0))
    enc.fit_transform(X.iloc[:1000], y[:1000])                    # warm-up: module load, allocator
    out, t_ft = timed(lambda: enc.fit_transform(X, y), rounds)
    _, t_tr = timed(lambda: enc.transform(X), rounds)
    st = Stages()
    staged = staged_fit_transform(X, y, st)
    st = Stages()
    for _ in range(rounds):
        staged_fit_transform(X, y, st)
    res = {'frame': name, 'rows': len(X), 'cols': X.shape[1], 'card': card(), 'rounds': rounds,
           'fit_transform_s': [round(t, 3) for t in t_ft], 'transform_s': [round(t, 3) for t in t_tr],
           'staged_equals_encoder': bool(staged.tobytes() == out.tobytes()),
           'stages_ms': {k: round(v / rounds, 3) for k, v in st.t.items()}}
    res['kernel_hbm_share'] = {k: round(st.bytes[k] / (st.t[k] * 1e-3) / HBM_BYTES_PER_S, 3)
                               for k in st.t if st.bytes.get(k) and st.t[k] > 0}
    if sklearn_too:
        from sklearn.preprocessing import TargetEncoder as Sk
        sk = Sk(cv=StratifiedKFold(5, shuffle=True, random_state=0))
        t0 = time.perf_counter()
        want = sk.fit_transform(X, y)
        res['sklearn_fit_transform_s'] = round(time.perf_counter() - t0, 3)
        t0 = time.perf_counter()
        sk.transform(X)
        res['sklearn_transform_s'] = round(time.perf_counter() - t0, 3)
        res['max_abs_diff_vs_sklearn'] = float(np.max(np.abs(want - out)))
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=1_000_000)
    ap.add_argument('--big-rows', type=int, default=10_000_000)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--skip-sklearn', action='store_true')
    ap.add_argument('--out', default=None, help='also append the JSON lines to this file')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_target_encoding: no CUDA device')
    results = []
    X, y = frame(a.rows, 26)
    results.append(run(f'{a.rows} x 26 int Zipf(1.2)', X, y, a.rounds, not a.skip_sklearn))
    Xs, _ = frame(a.rows, 26, strings=True)
    results.append(run(f'{a.rows} x 4 strings', Xs, y, a.rounds, not a.skip_sklearn))
    if a.big_rows:
        Xb, yb = frame(a.big_rows, 26, seed=1)
        results.append(run(f'{a.big_rows} x 26 int Zipf(1.2)', Xb, yb, a.rounds, False))
    if a.out:
        with open(a.out, 'a') as f:
            for r in results:
                f.write(json.dumps(r) + '\n')


if __name__ == '__main__':
    main()
