"""Benchmark of the gradient-boosted leaf features (deeptables_b200/gbm.py, csrc/gbdt.cu) on a Criteo-shaped frame:
26 categorical + 13 continuous columns, a label that depends on several of them, the default booster parameters.

    python tools/bench_gbm.py [--rows 1000000] [--out FILE]

Prints, with the card's name and power limit:
- the booster fit on the encoded device inputs, split into bin / grad / hist / split / partition / update (CUDA events
  around each launch, in a second fit) and the host's share;
- the histogram kernel on the root (all rows) over 20 launches: bytes/s of the algorithmic bytes, the feature bins, the
  row index and the two int64 fixed-point values per row;
- dtb_gbdt_leaves rows/s for the fitted trees (100 at the defaults);
- DefaultPreprocessor.fit_transform seconds with and without apply_gbm_features;
- the CPU baseline: scikit-learn's HistGradientBoostingClassifier with matched parameters.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def frame(rows, seed=0):
    g = np.random.default_rng(seed)
    vocab = [1460, 583, 10131227, 2202608, 305, 24, 12517, 633, 3, 93145, 5683, 8351593, 3194, 27, 14992, 5461306, 10,
             5652, 2173, 4, 7046547, 18, 15, 286181, 105, 142572]
    X = pd.DataFrame({f'C{i + 1}': g.integers(0, min(v, rows // 4 + 2), rows).astype(str) for i, v in enumerate(vocab)})
    for i in range(13):
        X[f'I{i + 1}'] = np.where(g.random(rows) < 0.05, np.nan, np.round(g.exponential(size=rows) * 10 ** (i % 3), 0))
    z = (X['C9'] == '1') * 1.0 + np.log1p(X['I1'].fillna(0)) * 0.5 - (X['C20'] == '2') * 0.7 + \
        np.log1p(X['I5'].fillna(0)) * (X['C14'].astype(int) % 3 == 0) * 0.3 + g.normal(size=rows)
    y = (z > np.quantile(z, 0.75)).astype(np.int64)
    return X, y


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:        # the numbers are still printed; the card is then unknown
        return f'unknown ({e})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=1_000_000)
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-sklearn', action='store_true')
    args = ap.parse_args()
    import torch
    from deeptables_b200 import _native as N, deeptable, gbm
    from deeptables_b200._native import ptr, stream_ptr
    if not torch.cuda.is_available():
        raise SystemExit('bench_gbm needs a GPU')
    res = {'card': card(), 'rows': args.rows}
    X, y = frame(args.rows)

    t0 = time.perf_counter()
    pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig())
    Xt, yt = pre.fit_transform(X, y)
    res['preprocess_s_without'] = time.perf_counter() - t0
    t0 = time.perf_counter()
    pre_g = deeptable.DefaultPreprocessor(deeptable.ModelConfig(apply_gbm_features=True))
    pre_g.fit_transform(X, y)
    torch.cuda.synchronize()
    res['preprocess_s_with'] = time.perf_counter() - t0

    enc = gbm.GbmLeavesEncoder(pre._cat_names, pre._cont_names, 'binary')
    p = gbm.resolve_params({}, 'binary')
    cat_np, cont_np = enc._arrays(Xt)
    sample = gbm.sample_rows(len(Xt), p['subsample_for_bin'], p['random_state'])
    cols = [cat_np[sample, j].astype(np.float32) for j in range(cat_np.shape[1])] + \
           [cont_np[sample, j] for j in range(cont_np.shape[1])]
    edges = [gbm.bin_edges(v, p['max_bin']) for v in cols]
    cat, cont = torch.as_tensor(cat_np).cuda(), torch.as_tensor(cont_np).cuda()
    dev = torch.device('cuda')
    label = np.asarray(yt)
    gbm.Booster(dict(p, n_estimators=2), 'binary', 2, enc.feat_col, edges, dev).fit(cat, cont, label)   # warm-up
    booster = gbm.Booster(p, 'binary', 2, enc.feat_col, edges, dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    trees = booster.fit(cat, cont, label)
    torch.cuda.synchronize()
    res['fit_s'] = time.perf_counter() - t0
    res['trees'] = trees.n_trees
    stages = {}
    booster.fit(cat, cont, label, stages=stages)
    res['fit_stages_s'] = stages
    res['fit_host_and_sync_s'] = res['fit_s'] - sum(stages.values())

    nf, rows = booster.nf, args.rows
    bins = booster.bin(cat, cont, rows)
    index = torch.as_tensor(np.random.default_rng(0).permutation(rows).astype(np.int32)).cuda()
    gq = torch.randint(-2 ** 40, 2 ** 40, (rows,), dtype=torch.int64, device='cuda')
    hq = torch.randint(0, 2 ** 40, (rows,), dtype=torch.int64, device='cuda')
    out = [torch.empty(nf, booster.nb, dtype=d, device='cuda') for d in (torch.int64, torch.int64, torch.int32)]

    def hist():
        N.check(N.lib.dtb_gbdt_hist(ptr(bins), ptr(index), 0, rows, ptr(gq), ptr(hq), nf, booster.nb, ptr(out[0]),
                                    ptr(out[1]), ptr(out[2]), stream_ptr()))
    for _ in range(3):
        hist()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(20):
        hist()
    e.record()
    e.synchronize()
    t_hist = s.elapsed_time(e) / 1e3 / 20
    algo = rows * (nf + 4 + 16)
    res['hist_root_ms'] = t_hist * 1e3
    res['hist_algorithmic_GBps'] = algo / t_hist / 1e9

    leaves = torch.empty(rows, max(trees.n_trees, 1), dtype=torch.int32, device='cuda')
    gbm.write_leaves(trees, enc.feat_col, cat, cont, rows, out_cat=leaves)
    s.record()
    for _ in range(5):
        gbm.write_leaves(trees, enc.feat_col, cat, cont, rows, out_cat=leaves)
    e.record()
    e.synchronize()
    res['leaves_rows_per_s'] = rows / (s.elapsed_time(e) / 1e3 / 5)

    if not args.skip_sklearn:
        from sklearn.ensemble import HistGradientBoostingClassifier
        Xs = np.concatenate([cat_np.astype(np.float32), cont_np], axis=1)
        t0 = time.perf_counter()
        HistGradientBoostingClassifier(max_iter=100, max_leaf_nodes=31, min_samples_leaf=20, l2_regularization=0,
                                       max_bins=255, early_stopping=False).fit(Xs, label)
        res['sklearn_cpu_fit_s'] = time.perf_counter() - t0
        res['cpu_count'] = os.cpu_count()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
