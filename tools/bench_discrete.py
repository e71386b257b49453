"""Benchmark of the quantile-bin columns of auto_discrete (deeptables_b200/discrete.py, csrc/discrete.cu) on a
Criteo-shaped frame: 26 categorical columns and 13 N(0,1) continuous ones, so each continuous column has about 10^6
distinct values and 10^5 bins (13 columns of 10^5 float64 edges: 10 MB, searched from L2).

    python tools/bench_discrete.py [--rows 1000000] [--out FILE]

Prints one JSON line, with the card's name and power limit:
- the device fit of the 13 columns (one sort, the order statistics, the host interpolation);
- dtb_discretize alone: CUDA events over 100 graph-replayed launches, GB/s of the algorithmic bytes (a float32 read
  and an int32 write per element), beside the least time HBM would need for them at the data sheet's 3.35 TB/s and
  the float64 edge loads the binary searches make;
- DefaultPreprocessor.transform_X seconds with the option on and off;
- one get_score_importances call (accuracy, n_iter=1) on a DeepFM fitted with the option on and off;
- the CPU baseline: scikit-learn's KBinsDiscretizer fit and transform on the same float64 columns.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import pandas as pd

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:        # the numbers are still printed; the card is then unknown
        return f'unknown ({e})'


def frame(rows, seed=0):
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'C{i + 1}': g.integers(0, 10 ** (1 + i % 4), rows).astype(str) for i in range(26)})
    for i in range(13):
        X[f'I{i + 1}'] = g.normal(size=rows)
    z = (X['C2'] == '1') * 1.0 + X['I1'] * 0.8 - (X['I2'] > 0.5) * 0.7 + g.normal(size=rows)
    y = (z > np.quantile(z, 0.75)).astype(np.int64)
    return X, y


def synced(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=1_000_000)
    ap.add_argument('--train-rows', type=int, default=200_000)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    from deeptables_b200 import deepnets, deeptable
    from deeptables_b200.discrete import MultiKBinsDiscretizer
    from deeptables_b200.utils.feature_importance import get_score_importances
    if not torch.cuda.is_available():
        raise SystemExit('bench_discrete needs a GPU')
    res = {'card': card(), 'rows': args.rows}
    X, y = frame(args.rows)
    pre_off = deeptable.DefaultPreprocessor(deeptable.ModelConfig())
    Xt, _ = pre_off.fit_transform(X, y)
    conts = pre_off._cont_names
    assert len(conts) == 13

    MultiKBinsDiscretizer(conts).fit(Xt.iloc[:1000])                                  # warm-up
    res['fit_s'], disc = synced(lambda: MultiKBinsDiscretizer(conts).fit(Xt))
    res['n_bins'] = [int(b) for b in disc.n_bins]
    res['edge_MB'] = disc._edges.nbytes / 1e6

    rows, C = args.rows, len(conts)
    cont = torch.as_tensor(np.ascontiguousarray(Xt[conts].to_numpy(np.float32))).cuda()
    out = torch.empty(rows, C, dtype=torch.int32, device='cuda')
    disc.write_device(out, cont, 0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        disc.write_device(out, cont, 0)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        disc.write_device(out, cont, 0)
    for _ in range(5):
        graph.replay()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(100):
        graph.replay()
    e.record()
    e.synchronize()
    t = s.elapsed_time(e) / 1e3 / 100
    algo = rows * C * 8
    res['kernel_ms'] = t * 1e3
    res['kernel_algorithmic_GBps'] = algo / t / 1e9
    res['kernel_hbm_bound_ms'] = algo / HBM_BYTES_PER_S * 1e3
    probes = sum(math.ceil(math.log2(len(b) - 1)) if len(b) > 2 else 0 for b in disc.bin_edges)
    res['search_edge_loads_per_row'] = probes
    res['search_edge_GBps'] = rows * probes * 8 / t / 1e9
    res['bound'] = 'search (L2 / load latency)' if t > 2 * algo / HBM_BYTES_PER_S else 'HBM'
    codes = out.cpu().numpy()
    for j in (0, C - 1):
        want = np.searchsorted(disc.bin_edges[j][1:-1], Xt[conts[j]].to_numpy(np.float32).astype(np.float64),
                               side='right')
        assert np.array_equal(codes[:, j], want), j

    pre_on = deeptable.DefaultPreprocessor(deeptable.ModelConfig(auto_discrete=True))
    pre_on.fit_transform(X, y)
    pre_on.transform_X(X.iloc[:1000])
    res['transform_X_s_off'], _ = synced(lambda: pre_off.transform_X(X))
    res['transform_X_s_on'], _ = synced(lambda: pre_on.transform_X(X))

    for name, on in (('off', False), ('on', True)):
        conf = deeptable.ModelConfig(nets=deepnets.DeepFM, auto_discrete=on, earlystopping_patience=1)
        dt = deeptable.DeepTable(config=conf)
        dt.fit(X.iloc[:args.train_rows], y[:args.train_rows], epochs=1, batch_size=4096, verbose=0)
        get_score_importances(dt, X.iloc[:10_000], y[:10_000], 'accuracy', n_iter=1, random_state=0)   # warm-up
        res[f'importance_s_{name}'], _ = synced(
            lambda: get_score_importances(dt, X, y, 'accuracy', n_iter=1, random_state=0))

    from sklearn.preprocessing import KBinsDiscretizer
    Xs = Xt[conts].to_numpy(np.float32).astype(np.float64)
    sk = KBinsDiscretizer(disc.n_bins, encode='ordinal', strategy='quantile', quantile_method='averaged_inverted_cdf',
                          subsample=None)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        t0 = time.perf_counter()
        sk.fit(Xs)
        res['sklearn_cpu_fit_s'] = time.perf_counter() - t0
        t0 = time.perf_counter()
        sk.transform(Xs)
        res['sklearn_cpu_transform_s'] = time.perf_counter() - t0
    res['cpu_count'] = os.cpu_count()
    res['edges_equal_sklearn'] = all(np.array_equal(a, b) for a, b in zip(disc.bin_edges, sk.bin_edges_))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
