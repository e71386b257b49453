"""Gradient-boosted leaf features on the GPU: each gbdt kernel exactly against the numpy restatement (tests/gbm_ref.py),
whole boosters against the restated booster, determinism, and apply_gbm_features end to end (DeepTable fit / predict /
evaluate / save / load, permutation importance, SHAP, data parallel)."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import gbm_ref as R

pytestmark = pytest.mark.gpu


def _features(rows, nf, seed, nan=False):
    """float32 features: every third an integer code, the rest continuous (some NaN)."""
    g = np.random.default_rng(seed)
    X = np.empty((rows, nf), np.float32)
    for j in range(nf):
        X[:, j] = g.integers(0, 3 + j % 40, rows) if j % 3 == 0 else g.normal(size=rows)
        if nan and j % 3 == 1:
            X[g.random(rows) < 0.1, j] = np.nan
    return X


def _split_inputs(X):
    """The device inputs of a booster over X: codes in an int32 cat tensor, the rest in cont, and the column map."""
    cat_cols = [j for j in range(X.shape[1]) if j % 3 == 0]
    cont_cols = [j for j in range(X.shape[1]) if j % 3 != 0]
    cat = torch.as_tensor(np.ascontiguousarray(X[:, cat_cols], np.int32)).cuda() if cat_cols else None
    cont = torch.as_tensor(np.ascontiguousarray(X[:, cont_cols])).cuda() if cont_cols else None
    feat_col = [cat_cols.index(j) if j in cat_cols else -1 - cont_cols.index(j) for j in range(X.shape[1])]
    return cat, cont, feat_col


def _booster(X, task, K, params):
    from deeptables_b200 import gbm
    p = gbm.resolve_params(params, task, K)
    edges = [gbm.bin_edges(X[:, j], p['max_bin']) for j in range(X.shape[1])]
    cat, cont, feat_col = _split_inputs(X)
    return gbm.Booster(p, task, K, feat_col, edges, torch.device('cuda')), p, edges, cat, cont, feat_col


@pytest.mark.parametrize('rows,nf', [(1, 1), (19, 39), (65537, 39), (1_000_000, 39), (3000, 300)])
def test_bins_and_histograms_equal_numpy(rows, nf):
    from deeptables_b200 import _native as N
    from deeptables_b200._native import ptr, stream_ptr
    X = _features(rows, nf, rows + nf, nan=True)
    b, p, edges, cat, cont, _ = _booster(X, 'binary', 1, {})
    bins = b.bin(cat, cont, rows)
    want = R.bins(X, edges)
    assert np.array_equal(bins.cpu().numpy(), want)
    g = np.random.default_rng(1)
    gq = g.integers(-2 ** 40, 2 ** 40, rows)
    hq = g.integers(0, 2 ** 40, rows)
    index = torch.as_tensor(g.permutation(rows).astype(np.int32)).cuda()
    gq_d, hq_d = torch.as_tensor(gq).cuda(), torch.as_tensor(hq).cuda()
    for begin, count in [(0, rows), (rows // 3, rows - rows // 3), (rows - 1, 1)]:
        out = [torch.empty(nf, b.nb, dtype=dt, device='cuda') for dt in (torch.int64, torch.int64, torch.int32)]
        N.check(N.lib.dtb_gbdt_hist(ptr(bins), ptr(index), begin, count, ptr(gq_d), ptr(hq_d), nf, b.nb, ptr(out[0]),
                                    ptr(out[1]), ptr(out[2]), stream_ptr()))
        sel = index.cpu().numpy()[begin:begin + count]
        G, H, C = R.histogram(want, sel, gq, hq, b.nb)
        assert np.array_equal(out[0].cpu().numpy(), G)
        assert np.array_equal(out[1].cpu().numpy(), H)
        assert np.array_equal(out[2].cpu().numpy(), C)


def test_partition_membership():
    from deeptables_b200 import _native as N
    from deeptables_b200._native import ptr, stream_ptr
    rows, nf = 50_000, 5
    X = _features(rows, nf, 4)
    b, p, edges, cat, cont, _ = _booster(X, 'binary', 1, {})
    bins = b.bin(cat, cont, rows)
    B = bins.cpu().numpy()
    index = torch.arange(rows, dtype=torch.int32, device='cuda')
    scratch = torch.empty(rows + 2, dtype=torch.int32, device='cuda')
    begin, count, f, t = 1000, 30_000, 1, 7
    seg = np.arange(begin, begin + count)
    left = int((B[seg, f] <= t).sum())
    N.check(N.lib.dtb_gbdt_partition(ptr(bins), nf, ptr(index), begin, count, f, t, left, ptr(scratch),
                                     stream_ptr()))
    out = index.cpu().numpy()
    assert np.array_equal(out[:begin], np.arange(begin)) and np.array_equal(out[begin + count:],
                                                                             np.arange(begin + count, rows))
    assert set(out[begin:begin + left]) == set(seg[B[seg, f] <= t])
    assert set(out[begin + left:begin + count]) == set(seg[B[seg, f] > t])


def _compare(trees, ref, what):
    """Identical structure and leaf values within 1e-6 relative; a flipped split prints both gains."""
    assert trees.n_trees == len(ref), f'{what}: {trees.n_trees} trees, restatement {len(ref)}'
    for t, r in enumerate(ref):
        a, b = trees.node_off[t], trees.node_off[t + 1]
        got = [trees.node_feature[a:b].tolist(), trees.node_bin[a:b].tolist(), trees.node_left[a:b].tolist(),
               trees.node_right[a:b].tolist()]
        want = [r['feature'], r['bin'], r['left'], r['right']]
        if got != want:
            raise AssertionError(f'{what}: tree {t} differs\n device  {got}\n  gains {trees.node_gain[a:b].tolist()}\n'
                                 f' numpy   {want}\n  gains {r["gain"]}')
        lv = trees.leaf_value[trees.leaf_off[t]:trees.leaf_off[t + 1]]
        np.testing.assert_allclose(lv, np.asarray(r['values'], np.float32), rtol=1e-6, atol=0, err_msg=what)


CASES = [('binary', 2, {}), ('regression', 1, {}), ('multiclass', 5, {}),
         ('binary', 2, {'num_leaves': 2}), ('binary', 2, {'num_leaves': 7, 'max_depth': 2}),
         ('regression', 1, {'num_leaves': 255, 'n_estimators': 5, 'min_child_samples': 5}),
         ('binary', 2, {'min_child_samples': 800}), ('regression', 1, {'reg_lambda': 3.0, 'reg_alpha': 0.5}),
         ('binary', 2, {'max_bin': 15}), ('multiclass', 5, {'max_bin': 15, 'num_leaves': 7})]


def _task_frame(task, K, rows=20_000, seed=0):
    X = _features(rows, 12, seed, nan=True)
    g = np.random.default_rng(seed + 1)
    z = np.nan_to_num(X[:, 1]) + (X[:, 0] == 2) - np.nan_to_num(X[:, 2]) * X[:, 5] + 0.5 * g.normal(size=rows)
    if task == 'binary':
        y = (z > 0.3).astype(np.float32)
    elif task == 'regression':
        y = (3 * z).astype(np.float32)
    else:
        y = np.digitize(z, np.quantile(z, np.linspace(0, 1, K + 1)[1:-1])).astype(np.float32)
    return X, y


@pytest.mark.parametrize('task,K,params', CASES)
def test_booster_equals_the_restatement(task, K, params):
    params = dict({'n_estimators': 20}, **params)
    X, y = _task_frame(task, K)
    b, p, edges, cat, cont, feat_col = _booster(X, task, K if task == 'multiclass' else None, params)
    log = torch.full((len(y), 200), -1, dtype=torch.int32, device='cuda')
    trees = b.fit(cat, cont, y, leaf_log=log)
    ref = R.fit(X, y, task, b.K, p, edges)
    _compare(trees, ref, f'{task} {params}')
    from deeptables_b200 import gbm
    out = torch.zeros(len(y), trees.n_trees, dtype=torch.int32, device='cuda')
    gbm.write_leaves(trees, feat_col, cat, cont, len(y), out_cat=out)
    leaves = out.cpu().numpy()
    for t, r in enumerate(ref):
        assert np.array_equal(leaves[:, t], R.traverse(r, X, edges)), f'tree {t}: traversal'
    assert np.array_equal(leaves, log[:, :trees.n_trees].cpu().numpy()), 'traversal differs from the partition'


def test_no_split_stops_boosting():
    X = _features(500, 4, 3)
    y = np.full(500, 2.5, np.float32)                       # constant target: zero gradients, no gain
    b, *_, cat, cont, _ = _booster(X, 'regression', None, {})
    assert b.fit(cat, cont, y).n_trees == 0
    X, y = _task_frame('binary', 2, rows=300)
    b, p, edges, cat, cont, _ = _booster(X, 'binary', None, {'min_child_samples': 140, 'n_estimators': 50})
    trees = b.fit(cat, cont, y)
    ref = R.fit(X, y, 'binary', 1, p, edges)
    _compare(trees, ref, 'min_child_samples=140')


def test_two_fits_are_bit_identical():
    X, y = _task_frame('multiclass', 5, rows=30_000, seed=9)
    runs = []
    for _ in range(2):
        b, *_, cat, cont, _ = _booster(X, 'multiclass', 5, {'n_estimators': 6})
        runs.append(b.fit(cat, cont, y).arrays())
    for k in runs[0]:
        assert np.array_equal(runs[0][k], runs[1][k]), k


def _frame(task, rows, seed):
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'c{i}': g.choice(list('abcdef')[:3 + i], rows) for i in range(3)})
    for i in range(4):
        X[f'n{i}'] = g.normal(size=rows)
    lead = (X['c0'] == 'a') * 1.5 + X['n0'] - X['n1'] * (X['c1'] == 'b')
    if task == 'binary':
        y = np.where(lead + 0.3 * g.normal(size=rows) > 0.5, 'yes', 'no')
    elif task == 'multiclass':
        y = np.digitize(lead + 0.3 * g.normal(size=rows), [-0.5, 0.5, 1.5])
    else:
        y = 2.0 * lead + 0.1 * g.normal(size=rows)
    return X, pd.Series(y)


_CACHE = {}


def _fitted(task, feature_type):
    key = (task, feature_type)
    if key not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        X, y = _frame(task, 2600, 5)
        conf = deeptable.ModelConfig(nets=deepnets.DeepFM, metrics=['accuracy' if task != 'regression' else 'mse'],
                                     embeddings_output_dim=4, earlystopping_patience=1, apply_gbm_features=True,
                                     gbm_feature_type=feature_type, gbm_params={'n_estimators': 8, 'num_leaves': 7})
        dt = deeptable.DeepTable(config=conf)
        dt.fit(X.iloc[:2000], y.iloc[:2000], epochs=2, batch_size=128, verbose=0)
        _CACHE[key] = (dt, X.iloc[2000:].reset_index(drop=True), y.iloc[2000:].reset_index(drop=True))
    return _CACHE[key]


@pytest.mark.parametrize('task', ['binary', 'regression', 'multiclass'])
@pytest.mark.parametrize('feature_type', ['embedding', 'dense'])
def test_end_to_end_fit_predict_evaluate_save_load(task, feature_type, tmp_path):
    from deeptables_b200 import deeptable
    dt, X, y = _fitted(task, feature_type)
    pre = dt.preprocessor
    enc = pre.gbm_encoder_
    T = enc.trees.n_trees
    assert T > 0 and enc.new_columns == [f'lgbm_leaf_{i}' for i in range(T)]
    desc = str(dt.get_model().model_desc)
    if feature_type == 'embedding':
        leaf_cols = [c for c in pre.categorical_columns if c.name.startswith('lgbm_leaf_')]
        assert [c.vocabulary_size for c in leaf_cols] == enc.trees.num_leaves.tolist()
        Xt = pre.transform_X(X)
        assert all(Xt[c.name].max() < c.vocabulary_size for c in leaf_cols)
        assert f'all_categorical_vars: ({len(pre.categorical_columns)})' in desc
    else:
        assert pre.continuous_columns[-1].name == 'input_continuous_gbm_leaves'
        assert pre.continuous_columns[-1].column_names == enc.new_columns
        assert 'input_continuous_gbm_leaves' in desc
    proba = dt.predict_proba(X)
    assert np.all(np.isfinite(proba))
    dt.evaluate(X, y)
    dt.save(str(tmp_path / 'm'))
    dt2 = deeptable.DeepTable.load(str(tmp_path / 'm'))
    assert np.array_equal(dt2.predict_proba(X), proba)


def test_permutation_importance_equals_the_host_loop():
    """Accuracy, exactly: the device passes against the same permutations applied to the raw DataFrame column."""
    from deeptables_b200 import importance
    from deeptables_b200.utils.feature_importance import get_score_importances
    from importance_ref import permutation
    dt, X, y = _fitted('multiclass', 'embedding')
    seed = 11
    got = importance.score_decreases(dt, X, y, 'accuracy', n_iter=2, random_state=seed, batch_size=97)
    assert got.columns == X.columns.to_list()
    base = np.mean(dt.predict(X) == np.asarray(y))
    for it in range(2):
        for j, c in enumerate(X.columns):
            Xp = X.copy()
            Xp[c] = X[c].to_numpy()[permutation(seed, it, j, len(X))]
            want = np.mean(dt.predict(Xp) == np.asarray(y))
            assert got.decreases[it, j] == -base - (-want), (it, c)
    assert get_score_importances(dt, X, y, 'accuracy', n_iter=1, random_state=3).shape == (X.shape[1], 2)


@pytest.mark.parametrize('feature_type', ['embedding', 'dense'])
def test_shap_coalition_values_equal_model_fn_on_composed_frames(feature_type):
    from deeptables_b200 import explain
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X, _ = _fitted('binary', feature_type)
    columns = X.columns.to_list()
    bg = X.iloc[:25].reset_index(drop=True)
    ex = DeepTablesExplainer(dt, bg, num_samples=None, random_state=0)
    x = X.iloc[100:102].reset_index(drop=True)
    trace = {}
    phi = explain.shap_values(ex._background, x, 30, 3, 65536, trace=trace)
    assert phi.shape == (2, len(columns))
    for i in range(2):
        r = trace[i]
        for pk in [0, 1, len(r.masks) // 2, len(r.masks) - 1]:
            S = [r.varying[k] for k in np.flatnonzero(r.masks[pk])]
            f = bg.copy()
            for j in S:
                f[columns[j]] = x.iloc[i][columns[j]]
            want = np.mean(np.asarray(ex.model_fn(f.to_numpy(dtype=object)), np.float64))
            assert r.values[pk] == pytest.approx(want, abs=1e-12)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, backend, data, out_dir):
    import torch.distributed as dist
    from deeptables_b200 import deeptable
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    kw = {'device_id': torch.device('cuda', rank)} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        X, y = pd.read_pickle(data)
        conf = deeptable.ModelConfig(apply_gbm_features=True, gbm_params={'n_estimators': 5}, task='binary')
        pre = deeptable.DefaultPreprocessor(conf)
        Xt, _ = pre.fit_transform(X, y)
        np.savez(os.path.join(out_dir, f'trees{rank}.npz'), **pre.gbm_encoder_.trees.arrays(),
                 leaves=Xt[pre.gbm_encoder_.new_columns].to_numpy())
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_data_parallel_ranks_have_identical_trees(tmp_path, backend):
    """World size 2; over gloo both ranks may share one GPU."""
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    X, y = _frame('binary', 3000, 2)
    pd.to_pickle((X, y), str(tmp_path / 'data.pkl'))
    mp.spawn(_dp_worker, args=(2, _free_port(), backend, str(tmp_path / 'data.pkl'), str(tmp_path)), nprocs=2,
             join=True)
    a, b = np.load(tmp_path / 'trees0.npz'), np.load(tmp_path / 'trees1.npz')
    assert a.files == b.files
    for k in a.files:
        assert np.array_equal(a[k], b[k]), k
