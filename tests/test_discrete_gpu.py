"""auto_discrete on the GPU: dtb_discretize exactly against scikit-learn's KBinsDiscretizer.transform, the device fit
against the scikit-learn oracle bit for bit, and the option end to end (fit / predict / evaluate / save / load, with
gradient-boosted leaves, permutation importance, SHAP coalitions, data parallel)."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import discrete_ref as R

pytestmark = pytest.mark.gpu


def _disc(columns, edges):
    """A discretiser holding the given (oracle) bin edges."""
    from deeptables_b200.discrete import MultiKBinsDiscretizer
    d = MultiKBinsDiscretizer(columns)
    d.bin_edges = [np.asarray(e, np.float64) for e in edges]
    d.n_bins = np.array([len(e) - 1 for e in edges], np.int64)
    d._stage()
    return d


def _kernel_case(kind):
    g = np.random.default_rng(len(kind))
    n = {'one_row': 1, 'odd_rows': 1_000_003, 'many_bins': 1_000_000}.get(kind, 20_011)
    if kind == 'ties':
        fit = np.minimum(g.zipf(1.4, n), 50).astype(np.float32)
    elif kind == 'signed_zero':
        fit = g.choice([-0.0, 0.0, -1.5, 1.5, 3.0], n).astype(np.float32)
    elif kind == 'two':
        fit = g.choice([0.25, 0.75], n).astype(np.float32)
    elif kind == 'const':
        fit = np.full(n, 3.5, np.float32)
    else:
        fit = g.normal(size=n).astype(np.float32)
    nb = 100_000 if kind == 'many_bins' else R.n_bins(fit)
    e = R.edges(fit, nb)
    x = fit.copy()
    if kind not in ('one_row', 'const'):                      # values exactly on the edges, and both zeros
        inner = e[1:-1].astype(np.float32)
        on = inner[inner.astype(np.float64) == e[1:-1]]
        x[:len(on)] = on[:n]
        x[len(on):len(on) + 2] = [-0.0, 0.0]
    if kind == 'many_bins':
        assert len(e) - 1 > 90_000
    return fit, x, nb, e


@pytest.mark.parametrize('kind', ['ties', 'signed_zero', 'two', 'const', 'one_row', 'odd_rows', 'many_bins',
                                  'normal'])
def test_kernel_codes_equal_kbins_transform(kind):
    fit, x, nb, e = _kernel_case(kind)
    d = _disc(['a', 'b'], [e, R.edges(fit[::-1].copy() * 2, 7)])
    frame = pd.DataFrame({'a': x, 'b': x * 2})
    got = d.codes(frame)
    assert got.dtype == np.int32
    assert np.array_equal(got[:, 0], R.codes(e, x))
    assert np.array_equal(got[:, 1], R.codes(d.bin_edges[1], x * 2))
    assert np.array_equal(got[:, 0], R.kbins(fit, nb).transform(x.astype(np.float64)[:, None])[:, 0])


def test_kernel_reads_src_col_and_writes_only_its_columns():
    from deeptables_b200 import _native as N
    from deeptables_b200._native import ptr, stream_ptr
    g = np.random.default_rng(5)
    rows = 4097
    cont = g.normal(size=(rows, 5)).astype(np.float32)
    edges = [R.edges(cont[:, j], 20 + j) for j in range(5)]
    d = _disc([f'c{j}' for j in range(5)], edges)
    src = torch.tensor([4, 0, 2], dtype=torch.int32, device='cuda')
    inner = [edges[j][1:-1] for j in (4, 0, 2)]
    flat = torch.as_tensor(np.concatenate(inner)).cuda()
    off = torch.as_tensor(np.cumsum([0] + [len(i) for i in inner]).astype(np.int64)).cuda()
    out = torch.full((rows, 7), -7, dtype=torch.int32, device='cuda')
    cont_d = torch.as_tensor(cont).cuda()
    N.check(N.lib.dtb_discretize(ptr(cont_d), 5, rows, ptr(src), ptr(flat), ptr(off), 3, ptr(out), 7, 2,
                                 stream_ptr()))
    o = out.cpu().numpy()
    assert np.all(o[:, :2] == -7) and np.all(o[:, 5:] == -7)
    for k, j in enumerate((4, 0, 2)):
        assert np.array_equal(o[:, 2 + k], R.codes(edges[j], cont[:, j]))
    assert np.array_equal(d.codes(pd.DataFrame(cont, columns=d.columns)),
                          np.stack([R.codes(edges[j], cont[:, j]) for j in range(5)], 1))
    with pytest.raises(RuntimeError, match='bad shape'):
        N.check(N.lib.dtb_discretize(ptr(cont_d), 5, rows, ptr(src), ptr(flat), ptr(off), 3, ptr(out), 7, 5,
                                     stream_ptr()))


@pytest.mark.parametrize('rows', [1, 3, 1000, 200_001])
def test_device_fit_equals_the_oracle(rows):
    from deeptables_b200.discrete import MultiKBinsDiscretizer
    g = np.random.default_rng(rows)
    frame = pd.DataFrame({
        'random': g.normal(size=rows).astype(np.float32),
        'zipf': (np.minimum(g.zipf(1.5, rows), 5000) * 0.1).astype(np.float32),
        'integers': g.integers(-50, 3000, rows).astype(np.float32),
        'scaled': ((lambda v: (v - v.min()) / (np.ptp(v) or 1.0))(g.lognormal(size=rows))).astype(np.float32),
        'signed_zero': g.choice([-0.0, 0.0, 2.0], rows).astype(np.float32)})
    d = MultiKBinsDiscretizer(frame.columns).fit(frame)
    for j, c in enumerate(frame.columns):
        col = frame[c].to_numpy()
        assert d.n_bins[j] == R.n_bins(col), c
        want = R.edges(col)
        got = d.bin_edges[j]
        assert got.dtype == np.float64 and len(got) == len(want), c
        assert np.array_equal(got, want), c
        zero = want == 0                                   # the oracle may keep -0.0 where the fit writes 0.0
        assert np.array_equal(got[~zero].view(np.int64), want[~zero].view(np.int64)), c
    Xt = d.transform(frame)
    for j, c in enumerate(frame.columns):
        assert np.array_equal(Xt[f'{c}_discrete'].to_numpy(), R.codes(d.bin_edges[j], frame[c].to_numpy()))


def _frame(task, rows, seed):
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'c{i}': g.choice(list('abcdef')[:3 + i], rows) for i in range(2)})
    for i in range(3):
        X[f'n{i}'] = g.normal(size=rows)
    X['n3'] = g.integers(0, 60, rows).astype(float)
    lead = (X['c0'] == 'a') * 1.0 + 1.5 * (X['n0'] > 0.3) - (X['n1'] > 0) * (X['c1'] == 'b') + 0.02 * X['n3']
    if task == 'binary':
        y = np.where(lead + 0.3 * g.normal(size=rows) > 0.8, 'yes', 'no')
    elif task == 'multiclass':
        y = np.digitize(lead + 0.3 * g.normal(size=rows), [0.0, 1.0, 2.0])
    elif task == 'multilabel':
        return X, np.stack([lead > 0.8, X['n2'] > 0, X['n3'] > 30], 1).astype(np.float32)
    else:
        y = 2.0 * lead + 0.1 * g.normal(size=rows)
    return X, pd.Series(y)


_CACHE = {}


def _fitted(task, gbm=False):
    key = (task, gbm)
    if key not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        X, y = _frame(task, 2600, 5)
        conf = deeptable.ModelConfig(nets=deepnets.DeepFM, metrics=['accuracy' if task != 'regression' else 'mse'],
                                     embeddings_output_dim=4, earlystopping_patience=1, auto_discrete=True,
                                     apply_gbm_features=gbm, gbm_params={'n_estimators': 6, 'num_leaves': 7})
        dt = deeptable.DeepTable(config=conf)
        dt.fit(X.iloc[:2000], y.iloc[:2000], epochs=2, batch_size=128, verbose=0)
        _CACHE[key] = (dt, X.iloc[2000:].reset_index(drop=True), y.iloc[2000:].reset_index(drop=True))
    return _CACHE[key]


@pytest.mark.parametrize('task', ['binary', 'regression', 'multiclass'])
@pytest.mark.parametrize('gbm', [False, True])
def test_end_to_end_fit_predict_evaluate_save_load(task, gbm, tmp_path):
    from deeptables_b200 import deeptable
    dt, X, y = _fitted(task, gbm)
    pre = dt.preprocessor
    disc = pre.discretizer_
    names = ['n0_discrete', 'n1_discrete', 'n2_discrete', 'n3_discrete']
    assert disc.new_columns == names
    cats = [c.name for c in pre.categorical_columns]
    assert cats[:2] == ['c0', 'c1'] and cats[2:6] == names
    assert [c.vocabulary_size for c in pre.categorical_columns[2:6]] == [int(b) + 1 for b in disc.n_bins]
    desc = str(dt.get_model().model_desc)
    assert f'all_categorical_vars: ({len(cats)})' in desc
    assert str([c.vocabulary_size for c in pre.categorical_columns]) in desc
    Xt = pre.transform_X(X)
    assert all(Xt[c.name].max() < c.vocabulary_size for c in pre.categorical_columns[2:6])
    if gbm:
        assert cats[6:] == pre.gbm_encoder_.new_columns
        assert pre.gbm_encoder_.cat_vars == ['c0', 'c1'] + names
    proba = dt.predict_proba(X)
    assert np.all(np.isfinite(proba))
    dt.evaluate(X, y)
    dt.save(str(tmp_path / 'm'))
    dt2 = deeptable.DeepTable.load(str(tmp_path / 'm'))
    assert np.array_equal(dt2.predict_proba(X), proba)
    assert np.array_equal(dt2.preprocessor.transform_X(X).to_numpy(), Xt.to_numpy())


def test_end_to_end_multilabel(tmp_path):
    """DefaultPreprocessor discretises a multilabel frame (the bins do not depend on y); the model trains, scores and
    reloads on it."""
    from deeptables_b200 import deepnets, deeptable
    from deeptables_b200.deepmodel import DeepModel
    X, y = _frame('multilabel', 2600, 6)
    conf = deeptable.ModelConfig(nets=deepnets.DeepFM, task='multilabel', metrics=['binary_accuracy'],
                                 auto_discrete=True, embeddings_output_dim=4)
    pre = deeptable.DefaultPreprocessor(conf)
    Xt, _ = pre.fit_transform(X.iloc[:2000], y[:2000])
    assert pre.task == 'multilabel' and Xt.columns[-4:].tolist() == pre.discretizer_.new_columns
    model = DeepModel('multilabel', 3, conf, pre.categorical_columns, pre.continuous_columns)
    model.fit(Xt, y[:2000], epochs=2, batch_size=128, verbose=0, validation_split=0.2)
    Xv = pre.transform_X(X.iloc[2000:])
    proba = model.predict(Xv)
    assert proba.shape == (600, 3) and np.all(np.isfinite(proba))
    model.evaluate(Xv, y[2000:])
    model.save(str(tmp_path / 'm.npz'))
    again = DeepModel('multilabel', 3, conf, pre.categorical_columns, pre.continuous_columns,
                      model_file=str(tmp_path / 'm.npz'))
    assert np.array_equal(again.predict(Xv), proba)


def test_gradient_boosted_trees_read_the_bin_columns():
    """y is the side of n0's median: the bin split at the median edge separates it exactly, a split of n0's own
    max_bin bins does not, so the first tree's root splits a bin column (feature positions 2..5)."""
    from deeptables_b200 import deeptable
    X, _ = _frame('binary', 2000, 8)
    y = (X['n0'] > X['n0'].median()).astype(int).to_numpy()
    conf = deeptable.ModelConfig(auto_discrete=True, apply_gbm_features=True, gbm_params={'n_estimators': 3})
    pre = deeptable.DefaultPreprocessor(conf)
    Xt, _ = pre.fit_transform(X, y)
    trees = pre.gbm_encoder_.trees
    assert trees.node_feature[0] == 2, trees.node_feature[:trees.node_off[1]]
    assert np.array_equal(pre.transform_X(X).to_numpy(), Xt.to_numpy())


@pytest.mark.parametrize('gbm', [False, True])
def test_permutation_importance_equals_the_host_loop(gbm):
    """Accuracy, exactly: the device passes against the same permutations applied to the raw DataFrame column."""
    from deeptables_b200 import importance
    from importance_ref import permutation
    dt, X, y = _fitted('multiclass', gbm)
    seed = 13
    got = importance.score_decreases(dt, X, y, 'accuracy', n_iter=2, random_state=seed, batch_size=97)
    assert got.columns == X.columns.to_list()
    base = np.mean(dt.predict(X) == np.asarray(y))
    for it in range(2):
        for j, c in enumerate(X.columns):
            Xp = X.copy()
            Xp[c] = X[c].to_numpy()[permutation(seed, it, j, len(X))]
            want = np.mean(dt.predict(Xp) == np.asarray(y))
            assert got.decreases[it, j] == -base - (-want), (it, c)


@pytest.mark.parametrize('gbm', [False, True])
def test_shap_coalition_values_equal_model_fn_on_composed_frames(gbm):
    from deeptables_b200 import explain
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X, _ = _fitted('binary', gbm)
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
        pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig(auto_discrete=True, task='binary'))
        Xt, _ = pre.fit_transform(X, y)
        disc = pre.discretizer_
        np.savez(os.path.join(out_dir, f'edges{rank}.npz'), n_bins=disc.n_bins,
                 **{f'edges_{j}': e for j, e in enumerate(disc.bin_edges)}, codes=Xt[disc.new_columns].to_numpy())
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_data_parallel_ranks_have_identical_edges(tmp_path, backend):
    """World size 2; over gloo both ranks may share one GPU."""
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    X, y = _frame('binary', 3000, 2)
    pd.to_pickle((X, y), str(tmp_path / 'data.pkl'))
    mp.spawn(_dp_worker, args=(2, _free_port(), backend, str(tmp_path / 'data.pkl'), str(tmp_path)), nprocs=2,
             join=True)
    a, b = np.load(tmp_path / 'edges0.npz'), np.load(tmp_path / 'edges1.npz')
    assert a.files == b.files and len(a.files) == 2 + 4
    for k in a.files:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k
