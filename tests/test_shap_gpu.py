"""Kernel SHAP on the GPU against the host: the exact Shapley values of coalition values taken from the reference's
``model_fn`` (pandas composition + ``predict``), the closed form of an additive model, the restated shap loops run on
the device path's own coalition values, the estimator's properties, composition with unseen categories and NaN,
determinism, the reference notebook's calls, the model left as it was, and data parallel."""
import itertools
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import shap_ref

pytestmark = pytest.mark.gpu

ROWS, TEST_ROWS = 3000, 300


def _frame(rows, seed, n_cat=3, n_cont=3, extra=True):
    """``n_cat`` categorical and ``n_cont`` continuous columns, plus (``extra``) a constant column that
    auto_discard_unique drops and an excluded one.  The label is decided by c0, n0 and n1."""
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'c{i}': g.choice(['a', 'b', 'c', 'd', 'e', 'f'][:3 + i % 4], rows) for i in range(n_cat)})
    for i in range(n_cont):
        X[f'n{i}'] = g.normal(size=rows)
    if extra:
        X['const'] = 'k'
        X['skip'] = g.normal(size=rows)
    lead = (X['c0'] == 'a').astype(float) * 2 + X['n0'] + 0.5 * X['n1'] * (X['c1'] == 'b')
    return X, lead + 0.3 * g.normal(size=rows)


_CACHE = {}


def _fitted(task, nets='DeepFM', n_cat=3, n_cont=3, extra=True):
    key = (task, tuple(nets) if isinstance(nets, list) else nets, n_cat, n_cont, extra)
    if key not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        X, lead = _frame(ROWS + TEST_ROWS, 5, n_cat, n_cont, extra)
        y = pd.Series(np.where(lead > 0.8, 'yes', 'no') if task == 'binary' else 3.0 * lead)
        nets = getattr(deepnets, nets) if isinstance(nets, str) else nets
        conf = deeptable.ModelConfig(nets=nets, metrics=['AUC' if task == 'binary' else 'mse'],
                                     exclude_columns=['skip'], embeddings_output_dim=4, earlystopping_patience=1,
                                     cin_params={'cross_layer_size': (16, 16), 'activation': 'relu',
                                                 'use_residual': False, 'use_bias': False, 'direct': False,
                                                 'reduce_D': False})
        dt = deeptable.DeepTable(config=conf)
        dt.fit(X.iloc[:ROWS], y.iloc[:ROWS], epochs=2, batch_size=128, verbose=0)
        _CACHE[key] = (dt, X.iloc[ROWS:].reset_index(drop=True))
    return _CACHE[key]


def _host_f(ex, frame):
    return np.asarray(ex.model_fn(frame.to_numpy(dtype=object)), np.float64).reshape(-1)


def _host_values(ex, bg, x, columns, coalitions):
    """Coalition values by the host: the background with the coalition's columns set to x's, through model_fn."""
    parts = []
    for S in coalitions:
        f = bg.copy()
        for j in S:
            f[columns[j]] = x[columns[j]]
        parts.append(f)
    f = _host_f(ex, pd.concat(parts, ignore_index=True))
    return f.reshape(len(coalitions), len(bg)).mean(axis=1)


def _explain(ex, X, **kw):
    from deeptables_b200 import explain
    trace = {}
    phi = explain.shap_values(ex._background, X, kw.get('nsamples', 'auto'), kw.get('seed', 0),
                              kw.get('batch_size', 65536), trace=trace)
    return phi, trace


def _explained_rows(X):
    """Three rows: as drawn; with the discarded column changed (so it varies) and an unseen category; with NaN in a
    continuous column."""
    x = X.iloc[:3].copy()
    x.loc[1, 'const'] = 'q'
    x.loc[1, 'c2'] = 'never-seen'
    x.loc[2, 'n1'] = np.nan
    return x.reset_index(drop=True)


@pytest.mark.parametrize('task', ['regression', 'binary'])
def test_exact_case_equals_the_brute_force_shapley_values(task):
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted(task)
    columns = X.columns.to_list()
    ex = DeepTablesExplainer(dt, X.iloc[10:], num_samples=10, random_state=0)
    bg = ex._background
    bg_frame = pd.DataFrame({c: v for c, v in zip(bg.columns, bg.values)})
    E = _host_f(ex, bg_frame).mean()
    tol = dict(rtol=0, atol=1e-9) if task == 'binary' else dict(rtol=1e-6, atol=1e-6 * max(1.0, abs(E)))
    np.testing.assert_allclose(ex.explainer.expected_value, E, **tol)
    assert isinstance(ex.explainer.expected_value, np.float64)
    x = _explained_rows(X)
    phi = ex.get_shap_values(x)
    assert phi.shape == (3, 8) and phi.dtype == np.float64
    fx = _host_f(ex, x)
    for i in range(3):
        vary = [j for j in range(8) if not all(shap_ref.not_equal(x.iloc[i, j], b) == 0 for b in bg_frame.iloc[:, j])]
        M = len(vary)
        subsets = [S for r in range(M + 1) for S in itertools.combinations(range(M), r)]
        vals = _host_values(ex, bg_frame, x.iloc[i], columns, [[vary[k] for k in S] for S in subsets])
        table = dict(zip(subsets, vals))
        want = np.zeros(8)
        want[vary] = shap_ref.exact_shapley(lambda S: table[tuple(sorted(S))], M)
        tol_i = dict(rtol=0, atol=1e-9) if task == 'binary' else dict(rtol=1e-6, atol=1e-6 * np.abs(want).max())
        np.testing.assert_allclose(phi[i], want, **tol_i)
        np.testing.assert_allclose(phi[i].sum() + ex.explainer.expected_value, fx[i], rtol=0, atol=1e-9 * max(1, abs(fx[i])))
        assert all(phi[i, j] == 0.0 for j in range(8) if j not in vary)        # non-varying: exactly 0
        for c in ('const', 'skip'):                                           # not read by the model
            assert abs(phi[i, columns.index(c)]) < 1e-9
    assert phi[0, columns.index('const')] == 0.0                              # const does not vary in row 0


def test_additive_model_gives_the_closed_form():
    """nets=['linear'] on regression is additive over columns, so any full-rank sample gives
    phi_i = mean_j [f_i(x_i) - f_i(bg_ji)]; each term is read off the model by changing one column of a background
    row.  20 varying columns: the sampled path."""
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted('regression', ['linear'], n_cat=10, n_cont=10, extra=False)
    columns = X.columns.to_list()
    ex = DeepTablesExplainer(dt, X.iloc[5:], num_samples=8, random_state=1)
    bg_frame = pd.DataFrame({c: v for c, v in zip(ex._background.columns, ex._background.values)})
    x = X.iloc[:2].reset_index(drop=True)
    phi, trace = _explain(ex, x, seed=4)
    base = _host_f(ex, bg_frame)
    for i in range(2):
        assert len(trace[i].varying) == 20 and len(trace[i].masks) == 2 * 20 + 2048
        want = np.array([(_host_values(ex, bg_frame, x.iloc[i], columns, [[j]])[0] - base.mean()) for j in range(20)])
        np.testing.assert_allclose(phi[i], want, rtol=0, atol=1e-4 * np.abs(want).max())


def test_sampled_path_equals_the_restated_loops():
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt16, X16 = _fitted('regression', n_cat=7, n_cont=7)
    ex = DeepTablesExplainer(dt16, X16.iloc[20:], num_samples=30, random_state=0)
    x = X16.iloc[:4].reset_index(drop=True)
    for nsamples in ('auto', 300):
        phi, trace = _explain(ex, x, nsamples=nsamples, seed=77)
        for i in range(4):
            r = trace[i]
            M = len(r.varying)
            assert M >= 12
            masks, weights = shap_ref.coalitions(M, nsamples, np.random.RandomState([77, i]))
            np.testing.assert_array_equal(r.masks, masks.astype(bool))
            np.testing.assert_array_equal(r.weights, weights)
            want = shap_ref.solve(masks, weights, r.values, r.fx, ex.explainer.expected_value)
            np.testing.assert_allclose(phi[i, r.varying], want, rtol=0, atol=1e-9 * max(1.0, np.abs(want).max()))
            assert abs(phi[i].sum() + ex.explainer.expected_value - r.fx) < 1e-9 * max(1.0, abs(r.fx))


@pytest.mark.parametrize('task', ['regression', 'binary'])
def test_device_coalition_values_equal_model_fn_on_host_composed_frames(task):
    """A few coalitions of rows holding an unseen category and NaN continuous values (also in the background)."""
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted(task)
    columns = X.columns.to_list()
    bgX = X.iloc[10:40].copy()
    bgX.iloc[0, columns.index('n0')] = np.nan
    bgX.iloc[1, columns.index('c0')] = 'also-unseen'
    ex = DeepTablesExplainer(dt, bgX, num_samples=None, random_state=0)
    bg_frame = bgX.reset_index(drop=True)
    x = _explained_rows(X)
    _, trace = _explain(ex, x, nsamples=40, seed=3)
    for i in range(3):
        r = trace[i]
        pick = [0, 1, 2, 3, len(r.masks) // 2, len(r.masks) - 1]
        coalitions = [[r.varying[k] for k in np.flatnonzero(r.masks[p])] for p in pick]
        host = _host_values(ex, bg_frame, x.iloc[i], columns, coalitions)
        tol = dict(rtol=0, atol=1e-12) if task == 'binary' else dict(rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(r.values[pick], host, **tol)
        np.testing.assert_allclose(r.fx, _host_f(ex, x.iloc[i:i + 1])[0], **tol)


def test_determinism_across_calls_and_batch_sizes():
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted('regression')
    x = _explained_rows(X)
    a = DeepTablesExplainer(dt, X.iloc[10:], num_samples=40, random_state=5).get_shap_values(x, nsamples=100)
    b = DeepTablesExplainer(dt, X.iloc[10:], num_samples=40, random_state=5).get_shap_values(x, nsamples=100)
    c = DeepTablesExplainer(dt, X.iloc[10:], num_samples=40, random_state=5, batch_size=200).get_shap_values(
        x, nsamples=100)
    assert np.array_equal(a, b) and np.array_equal(a, c)
    d = DeepTablesExplainer(dt, X.iloc[10:], num_samples=40, random_state=6).get_shap_values(x, nsamples=100)
    assert not np.array_equal(a, d)


def test_xdeepfm_at_39_columns():
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted('binary', 'xDeepFM', n_cat=26, n_cont=11)
    ex = DeepTablesExplainer(dt, X.iloc[5:], num_samples=50, random_state=0)
    x = X.iloc[:2].reset_index(drop=True)
    phi = ex.get_shap_values(x)
    assert phi.shape == (2, 39)
    fx = _host_f(ex, x)
    np.testing.assert_allclose(phi.sum(1) + ex.explainer.expected_value, fx, rtol=0, atol=1e-9)


def test_reference_notebook_calls_and_the_model_left_as_it_was(tmp_path):
    """DeepTablesExplainer(dt, df, num_samples=100), get_shap_values(df[:1], nsamples='auto'),
    explainer.expected_value; predictions and saved weights are the same bits afterwards."""
    from deeptables_b200 import deeptable
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted('binary')
    dt.save(str(tmp_path / 'm'))
    a, b = deeptable.DeepTable.load(str(tmp_path / 'm')), deeptable.DeepTable.load(str(tmp_path / 'm'))
    before = a.predict_proba(X)
    explainer = DeepTablesExplainer(a, X, num_samples=100)
    shap_values = explainer.get_shap_values(X[:1], nsamples='auto')
    assert shap_values.shape == (1, X.shape[1])
    assert np.isfinite(explainer.explainer.expected_value)
    assert 0.0 <= explainer.explainer.expected_value <= 1.0
    np.testing.assert_array_equal(a.predict_proba(X), before)
    a.get_model().save(str(tmp_path / 'a.npz'))
    b.get_model().save(str(tmp_path / 'b.npz'))
    with np.load(tmp_path / 'a.npz') as sa, np.load(tmp_path / 'b.npz') as sb:
        assert sa.files == sb.files
        for k in sa.files:
            np.testing.assert_array_equal(sa[k], sb[k], err_msg=k)


def test_refusals():
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted('binary')
    ex = DeepTablesExplainer(dt, X.iloc[5:], num_samples=10, random_state=0)
    with pytest.raises(ValueError, match='columns'):
        ex.get_shap_values(X.iloc[:1, ::-1])
    for bad in (0, 'full', 2.5):
        with pytest.raises(ValueError):
            ex.get_shap_values(X.iloc[:1], nsamples=bad)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, backend, model_dir, data, out_dir):
    import torch.distributed as dist
    from deeptables_b200 import deeptable
    from deeptables_b200.utils.shap import DeepTablesExplainer
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    kw = {'device_id': torch.device('cuda', rank)} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        dt = deeptable.DeepTable.load(model_dir)
        X, x = pd.read_pickle(data)
        np.random.seed(rank)                         # rank 0's seed is the one every rank uses
        phi = DeepTablesExplainer(dt, X, num_samples=20).get_shap_values(x, nsamples=200)
        np.save(os.path.join(out_dir, f'phi{rank}.npy'), phi)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_data_parallel_ranks_return_the_single_process_array(tmp_path, backend):
    """World size 2; over gloo both ranks may share one GPU."""
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    from deeptables_b200.utils.shap import DeepTablesExplainer
    dt, X = _fitted('regression')
    x = _explained_rows(X)
    dt.save(str(tmp_path / 'm'))
    pd.to_pickle((X, x), str(tmp_path / 'data.pkl'))
    np.random.seed(0)
    single = DeepTablesExplainer(dt, X, num_samples=20).get_shap_values(x, nsamples=200)
    mp.spawn(_dp_worker, args=(2, _free_port(), backend, str(tmp_path / 'm'), str(tmp_path / 'data.pkl'),
                               str(tmp_path)), nprocs=2, join=True)
    for rank in range(2):
        assert np.array_equal(np.load(tmp_path / f'phi{rank}.npy'), single)
