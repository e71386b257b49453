"""Partial dependence on the GPU against the host: scikit-learn's ``partial_dependence(method='brute')`` over an adapter
of the DeepTable, a host loop for multilabel and for the derived quantile-bin and boosted-leaf columns, columns the
model does not read, determinism across calls and batch sizes, the kernel's order restated in numpy, the model left as
it was, data parallel, and xDeepFM at 39 columns."""
import ctypes
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import pdp_ref

pytestmark = pytest.mark.gpu

ROWS, TEST_ROWS = 3000, 300
AVG_TOL = dict(rtol=1e-6, atol=1e-7)
ICE_TOL = dict(rtol=1e-6, atol=1e-6)


def _frame(rows, seed, n_cat=3, n_cont=3, extra=True):
    """``n_cat`` categorical and ``n_cont`` continuous columns, plus (``extra``) an integer-coded categorical column, a
    constant column that auto_discard_unique drops and an excluded one."""
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'c{i}': g.choice(['a', 'b', 'c', 'd', 'e', 'f'][:3 + i % 4], rows) for i in range(n_cat)})
    for i in range(n_cont):
        X[f'n{i}'] = g.normal(size=rows)
    lead = (X['c0'] == 'a').astype(float) * 2 + X['n0'] + 0.5 * X['n1'] * (X['c1'] == 'b')
    if extra:
        X['icode'] = g.integers(0, 8, rows)
        X['const'] = 'k'
        X['skip'] = g.normal(size=rows)
        lead = lead + 0.2 * (X['icode'] % 3)
    return X, lead + 0.3 * g.normal(size=rows)


_CACHE = {}


def _fitted(task, nets='DeepFM', n_cat=3, n_cont=3, extra=True, **conf_kw):
    key = (task, nets, n_cat, n_cont, extra, tuple(sorted(conf_kw)))
    if key not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        X, lead = _frame(ROWS + TEST_ROWS, 5, n_cat, n_cont, extra)
        y = {'binary': lambda: np.where(lead > 0.8, 'yes', 'no'),
             'multiclass': lambda: np.array(['lo', 'mid', 'hi'])[np.digitize(lead, [0.0, 1.5])],
             'regression': lambda: 3.0 * lead}[task]()
        conf = deeptable.ModelConfig(nets=getattr(deepnets, nets), metrics=['mse' if task == 'regression' else 'AUC'],
                                     exclude_columns=['skip'], embeddings_output_dim=4, earlystopping_patience=1,
                                     auto_categorize=True,
                                     cin_params={'cross_layer_size': (16, 16), 'activation': 'relu',
                                                 'use_residual': False, 'use_bias': False, 'direct': False,
                                                 'reduce_D': False}, **conf_kw)
        dt = deeptable.DeepTable(config=conf)
        y = pd.Series(y)
        dt.fit(X.iloc[:ROWS], y.iloc[:ROWS], epochs=2, batch_size=128, verbose=0)
        _CACHE[key] = (dt, X.iloc[ROWS:].reset_index(drop=True), X.iloc[:ROWS])
    return _CACHE[key]


def _multilabel():
    if 'multilabel' not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        from deeptables_b200.deepmodel import DeepModel
        X, lead = _frame(ROWS + TEST_ROWS, 6)
        y = np.stack([lead > 0.8, X['n2'] > 0, X['icode'] > 3], 1).astype(np.float32)
        conf = deeptable.ModelConfig(nets=deepnets.DeepFM, task='multilabel', metrics=['binary_accuracy'],
                                     exclude_columns=['skip'], embeddings_output_dim=4, auto_categorize=True)
        pre = deeptable.DefaultPreprocessor(conf)
        Xt, _ = pre.fit_transform(X.iloc[:ROWS], y[:ROWS])
        model = DeepModel('multilabel', 3, conf, pre.categorical_columns, pre.continuous_columns)
        model.fit(Xt, y[:ROWS], epochs=2, batch_size=128, verbose=0)
        dt = deeptable.DeepTable(conf, preprocessor=pre)
        dt._DeepTable__current_model = model
        _CACHE['multilabel'] = (dt, X.iloc[ROWS:].reset_index(drop=True))
    return _CACHE['multilabel']


def _pd(dt, X, features, **kw):
    from deeptables_b200.utils.partial_dependence import partial_dependence
    return partial_dependence(dt, X, features, **kw)


def _grid(values):
    from sklearn.utils.extmath import cartesian
    return cartesian(values)


CASES = {
    'continuous': ('n0', {}),
    'categorical': ('c0', dict(categorical_features=['c0'])),
    'integer_categorical': ('icode', dict(categorical_features=['icode'])),
    'two_way_mixed': (['c1', 'n1'], dict(categorical_features=['c1'], grid_resolution=8)),
    'both_weighted': ('n1', dict(kind='both', grid_resolution=20, sample_weight='w')),
    'custom_values': ('c2', dict(kind='both', categorical_features=['c2'],
                                 custom_values={'c2': ['a', 'zz-unseen', 'b']})),
}


@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('task', ['binary', 'multiclass', 'regression'])
def test_matches_scikit_learn_brute(task, case):
    from sklearn.inspection import partial_dependence as sk_pd
    dt, X, _ = _fitted(task)
    features, kw = CASES[case]
    kw = dict(kw)
    if kw.get('sample_weight') == 'w':
        kw['sample_weight'] = np.random.default_rng(1).random(len(X)) * 2
    ours = _pd(dt, X, features, **kw)
    theirs = sk_pd(pdp_ref.adapter(dt), X, features, method='brute', **kw)
    assert list(ours.keys()) == list(theirs.keys())
    assert len(ours.grid_values) == len(theirs.grid_values)
    for a, b in zip(ours.grid_values, theirs.grid_values):
        assert a.dtype == b.dtype and np.array_equal(a, b)
    if 'average' in theirs:
        assert ours.average.shape == theirs.average.shape and ours.average.dtype == np.float64
        np.testing.assert_allclose(ours.average, theirs.average, **AVG_TOL)
    if 'individual' in theirs:
        assert ours.individual.shape == theirs.individual.shape and ours.individual.dtype == np.float32
        np.testing.assert_allclose(ours.individual, theirs.individual, **ICE_TOL)
    n_out = {'binary': 1, 'multiclass': 3, 'regression': 1}[task]
    assert ours.average.shape[0] == n_out if 'average' in ours else ours.individual.shape[0] == n_out


def _against_host(dt, X, features, **kw):
    out = _pd(dt, X, features, kind='both', **kw)
    names = [features] if isinstance(features, str) else features
    avg, ind = pdp_ref.host_loop(dt, X, names, _grid(out.grid_values), kw.get('sample_weight'))
    if dt.task == 'binary':
        avg, ind = avg[-1:], ind[-1:]
    shape = [len(v) for v in out.grid_values]
    np.testing.assert_allclose(out.average, avg.reshape(-1, *shape), **AVG_TOL)
    np.testing.assert_allclose(out.individual, ind.reshape(-1, len(X), *shape), **ICE_TOL)
    return out


def test_derived_bin_and_leaf_columns_are_recomputed():
    dt, X, _ = _fitted('binary', auto_discrete=True, apply_gbm_features=True,
                       gbm_params={'n_estimators': 6, 'num_leaves': 7})
    assert dt.preprocessor.discretizer_ is not None and dt.preprocessor.gbm_encoder_ is not None
    out = _against_host(dt, X, 'n0', grid_resolution=15)
    assert np.ptp(out.average) > 0
    _against_host(dt, X, ['c0', 'n1'], categorical_features=['c0'], grid_resolution=6)


def test_multilabel_matches_the_host_loop():
    dt, X = _multilabel()
    out = _against_host(dt, X, 'n2', grid_resolution=12)
    assert out.average.shape == (3, 12) and out.individual.shape == (3, len(X), 12)
    _against_host(dt, X, 'icode', categorical_features=['icode'],
                  sample_weight=np.random.default_rng(2).random(len(X)))


@pytest.mark.parametrize('task', ['binary', 'multiclass'])
def test_unread_columns_give_the_mean_prediction(task):
    """'skip' is excluded, 'const' dropped by auto_discard_unique: the model reads neither."""
    dt, X, _ = _fitted(task)
    proba = dt.predict_proba(X)
    mean = (proba[:, -1:] if task == 'binary' else proba).astype(np.float64).mean(axis=0)
    for feature, kw in (('skip', {}), ('const', dict(custom_values={'const': ['k', 'q', 'r']}))):
        out = _pd(dt, X, feature, kind='both', **kw)
        avg = out.average
        assert np.all(avg == avg[:, :1])
        np.testing.assert_allclose(avg[:, 0], mean, **AVG_TOL)
        np.testing.assert_allclose(out.individual, np.repeat((proba[:, -1:] if task == 'binary' else proba).T[:, :, None],
                                                             avg.shape[1], axis=2), **ICE_TOL)


def test_determinism_and_the_block_order_past_one_chunk():
    """3000 rows: at batch_size=257 every grid point runs over three chunks of rows; at 65536 grid points share
    chunks.  Both give the same bits, equal to the restated block order over the call's own ICE."""
    from deeptables_b200.utils.partial_dependence import _BLOCK_ROWS
    dt, _, X = _fitted('multiclass')
    w = np.random.default_rng(4).random(len(X))
    for weight in (None, w):
        a = _pd(dt, X, ['c0', 'n0'], categorical_features=['c0'], kind='both', sample_weight=weight,
                grid_resolution=30)
        b = _pd(dt, X, ['c0', 'n0'], categorical_features=['c0'], kind='both', sample_weight=weight,
                grid_resolution=30)
        c = _pd(dt, X, ['c0', 'n0'], categorical_features=['c0'], kind='both', sample_weight=weight,
                grid_resolution=30, batch_size=257)
        assert np.array_equal(a.average, b.average) and np.array_equal(a.individual, b.individual)
        assert np.array_equal(a.average, c.average)
        np.testing.assert_allclose(a.individual, c.individual, **ICE_TOL)
        ice = a.individual.reshape(3, len(X), -1)
        avg = a.average.reshape(3, -1)
        for g in range(ice.shape[2]):
            want = pdp_ref.block_order_mean(ice[:, :, g].T.copy(), weight, _BLOCK_ROWS)
            assert np.array_equal(avg[:, g], want), g


@pytest.mark.parametrize('weighted', [False, True])
def test_block_sums_kernel_equals_the_restated_order(weighted):
    """6001 groups x 4 blocks (the last short) x 3 columns: 72 012 sums, several passes of the capped grid."""
    from deeptables_b200 import _native as N
    groups, rows, cols, block = 6001, 200, 3, 64
    g = np.random.default_rng(7)
    prob = g.normal(size=(groups, rows, cols)).astype(np.float32)
    weight = g.random(rows) * 4 if weighted else None
    sm = ctypes.c_int()
    N.lib.dtb_device_sm_count(ctypes.byref(sm))
    assert groups * 4 * cols > 3 * sm.value * 16 * 8
    p = torch.as_tensor(prob).cuda().view(-1, cols)
    w = torch.as_tensor(weight).cuda() if weighted else None
    out = torch.full((groups * 4 * cols,), float('nan'), dtype=torch.float64, device='cuda')
    N.check(N.lib.dtb_pdp_block_sums(N.ptr(p), N.ptr(w), groups, rows, cols, block, N.ptr(out), N.stream_ptr()))
    got = out.cpu().numpy().reshape(groups, 4, cols)
    assert np.array_equal(got, pdp_ref.block_sums_restated(prob, weight, block))


def test_model_left_as_it_was(tmp_path):
    from deeptables_b200 import deeptable
    dt, X, _ = _fitted('binary')
    dt.save(str(tmp_path / 'm'))
    a, b = deeptable.DeepTable.load(str(tmp_path / 'm')), deeptable.DeepTable.load(str(tmp_path / 'm'))
    before = a.predict_proba(X)
    out = _pd(a, X, ['c0', 'n0'], categorical_features=['c0'], kind='both', grid_resolution=10)
    assert np.isfinite(out.average).all()
    np.testing.assert_array_equal(a.predict_proba(X), before)
    a.get_model().save(str(tmp_path / 'a.npz'))
    b.get_model().save(str(tmp_path / 'b.npz'))
    with np.load(tmp_path / 'a.npz') as sa, np.load(tmp_path / 'b.npz') as sb:
        assert sa.files == sb.files
        for k in sa.files:
            np.testing.assert_array_equal(sa[k], sb[k], err_msg=k)


def test_array_input_with_feature_names():
    dt, X, _ = _fitted('regression')
    a = _pd(dt, X, 'n1', grid_resolution=9)
    b = _pd(dt, X.to_numpy(dtype=object), 'n1', grid_resolution=9, feature_names=list(X.columns))
    assert np.array_equal(a.grid_values[0], b.grid_values[0]) and np.array_equal(a.average, b.average)
    with pytest.raises(ValueError, match='columns'):
        _pd(dt, X.drop(columns=['skip']), 'n1')


def test_xdeepfm_at_39_columns():
    dt, X, _ = _fitted('binary', 'xDeepFM', n_cat=26, n_cont=10)
    assert X.shape[1] == 39
    sample = X.iloc[:100].reset_index(drop=True)
    _against_host(dt, sample, 'n3', grid_resolution=10)
    _against_host(dt, sample, 'c7', categorical_features=['c7'])


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_args(X):
    return dict(features=['c0', 'n0'], categorical_features=['c0'], kind='both', grid_resolution=7,
                sample_weight=np.linspace(0.5, 2.0, len(X)))


def _dp_worker(rank, world, port, backend, model_dir, data, out_dir):
    import torch.distributed as dist
    from deeptables_b200 import deeptable
    from deeptables_b200.utils.partial_dependence import partial_dependence
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    kw = {'device_id': torch.device('cuda', rank)} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        dt = deeptable.DeepTable.load(model_dir)
        X = pd.read_pickle(data)
        out = partial_dependence(dt, X, **_dp_args(X))
        np.save(os.path.join(out_dir, f'avg{rank}.npy'), out.average)
        np.save(os.path.join(out_dir, f'ind{rank}.npy'), out.individual)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_data_parallel_ranks_return_the_single_process_arrays(tmp_path, backend):
    """World size 2; over gloo both ranks may share one GPU."""
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    from deeptables_b200.utils.partial_dependence import partial_dependence
    dt, X, _ = _fitted('multiclass')
    dt.save(str(tmp_path / 'm'))
    pd.to_pickle(X, str(tmp_path / 'data.pkl'))
    single = partial_dependence(dt, X, **_dp_args(X))
    mp.spawn(_dp_worker, args=(2, _free_port(), backend, str(tmp_path / 'm'), str(tmp_path / 'data.pkl'),
                               str(tmp_path)), nprocs=2, join=True)
    for rank in range(2):
        assert np.array_equal(np.load(tmp_path / f'avg{rank}.npy'), single.average)
        assert np.array_equal(np.load(tmp_path / f'ind{rank}.npy'), single.individual)
