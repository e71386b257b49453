"""Permutation feature importance on the GPU against the host algorithm: the device permutations applied to the
DataFrame, DeepTable.predict_proba / predict and deeptable._calc_scores (or DeepModel.streaming_scores) give the same
score decreases.  Also: the reference's own test, the ranking of a decisive column, unread columns, determinism, the
model left as it was, and data parallel."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

from importance_ref import perm_keys

pytestmark = pytest.mark.gpu

ROWS, TEST_ROWS, BS = 3000, 700, 256


def _frame(task, rows, seed):
    """16 columns: 7 categorical, 7 continuous, one constant (dropped by auto_discard_unique) and one excluded.  The
    label is decided by c0 and n0 (regression: also n1)."""
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'c{i}': g.choice(['a', 'b', 'c', 'd', 'e', 'f'][:3 + i % 4], rows) for i in range(7)})
    for i in range(7):
        X[f'n{i}'] = g.normal(size=rows)
    X['const'] = 'k'
    X['skip'] = g.normal(size=rows)
    lead = (X['c0'] == 'a').astype(float) * 2 + X['n0']
    if task == 'binary':
        y = np.where(lead + 0.3 * g.normal(size=rows) > 0.8, 'yes', 'no')
    elif task == 'multiclass':
        y = np.digitize(lead + 0.3 * g.normal(size=rows), [0.0, 1.0, 2.0])
    else:
        y = 3.0 * lead + X['n1'] + 0.1 * g.normal(size=rows)
    return X, pd.Series(y)


_CACHE = {}


def _fitted(task, nets='DeepFM'):
    key = (task, nets)
    if key not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        X, y = _frame(task, ROWS + TEST_ROWS, 5)
        metric = {'binary': 'AUC', 'multiclass': 'accuracy', 'regression': 'mse'}[task]
        conf = deeptable.ModelConfig(nets=getattr(deepnets, nets), metrics=[metric], exclude_columns=['skip'],
                                     embeddings_output_dim=4, earlystopping_patience=1,
                                     cin_params={'cross_layer_size': (16, 16), 'activation': 'relu',
                                                 'use_residual': False, 'use_bias': False, 'direct': False,
                                                 'reduce_D': False})
        dt = deeptable.DeepTable(config=conf)
        dt.fit(X.iloc[:ROWS], y.iloc[:ROWS], epochs=2, batch_size=128, verbose=0)
        _CACHE[key] = (dt, X.iloc[ROWS:].reset_index(drop=True), y.iloc[ROWS:].reset_index(drop=True))
    return _CACHE[key]


def _host_score(dt, X, y, metric):
    """One pass of the host algorithm: the reference's routing, scored as fit_cross_validation scores oof_metrics."""
    from deeptables_b200 import deeptable
    if deeptable._is_streaming_metric(metric):
        model = dt.get_model()
        raw = model.predict(dt.preprocessor.transform_X(X), batch_size=BS)
        enc = dt.preprocessor.transform_y(y) if dt.task != 'regression' else np.asarray(y)
        (v,) = model.streaming_scores([metric], enc, raw).values()
        return float(v)
    proba = dt.predict_proba(X, batch_size=BS)
    pred = dt.proba2predict(proba) if dt.task != 'regression' else proba
    (v,) = deeptable._calc_scores(np.asarray(y), pred, proba, dt.task, [metric], dt.pos_label, dt.classes_).values()
    return float(v)


def _log_loss_f64(dt, X, y):
    """sklearn's log loss formula (float32 probabilities clipped at float32's eps) evaluated in float64."""
    proba = dt.predict_proba(X, batch_size=BS).astype(np.float32)
    eps = np.finfo(np.float32).eps
    q = np.clip(proba, eps, np.float32(1) - eps)
    enc = dt.preprocessor.transform_y(y)
    return float(np.mean(-np.log(q[np.arange(len(enc)), enc].astype(np.float64))))


def _host_decreases(dt, X, y, metric, n_iter, mode, seed, score=_host_score):
    from deeptables_b200 import importance
    sign = -1.0 if mode == 'min' else 1.0
    base = sign * score(dt, X, y, metric)
    read = set(dt.preprocessor.get_categorical_columns()) | set(dt.preprocessor.get_continuous_columns())
    out = np.zeros((n_iter, X.shape[1]))
    for it in range(n_iter):
        for j, c in enumerate(X.columns):
            if c not in read:
                continue
            perm = importance.permutation(len(X), seed, it, j, dt.get_model().device).cpu().numpy()
            Xs = X.copy()
            Xs[c] = X[c].values[perm]
            out[it, j] = base - sign * score(dt, Xs, y, metric)
    return base, out


CASES = [
    ('binary', 'DeepFM', 'auc', 'max'), ('binary', 'DeepFM', 'accuracy', 'max'), ('binary', 'DeepFM', 'f1', 'max'),
    ('binary', 'DeepFM', 'precision', 'max'), ('binary', 'xDeepFM', 'roc_auc', 'max'),
    ('multiclass', 'DeepFM', 'accuracy', 'max'), ('multiclass', 'DeepFM', 'f1', 'max'),
    ('multiclass', 'DeepFM', 'auc', 'max'),
    ('regression', 'DeepFM', 'mse', 'min'), ('regression', 'DeepFM', 'rmse', 'min'),
    ('regression', 'DeepFM', 'mae', 'min'), ('regression', 'DeepFM', 'r2', 'max'),
    ('regression', 'DeepFM', 'r2_score', 'max'),
]


@pytest.mark.parametrize('task,nets,metric,mode', CASES)
def test_decreases_equal_the_host_algorithm(task, nets, metric, mode):
    from deeptables_b200 import importance
    dt, X, y = _fitted(task, nets)
    res = importance.score_decreases(dt, X, y, metric, n_iter=2, mode=mode, random_state=11, batch_size=BS)
    base, host = _host_decreases(dt, X, y, metric, 2, mode, 11)
    assert res.columns == X.columns.to_list()
    if metric in ('accuracy', 'f1', 'precision'):       # counts: the same bits
        np.testing.assert_array_equal(res.decreases, host)
    else:                                               # float64 sums in another order (AUC: one rounding)
        np.testing.assert_allclose(res.decreases, host, rtol=1e-12, atol=1e-12 * abs(base))
    assert np.abs(host).max() > 0


@pytest.mark.parametrize('task', ['binary', 'multiclass'])
def test_log_loss(task):
    """The device evaluates sklearn's log-loss formula in float64: equal to a float64 restatement within 1e-12, and to
    sklearn, which sums float32 logs, within float32 rounding."""
    from deeptables_b200 import importance
    dt, X, y = _fitted(task)
    res = importance.score_decreases(dt, X, y, 'log_loss', n_iter=1, mode='min', random_state=3, batch_size=BS)
    base, exact = _host_decreases(dt, X, y, None, 1, 'min', 3, score=lambda d, Xs, ys, m: _log_loss_f64(d, Xs, ys))
    np.testing.assert_allclose(res.decreases, exact, rtol=1e-12, atol=1e-12 * abs(base))
    base, sk = _host_decreases(dt, X, y, 'log_loss', 1, 'min', 3)
    np.testing.assert_allclose(res.decreases, sk, rtol=0, atol=4e-6 * abs(base))


def test_device_keys_match_the_restatement():
    from deeptables_b200 import _native as N
    from deeptables_b200._native import ptr, stream_ptr
    for seed, it, col, rows in [(11, 0, 0, 1000), (2 ** 32 - 1, 4, 15, 70001)]:
        keys = torch.empty(rows, dtype=torch.int64, device='cuda')
        N.check(N.lib.dtb_perm_keys(ptr(keys), rows, seed, it, col, stream_ptr()))
        np.testing.assert_array_equal(keys.cpu().numpy(), perm_keys(seed, it, col, rows))


def test_reference_shape():
    """The reference's tests/utils/feature_importance_test.py."""
    from deeptables_b200.utils.feature_importance import get_score_importances
    dt, X, y = _fitted('binary')
    fi = get_score_importances(dt, X, y, 'AUC', 1, mode='max')
    assert fi.shape == (16, 2)
    fi2 = get_score_importances(dt, X, y, 'log_loss', 1, mode='min')
    assert fi2.shape == (16, 2)


def test_ranking_and_unread_columns():
    from deeptables_b200 import importance
    from deeptables_b200.utils.feature_importance import get_score_importances, select_features
    dt, X, y = _fitted('binary')
    y2 = pd.Series(np.where(X['c0'] == 'a', 'yes', 'no'))      # c0 alone decides this label
    fi = get_score_importances(dt, X, y2, 'auc', 3, mode='max', random_state=1)
    assert fi[0, 0] == 'c0'
    values = dict(fi.tolist())
    assert values['const'] == '0.0' and values['skip'] == '0.0'
    res = importance.score_decreases(dt, X, y2, 'auc', n_iter=3, mode='max', random_state=1)
    assert res.passes == 3 * 14
    assert select_features(fi, threshold=0.0)[0][0] == 'c0'


def test_determinism():
    from deeptables_b200.utils.feature_importance import get_score_importances
    dt, X, y = _fitted('binary')
    a = get_score_importances(dt, X, y, 'auc', 2, mode='max', random_state=5)
    assert np.array_equal(a, get_score_importances(dt, X, y, 'auc', 2, mode='max', random_state=5))
    assert not np.array_equal(a, get_score_importances(dt, X, y, 'auc', 2, mode='max', random_state=6))
    b = get_score_importances(dt, X, y, 'auc', 2, mode='max', random_state=5, batch_size=300)
    assert np.array_equal(a, b)


def test_model_left_as_it_was(tmp_path):
    """predict_proba and evaluate give the same bits after the call, and so does the saved state (weights, optimiser
    step and moments).  A train step from that state is compared within float32 rounding: the Dense weight gradient
    adds its split-K partial sums with float atomics, so two runs of one step may differ in the last bits."""
    from deeptables_b200 import deeptable
    from deeptables_b200.utils.feature_importance import get_score_importances
    dt, X, y = _fitted('binary')
    dt.save(str(tmp_path / 'm'))
    a, b = deeptable.DeepTable.load(str(tmp_path / 'm')), deeptable.DeepTable.load(str(tmp_path / 'm'))
    before = a.predict_proba(X)
    get_score_importances(a, X, y, 'auc', 1, mode='max', random_state=2)
    np.testing.assert_array_equal(a.predict_proba(X), before)
    np.testing.assert_array_equal(a.evaluate(X, y)['loss'], b.evaluate(X, y)['loss'])
    a.get_model().save(str(tmp_path / 'a.npz'))
    b.get_model().save(str(tmp_path / 'b.npz'))
    with np.load(tmp_path / 'a.npz') as sa, np.load(tmp_path / 'b.npz') as sb:
        assert sa.files == sb.files
        for k in sa.files:
            np.testing.assert_array_equal(sa[k], sb[k], err_msg=k)
    Xt, yt = a.preprocessor.transform(X.iloc[:128], y.iloc[:128])
    cats = a.preprocessor.get_categorical_columns()
    conts = a.preprocessor.get_continuous_columns()
    for dt_ in (a, b):
        dt_.get_model()._scope.generator.manual_seed(7)          # the same embedding-dropout masks in both steps
        dt_.get_model().train_on_batch(Xt[cats].values, Xt[conts].values, yt)
    sa, sb = a.get_model().state_dict(), b.get_model().state_dict()
    for k in sa:
        torch.testing.assert_close(sa[k], sb[k], rtol=1e-5, atol=1e-7, msg=k)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, backend, model_dir, data, out_dir):
    import torch.distributed as dist
    from deeptables_b200 import deeptable
    from deeptables_b200.utils.feature_importance import get_score_importances
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    kw = {'device_id': torch.device('cuda', rank)} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        dt = deeptable.DeepTable.load(model_dir)
        X, y = pd.read_pickle(data)
        np.random.seed(rank)                         # rank 0's seed is the one every rank uses
        fi = get_score_importances(dt, X, y, 'auc', 2, mode='max')
        np.save(os.path.join(out_dir, f'fi{rank}.npy'), fi)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_data_parallel_ranks_return_the_single_process_array(tmp_path, backend):
    """World size 2; over gloo both ranks may share one GPU."""
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    from deeptables_b200.utils.feature_importance import get_score_importances
    dt, X, y = _fitted('binary')
    dt.save(str(tmp_path / 'm'))
    pd.to_pickle((X, y), str(tmp_path / 'data.pkl'))
    np.random.seed(0)
    single = get_score_importances(dt, X, y, 'auc', 2, mode='max')
    mp.spawn(_dp_worker, args=(2, _free_port(), backend, str(tmp_path / 'm'), str(tmp_path / 'data.pkl'),
                               str(tmp_path)), nprocs=2, join=True)
    for rank in range(2):
        assert np.array_equal(np.load(tmp_path / f'fi{rank}.npy'), single)
