"""Linear probes without a GPU: the numpy restatement of the objective against scikit-learn's own LinearModelLoss, the
estimator driven by it against scikit-learn's float64 optimum, every refusal of probe_evaluate, and the dealing of
layers over a gloo world of two."""
import os
import socket
import warnings

import numpy as np
import pandas as pd
import pytest
import torch

import probe_ref


def _data(n, d, classes, seed):
    g = np.random.default_rng(seed)
    X = g.normal(size=(n, d)).astype(np.float32)
    w = g.normal(size=(d, classes))
    codes = np.argmax(X @ w + 1.5 * g.normal(size=(n, classes)), axis=1)
    return X, codes


@pytest.mark.parametrize('classes', [2, 4])
@pytest.mark.parametrize('fit_intercept', [True, False])
def test_restated_objective_matches_sklearn_linear_model_loss(classes, fit_intercept):
    from sklearn._loss.loss import HalfBinomialLoss, HalfMultinomialLoss
    from sklearn.linear_model._linear_loss import LinearModelLoss
    n, d, C = 500, 7, 0.7
    X, codes = _data(n, d, classes, 1)
    K = 1 if classes == 2 else classes
    cols = d + 1 if fit_intercept else d
    w = np.random.default_rng(2).normal(size=K * cols)
    f, g = probe_ref.objective(X, codes, w, K, C, fit_intercept)
    if K == 1:
        lml = LinearModelLoss(base_loss=HalfBinomialLoss(), fit_intercept=fit_intercept)
        want_f, want_g = lml.loss_gradient(w, X.astype(np.float64), codes.astype(np.float64),
                                           l2_reg_strength=1.0 / (C * n))
    else:
        lml = LinearModelLoss(base_loss=HalfMultinomialLoss(n_classes=K), fit_intercept=fit_intercept)
        want_f, want_g = lml.loss_gradient(w.reshape(K, cols), X.astype(np.float64), codes.astype(np.float64),
                                           l2_reg_strength=1.0 / (C * n))
    assert abs(f - want_f) <= 1e-12 * abs(want_f)
    np.testing.assert_allclose(g, np.ravel(want_g), rtol=0, atol=1e-12 * np.abs(want_g).max())


@pytest.mark.parametrize('classes', [2, 3])
@pytest.mark.parametrize('fit_intercept', [True, False])
def test_estimator_reaches_the_float64_optimum(monkeypatch, classes, fit_intercept):
    from sklearn.linear_model import LogisticRegression
    from deeptables_b200 import probe
    monkeypatch.setattr(probe.LogisticProbe, 'objective', probe_ref.HostObjective)
    X, codes = _data(800, 6, classes, 3)
    labels = np.array([3, 7, 9])[codes]
    clf = probe.LogisticProbe(C=0.5, fit_intercept=fit_intercept, tol=1e-10, max_iter=10_000).fit(torch.tensor(X),
                                                                                                 labels)
    ref = LogisticRegression(C=0.5, fit_intercept=fit_intercept, tol=1e-10, max_iter=10_000).fit(
        X.astype(np.float64), labels)
    np.testing.assert_array_equal(clf.classes_, ref.classes_)
    assert clf.coef_.shape == ref.coef_.shape and clf.intercept_.shape == ref.intercept_.shape
    np.testing.assert_allclose(clf.coef_, ref.coef_, rtol=0, atol=1e-6 * max(1.0, np.abs(ref.coef_).max()))
    np.testing.assert_allclose(clf.intercept_, ref.intercept_, rtol=0,
                               atol=1e-6 * max(1.0, np.abs(ref.intercept_).max()))
    assert clf.n_iter_.shape == (1,) and 0 < clf.n_iter_[0] < 10_000


def test_estimator_warns_at_max_iter(monkeypatch):
    from sklearn.exceptions import ConvergenceWarning
    from deeptables_b200 import probe
    monkeypatch.setattr(probe.LogisticProbe, 'objective', probe_ref.HostObjective)
    X, codes = _data(300, 5, 3, 4)
    with pytest.warns(ConvergenceWarning):
        clf = probe.LogisticProbe(max_iter=2).fit(torch.tensor(X), codes)
    assert clf.n_iter_[0] == 2
    with pytest.raises(ValueError, match='y:'):
        probe.LogisticProbe().fit(torch.tensor(X), np.zeros(300, np.int64))


class _Pre:
    def __init__(self, task):
        self.task = task

    def transform_y(self, y):
        return np.asarray(y).astype(np.int64)


class _Model:
    model = object()

    def layer_widths(self):
        return {'flatten_embeddings': 16, 'dnn_dense_1': 20_000}


class _DT:
    def __init__(self, task='binary'):
        self.task = task
        self.preprocessor = _Pre(task)

    def get_model(self):
        return _Model()


@pytest.mark.parametrize('kwargs, match', [
    (dict(layers=[]), 'layers'),
    (dict(layers='dnn_dense_1'), 'layers'),
    (dict(layers=['dnn_dense_1', 'nope']), 'layers'),
    (dict(layers=['flatten_embeddings', 'dnn_dense_1']), 'too wide'),
    (dict(y=np.array([0, 1, 1])), 'y has'),
    (dict(y_test=np.array([0, 1])), 'y_test has'),
    (dict(score_fn=[len]), 'score_fn'),
    (dict(score_fn={'a': 3}), 'score_fn'),
    (dict(dt=_DT('regression')), 'y: '),
    (dict(dt=_DT('multilabel')), 'y: '),
    (dict(y=np.array([1, 1, 1, 1])), 'y: '),
    (dict(batch_size=0), 'batch_size'),
    (dict(dt=None), 'dt_model'),
])
def test_refusals_name_their_argument(kwargs, match):
    from deeptables_b200 import deeptable
    X = pd.DataFrame({'a': [1, 2, 3, 4]})
    args = dict(dt=_DT(), X=X, y=np.array([0, 1, 0, 1]), X_test=X.head(3), y_test=np.array([0, 1, 1]),
                layers=['flatten_embeddings'], score_fn={})
    args.update(kwargs)
    with pytest.raises(ValueError, match=match):
        deeptable.probe_evaluate(**args)


def test_more_classes_than_the_kernels_take_are_refused():
    from deeptables_b200 import deeptable
    X = pd.DataFrame({'a': np.arange(65)})
    with pytest.raises(ValueError, match='y: a probe takes at most 64 classes'):
        deeptable.probe_evaluate(_DT('multiclass'), X, np.arange(65), X, np.arange(65), ['flatten_embeddings'])


def test_reachable_from_the_reference_module_path():
    from deeptables_b200 import deeptable, models
    assert models.deeptable.probe_evaluate is deeptable.probe_evaluate


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _worker(rank, world, port, results):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from deeptables_b200 import probe
        calls = []

        def fit(i):
            calls.append(i)
            return {'accuracy': 0.5 + i / 100, 'layer': i}

        results[rank] = (probe.deal(5, fit), calls)
    finally:
        dist.destroy_process_group()


def test_layers_are_dealt_over_ranks_and_every_rank_returns_the_whole_result():
    import torch.multiprocessing as mp
    from deeptables_b200 import probe
    world = 2
    with mp.Manager() as manager:
        results = manager.dict()
        mp.spawn(_worker, args=(world, _free_port(), results), nprocs=world, join=True)
        got = dict(results)
    want = probe.deal(5, lambda i: {'accuracy': 0.5 + i / 100, 'layer': i})
    for rank in range(world):
        lst, calls = got[rank]
        assert lst == want
        assert calls == list(range(rank, 5, world))
