"""Permutation feature importance, host side: select_features, the result's shape, dtype and numeric order, the mode /
metric / seed validation and routing, and the numpy restatement of the permutation keys."""
import numpy as np
import pytest

from importance_ref import perm_keys, permutation


def test_select_features_splits_at_threshold():
    from deeptables_b200.utils.feature_importance import select_features
    fi = np.array([['a', '0.5'], ['b', '0.0'], ['c', '-0.1'], ['d', '2e-05']])
    assert select_features(fi) == (['a', 'd'], ['b', 'c'])
    assert select_features(fi, threshold=0.1) == (['a'], ['b', 'c', 'd'])


def test_result_is_a_string_array_sorted_by_value(monkeypatch):
    from deeptables_b200 import importance
    from deeptables_b200.utils import feature_importance as F
    cols = ['x', 'y', 'z', 'w']
    dec = np.array([[9.0, 10.0, -1.0, 0.0], [9.0, 12.0, -3.0, 0.0]])

    def fake(dt_model, X, y, metric, **kw):
        assert metric == 'auc'                   # the name is lower-cased, as the reference does
        return importance.Result(cols, dec, 6, 1)
    monkeypatch.setattr(importance, 'score_decreases', fake)
    fi = F.get_score_importances(None, None, None, 'AUC', n_iter=2, mode='max')
    assert fi.shape == (4, 2) and fi.dtype.kind == 'U'
    # numeric order: 11 > 9 > 0 > -2 (the reference's string sort would put '9.0' before '11.0')
    assert fi[:, 0].tolist() == ['y', 'x', 'w', 'z']
    assert [float(v) for v in fi[:, 1]] == [11.0, 9.0, 0.0, -2.0]
    assert fi[2, 1] == '0.0'


def test_mode_is_checked_first():
    from deeptables_b200.utils.feature_importance import get_score_importances
    with pytest.raises(ValueError, match='Unsupported mode:avg'):
        get_score_importances(None, None, None, 'auc', mode='avg')


def test_sklearn_names_are_the_oof_metric_names():
    from deeptables_b200 import deeptable, importance
    assert set(importance.SKLEARN_METRICS) == set(deeptable._OOF_SKLEARN_NAMES)


@pytest.mark.parametrize('metric,proba', [('auc', True), ('AUC', True), ('roc_auc', True), ('log_loss', True),
                                          ('logloss', True), ('accuracy', False), ('f1', False), ('mse', False),
                                          ('r2', False), ('precision', True)])
def test_routing(metric, proba):
    from deeptables_b200 import importance
    assert importance.uses_probabilities(metric) is proba


def test_metric_validation():
    from deeptables_b200 import importance as I, metrics as M
    assert I.resolve_metric('f1', 'binary', 2).kind == I.F1
    assert I.resolve_metric('f1', 'multiclass', 3).kind == I.F1_MACRO
    assert I.resolve_metric('rmse', 'regression', None).kind == I.RMSE
    s = I.resolve_metric(M.Precision(thresholds=0.5), 'binary', 2)
    assert s.kind == I.STREAMING and s.name == 'precision'
    assert I.resolve_metric('precision', 'multilabel', 3).kind == I.STREAMING
    for bad, task in [('auc', 'multilabel'), ('accuracy', 'multilabel'), ('mse', 'binary'), ('auc', 'regression'),
                      ('no_such_metric', 'binary'), (len, 'binary')]:
        with pytest.raises(ValueError):
            I.resolve_metric(bad, task, 3)
    with pytest.raises(ValueError, match='vector'):
        I.resolve_metric(M.Precision(thresholds=[0.3, 0.6]), 'binary', 2)


def test_seed_validation():
    from deeptables_b200.analysis import draw_seed
    assert draw_seed(0) == 0 and draw_seed(2 ** 32 - 1) == 2 ** 32 - 1
    np.random.seed(3)
    a = draw_seed(None)
    np.random.seed(3)
    assert draw_seed(None) == a
    for bad in (-1, 2 ** 32, 1.5, True, 'x'):
        with pytest.raises(ValueError):
            draw_seed(bad)


def test_a_model_set_is_not_a_fitted_model():
    from deeptables_b200 import importance

    class ModelSet:
        def get_model(self):
            return [object()]
    with pytest.raises(ValueError, match='no fitted model'):
        importance.score_decreases(ModelSet(), None, None, 'auc')


def test_restated_keys_give_a_permutation_that_depends_on_every_input():
    k = perm_keys(7, 0, 3, 1000)
    assert k.dtype == np.int64 and np.array_equal(k & 0xFFFFFFFF, np.arange(1000))
    p = permutation(7, 0, 3, 1000)
    assert np.array_equal(np.sort(p), np.arange(1000))
    assert not np.array_equal(p, np.arange(1000))
    for other in [(8, 0, 3), (7, 1, 3), (7, 0, 4)]:
        assert not np.array_equal(permutation(*other, 1000), p)
    assert np.array_equal(permutation(7, 0, 3, 1000), p)
