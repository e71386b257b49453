"""Partial dependence, the parts that need no GPU: the restated grid against scikit-learn's ``_grid_from_X``, the
feature and argument checks, the block-sum order against math.fsum, and the C ABI of ``dtb_pdp_block_sums``."""
import ctypes
import math

import numpy as np
import pandas as pd
import pytest

import pdp_ref


def _X(rows=400, seed=0):
    g = np.random.default_rng(seed)
    return pd.DataFrame({'cont': g.normal(size=rows), 'few': g.choice([0.5, 1.5, 2.5], rows),
                         'cat': g.choice(list('abcde'), rows), 'code': g.integers(0, 7, rows),
                         'words': [f'w{i}' for i in g.integers(0, 150, rows)]})


def _ours(X, features, **kw):
    from deeptables_b200.utils import partial_dependence as P
    idx, keys = P.feature_indices(X.columns, features)
    is_cat = P.categorical_mask(X.columns, idx, kw.pop('categorical_features', None))
    custom = kw.pop('custom_values', {}) or {}
    custom = {i: custom[k] for i, k in enumerate(keys) if k in custom}
    return P.grid_from_columns([(X.columns[j], X.iloc[:, j]) for j in idx], kw.get('percentiles', (0.05, 0.95)),
                               is_cat, kw.get('grid_resolution', 100), custom)


def _sklearn(X, features, **kw):
    from sklearn.inspection._partial_dependence import _grid_from_X
    from deeptables_b200.utils import partial_dependence as P
    idx, keys = P.feature_indices(X.columns, features)
    is_cat = P.categorical_mask(X.columns, idx, kw.pop('categorical_features', None))
    custom = kw.pop('custom_values', {}) or {}
    custom = {i: custom[k] for i, k in enumerate(keys) if k in custom}
    return _grid_from_X(X.iloc[:, idx], kw.get('percentiles', (0.05, 0.95)), is_cat, kw.get('grid_resolution', 100),
                        custom)


def _same(a, b):
    assert len(a[1]) == len(b[1])
    for u, v in zip(a[1], b[1]):
        assert u.dtype == v.dtype and np.array_equal(u, v)
    assert a[0].dtype == b[0].dtype and np.array_equal(a[0], b[0])


@pytest.mark.parametrize('case', [
    dict(features='cont'),                                             # many uniques: quantile branch
    dict(features='cont', grid_resolution=7, percentiles=(0.1, 0.8)),
    dict(features='few'),                                              # fewer uniques than the resolution
    dict(features='cat', categorical_features=['cat']),                # string categories
    dict(features=2, categorical_features=[False, False, True, False, False]),
    dict(features='code', categorical_features=['code']),              # integer categories
    dict(features='words', grid_resolution=10, categorical_features=[4]),   # more categories than the resolution
    dict(features='cat', categorical_features=['cat'], custom_values={'cat': ['a', 'zz-unseen']}),
    dict(features='cont', custom_values={'cont': [-1.0, 0.0, 2.5]}),
    dict(features=['cat', 'cont'], categorical_features=['cat'], grid_resolution=5),    # two-way product
    dict(features=['code', 'few'], categorical_features=['code']),
    dict(features=[True, False, True, False, False], categorical_features=['cat'], grid_resolution=4),
], ids=lambda c: repr(c)[:60])
def test_grid_equals_scikit_learn(case):
    X = _X()
    _same(_ours(X, **case), _sklearn(X, **case))


def test_grid_errors_match_scikit_learn():
    X = _X()
    X['flat'] = np.r_[np.zeros(396), np.arange(1.0, 5.0)]
    for kw in (dict(features='flat', grid_resolution=3), dict(features='cont', percentiles=(0.5, 0.5)),
               dict(features='cont', percentiles=(0.1,)), dict(features='cont', percentiles=(-0.1, 0.5)),
               dict(features='cont', grid_resolution=1),
               dict(features='cont', custom_values={'cont': [[1.0, 2.0]]})):
        with pytest.raises(ValueError):
            _sklearn(X, **dict(kw))
        with pytest.raises(ValueError):
            _ours(X, **dict(kw))
    # a string column that needs the quantile branch: scikit-learn fails inside mquantiles
    with pytest.raises(TypeError):
        _sklearn(X, features='words', grid_resolution=10)
    with pytest.raises(ValueError, match="'words'"):
        _ours(X, features='words', grid_resolution=10)
    # NaN among strings cannot be sorted
    X.loc[3, 'cat'] = np.nan
    with pytest.raises(ValueError, match='mixed data types'):
        _sklearn(X, features='cat', categorical_features=['cat'])
    with pytest.raises(ValueError, match='mixed data types'):
        _ours(X, features='cat', categorical_features=['cat'])


def test_feature_indices():
    from deeptables_b200.utils.partial_dependence import feature_indices
    cols = ['a', 'b', 'c']
    assert feature_indices(cols, 'b') == ([1], ['b'])
    assert feature_indices(cols, 2) == ([2], [2])
    assert feature_indices(cols, ['c', 'a']) == ([2, 0], ['c', 'a'])
    assert feature_indices(cols, [False, True, True]) == ([1, 2], [1, 2])
    for bad in ('zz', 3, -1, ['a', 1], [], [True, False], [False, False, False], 1.5):
        with pytest.raises(ValueError, match='features'):
            feature_indices(cols, bad)


class _Model:
    task, model = 'binary', object()


class _FakeDeepTable:
    """What the checks read of a fitted DeepTable; any device work would fail on it."""

    def __init__(self, columns, task='binary'):
        from deeptables_b200 import deeptable
        self.preprocessor = deeptable.DefaultPreprocessor(deeptable.ModelConfig())
        self.preprocessor.feature_names_in_ = list(columns)
        self._model = _Model()
        self._model.task = task

    def get_model(self):
        return self._model


def test_refusals_fire_before_any_device_work():
    from deeptables_b200.utils.partial_dependence import partial_dependence
    X = _X().drop(columns=['words'])
    dt, reg = _FakeDeepTable(X.columns), _FakeDeepTable(X.columns, 'regression')
    cases = [
        (dt, dict(method='recursion'), 'method'),
        (dt, dict(method='fast'), 'method'),
        (dt, dict(response_method='decision_function'), 'response_method'),
        (reg, dict(response_method='predict_proba'), 'response_method'),
        (dt, dict(kind='mean'), 'kind'),
        (dt, dict(grid_resolution=1), 'grid_resolution'),
        (dt, dict(grid_resolution=2.5), 'grid_resolution'),
        (dt, dict(percentiles=(0.5, 0.2)), 'percentiles'),
        (dt, dict(percentiles=(0.1, 1.5)), 'percentiles'),
        (dt, dict(percentiles=(0.1, 0.5, 0.9)), 'percentiles'),
        (dt, dict(sample_weight=np.ones(3)), 'sample_weight'),
        (dt, dict(sample_weight=-np.ones(len(X))), 'sample_weight'),
        (dt, dict(sample_weight=np.zeros(len(X))), 'sample_weight'),
        (dt, dict(features='nope'), 'features'),
        (dt, dict(features=9), 'features'),
        (dt, dict(features='code'), "'code'"),                        # integer data that is not categorical
        (dt, dict(batch_size=0), 'batch_size'),
        (_FakeDeepTable(list(X.columns)[::-1]), {}, 'columns'),
        (_FakeDeepTable(list(X.columns) + ['extra']), {}, 'columns'),
    ]
    for model, kw, match in cases:
        args = dict(features='cont')
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            partial_dependence(model, X, **args)
    unfitted = _FakeDeepTable(X.columns)
    unfitted._model = None
    with pytest.raises(ValueError, match='dt_model'):
        partial_dependence(unfitted, X, 'cont')
    with pytest.raises(ValueError, match='feature_names'):
        partial_dependence(dt, X.to_numpy(), 'cont')


def test_block_order_restatement_against_fsum():
    g = np.random.default_rng(3)
    for rows, block in ((1, 1024), (1000, 1024), (5000, 1024), (3000, 64)):
        p = g.random((rows, 2), dtype=np.float32)
        w = g.random(rows) * 3
        for weight in (None, w):
            got = pdp_ref.block_order_mean(p, weight, block)
            ww = np.ones(rows) if weight is None else weight
            for c in range(2):
                want = math.fsum(ww * p[:, c].astype(np.float64)) / math.fsum(ww)
                assert abs(got[c] - want) <= 1e-14 * abs(want)
    # the lane and butterfly order on 64 rows, written out
    p = g.random((1, 64, 1), dtype=np.float32).astype(np.float64)
    lanes = [0.0 + p[0, l, 0] + p[0, l + 32, 0] for l in range(32)]
    for o in (16, 8, 4, 2, 1):
        lanes = [lanes[l] + lanes[l ^ o] for l in range(32)]
    assert pdp_ref.block_sums_restated(p.astype(np.float32), None, 1024)[0, 0, 0] == lanes[0]


def test_block_sums_symbol_is_declared_and_bound():
    from deeptables_b200 import _native
    sym = 'dtb_pdp_block_sums'
    assert sym in _native.declared_symbols() and sym in _native._SIGNATURES and hasattr(_native.lib, sym)


def test_block_sums_refuses_bad_arguments_without_a_gpu():
    """Argument checks run on the host before any launch."""
    from deeptables_b200 import _native as nat
    p = ctypes.c_void_p(16)
    for args in ((None, None, 1, 10, 1, 4, p), (p, None, 1, 10, 1, 4, None), (p, None, 0, 10, 1, 4, p),
                 (p, p, 1, 0, 1, 4, p), (p, p, 1, 10, 0, 4, p), (p, None, 1, 10, 1, 0, p),
                 (p, None, 2 ** 60, 10, 1, 1, p)):
        assert nat.lib.dtb_pdp_block_sums(*args, None) != 0
        assert 'invalid argument' in nat.last_error()
