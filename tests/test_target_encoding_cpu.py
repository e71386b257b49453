"""Target encoding, the parts that need no GPU: the numpy restatement (tests/te_ref.py) against the installed
scikit-learn, scikit-learn's category order, every refusal (all raised before any device work), and the reference
helper's quirks on the restatement."""
import warnings

import numpy as np
import pandas as pd
import pytest
from sklearn.model_selection import KFold, StratifiedKFold
from sklearn.preprocessing import TargetEncoder as SkTargetEncoder

import te_ref


def _frame(rows=3000, seed=0):
    g = np.random.default_rng(seed)
    f = g.normal(size=rows).round(1)
    f[g.random(rows) < 0.05] = np.nan
    s = g.choice(['a', 'b', 'c', 'd', None], rows).astype(object)
    s[g.random(rows) < 0.03] = np.nan
    return pd.DataFrame({'zipf': np.minimum(g.zipf(1.3, rows), 400), 'few': g.integers(0, 5, rows), 'f': f, 's': s})


def _target(kind, rows, seed=1):
    g = np.random.default_rng(seed)
    if kind == 'binary':
        return np.where(g.random(rows) < 0.3, 'yes', 'no')
    if kind == 'multiclass':
        return g.integers(0, 4, rows)
    return g.normal(size=rows) * 3 + 1


def _cv(kind):
    return (KFold if kind == 'continuous' else StratifiedKFold)(5, shuffle=True, random_state=0)


def _close(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape
    np.testing.assert_array_less(np.abs(a - b), 1e-12 * np.maximum(1.0, np.abs(b)) + 1e-300)


@pytest.mark.parametrize('smooth', ['auto', 0.0, 10.0])
@pytest.mark.parametrize('kind', ['binary', 'multiclass', 'continuous'])
def test_restatement_matches_sklearn(kind, smooth):
    X, Xt = _frame(), _frame(700, seed=5)
    Xt.loc[:10, 'zipf'] = 10 ** 6                        # unseen at transform
    y = _target(kind, len(X))
    sk = SkTargetEncoder(smooth=smooth, cv=_cv(kind))
    want = sk.fit_transform(X, y)
    want_t = sk.transform(Xt)
    codes = np.stack([te_ref.codes_of(X.iloc[:, i].to_numpy(), c) for i, c in enumerate(sk.categories_)], axis=1)
    Vs = [len(c) for c in sk.categories_]
    Y = te_ref.indicators(y, sk.target_type_, sk.classes_)
    fold = te_ref.fold_ids(_cv(kind).split(X, y), len(X))
    _close(te_ref.cross_fit(codes, Y, Vs, fold, smooth), want)
    encs, prior = te_ref.fit(codes, Y, Vs, smooth)
    for a, b in zip(encs, sk.encodings_):
        _close(a, b)
    _close(prior, np.atleast_1d(sk.target_mean_))
    tcodes = np.stack([te_ref.codes_of(Xt.iloc[:, i].to_numpy(), c) for i, c in enumerate(sk.categories_)], axis=1)
    _close(te_ref.transform(tcodes, encs, prior), want_t)


def test_restatement_absent_category_gets_the_fold_mean():
    # category 7 lives only in fold 0: its rows are encoded by the other folds, where it has no row
    X = pd.DataFrame({'c': [7] * 4 + [1, 2] * 18})
    y = np.r_[[1, 0, 1, 1], np.tile([0, 1, 1, 0], 9)]
    folds = [(np.arange(4, 40), np.arange(4))] + [
        (np.setdiff1d(np.arange(40), te), te) for te in np.array_split(np.arange(4, 40), 4)]
    for smooth in ('auto', 0.0, 3.0):
        want = SkTargetEncoder(smooth=smooth, cv=folds).fit_transform(X, y)
        codes = te_ref.codes_of(X['c'].to_numpy(), [1, 2, 7])[:, None]
        got = te_ref.cross_fit(codes, y[:, None].astype(float), [3], te_ref.fold_ids(folds, 40), smooth)
        _close(got, want)
        np.testing.assert_array_equal(want[:4, 0], y[4:].mean())


def test_sklearn_category_order():
    """The categories_ the device path must reproduce: sorted; NaN last; None before NaN; bool and category dtypes."""
    X = pd.DataFrame({
        'i': [3, -1, 3, 2, 7, -1],
        'f': [1.5, np.nan, -2.0, 1.5, np.nan, 0.0],
        's': pd.Series(['b', None, 'a', np.nan, 'b', 'c'], dtype=object),
        'b': [True, False, True, True, False, False],
        'cat': pd.Categorical([2, 1, 2, np.nan, 1, 5]),
        'scat': pd.Categorical(['y', 'x', 'y', 'x', None, 'x']),
    })
    sk = SkTargetEncoder(cv=2).fit(X, [0, 1, 0, 1, 1, 0])
    want = [np.array([-1, 2, 3, 7]), np.array([-2.0, 0.0, 1.5, np.nan]),
            np.array(['a', 'b', 'c', None, np.nan], dtype=object), np.array([False, True]),
            np.array([1.0, 2.0, 5.0, np.nan]), np.array(['x', 'y', np.nan], dtype=object)]
    for got, w in zip(sk.categories_, want):
        assert got.dtype == w.dtype
        assert len(got) == len(w)
        for a, b in zip(got, w):
            assert (a is b) or (a == b) or (te_ref._is_nan(a) and te_ref._is_nan(b))


# ---- refusals: each raises ValueError naming the argument, before any device work ----------------------------------

def _enc(**kw):
    from deeptables_b200.preprocessing import TargetEncoder
    return TargetEncoder(**kw)


@pytest.mark.parametrize('call, match', [
    (lambda: _enc().fit_transform(_frame(50), np.zeros(49)), 'lengths'),
    (lambda: _enc().fit(_frame(50), np.zeros((50, 2))), 'multilabel'),
    (lambda: _enc().fit(_frame(50), np.r_[np.nan, np.zeros(49)]), 'NaN'),
    (lambda: _enc().fit(_frame(50), np.array([None] + ['a'] * 49, dtype=object)), 'NaN'),
    (lambda: _enc(smooth=-1.0).fit(_frame(50), np.arange(50) % 2), 'smooth'),
    (lambda: _enc(smooth='high').fit(_frame(50), np.arange(50) % 2), 'smooth'),
    (lambda: _enc(target_type='binary').fit(_frame(50), np.arange(50) % 3), 'target_type'),
    (lambda: _enc(target_type='multiclass').fit(_frame(50), np.arange(50) % 2), 'target_type'),
    (lambda: _enc(target_type='continuous').fit(_frame(50), np.array(['a', 'b'] * 25)), 'target_type'),
    (lambda: _enc(target_type='other').fit(_frame(50), np.arange(50) % 2), 'target_type'),
    (lambda: _enc(categories=[[1, 2]]).fit(_frame(50), np.arange(50) % 2), 'categories'),
    (lambda: _enc(categories=[[3, 1, 2], [0], [0.0], ['a']]).fit(_frame(50), np.arange(50) % 2), 'categories'),
    (lambda: _enc(cv=[(np.arange(25, 50), np.arange(25)), (np.arange(20), np.arange(20, 50))]).fit_transform(
        _frame(50), np.arange(50) % 2), 'cv'),
    (lambda: _enc(cv=[(np.arange(25, 50), np.arange(25)), (np.arange(25), np.arange(24, 50))]).fit_transform(
        _frame(50), np.arange(50) % 2), 'cv'),
    (lambda: _enc(cv=[(np.arange(40, 50), np.arange(25)), (np.arange(25), np.arange(25, 50))]).fit_transform(
        _frame(50), np.arange(50) % 2), 'cv'),
])
def test_refusals(call, match):
    with pytest.raises(ValueError, match=match):
        call()


def _fitted():
    enc = _enc()
    enc.n_features_in_ = 4
    enc.feature_names_in_ = np.array(['zipf', 'few', 'f', 's'], dtype=object)
    enc.target_type_, enc.classes_ = 'binary', np.array([0, 1])
    enc.categories_ = [np.array([1])] * 4
    enc.encodings_ = [np.array([0.5])] * 4
    enc.target_mean_ = np.float64(0.5)
    return enc


def test_transform_refuses_other_columns():
    enc = _fitted()
    with pytest.raises(ValueError, match='X has 3 features'):
        enc.transform(_frame(20).iloc[:, :3])
    with pytest.raises(ValueError, match='feature names'):
        enc.transform(_frame(20).rename(columns={'s': 't'}))
    with pytest.raises(ValueError, match='not fitted'):
        _enc().transform(_frame(20))


def test_params_and_feature_names():
    enc = _enc(smooth=2.0, cv=3, shuffle=False)
    assert enc.get_params() == {'categories': 'auto', 'target_type': 'auto', 'smooth': 2.0, 'cv': 3,
                                'shuffle': False, 'random_state': None}
    fitted = _fitted()
    assert list(fitted.get_feature_names_out()) == ['zipf', 'few', 'f', 's']
    fitted.target_type_, fitted.classes_ = 'multiclass', np.array(['p', 'q', 'r'])
    assert list(fitted.get_feature_names_out())[:4] == ['zipf_p', 'zipf_q', 'zipf_r', 'few_p']
    del fitted.feature_names_in_
    assert list(fitted.get_feature_names_out())[-1] == 'x3_r'


def test_helper_refusals():
    from deeptables_b200.preprocessing.utils import target_encoding
    df = _frame(50).assign(y=np.array(['u', 'v'] * 25))
    with pytest.raises(ValueError, match='numeric'):
        target_encoding(df, 'y')
    with pytest.raises(ValueError, match='feat_to_encode'):
        target_encoding(_frame(50).assign(y=np.arange(50) % 2), 'y', feat_to_encode=['nope'])
    with pytest.raises(ValueError, match='smooth'):
        target_encoding(_frame(50).assign(y=np.arange(50) % 2), 'y', smooth=-1.0)


def test_no_future_warning_for_shuffle_and_random_state():
    with warnings.catch_warnings():
        warnings.simplefilter('error')
        _enc(shuffle=True, random_state=0).get_params()


# ---- the reference helper's quirks, on the restatement ------------------------------------------------------------

def test_reference_helper_quirks():
    g = np.random.default_rng(3)
    rows = 400
    train = pd.DataFrame({'a': g.integers(0, 30, rows), 'keep': g.normal(size=rows),
                          'b': g.choice(['x', 'y', None], rows), 'label': g.integers(0, 2, rows)},
                         index=g.permutation(rows) + 1000)
    test = pd.DataFrame({'a': [1, 2, 999], 'keep': [0.0, 1.0, 2.0], 'b': ['x', None, 'zz']})
    before = train.copy()
    out, tout, feats, target = te_ref.target_encoding(train, 'label', test, feat_to_encode=['a', 'b'], smooth=0.5)
    assert list(train.columns) == ['a', 'keep', 'b']                   # target popped in place
    assert train.index.is_monotonic_increasing                         # sorted in place
    assert target.name == 'label' and target.index.equals(train.index)
    np.testing.assert_array_equal(target.to_numpy(), before.sort_index()['label'].to_numpy())
    assert feats == ['a', 'keep', 'b'] and list(out.columns) == feats and out.index.equals(train.index)
    np.testing.assert_array_equal(out['keep'].to_numpy(), train['keep'].to_numpy())     # passes through
    assert out['a'].dtype == np.float64 and out['b'].dtype == np.float64
    prior = target.mean()
    assert tout['a'].iloc[2] == prior and tout['b'].iloc[1] == prior and tout['b'].iloc[2] == prior
    np.testing.assert_array_equal(tout['keep'].to_numpy(), test['keep'].to_numpy())


@pytest.mark.parametrize('smooth', ['auto', 2.0])
def test_restatement_given_categories_matches_sklearn(smooth):
    """Rows outside given categories: scikit-learn fits them as the first category, and fit_transform gives each of
    them the last fold's mean."""
    X, Xt = _frame(), _frame(500, seed=9)
    cats = [np.array([1, 2, 3, 4, 5]), np.array([0, 1, 2]), np.array([-1.0, 0.0, 0.5, np.nan]),
            np.array(['c', 'a', None], dtype=object)]
    y = _target('continuous', len(X))
    sk = SkTargetEncoder(categories=cats, smooth=smooth, cv=_cv('continuous'))
    want = sk.fit_transform(X, y)
    codes = np.stack([te_ref.codes_of(X.iloc[:, i].to_numpy(), c) for i, c in enumerate(cats)], axis=1)
    assert (codes < 0).any(axis=0).all()
    Vs, Y = [len(c) for c in cats], y[:, None]
    _close(te_ref.cross_fit(codes, Y, Vs, te_ref.fold_ids(_cv('continuous').split(X, y), len(X)), smooth), want)
    encs, prior = te_ref.fit(codes, Y, Vs, smooth)
    for a, b in zip(encs, sk.encodings_):
        _close(a, b)
    tcodes = np.stack([te_ref.codes_of(Xt.iloc[:, i].to_numpy(), c) for i, c in enumerate(cats)], axis=1)
    _close(te_ref.transform(tcodes, encs, prior), sk.transform(Xt))
