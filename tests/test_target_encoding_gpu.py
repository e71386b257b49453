"""Target encoding on the GPU against scikit-learn 1.9's TargetEncoder and the numpy restatement tests/te_ref.py:
every output and encodings_ entry to 1e-12 * max(1, |x|); categories_, classes_, target_type_ and the folds exactly;
the same bits across runs, tile sizes and column groups."""
import numpy as np
import pandas as pd
import pytest
from sklearn.model_selection import KFold, StratifiedKFold
from sklearn.preprocessing import TargetEncoder as SkTargetEncoder

import te_ref

pytestmark = pytest.mark.gpu


def _enc(**kw):
    from deeptables_b200.preprocessing import TargetEncoder
    return TargetEncoder(**kw)


def _frame(rows=6000, seed=0):
    g = np.random.default_rng(seed)
    f = g.normal(size=rows).round(1)
    f[g.random(rows) < 0.05] = np.nan
    s = g.choice(['a', 'b', 'c', 'd', None], rows).astype(object)
    s[g.random(rows) < 0.03] = np.nan
    return pd.DataFrame({'zipf': np.minimum(g.zipf(1.3, rows), 400), 'few': g.integers(0, 5, rows), 'f': f, 's': s,
                         'b': g.random(rows) < 0.4, 'cat': pd.Categorical(g.choice([3, 1, 2], rows)),
                         'str': pd.Series(g.choice(['u', 'v', 'w'], rows), dtype='str')})


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
    bad = ~(np.abs(a - b) <= 1e-12 * np.maximum(1.0, np.abs(b)))
    assert not bad.any(), f'{bad.sum()} entries differ; worst {np.nanmax(np.abs(a - b))}'


def _same_cats(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and len(a) == len(b), (a, b)
        for u, v in zip(a, b):
            assert (u is v) or (u == v) or (te_ref._is_nan(u) and te_ref._is_nan(v)), (a, b)


def _check_fitted(ours, sk):
    _same_cats(ours.categories_, sk.categories_)
    assert ours.target_type_ == sk.target_type_
    if sk.classes_ is None:
        assert ours.classes_ is None
    else:
        np.testing.assert_array_equal(ours.classes_, sk.classes_)
    assert len(ours.encodings_) == len(sk.encodings_)
    for a, b in zip(ours.encodings_, sk.encodings_):
        _close(a, b)
    _close(np.atleast_1d(ours.target_mean_), np.atleast_1d(sk.target_mean_))
    assert ours.n_features_in_ == sk.n_features_in_
    np.testing.assert_array_equal(ours.get_feature_names_out(), sk.get_feature_names_out())


@pytest.mark.parametrize('smooth', ['auto', 0.0, 10.0])
@pytest.mark.parametrize('kind', ['binary', 'multiclass', 'continuous'])
def test_matches_sklearn(kind, smooth):
    X, Xt = _frame(), _frame(900, seed=5)
    Xt.loc[:10, 'zipf'] = 10 ** 6                         # unseen at transform
    Xt.loc[:5, 's'] = 'zz'
    y = _target(kind, len(X))
    sk = SkTargetEncoder(smooth=smooth, cv=_cv(kind))
    want = sk.fit_transform(X, y)
    ours = _enc(smooth=smooth, cv=_cv(kind))
    got = ours.fit_transform(X, y, _tile_rows=256)
    _close(got, want)
    _check_fitted(ours, sk)
    _close(ours.transform(Xt), sk.transform(Xt))
    refit = _enc(smooth=smooth).fit(X, y)
    _check_fitted(refit, sk)
    _close(refit.transform(Xt), sk.transform(Xt))


def test_shuffle_and_random_state_pick_sklearn_folds():
    X, y = _frame(3000), _target('binary', 3000)
    want = SkTargetEncoder(cv=StratifiedKFold(4, shuffle=True, random_state=7)).fit_transform(X, y)
    _close(_enc(cv=4, random_state=7).fit_transform(X, y), want)
    want = SkTargetEncoder(cv=StratifiedKFold(3)).fit_transform(X, y)
    _close(_enc(cv=3, shuffle=False).fit_transform(X, y), want)


def test_category_order_and_dtypes():
    X = pd.DataFrame({
        'i': [3, -1, 3, 2, 7, -1], 'f': [1.5, np.nan, -2.0, 1.5, np.nan, 0.0],
        's': pd.Series(['b', None, 'a', np.nan, 'b', 'c'], dtype=object),
        'b': [True, False, True, True, False, False], 'cat': pd.Categorical([2, 1, 2, np.nan, 1, 5]),
        'scat': pd.Categorical(['y', 'x', 'y', 'x', None, 'x']), 'f32': np.array([1, 2, 2, 1, 3, 3], np.float32),
    })
    y = [0, 1, 0, 1, 1, 0]
    _same_cats(_enc(cv=2).fit(X, y).categories_, SkTargetEncoder(cv=2).fit(X, y).categories_)
    arr = X[['s']].to_numpy()
    _same_cats(_enc(cv=2).fit(arr, y).categories_, SkTargetEncoder(cv=2).fit(arr, y).categories_)


@pytest.mark.parametrize('kind', ['binary', 'multiclass', 'continuous'])
def test_hard_columns(kind):
    """A category holding 60 % of the rows, a column with V close to N, a single-category column, across many tiles
    and several column groups."""
    rows = 40000
    g = np.random.default_rng(11)
    X = pd.DataFrame({'heavy': np.where(g.random(rows) < 0.6, 7, g.integers(0, 50, rows)),
                      'wide': g.permutation(rows) // 1 + (g.random(rows) < 0.05),
                      'one': np.full(rows, 'k', dtype=object), 'zipf': g.zipf(1.2, rows) % 5000})
    y = _target(kind, rows, seed=2)
    for smooth in ('auto', 0.0):
        sk = SkTargetEncoder(smooth=smooth, cv=_cv(kind))
        want = sk.fit_transform(X, y)
        ours = _enc(smooth=smooth, cv=_cv(kind))
        _close(ours.fit_transform(X, y, _tile_rows=64, _group_cols=3), want)
        _check_fitted(ours, sk)
        codes = np.stack([te_ref.codes_of(X.iloc[:, i].to_numpy(), c) for i, c in enumerate(sk.categories_)], axis=1)
        Y = te_ref.indicators(y, sk.target_type_, sk.classes_)
        ref = te_ref.cross_fit(codes, Y, [len(c) for c in sk.categories_],
                               te_ref.fold_ids(_cv(kind).split(X, y), rows), smooth)
        _close(ours.fit_transform(X, y, _group_cols=1, _workspace_bytes=1), ref)


def test_category_absent_from_a_fold():
    X = pd.DataFrame({'c': [7] * 4 + [1, 2] * 18, 'd': np.arange(40) % 3})
    for kind, y in (('binary', np.r_[[1, 0, 1, 1], np.tile([0, 1, 1, 0], 9)]),
                    ('continuous', np.linspace(-1, 2, 40) ** 2)):
        folds = [(np.arange(4, 40), np.arange(4))] + [
            (np.setdiff1d(np.arange(40), te), te) for te in np.array_split(np.arange(4, 40), 4)]
        for smooth in ('auto', 0.0, 3.0):
            sk = SkTargetEncoder(smooth=smooth, cv=folds)
            want = sk.fit_transform(X, y)
            ours = _enc(smooth=smooth, cv=folds)
            _close(ours.fit_transform(X, y), want)
            _check_fitted(ours, sk)
            _close(ours.fit_transform(X, y)[:4, 0], np.full(4, y[4:].mean()))


def test_given_categories_and_unknowns():
    X, Xt = _frame(3000), _frame(500, seed=9)
    cats = [np.array([1, 2, 3, 4, 5]), np.array([0, 1, 2]), np.array([-1.0, 0.0, 0.5, np.nan]),
            np.array(['c', 'a', None], dtype=object), np.array([False, True]), np.array([1, 3]),
            np.array(['w', 'u'], dtype=object)]
    y = _target('continuous', 3000)
    for smooth in ('auto', 2.0):
        sk = SkTargetEncoder(categories=cats, smooth=smooth, cv=_cv('continuous'))
        want = sk.fit_transform(X, y)
        ours = _enc(categories=cats, smooth=smooth, cv=_cv('continuous'))
        _close(ours.fit_transform(X, y), want)
        _check_fitted(ours, sk)
        _close(ours.transform(Xt), sk.transform(Xt))


def test_same_bits_across_runs_tiles_and_groups():
    rows = 30000
    g = np.random.default_rng(4)
    X = pd.DataFrame({f'c{i}': g.zipf(1.1 + 0.1 * i, rows) % (10 ** (i + 1)) for i in range(5)})
    X['s'] = g.choice(['p', 'q', 'r'], rows)
    y = g.standard_cauchy(rows)
    base = _enc(cv=_cv('continuous')).fit_transform(X, y)
    for tile, group, ws in ((4096, None, 1 << 30), (32, 2, 1 << 30), (1024, 1, 1), (96, 4, 1 << 20)):
        for _ in range(2):
            got = _enc(cv=_cv('continuous')).fit_transform(X, y, _tile_rows=tile, _group_cols=group,
                                                           _workspace_bytes=ws)
            assert got.tobytes() == base.tobytes(), (tile, group, ws)
    enc = _enc(cv=_cv('continuous')).fit(X, y)
    assert enc.transform(X).tobytes() == enc.transform(X, _group_cols=1).tobytes()


def test_set_output_pandas():
    X, y = _frame(2000), _target('multiclass', 2000)
    enc = _enc(cv=_cv('multiclass')).set_output(transform='pandas')
    out = enc.fit_transform(X, y)
    assert isinstance(out, pd.DataFrame) and list(out.columns) == list(enc.get_feature_names_out())
    assert out.index.equals(X.index)


def test_reference_helper_against_restatement():
    from deeptables_b200.preprocessing.utils import target_encoding
    rows = 5000
    g = np.random.default_rng(8)
    b = g.choice(['x', 'y', 'z', None], rows).astype(object)
    b[g.random(rows) < 0.02] = np.nan
    f = g.integers(0, 60, rows).astype(float)
    f[g.random(rows) < 0.05] = np.nan
    train = pd.DataFrame({'a': g.zipf(1.4, rows) % 300, 'keep': g.normal(size=rows), 'b': b, 'f': f,
                          'label': (g.random(rows) < 0.35).astype(int)}, index=g.permutation(rows) + 7)
    test = train.drop(columns='label').iloc[:700].copy()
    test.iloc[:20, 0] = 10 ** 6
    test.iloc[20:30, 2] = 'new'
    for smooth in (0.2, 5.0):
        t1, t2 = train.copy(), train.copy()
        want = te_ref.target_encoding(t1, 'label', test, feat_to_encode=['a', 'b', 'f'], smooth=smooth,
                                      random_state=9527)
        got = target_encoding(t2, 'label', test, feat_to_encode=['a', 'b', 'f'], smooth=smooth, _tile_rows=64)
        pd.testing.assert_frame_equal(t1, t2)
        assert got[2] == want[2] and list(got[0].columns) == want[2]
        pd.testing.assert_series_equal(got[3], want[3])
        for a, w in ((got[0], want[0]), (got[1], want[1])):
            assert a.index.equals(w.index)
            np.testing.assert_array_equal(a['keep'].to_numpy(), w['keep'].to_numpy())
            for c in ('a', 'b', 'f'):
                _close(a[c].to_numpy(), w[c].to_numpy())
    t = train.copy()
    out, none, feats, _ = target_encoding(t, 'label')
    assert none is None and feats == ['a', 'keep', 'b', 'f'] and out['keep'].dtype == np.float64
