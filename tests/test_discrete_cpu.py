"""auto_discrete without a GPU: the host quantile arithmetic against numpy and scikit-learn, the bin-count rule, the
preprocessor's columns (vocabularies, widths, order with and without gradient-boosted leaves), the refusals, the
unchanged output with the option off, and the C ABI of dtb_discretize."""
import numpy as np
import pandas as pd
import pytest

import discrete_ref as R

NBINS = range(2, 301)
LEVELS = np.concatenate([np.linspace(0, 100, nb + 1) for nb in NBINS])


def _D():
    from deeptables_b200 import discrete
    return discrete


def _host_percentiles(v, n):
    D = _D()
    out = []
    for nb in NBINS:
        prev, nxt, gamma = D.quantile_plan(n, nb)
        out.append(D.lerp(v[prev], v[nxt], gamma))
    return np.concatenate(out)


@pytest.mark.parametrize('first', [1, 501, 1001, 1501])
def test_quantile_arithmetic_equals_numpy_percentile(first):
    """Every n_bins in 2..300 and every n in 1..2000 (four chunks of n), bit for bit.  The chunk holds levels where
    n*q in float64 is not the exact n*k/n_bins (the rounding boundaries the virtual index depends on)."""
    g = np.random.default_rng(first)
    boundary = 0
    for n in range(first, first + 500):
        v = np.sort(g.normal(size=n).astype(np.float32)).astype(np.float64)
        want = np.percentile(v, LEVELS, method='averaged_inverted_cdf')
        got = _host_percentiles(v, n)
        assert np.array_equal(want.view(np.int64), got.view(np.int64)), n
        for nb in (3, 7, 10, 100):
            k = np.arange(nb + 1)
            vi = n * (np.linspace(0, 100, nb + 1) / 100) - 1
            boundary += int(np.sum((vi == np.floor(vi)) != ((n * k) % nb == 0)))
    assert boundary > 0


@pytest.mark.parametrize('n', [1_000_000, 2 ** 24 + 1, 3_000_017])
def test_quantile_arithmetic_at_large_n(n):
    D = _D()
    g = np.random.default_rng(n)
    v = np.sort(g.standard_t(3, size=n).astype(np.float32)).astype(np.float64)
    for nb in (2, 3, 7, 1000, 99_991, 100_000):
        want = np.percentile(v, np.linspace(0, 100, nb + 1), method='averaged_inverted_cdf')
        prev, nxt, gamma = D.quantile_plan(n, nb)
        assert np.array_equal(want.view(np.int64), D.lerp(v[prev], v[nxt], gamma).view(np.int64)), nb


def _column(kind, n, seed):
    g = np.random.default_rng(seed)
    return {'normal': lambda: g.normal(size=n),
            'zipf': lambda: np.minimum(g.zipf(1.6, size=n), 1000) * 0.25,
            'integers': lambda: g.integers(-20, 400, n),
            'rounded': lambda: np.round(g.exponential(size=n), 2),
            'two': lambda: g.choice([0.0, 1.0], n),
            'const': lambda: np.full(n, 0.5),
            'signed_zero': lambda: g.choice([-0.0, 0.0, 1.0, -1.0, 2.5], n),
            'scaled': lambda: (lambda x: (x - x.min()) / (np.ptp(x) or 1.0))(g.lognormal(size=n))}[kind]().astype(
        np.float32)


@pytest.mark.parametrize('kind', ['normal', 'zipf', 'integers', 'rounded', 'two', 'const', 'signed_zero', 'scaled'])
@pytest.mark.parametrize('n', [1, 2, 19, 1000, 54_321])
def test_edges_after_the_width_filter_equal_kbins_discretizer(kind, n):
    col = _column(kind, n, n)
    nb, got = R.host_edges(col)
    assert nb == R.n_bins(col)
    want = R.edges(col)
    assert got.dtype == np.float64 and np.array_equal(got, want), (got, want)
    assert np.array_equal(R.codes(got, col), R.kbins(col, nb).transform(col.astype(np.float64)[:, None])[:, 0])


def test_requested_bin_counts_past_the_rule():
    """Many more bins than distinct values: narrow bins are removed as scikit-learn removes them."""
    col = _column('zipf', 5000, 3)
    for nb in (2, 50, 400, 4999):
        assert np.array_equal(R.host_edges(col, nb)[1], R.edges(col, nb)), nb


def test_n_bins_rule():
    D = _D()
    assert [D.n_bins_for(u) for u in (0, 1, 19, 20, 29, 30, 1000, 1_000_003)] == [2, 2, 2, 2, 2, 3, 100, 100_000]


def _frame(rows=400, seed=0):
    g = np.random.default_rng(seed)
    X = pd.DataFrame({'c0': g.choice(list('abc'), rows), 'n0': g.normal(size=rows), 'c1': g.choice(list('xy'), rows),
                      'n1': g.integers(0, 1000, rows) * 0.5, 'n2': g.choice([1.0, 2.0], rows)})
    return X, g.integers(0, 2, rows)


@pytest.mark.parametrize('fixed,dim', [(True, 0), (True, 8), (False, 0)])
def test_columns_vocabularies_and_widths(monkeypatch, fixed, dim):
    from deeptables_b200 import deeptable
    R.patch_host(monkeypatch)
    X, y = _frame()
    pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig(auto_discrete=True, fixed_embedding_dim=fixed,
                                                              embeddings_output_dim=dim))
    Xt, _ = pre.fit_transform(X, y)
    names = ['n0_discrete', 'n1_discrete', 'n2_discrete']
    assert [c.name for c in pre.categorical_columns] == ['c0', 'c1'] + names
    assert pre.continuous_columns[0].column_names == ['n0', 'n1', 'n2'] and len(pre.continuous_columns) == 1
    assert Xt.columns.tolist() == ['c0', 'c1', 'n0', 'n1', 'n2'] + names
    Xe = pre._encode(X)
    vocab = [R.n_bins(Xe[c].to_numpy()) + 1 for c in ('n0', 'n1', 'n2')]
    assert [c.vocabulary_size for c in pre.categorical_columns[2:]] == vocab
    width = [(dim or 4) if fixed else min(4 * int(v ** 0.25), 20) for v in vocab]
    assert [c.embeddings_output_dim for c in pre.categorical_columns[2:]] == width
    for c, e in zip(('n0', 'n1', 'n2'), pre.discretizer_.bin_edges):
        assert np.array_equal(Xt[f'{c}_discrete'].to_numpy(), R.codes(e, Xe[c].to_numpy()))
        assert Xt[f'{c}_discrete'].dtype == np.int32
    assert pre.transform_X(X).equals(Xt)


def test_column_order_with_gradient_boosted_leaves(monkeypatch):
    """Raw categoricals, then <col>_discrete, then the leaf columns; the trees take the bin columns as categorical
    inputs, so their feature positions match the model's layout."""
    from deeptables_b200 import deeptable, gbm
    R.patch_host(monkeypatch)
    trees = gbm._trees_from_lists([{'feature': [2], 'bin': [0], 'threshold': [1.0], 'left': [-1], 'right': [-2],
                                    'gain': [1.0], 'values': [0.0, 0.1]}] * 2)
    monkeypatch.setattr(gbm.GbmLeavesEncoder, '_fit', lambda self, X, label, params, K: ([], trees))
    monkeypatch.setattr(gbm.GbmLeavesEncoder, 'leaves', lambda self, X: np.zeros((len(X), 2), np.int32))
    X, y = _frame()
    pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig(auto_discrete=True, apply_gbm_features=True))
    Xt, _ = pre.fit_transform(X, y)
    disc = ['n0_discrete', 'n1_discrete', 'n2_discrete']
    assert [c.name for c in pre.categorical_columns] == ['c0', 'c1'] + disc + ['lgbm_leaf_0', 'lgbm_leaf_1']
    assert Xt.columns.tolist() == ['c0', 'c1', 'n0', 'n1', 'n2'] + disc + ['lgbm_leaf_0', 'lgbm_leaf_1']
    assert pre.gbm_encoder_.cat_vars == ['c0', 'c1'] + disc and pre.gbm_encoder_.cont_vars == ['n0', 'n1', 'n2']
    assert pre.transform_X(X).columns.tolist() == Xt.columns.tolist()


@pytest.mark.parametrize('bad', [np.nan, np.inf, -np.inf])
def test_non_finite_values_are_refused_naming_the_column(monkeypatch, bad):
    from deeptables_b200 import deeptable
    R.patch_host(monkeypatch)
    X, y = _frame()
    Xb = X.copy()
    Xb.loc[7, 'n1'] = bad
    conf = deeptable.ModelConfig(auto_discrete=True, auto_imputation=False)
    with pytest.raises(ValueError, match=r"\['n1'\].*fit"):
        deeptable.DefaultPreprocessor(conf).fit_transform(Xb, y)
    pre = deeptable.DefaultPreprocessor(conf)
    pre.fit_transform(X, y)
    with pytest.raises(ValueError, match=r"\['n1'\].*transform"):
        pre.transform_X(Xb)


def test_clashing_names_are_refused(monkeypatch):
    from deeptables_b200 import deeptable
    R.patch_host(monkeypatch)
    X, y = _frame()
    conf = deeptable.ModelConfig(auto_discrete=True)
    with pytest.raises(ValueError, match='n0_discrete'):
        deeptable.DefaultPreprocessor(conf).fit_transform(X.assign(n0_discrete=1.0), y)
    pre = deeptable.DefaultPreprocessor(conf)
    pre.fit_transform(X.assign(c0_discrete=1.0, other_discrete=2.0), y)      # stems that are not continuous columns
    with pytest.raises(ValueError, match='n2_discrete'):
        pre.transform_X(X.assign(n2_discrete=1.0))


def test_option_off_leaves_the_output_unchanged():
    from deeptables_b200 import deeptable
    X, y = _frame()
    for conf in (deeptable.ModelConfig(), deeptable.ModelConfig(auto_discrete=False)):
        pre = deeptable.DefaultPreprocessor(conf)
        Xt, _ = pre.fit_transform(X, y)
        assert Xt.columns.tolist() == ['c0', 'c1', 'n0', 'n1', 'n2'] and pre.discretizer_ is None
        assert [c.name for c in pre.categorical_columns] == ['c0', 'c1']
        assert [(c.name, c.column_names) for c in pre.continuous_columns] == [('input_continuous_all',
                                                                               ['n0', 'n1', 'n2'])]
        assert Xt.equals(pre._encode(X)) and pre.transform_X(X).equals(Xt)
    pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig(auto_discrete=True))
    Xt, _ = pre.fit_transform(X[['c0', 'c1']], y)            # no continuous column: nothing to discretise
    assert pre.discretizer_ is None and Xt.columns.tolist() == ['c0', 'c1']


def test_dtb_discretize_signature_matches_the_header():
    """The C-ABI method of test_host_cpu: same arity and scalar class per argument as the header prototype."""
    import ctypes
    import re
    from deeptables_b200 import _native as nat
    with open(nat.HEADER_PATH) as f:
        text = re.sub(r'/\*.*?\*/', '', f.read(), flags=re.S)
    (args,) = re.findall(r'\bint\s+dtb_discretize\s*\(([^)]*)\)\s*;', text)
    kinds = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64}
    want = []
    for a in args.split(','):
        decl = a.strip()
        want.append(ctypes.c_void_p if '*' in decl else kinds[decl.rsplit(None, 1)[0].replace('const', '').strip()])
    res, argtypes = nat._SIGNATURES['dtb_discretize']
    assert res is ctypes.c_int and argtypes == want
    assert 'dtb_discretize' in nat.declared_symbols() and hasattr(nat.lib, 'dtb_discretize')
