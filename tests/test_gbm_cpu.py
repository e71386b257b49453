"""Gradient-boosted leaf features without a GPU: the restatement's split search against brute force, the binning rules,
gbm_params parsing, column naming and widths, and a sanity check that the restated booster is a real GBDT."""
import itertools

import numpy as np
import pandas as pd
import pytest

import gbm_ref as R


def _gbm():
    from deeptables_b200 import gbm
    return gbm


@pytest.mark.parametrize('seed', range(6))
@pytest.mark.parametrize('alpha,lam,msc', [(0.0, 0.0, 1), (0.3, 2.0, 3), (0.0, 1.0, 5)])
def test_split_search_equals_brute_force(seed, alpha, lam, msc):
    g = np.random.default_rng(seed)
    rows, nf = 40, 3
    B = g.integers(0, 5, size=(rows, nf)).astype(np.uint8)
    gq, hq = g.integers(-1000, 1000, rows), g.integers(1, 500, rows)
    n_bins = [5] * nf
    p = dict(reg_alpha=alpha, reg_lambda=lam, min_split_gain=0.0, min_child_samples=msc, min_child_weight=1e-3)
    sg, sh = 2.0 ** -10, 2.0 ** -10
    got = R.best_split(*R.histogram(B, np.arange(rows), gq, hq, 5), n_bins, p, sg, sh)

    def T(G):
        return np.sign(G) * max(abs(G) - alpha, 0.0)

    def term(G, H):
        return T(G) ** 2 / (H + lam)

    G, H = gq.sum() * sg, hq.sum() * sh
    best = None
    for f, t in itertools.product(range(nf), range(4)):
        left = B[:, f] <= t
        if left.sum() < msc or (~left).sum() < msc:
            continue
        GL, HL = gq[left].sum() * sg, hq[left].sum() * sh
        gain = term(GL, HL) + term(G - GL, H - HL) - term(G, H)
        if gain > 0 and (best is None or gain > best[0] + 1e-12):
            best = (gain, f, t)
    if best is None:
        assert got is None
    else:
        assert got[1:3] == best[1:3] and got[0] == pytest.approx(best[0], rel=1e-12)


@pytest.mark.parametrize('max_bin', [2, 15, 255])
@pytest.mark.parametrize('kind', ['few', 'many', 'ties', 'nan', 'const'])
def test_binning_properties(max_bin, kind):
    gbm = _gbm()
    g = np.random.default_rng(1)
    v = {'few': g.integers(0, 10, 5000).astype(np.float32),
         'many': g.normal(size=5000).astype(np.float32),
         'ties': np.round(g.exponential(size=5000), 1).astype(np.float32),
         'nan': np.where(g.random(5000) < 0.2, np.nan, g.normal(size=5000)).astype(np.float32),
         'const': np.full(5000, 3.0, np.float32)}[kind]
    e = gbm.bin_edges(v, max_bin)
    assert e.dtype == np.float32 and len(e) + 1 <= max_bin
    assert np.all(np.diff(e) > 0)
    b = R.bins(v[:, None], [e])[:, 0]
    finite = ~np.isnan(v)
    assert np.all(b[~finite] == len(e))
    for x in np.unique(v[finite]):                       # one value, one bin; x <= edge exactly when left of it
        bb = np.unique(b[v == x])
        assert len(bb) == 1
        assert np.all((x <= e) == (np.arange(len(e)) >= bb[0]))
    u = np.unique(v[finite])
    if len(u) <= max_bin:
        assert len(e) == max(len(u) - 1, 0)


def test_midpoint_never_reaches_the_upper_value():
    gbm = _gbm()
    a = np.float32(1.0)
    b = np.nextafter(a, np.float32(2))
    assert gbm.bin_edges(np.array([a, b], np.float32), 255).tolist() == [a]


def test_sample_rows_is_seeded_and_without_replacement():
    gbm = _gbm()
    a, b = gbm.sample_rows(10_000, 300, None), gbm.sample_rows(10_000, 300, None)
    assert np.array_equal(a, b) and len(np.unique(a)) == 300
    assert np.array_equal(gbm.sample_rows(50, 300, 7), np.arange(50))


def test_params_defaults_aliases_and_multiclass_rule():
    gbm = _gbm()
    p = gbm.resolve_params({}, 'binary')
    assert (p['n_estimators'], p['num_leaves'], p['min_child_samples'], p['max_bin']) == (100, 31, 20, 255)
    p = gbm.resolve_params({'num_iterations': 7, 'min_data_in_leaf': 3, 'min_sum_hessian_in_leaf': 0.5,
                            'lambda_l2': 1.0, 'lambda_l1': 0.1, 'seed': 4, 'n_jobs': 8, 'verbose': -1,
                            'verbosity': 0, 'boosting_type': 'gbdt', 'subsample': 1.0, 'colsample_bytree': 1.0},
                           'regression')
    assert (p['n_estimators'], p['min_child_samples'], p['min_child_weight'], p['reg_lambda'], p['reg_alpha'],
            p['random_state']) == (7, 3, 0.5, 1.0, 0.1, 4)
    assert gbm.resolve_params({}, 'multiclass', 5)['n_estimators'] == int(100 / 5) + 1
    assert gbm.resolve_params({}, 'multiclass', 3)['n_estimators'] == 34
    assert gbm.resolve_params({'n_estimators': 9}, 'multiclass', 5)['n_estimators'] == 9


@pytest.mark.parametrize('params', [{'boosting_type': 'dart'}, {'subsample': 0.8}, {'colsample_bytree': 0.5},
                                    {'objective': 'binary'}, {'class_weight': 'balanced'},
                                    {'categorical_feature': [0]}, {'max_bin': 511}, {'importance_type': 'gain'}])
def test_params_refused_by_name(params):
    with pytest.raises(NotImplementedError, match=list(params)[0]):
        _gbm().resolve_params(params, 'binary')


@pytest.mark.parametrize('params', [{'n_estimators': 0}, {'num_leaves': 1}, {'learning_rate': 0}, {'max_bin': 1},
                                    {'reg_lambda': -1}, {'min_child_samples': -1}, {'max_depth': 1.5},
                                    {'random_state': -3}, {'num_leaves': 5000}, {'n_estimators': 3,
                                                                                 'num_iterations': 4}])
def test_params_out_of_range(params):
    with pytest.raises(ValueError):
        _gbm().resolve_params(params, 'binary')


def test_fixed_point_sum_cannot_overflow():
    gbm = _gbm()
    for rows, m in [(1, 1.0), (19, 0.25), (1_000_000, 1.0), (3, 12345.678), (2 ** 20 + 1, 1e-30)]:
        s = gbm.fixed_shift(m, rows)
        assert rows * np.rint(m * 2.0 ** s) <= 2 ** 62
        assert rows * np.rint(m * 2.0 ** (s + 1)) > 2 ** 61        # and it uses the range
    assert gbm.fixed_shift(0.0, 10) == 0


def test_restated_booster_is_a_real_gbdt():
    """Training log loss within 2 % of scikit-learn's HistGradientBoostingClassifier at matched parameters."""
    from sklearn.ensemble import HistGradientBoostingClassifier
    gbm = _gbm()
    g = np.random.default_rng(3)
    n = 4000
    X = np.stack([g.normal(size=n), g.integers(0, 6, n), g.normal(size=n), g.uniform(size=n)], 1).astype(np.float32)
    z = X[:, 0] + (X[:, 1] == 2) - X[:, 2] * X[:, 3] + 0.5 * g.normal(size=n)
    y = (z > 0.3).astype(np.float32)
    p = gbm.resolve_params({'n_estimators': 30}, 'binary')
    edges = [gbm.bin_edges(X[:, j], p['max_bin']) for j in range(X.shape[1])]
    trees = R.fit(X, y, 'binary', 1, p, edges)
    s = np.full(n, np.log(y.mean() / (1 - y.mean())))
    for t in trees:
        s += np.asarray(t['values'], np.float64)[R.traverse(t, X, edges)]
    q = 1 / (1 + np.exp(-s))
    ours = -np.mean(y * np.log(q) + (1 - y) * np.log(1 - q))
    sk = HistGradientBoostingClassifier(max_iter=30, max_leaf_nodes=31, min_samples_leaf=20, l2_regularization=0,
                                        max_bins=255, early_stopping=False, learning_rate=0.1).fit(X, y)
    qs = sk.predict_proba(X)[:, 1]
    theirs = -np.mean(y * np.log(qs) + (1 - y) * np.log(1 - qs))
    assert abs(ours - theirs) <= 0.02 * theirs, (ours, theirs)
    # the partition's leaves are the traversal's on the training rows
    for t in trees:
        assert np.array_equal(t['leaf'], R.traverse(t, X, edges))


def test_leaf_columns_vocabularies_and_widths():
    """The preprocessor's columns from a fitted encoder (trees made by hand: no GPU needed)."""
    from deeptables_b200 import deeptable, gbm
    from deeptables_b200.metainfo import CategoricalColumn
    enc = gbm.GbmLeavesEncoder(['a'], ['b'], 'binary')
    enc.trees = gbm._trees_from_lists([{'feature': [], 'bin': [], 'threshold': [], 'left': [], 'right': [], 'gain': [],
                                        'values': [0.0]}] * 2 + [
        {'feature': [0] * 29, 'bin': [0] * 29, 'threshold': [0.0] * 29, 'left': [0] * 29, 'right': [0] * 29,
         'gain': [1.0] * 29, 'values': [0.0] * 30}])
    enc.new_columns = [f'lgbm_leaf_{i}' for i in range(3)]
    assert enc.new_columns == ['lgbm_leaf_0', 'lgbm_leaf_1', 'lgbm_leaf_2']
    assert enc.trees.num_leaves.tolist() == [1, 1, 30]
    for fixed, dim, want in [(True, 0, [4, 4, 4]), (True, 8, [8, 8, 8]), (False, 0, [4, 4, 8])]:
        conf = deeptable.ModelConfig(fixed_embedding_dim=fixed, embeddings_output_dim=dim)
        pre = deeptable.DefaultPreprocessor(conf)
        pre.categorical_columns = []
        d = (dim if dim > 0 else 4) if fixed else 0
        for name, leaves in zip(enc.new_columns, enc.trees.num_leaves):
            v = int(leaves)
            pre.categorical_columns.append(CategoricalColumn(name, v, d if fixed else min(4 * int(v ** 0.25), 20)))
        assert [c.embeddings_output_dim for c in pre.categorical_columns] == want
        assert [c.vocabulary_size for c in pre.categorical_columns] == [1, 1, 30]


def test_default_config_leaves_the_preprocessor_output_unchanged():
    from deeptables_b200 import deeptable
    g = np.random.default_rng(0)
    X = pd.DataFrame({'c': g.choice(list('abc'), 200), 'n': g.normal(size=200)})
    y = g.integers(0, 2, 200)
    pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig())
    Xt, _ = pre.fit_transform(X, y)
    assert Xt.columns.tolist() == ['c', 'n'] and pre.gbm_encoder_ is None
    assert [c.name for c in pre.continuous_columns] == ['input_continuous_all']


def test_multilabel_and_clashing_names_are_refused():
    from deeptables_b200 import deeptable
    g = np.random.default_rng(0)
    X = pd.DataFrame({'c': g.choice(list('abc'), 50), 'n': g.normal(size=50)})
    pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig(task='multilabel', apply_gbm_features=True))
    with pytest.raises(NotImplementedError, match='multilabel'):
        pre.fit_transform(X, g.integers(0, 2, (50, 3)))
    pre = deeptable.DefaultPreprocessor(deeptable.ModelConfig(apply_gbm_features=True))
    with pytest.raises(ValueError, match='lgbm_leaf_'):
        pre.fit_transform(X.assign(lgbm_leaf_0=1.0), g.integers(0, 2, 50))
