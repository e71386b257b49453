"""Kernel SHAP, host side: the coalition sampler against the restatement of shap's loops (budget and cap, enumerated
sizes, pairing, repeated draws, weights), varying-column detection, the constrained solve against numpy's least
squares, argument validation and the C ABI of the two kernels."""
import numpy as np
import pandas as pd
import pytest

import shap_ref


@pytest.mark.parametrize('M,nsamples,want', [(2, 'auto', 2), (5, 'auto', 30), (11, 'auto', 2046), (12, 'auto', 2072),
                                             (30, 'auto', 2108), (31, 'auto', 2110), (40, 'auto', 2128),
                                             (8, 100, 100), (8, 1000, 254), (35, 7, 7)])
def test_budget_rule_and_cap(M, nsamples, want):
    from deeptables_b200 import explain
    assert explain.budget(M, nsamples) == want == shap_ref.budget(M, nsamples)


@pytest.mark.parametrize('M,nsamples,seed', [(2, 'auto', 0), (3, 'auto', 1), (4, 'auto', 2), (7, 'auto', 3),
                                             (8, 40, 4), (9, 'auto', 5), (11, 'auto', 6), (12, 'auto', 7),
                                             (13, 300, 8), (16, 'auto', 9), (20, 'auto', 10), (39, 'auto', 11),
                                             (6, 13, 12), (10, 2000, 13)])
def test_sampler_equals_the_restated_loops(M, nsamples, seed):
    from deeptables_b200 import explain
    masks, weights = explain.sample_coalitions(M, nsamples, np.random.RandomState([seed, 3]))
    ref_masks, ref_weights = shap_ref.coalitions(M, nsamples, np.random.RandomState([seed, 3]))
    assert masks.dtype == bool and masks.shape == ref_masks.shape
    np.testing.assert_array_equal(masks, ref_masks.astype(bool))
    np.testing.assert_array_equal(weights, ref_weights)
    assert len(masks) <= explain.budget(M, nsamples)
    assert abs(weights.sum() - 1.0) < 1e-12
    sizes = masks.sum(1)
    assert sizes.min() >= 1 and sizes.max() <= M - 1
    assert len({m.tobytes() for m in masks}) == len(masks)           # repeated draws are merged into weights


def test_full_enumeration_has_every_coalition_at_the_shapley_kernel_weight():
    from math import comb
    from deeptables_b200 import explain
    for M in (2, 3, 6, 9, 11):
        masks, weights = explain.sample_coalitions(M, 'auto', np.random.RandomState(0))
        assert len(masks) == 2 ** M - 2
        s = masks.sum(1)
        kernel = (M - 1) / (np.array([comb(M, k) for k in s]) * s * (M - s))
        np.testing.assert_allclose(weights / weights[0], kernel / kernel[0], rtol=1e-12)


def test_enumerated_sizes_and_pairing():
    from deeptables_b200 import explain
    M = 20                                    # budget 2088: sizes 1 (40 with complements) and 2 (380) fit, 3 does not
    masks, weights = explain.sample_coalitions(M, 'auto', np.random.RandomState(1))
    s = masks.sum(1)
    assert len(masks) == 2088
    np.testing.assert_array_equal(s[:40], np.tile([1, 19], 20))
    np.testing.assert_array_equal(s[40:420], np.tile([2, 18], 190))
    np.testing.assert_array_equal(masks[0:40:2], ~masks[1:40:2])
    drawn = masks[420:]
    assert set(drawn.sum(1)) <= set(range(3, 18))
    i = 0
    while i < len(drawn):                     # a paired size (<= 9) is followed by its complement; size 10 is not
        if drawn[i].sum() <= 9:
            assert i + 1 == len(drawn) or np.array_equal(drawn[i + 1], ~drawn[i])
            i += 2
        else:
            assert drawn[i].sum() == 10
            i += 1
    assert weights[420:].max() > weights[420:].min()          # some draw was repeated
    np.testing.assert_allclose(weights[:420].sum() + weights[420:].sum(), 1.0, rtol=1e-12)


def test_varying_columns_rule():
    from deeptables_b200 import explain
    bg = pd.DataFrame({'s': ['a', 'a'], 's2': ['a', 'b'], 'f': [1.0, 1.0 + 1e-12], 'g': [1.0, 1.01],
                       'n': [np.nan, np.nan], 'n2': [np.nan, 0.5], 'i': [3, 3], 'o': ['x', 1.0]})
    cols = [bg[c].to_numpy() for c in bg.columns]
    x = np.array(['a', 'a', 1.0, 1.0, np.nan, np.nan, 3, 1.0], dtype=object)
    got = explain.varying_columns(x, cols).tolist()
    assert got == shap_ref.varying(x, bg.to_numpy(dtype=object)) == [1, 3, 5, 7]
    x2 = np.array(['b', 'a', 1.0 + 1e-9, 1.0, 0.0, 0.5, 4, 'x'], dtype=object)
    assert explain.varying_columns(x2, cols).tolist() == shap_ref.varying(x2, bg.to_numpy(dtype=object)) == \
        [0, 1, 3, 4, 5, 6, 7]


def test_solve_equals_lstsq_of_the_eliminated_system_and_shap():
    from deeptables_b200 import explain
    g = np.random.default_rng(0)
    for M in (2, 5, 12, 39):
        masks, weights = explain.sample_coalitions(M, 'auto', np.random.RandomState(M))
        values = g.normal(size=len(masks))
        fx, E = 1.7, 0.3
        phi = explain.solve(masks, weights, values, fx, E)
        Z = masks.astype(np.float64)
        Zt, y = Z[:, :-1] - Z[:, -1:], values - E - Z[:, -1] * (fx - E)
        sw = np.sqrt(weights)
        p, *_ = np.linalg.lstsq(Zt * sw[:, None], y * sw, rcond=None)
        np.testing.assert_allclose(phi[:-1], p, rtol=1e-9, atol=1e-12)
        assert abs(phi.sum() - (fx - E)) < 1e-12
        np.testing.assert_allclose(phi, shap_ref.solve(Z, weights, values, fx, E), rtol=1e-9, atol=1e-12)


def test_solve_recovers_an_additive_value_function():
    from deeptables_b200 import explain
    g = np.random.default_rng(1)
    M = 25
    a = g.normal(size=M)
    masks, weights = explain.sample_coalitions(M, 'auto', np.random.RandomState(2))
    E = 0.25
    phi = explain.solve(masks, weights, E + masks @ a, E + a.sum(), E)
    np.testing.assert_allclose(phi, a, atol=1e-10)


def test_argument_validation():
    from deeptables_b200 import explain
    from deeptables_b200.utils.shap import DeepTablesExplainer
    X = pd.DataFrame({'a': [1.0, 2.0]})
    for bad in (0, -1, 1.5, True, 'all', None):
        with pytest.raises(ValueError):
            explain.check_nsamples(bad)
    explain.check_nsamples('auto')
    explain.check_nsamples(5)
    for kw in ({'random_state': -1}, {'random_state': 2 ** 32}, {'random_state': 'x'}, {'batch_size': 0},
               {'batch_size': 2.0}, {'num_samples': 0}, {'num_samples': 1.5}):
        with pytest.raises(ValueError):
            DeepTablesExplainer(None, X, **kw)
    with pytest.raises(ValueError, match='no fitted model'):
        DeepTablesExplainer(None, X)

    class Unfitted:
        def get_model(self):
            return None
    with pytest.raises(ValueError, match='no fitted model'):
        DeepTablesExplainer(Unfitted(), X, num_samples=None)


def test_kernels_are_declared_and_bound():
    from deeptables_b200 import _native
    for sym in ('dtb_shap_compose', 'dtb_shap_means'):
        assert sym in _native.declared_symbols() and sym in _native._SIGNATURES and hasattr(_native.lib, sym)


def test_symmetric_columns_get_equal_values_in_the_exact_case():
    """Columns 0 and 1 enter the value function only through how many of them a coalition holds."""
    from deeptables_b200 import explain
    M = 7
    masks, weights = explain.sample_coalitions(M, 'auto', np.random.RandomState(0))
    a = np.array([0.0, 0.0, 0.3, -1.2, 0.7, 2.0, 0.1])

    def v(m):
        pair = m[..., 0].astype(float) + m[..., 1]
        return 0.5 + m @ a + 1.5 * pair ** 2 - 0.4 * pair * m[..., 3]
    full = np.ones(M, bool)
    phi = explain.solve(masks, weights, v(masks), v(full), v(np.zeros(M, bool)))
    assert abs(phi[0] - phi[1]) < 1e-12
    want = shap_ref.exact_shapley(lambda S: v(np.isin(np.arange(M), list(S))), M)
    np.testing.assert_allclose(phi, want, atol=1e-12)
