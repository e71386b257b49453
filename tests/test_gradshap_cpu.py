"""Expected gradients, host side: the draws, the numpy restatement of the interpolated inputs and of the reductions,
the refusals (which fire before any device work), the background rule and the C ABI of the kernels."""
import ctypes

import numpy as np
import pandas as pd
import pytest

import gradshap_ref

SYMBOLS = ('dtb_gradshap_compose', 'dtb_gradshap_reduce', 'dtb_gradshap_means', 'dtb_gradshap_output_grad',
           'dtb_batchnorm_infer_bwd', 'dtb_linear_dense_grad')


def test_draws_per_row_equal_the_restatement():
    from deeptables_b200 import explain
    for seed, i, n, bg in ((0, 0, 200, 100), (7, 12345, 37, 1), (2 ** 32 - 1, 3, 4096, 50)):
        j, a = explain.gradient_draws(seed, i, n, bg)
        rj, ra = gradshap_ref.draws(seed, i, n, bg)
        assert j.dtype == np.int32 and a.dtype == np.float32 and len(j) == len(a) == n
        np.testing.assert_array_equal(j, rj)
        np.testing.assert_array_equal(a, ra)
        assert j.min() >= 0 and j.max() < bg
        assert a.min() >= 0 and a.max() < 1
        assert np.all(a * np.float32(2 ** 24) == np.floor(a * np.float32(2 ** 24)))     # exact steps of 2^-24
    # a reseeded generator gives the same draws, whatever it drew before
    rng = np.random.RandomState(99)
    rng.random_sample(7)
    for i in (4, 0, 4):
        for got, want in zip(explain.gradient_draws(3, i, 50, 20, rng), gradshap_ref.draws(3, i, 50, 20)):
            np.testing.assert_array_equal(got, want)
    # a row's draws do not depend on the other rows drawn with it
    j0, _ = explain.gradient_draws(5, 9, 64, 30)
    assert not np.array_equal(j0, explain.gradient_draws(5, 10, 64, 30)[0])
    assert not np.array_equal(j0, explain.gradient_draws(6, 9, 64, 30)[0])


def test_draws_cover_the_background_uniformly():
    from deeptables_b200 import explain
    j, a = explain.gradient_draws(1, 0, 200_000, 10)
    counts = np.bincount(j, minlength=10)
    assert np.abs(counts / 20_000 - 1).max() < 0.03
    assert abs(a.mean() - 0.5) < 0.005


def test_composition_restates_one_rounding_per_operation():
    g = np.random.default_rng(0)
    vocab, dims, dmax = [5, 7, 3], [4, 2, 4], 4
    offs = np.concatenate([[0], np.cumsum(vocab)])
    table = g.normal(size=(offs[-1], dmax)).astype(np.float32)
    for f, d in enumerate(dims):
        table[offs[f]:offs[f + 1], d:] = 0
    x_cat = np.stack([g.integers(0, v, 6) for v in vocab], 1).astype(np.int32)
    bg_cat = np.stack([g.integers(0, v, 4) for v in vocab], 1).astype(np.int32)
    x_cat[0, 1] = 99                                      # out of range: reads as zeros
    x_cont, bg_cont = g.normal(size=(6, 2)).astype(np.float32), g.normal(size=(4, 2)).astype(np.float32)
    xi = np.array([0, 0, 1, 5, 3], np.int32)
    bi = np.array([0, 3, 1, 2, 2], np.int32)
    alpha = np.array([0.0, 0.25, 0.7, 1 - 2 ** -24, 0.5], np.float32)
    emb, cont = gradshap_ref.compose(x_cat, x_cont, bg_cat, bg_cont, table, offs, dims, xi, bi, alpha)
    for p in range(5):
        for f in range(3):
            for d in range(dmax):
                idx = x_cat[xi[p], f]
                ei = table[offs[f] + idx, d] if idx < vocab[f] and d < dims[f] else np.float32(0)
                ej = table[offs[f] + bg_cat[bi[p], f], d] if d < dims[f] else np.float32(0)
                want = np.float32(ej + np.float32(alpha[p] * np.float32(ei - ej)))
                assert emb[p, f, d].tobytes() == want.tobytes()
        for c in range(2):
            xv, bv = x_cont[xi[p], c], bg_cont[bi[p], c]
            assert cont[p, c].tobytes() == np.float32(bv + np.float32(alpha[p] * np.float32(xv - bv))).tobytes()
    np.testing.assert_array_equal(emb[0], gradshap_ref.rows_of(table, offs, bg_cat[[0]], dims)[0])   # alpha 0 is b

    # the per-pair values: a zero difference contributes exactly 0, even against a non-finite gradient
    g_emb = g.normal(size=emb.shape).astype(np.float32)
    g_cont = g.normal(size=cont.shape).astype(np.float32)
    xi2, bi2 = np.array([2, 2], np.int32), np.array([0, 1], np.int32)
    x_cont2 = x_cont.copy()
    x_cont2[2] = bg_cont[1]
    x_cat2 = x_cat.copy()
    x_cat2[2] = bg_cat[1]
    ge, gc = g_emb[:2].copy(), g_cont[:2].copy()
    ge[1] = np.inf
    gc[1] = np.nan
    v = gradshap_ref.reduce(x_cat2, x_cont2, bg_cat, bg_cont, table, offs, dims, xi2, bi2, ge, gc)
    assert np.all(v[1] == 0) and np.all(np.isfinite(v[0]))
    m = gradshap_ref.means(np.arange(12, dtype=np.float64).reshape(6, 2), 2, 3)
    np.testing.assert_array_equal(m, [[2.0, 3.0], [8.0, 9.0]])


class _Config:
    def __init__(self, **kw):
        self.apply_gbm_features = kw.get('apply_gbm_features', False)
        self.auto_discrete = kw.get('auto_discrete', False)


class _FakeDeepTable:
    def __init__(self, **kw):
        self.config = _Config(**kw)

    def get_model(self):
        return None


def test_refusals_fire_before_any_device_work():
    from deeptables_b200 import explain
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    X = pd.DataFrame({'a': [1.0, 2.0], 'b': ['x', 'y']})
    for kw, match in (({'random_state': -1}, 'random_state'), ({'random_state': 2 ** 32}, 'random_state'),
                      ({'random_state': 1.5}, 'random_state'), ({'batch_size': 0}, 'batch_size'),
                      ({'num_samples': 0}, 'num_samples')):
        with pytest.raises(ValueError, match=match):
            DeepTablesGradientExplainer(_FakeDeepTable(), X, **kw)
    for option in ('apply_gbm_features', 'auto_discrete'):
        with pytest.raises(NotImplementedError, match=option):
            DeepTablesGradientExplainer(_FakeDeepTable(**{option: True}), X)
    with pytest.raises(ValueError, match='no fitted model'):
        DeepTablesGradientExplainer(_FakeDeepTable(), X)

    class _Bg:
        columns = ['a', 'b']
        cols = 1
    ex = DeepTablesGradientExplainer.__new__(DeepTablesGradientExplainer)
    ex.feature_names, ex._background, ex.random_state, ex.batch_size = ['a', 'b'], _Bg(), 0, 16
    for bad in (0, -3, 2.0, True, 'auto', None):
        with pytest.raises(ValueError, match='nsamples'):
            ex.get_shap_values(X, nsamples=bad)
    with pytest.raises(ValueError, match='X_to_explain'):
        ex.get_shap_values(X[['a']], nsamples=4)
    with pytest.raises(ValueError, match='X_to_explain'):
        ex.get_shap_values(X[['b', 'a']], nsamples=4)
    with pytest.raises(ValueError, match='nsamples'):
        explain.gradient_values(_Bg(), X, nsamples=0)
    with pytest.raises(ValueError, match='batch_size'):
        explain.gradient_values(_Bg(), X, nsamples=3, batch_size=0)


def test_background_rule_is_the_kernel_explainers():
    from sklearn.utils import resample
    from deeptables_b200.utils import shap as S
    X = pd.DataFrame({'a': np.arange(30.0), 'b': [str(i) for i in range(30)]})
    pd.testing.assert_frame_equal(S._background_rows(X, 7), resample(X, n_samples=7, random_state=0, replace=False))
    assert S._background_rows(X, None) is X and S._background_rows(X, 30) is X and S._background_rows(X, 99) is X


def test_kernels_are_declared_and_bound():
    from deeptables_b200 import _native
    for sym in SYMBOLS:
        assert sym in _native.declared_symbols() and sym in _native._SIGNATURES and hasattr(_native.lib, sym)


def test_kernels_refuse_bad_arguments_without_a_gpu():
    """Argument checks run on the host before any launch."""
    from deeptables_b200 import _native as nat
    p = ctypes.c_void_p(16)
    t8 = (p, p, p, p, p, p, p, 4)                     # x_cat, x_cont, bg_cat, bg_cont, table, offsets, col offsets, dim
    compose = [
        t8 + (None, p, p, 10, 2, 3, 1, p, p),            # NULL x_index
        t8 + (p, p, None, 10, 2, 3, 1, p, p),            # NULL alpha
        t8 + (p, p, p, 0, 2, 3, 1, p, p),                # no pairs
        t8 + (p, p, p, 10, 0, 0, 1, p, p),               # no columns
        t8 + (p, p, p, 10, 2, 3, 1, None, p),            # NULL out_emb with fields
        t8 + (p, p, p, 10, 2, 3, 1, p, None),            # NULL out_cont with conts
        (p, p, p, p, p, p, p, 0) + (p, p, p, 10, 2, 3, 1, p, p),    # table width 0
        t8 + (p, p, p, 10, 2, 3, 2, p, p),               # bad layout flag
    ]
    for args in compose:
        assert nat.lib.dtb_gradshap_compose(*args, None) != 0
        assert 'invalid argument' in nat.last_error()
    reduce = [
        t8 + (None, p, 10, 2, 3, p, p, p),
        t8 + (p, p, 10, 2, 3, p, p, None),
        t8 + (p, p, -1, 2, 3, p, p, p),
        t8 + (p, p, 10, 2, 3, None, p, p),
        t8 + (p, p, 10, 2, 3, p, None, p),
    ]
    for args in reduce:
        assert nat.lib.dtb_gradshap_reduce(*args, None) != 0
        assert 'invalid argument' in nat.last_error()
    for args in ((None, 1, 1, 1, p), (p, 0, 1, 1, p), (p, 1, 0, 1, p), (p, 1, 1, 0, p), (p, 1, 1, 1, None)):
        assert nat.lib.dtb_gradshap_means(*args, None) != 0
        assert 'invalid argument' in nat.last_error()
    for args in ((None, 4, 2, 0, 1, p), (p, 4, 2, 2, 1, p), (p, 4, 2, -1, 1, p), (p, 4, 2, 0, 3, p), (p, 0, 2, 0, 1, p)):
        assert nat.lib.dtb_gradshap_output_grad(*args, None) != 0
        assert 'invalid argument' in nat.last_error()
    assert nat.lib.dtb_batchnorm_infer_bwd(None, p, p, p, 4, 2, 1e-3, None) != 0
    assert nat.lib.dtb_batchnorm_infer_bwd(p, p, p, p, 4, 0, 1e-3, None) != 0
    assert nat.lib.dtb_linear_dense_grad(p, None, p, 4, 2, None) != 0
    assert nat.lib.dtb_linear_dense_grad(p, p, p, 4, 0, None) != 0
    # Dense backward: a weight-gradient-free call needs dX, and a bias gradient needs dW
    assert nat.lib.dtb_dense_bwd(p, p, None, p, None, None, None, None, 0, 4, 2, 2, 0, None) != 0
    assert nat.lib.dtb_dense_bwd(p, p, None, p, p, None, p, None, 0, 4, 2, 2, 0, None) != 0
