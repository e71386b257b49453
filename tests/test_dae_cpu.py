"""Denoising auto-encoder (fe.dae) without a GPU: the layer plan, the swap count, the batch schedule, the refused inputs,
the distribution of the swapped columns and the C ABI of dtb_dae_swap_batch."""
import ctypes
import re

import numpy as np
import pandas as pd
import pytest
from scipy import stats

import dae_ref
from deeptables_b200 import dae
from deeptables_b200.fe.dae import DAE


@pytest.mark.parametrize('units', [(500, 500), (64,), (32, 64, 16)])
@pytest.mark.parametrize('act', ['relu', 'tanh', None])
def test_layer_plan_matches_build_dae(units, act):
    got = dae.layer_plan(units, 20, act, 37)
    assert got == dae_ref.layer_plan(units, 20, act, 37)
    names = [r[0] for r in got]
    assert names[len(units) - 1] == 'feature_layer' and names[-1] == 'output_layer'
    assert got[-1][2] == 37 and got[0][1] == 37


def test_layer_plan_shapes():
    assert dae.layer_plan((500, 500), 20, 'relu', 200) == [
        ('encoder_0', 200, 500, 'relu'), ('feature_layer', 500, 20, None), ('decoder_1', 20, 500, 'relu'),
        ('output_layer', 500, 200, 'relu')]
    assert dae.layer_plan((64,), 8, 'tanh', 5) == [('feature_layer', 5, 8, None), ('output_layer', 8, 5, 'tanh')]


@pytest.mark.parametrize('cols,rate,k', [(200, 0, 0), (200, 0.15, 30), (200, 1, 200), (200, 1.0, 200), (5, 0.15, 0),
                                         (7, 1 / 7, 1), (100, 0.29, 28), (10, 0.3, 3), (1, 0.999, 0), (221, 0.15, 33)])
def test_swap_count_is_the_references_float_truncation(cols, rate, k):
    assert dae.swap_count(cols, rate) == dae_ref.swap_count(cols, rate) == k


@pytest.mark.parametrize('n,bs,sizes', [(1, 128, [1]), (128, 128, [128]), (129, 128, [128, 1]), (300, 128, [128, 128, 44]),
                                        (5, 2, [2, 2, 1]), (7, 100, [7])])
def test_batch_schedule(n, bs, sizes):
    assert dae_ref.steps_per_epoch(n, bs) == len(sizes)
    assert dae_ref.batch_rows(n, bs) == sizes


X4 = np.zeros((3, 4))


@pytest.mark.parametrize('kw,fit_kw,match', [
    (dict(encoder_units=()), {}, 'encoder_units'),
    (dict(encoder_units=(8, 0)), {}, r'encoder_units\[1\]'),
    (dict(feature_units=0), {}, 'feature_units'),
    (dict(noise_rate=1.01), {}, 'noise_rate'),
    (dict(noise_rate=-0.1), {}, 'noise_rate'),
    (dict(noise_rate=float('nan')), {}, 'noise_rate'),
    (dict(random_state=2 ** 32), {}, 'random_state'),
    (dict(random_state=-1), {}, 'random_state'),
    ({}, dict(batch_size=0), 'batch_size'),
    ({}, dict(batch_size=2.0), 'batch_size'),
    ({}, dict(batch_size=True), 'batch_size'),
    ({}, dict(epochs=-1), 'epochs'),
    ({}, dict(epochs=1.5), 'epochs'),
])
def test_bad_arguments_raise_value_error_before_device_work(kw, fit_kw, match):
    for call in ('fit', 'fit_transform'):
        with pytest.raises(ValueError, match=match):
            getattr(DAE(**kw), call)(X4, **fit_kw)


@pytest.mark.parametrize('X,match', [
    (np.array([[1.0, np.nan], [2.0, 3.0]]), 'column 1 '),
    (np.array([[1.0, 2.0], [np.inf, 3.0]]), 'column 0 '),
    (pd.DataFrame({'a': [1.0, 2.0], 'b': ['x', 'y']}), "column 'b' is not numeric"),
    (pd.DataFrame({'a': [1.0, 2.0], 'c': pd.Categorical(['x', 'y'])}), "column 'c' is not numeric"),
    (pd.DataFrame({'a': [1.0, -np.inf], 'b': [1, 2]}), "column 'a' has NaN"),
    (np.array([['a', 'b']]), 'numeric'),
    (np.zeros(5), '2-D'),
    (np.zeros((0, 3)), 'at least one row'),
])
def test_bad_inputs_raise_value_error_naming_the_column(X, match):
    for call in ('fit', 'fit_transform', 'build_dae'):
        with pytest.raises(ValueError, match=match):
            getattr(DAE(), call)(X)


def test_unsupported_activation_raises_dense_error():
    with pytest.raises(NotImplementedError, match='activation'):
        DAE(activation='sigmoid').fit(X4)


def test_epochs_zero_is_accepted_by_the_checks():
    assert dae._count('epochs', 0, 0) == 0


def test_as_matrix_casts_to_float32():
    df = pd.DataFrame({'a': [1, 2], 'b': [0.5, 1.5], 'c': [True, False]})
    got = dae.as_matrix(df)
    assert got.dtype == np.float32 and got.flags.c_contiguous
    np.testing.assert_array_equal(got, [[1, 0.5, 1], [2, 1.5, 0]])


@pytest.mark.parametrize('cols,k', [(10, 3), (37, 5), (64, 64), (200, 30)])
def test_noise_choice_is_k_distinct_columns_uniformly(cols, k):
    counts = np.zeros(cols)
    trials = 0
    for step in range(1, 41):
        for row in range(100):
            c = dae_ref.swapped_columns(12345, step, row, cols, k)
            assert len(c) == k and len(np.unique(c)) == k and c.min() >= 0 and c.max() < cols
            counts[c] += 1
            trials += 1
    if k == cols:
        assert (counts == trials).all()
        return
    # each column is chosen with probability k / cols in every trial
    chi2, p = stats.chisquare(counts, np.full(cols, trials * k / cols))
    assert p > 1e-3, (chi2, p)


def test_noise_choice_breaks_hash_ties_by_column():
    h = dae_ref.row_hashes(7, 3, 11, 50)
    keys = (h << np.uint64(32)) | np.arange(50, dtype=np.uint64)
    assert len(np.unique(keys)) == 50
    np.testing.assert_array_equal(dae_ref.swapped_columns(7, 3, 11, 50, 50), np.arange(50))


def test_dtb_dae_swap_batch_signature_matches_the_header():
    from deeptables_b200 import _native as nat
    with open(nat.HEADER_PATH) as f:
        text = re.sub(r'/\*.*?\*/', '', f.read(), flags=re.S)
    (args,) = re.findall(r'\bint\s+dtb_dae_swap_batch\s*\(([^)]*)\)\s*;', text)
    kinds = {'int': ctypes.c_int, 'int64_t': ctypes.c_int64, 'unsigned long long': ctypes.c_ulonglong}
    want = []
    for a in args.split(','):
        decl = a.strip()
        want.append(ctypes.c_void_p if '*' in decl else kinds[decl.rsplit(None, 1)[0].replace('const', '').strip()])
    res, argtypes = nat._SIGNATURES['dtb_dae_swap_batch']
    assert res is ctypes.c_int and argtypes == want
    assert 'dtb_dae_swap_batch' in nat.declared_symbols() and hasattr(nat.lib, 'dtb_dae_swap_batch')
