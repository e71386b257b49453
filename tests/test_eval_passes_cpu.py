"""The numpy restatements of the fixed summation orders tests/test_eval_passes_gpu.py holds the device to: the
permutation-importance sums (sum_partials_kernel, then the finishing block) and the SHAP means (one warp per group).
Each must add every term exactly once: on integer-valued terms, where any order is exact, it equals math.fsum; on
random terms it stays within the rounding bound of a float64 sum; and a term left out or added twice shows."""
import math

import numpy as np
import pytest

from test_eval_passes_gpu import WARP, block_tree, shap_means_order, sum_partials_order


def _bound(terms):
    """the rounding bound of any float64 summation of `terms`"""
    return len(terms) * np.finfo(np.float64).eps * math.fsum(np.abs(terms))


def test_block_tree_adds_pairs_at_halving_strides():
    v = np.arange(256, dtype=np.float64)
    assert block_tree(v) == 255 * 256 / 2
    # the first step pairs i with i + 128: two values that cancel only when paired that way
    v = np.zeros(256)
    v[3], v[131] = 1e300, -1e300
    v[0] = 1.0
    assert block_tree(v) == 1.0


@pytest.mark.parametrize('n', [1, 255, 65536, 65537, 1_000_003])
def test_sum_partials_order_adds_every_term_once(n):
    g = np.random.default_rng(n)
    ints = g.integers(-1000, 1000, n).astype(np.float64)
    assert sum_partials_order(ints) == math.fsum(ints)
    x = g.random(n) * g.choice([1e-3, 1.0, 1e3], n)
    s = sum_partials_order(x)
    assert abs(s - math.fsum(x)) <= _bound(x)
    if n > 1:
        twice = x.copy()
        twice[n // 2] *= 2
        assert sum_partials_order(twice) != s


def test_sum_partials_order_is_per_thread_then_per_block():
    # thread 0 of block 0 adds rows 0 and 65 536 first: 1e300 and -1e300 cancel there, before any tree step
    n = 65536 + 10
    x = np.zeros(n)
    x[0], x[65536], x[1] = 1e300, -1e300, 2.0
    assert sum_partials_order(x) == 2.0


@pytest.mark.parametrize('groups,n', [(1, 1), (3, 31), (5, 32), (7, 100), (1000, 333)])
def test_shap_means_order_adds_every_row_once(groups, n):
    g = np.random.default_rng(groups * n)
    ints = g.integers(0, 50, (groups, n)).astype(np.float64)
    want = np.array([math.fsum(r) for r in ints]) / n
    assert np.array_equal(shap_means_order(ints), want)
    x = g.random((groups, n))
    got = shap_means_order(x)
    for r in range(groups):
        assert abs(got[r] * n - math.fsum(x[r])) <= _bound(x[r])


def test_shap_means_order_is_lane_stride_then_butterfly():
    # lane 0 adds rows 0 and 32 first, where 1e300 and -1e300 cancel; the butterfly's first step pairs lanes 16 apart
    v = np.zeros((1, 64))
    v[0, 0], v[0, 32], v[0, 5] = 1e300, -1e300, 3.0
    assert shap_means_order(v)[0] == 3.0 / 64
    v = np.zeros((1, WARP))
    v[0, 2], v[0, 18], v[0, 7] = 1e300, -1e300, 1.0
    assert shap_means_order(v)[0] == 1.0 / WARP
