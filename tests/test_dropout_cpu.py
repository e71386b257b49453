"""Dropout without a GPU: the attention layer accepts a rate, the mask formula against values worked out by hand, and
the bookkeeping that lets a captured train step read its seeds from device memory."""
import numpy as np
import pytest

import dropout_ref as D


def test_attention_layer_accepts_a_dropout_rate():
    from deeptables_b200 import layers as L
    layer = L.MultiheadAttention({'num_heads': 2, 'dropout_rate': 0.2, 'use_residual': True})
    assert layer.dropout_rate == 0.2
    assert L.MultiheadAttention({'num_heads': 1}).dropout_rate == 0
    for rate in (-0.1, 1, 1.5):
        with pytest.raises(ValueError):
            L.MultiheadAttention({'dropout_rate': rate})


def test_mask_bits_match_values_computed_by_hand():
    # mix32(seed * 0x9E3779B97F4A7C15 + i) evaluated step by step with unbounded integers reduced modulo 2^64
    assert D.bits(0, np.arange(4)).tolist() == [0, 885181228, 1694925799, 167303374]
    assert D.bits(12345, np.arange(6)).tolist() == [451982879, 1311178941, 3680713863, 4110786107, 2220720024,
                                                    3812423629]
    assert D.bits(0xFFFFFFFFFFFF, [0, 1, 2 ** 33 + 7]).tolist() == [2187474036, 2161992022, 4165166464]
    # the rate reaches the kernels as a float: 0.3f = 0.300000011920929, 0.1f = 0.100000001490116
    assert int(D.threshold(0.3)) == 1288490240 and int(D.threshold(0.1)) == 429496736
    assert int(D.threshold(0.5)) == 2 ** 31 and int(D.threshold(0.0)) == 0
    assert D.keep(12345, np.arange(6), 0.3).tolist() == [False, True, True, True, True, True]
    assert D.keep(12345, np.arange(6), 0.5).tolist() == [False, False, True, True, True, True]
    assert D.keep(0, np.arange(4), 0.1).tolist() == [False, True, True, False]


def test_attention_mask_index_does_not_depend_on_the_slice():
    whole = D.attention_keep(77, 0.3, rows=9, heads=2, fields=5)
    part = D.attention_keep(77, 0.3, rows=4, heads=2, fields=5, row_offset=3)
    assert np.array_equal(whole[3:7], part)
    # weight (b, h, q, k) = (2, 1, 3, 4)
    assert whole[2, 1, 3, 4] == D.keep(77, ((2 * 2 + 1) * 5 + 3) * 5 + 4, 0.3)


@pytest.mark.parametrize('near_wrap', [False, True])
def test_device_slots_follow_the_seeds_of_eager_passes(near_wrap):
    """A captured step reads slot k; dtb_seed_advance adds the number of sites modulo 2^48 at the end of every replay.
    The slots must hold what next_seed() returns in eager passes, also across the 48-bit wrap and when eager passes
    and replays alternate (the seed buffer of a scope on the CPU is host memory)."""
    from deeptables_b200.deepmodel import _Scope, SEED_MASK
    sites, passes = 5, 7
    eager, graphed = _Scope('cpu', seed=4242), _Scope('cpu', seed=4242)
    if near_wrap:
        start = SEED_MASK + 1 - eager.seed_at(0) - 2 * sites - 3        # the third pass crosses 2^48
        eager._seed_counter = graphed._seed_counter = start
    want = [[eager.next_seed() for _ in range(sites)] for _ in range(passes)]
    flat = [s for p in want for s in p]
    assert all(0 <= s <= SEED_MASK for s in flat) and len(set(flat)) == len(flat)
    if near_wrap:
        assert min(flat) < sites and max(flat) > SEED_MASK - 3 * sites
    graphed.seed_sites = sites
    got, buf = [], None
    for p in range(passes):
        if p in (0, 4):                          # an eager pass: the first step, or one with sample weights
            got.append([graphed.next_seed() for _ in range(sites)])
            continue
        if buf is None:                          # the capture: slot k goes to the k-th call site, nothing is drawn
            before = graphed._seed_counter
            with graphed.device_seeds() as buf:
                handed = [graphed.next_seed() for _ in range(sites)]
            assert graphed._seed_counter == before
            assert [h.data_ptr() for h in handed] == [buf[k:].data_ptr() for k in range(sites)]
        graphed.replay_seeds()
        got.append(buf.tolist())                 # what the replayed kernels read
        buf.copy_((buf + sites) & SEED_MASK)     # seed_advance_kernel at the end of the replay
    assert got == want
    assert graphed._seed_counter == eager._seed_counter
