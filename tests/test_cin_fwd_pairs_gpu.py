"""The fused CIN forward, whose CTA runs pairs of 64-row tiles on two consumer warpgroups that share each weight chunk
from a ring of shared-memory stages: `pooled` and every block of `saved` (x0t and each T_k) against the any-shape
forward (precision 1), for precision codes 2, 3 and 4, with bias on and off, relu and linear, `direct` on and off.  The
shapes reach NP = 16, 32, 64 and 128, D = 4 and 32, eight layers, and the largest shared-memory shape of the envelope
(F = 64, Lmax = 128); the batches give an odd tile count, a ragged last tile, fewer tiles than CTAs, and many pairs per
CTA, so that the ring wraps many times.  Bit-identity properties that hold for any build: training and inference give
the same bits, and the same rows at different batch offsets (shifted by one tile, by one pair, reversed) give the same
bits, whichever warpgroup or CTA ran them.  Out-of-range ids set their status bits and read as zero."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import layers_ref as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def make_inputs(f, d, sizes, direct, b, seed, use_bias=True):
    g = np.random.default_rng(seed)
    vocab = [53 + i for i in range(f)]
    table = torch.tensor(g.uniform(-0.5, 0.5, size=(sum(vocab), d)).astype(np.float32), device='cuda')
    offs = torch.tensor(np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64), device='cuda')
    idx = torch.tensor(np.stack([g.integers(0, v, size=b) for v in vocab], axis=1).astype(np.int32), device='cuda')
    fns = L.cin_field_nums(f, sizes, direct)
    w = torch.tensor(np.concatenate([(g.normal(size=(f * fns[k], s)) / np.sqrt(f * fns[k])).astype(np.float32).reshape(-1)
                                     for k, s in enumerate(sizes)]), device='cuda')
    bias = torch.tensor(g.normal(size=sum(sizes)).astype(np.float32) * 0.1, device='cuda') if use_bias else None
    return vocab, table, offs, idx, w, bias


def run_fwd(nat, f, d, sizes, direct, act, precision, table, offs, idx, w, bias, training=True, status=None):
    b = idx.shape[0]
    sizes_c, n = nat.int_array(sizes), len(sizes)
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=direct))
    pooled = torch.full((b, pw), float('nan'), device='cuda')
    ws_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, int(direct), int(training))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    saved = None
    if training:
        saved = torch.full((nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, int(direct)) // 4,), float('nan'),
                           device='cuda')
    nat.check(nat.lib.dtb_cin_fwd(P(idx), P(table), P(offs), P(w), P(bias), P(pooled), P(saved), P(ws), ws_bytes, b, f,
                                  d, sizes_c, n, int(direct), act, precision, P(status), None))
    torch.cuda.synchronize()
    return pooled, saved


def saved_blocks(saved, b, f, d, sizes):
    """x0t [B, D, F], then T_k [B, D, L_k]"""
    out, at = [saved[:b * d * f].view(b, d, f)], b * d * f
    for s in sizes:
        out.append(saved[at:at + b * d * s].view(b, d, s))
        at += b * d * s
    return out


CASES = [
    # (fields, D, cross_layer_size, direct, batch)
    (6, 4, (16, 16), False, 10),               # NP 16; 40 GEMM rows: one tile, shorter than 64 rows
    (30, 8, (32, 32), True, 17),               # NP 32; 3 tiles (odd), the last one ragged
    (25, 8, (64, 48), False, 325),             # NP 64; 41 tiles (odd), ragged; fewer pairs than CTAs
    (26, 16, (128, 128, 128), False, 20003),   # NP 128, the headline layers; 5001 tiles: ~19 pairs per CTA, ragged
    (12, 32, (16, 16), False, 3),              # D 32; 2 tiles, the second one half
    (10, 32, (64, 128), True, 205),            # D 32, NP 128, direct; 103 tiles (odd), ragged
    (9, 8, (32,) * 8, False, 250),             # eight layers; 32 tiles, the last one ragged
    (64, 16, (128, 128), False, 604),          # F 64 at NP 128: the largest shared-memory shape; 151 tiles
]


@pytest.mark.parametrize('precision', [2, 3, 4])
@pytest.mark.parametrize('act', [0, 1])
@pytest.mark.parametrize('use_bias', [False, True])
@pytest.mark.parametrize('f,d,sizes,direct,b', CASES)
def test_cin_fwd_pairs_match_any_shape(nat, f, d, sizes, direct, b, use_bias, act, precision):
    assert nat.lib.dtb_cin_tc_supported(f, d, nat.int_array(sizes), len(sizes), int(direct))
    _, table, offs, idx, w, bias = make_inputs(f, d, sizes, direct, b, seed=100 * f + d + b, use_bias=use_bias)
    args = (table, offs, idx, w, bias)
    pooled, saved = run_fwd(nat, f, d, sizes, direct, act, precision, *args)
    pooled1, saved1 = run_fwd(nat, f, d, sizes, direct, act, 1, *args)
    tol = 2e-5 if precision == 2 else 2e-2      # bf16x3 split: fp32-grade; one bf16 or fp16 pass: ~2^-8 per operand

    def close(got, want, what):
        assert torch.isfinite(got).all(), f'{what}: not finite'
        scale = float(want.abs().max())
        assert scale > 0, f'{what}: empty reference'
        e = float((got - want).abs().max()) / scale
        assert e < tol, f'{what}: {e:.2e} of max |any-shape|'

    close(pooled, pooled1, 'pooled')
    got, want = saved_blocks(saved, b, f, d, sizes), saved_blocks(saved1, b, f, d, sizes)
    assert torch.equal(got[0], want[0]), 'saved x0t'
    for k in range(len(sizes)):
        close(got[k + 1], want[k + 1], f'saved T_{k}')


@pytest.mark.parametrize('precision', [2, 3, 4])
def test_cin_fwd_pairs_bits_do_not_depend_on_position(nat, precision):
    f, d, sizes, act = 26, 16, (128, 128, 128), 1
    b = 2000                                   # 500 tiles: 250 pairs, more than the CTAs
    rows_tile, rows_pair = 64 // d, 128 // d
    _, table, offs, idx, w, bias = make_inputs(f, d, sizes, False, b + rows_pair, seed=7)
    base, pad = idx[:b], idx[b:]
    pooled, saved = run_fwd(nat, f, d, sizes, False, act, precision, table, offs, base, w, bias)
    pooled_inf, _ = run_fwd(nat, f, d, sizes, False, act, precision, table, offs, base, w, bias, training=False)
    assert torch.equal(pooled, pooled_inf), 'training and inference differ'
    ref = saved_blocks(saved, b, f, d, sizes)
    for name, ids, rows in [('shifted by one tile', torch.cat([pad[:rows_tile], base]), lambda t: t[rows_tile:]),
                            ('shifted by one pair', torch.cat([pad, base]), lambda t: t[rows_pair:]),
                            ('reversed', base.flip(0), lambda t: t.flip(0))]:
        p2, s2 = run_fwd(nat, f, d, sizes, False, act, precision, table, offs, ids.contiguous(), w, bias)
        n2 = ids.shape[0]
        assert torch.equal(rows(p2), pooled), f'pooled {name}'
        for k, (x, y) in enumerate(zip(saved_blocks(s2, n2, f, d, sizes), ref)):
            assert torch.equal(rows(x), y), f'saved block {k} {name}'


@pytest.mark.parametrize('precision', [2, 3, 4])
def test_cin_fwd_pairs_out_of_range_ids(nat, precision):
    f, d, sizes, b = 12, 8, (64, 64), 300
    vocab, table, offs, idx, w, bias = make_inputs(f, d, sizes, False, b, seed=11)
    bad = idx.clone()
    bad[5, 3] = -1
    bad[257, 7] = vocab[7]                     # one past the field's vocabulary
    status = torch.zeros(1, dtype=torch.int32, device='cuda')
    pooled, saved = run_fwd(nat, f, d, sizes, False, 1, precision, table, offs, bad, w, bias, status=status)
    assert int(status.item()) == (1 << 3) | (1 << 7)
    x0 = saved_blocks(saved, b, f, d, sizes)[0]
    assert torch.equal(x0[5, :, 3], torch.zeros(d, device='cuda'))
    assert torch.equal(x0[257, :, 7], torch.zeros(d, device='cuda'))
    st1 = torch.zeros(1, dtype=torch.int32, device='cuda')
    pooled1, _ = run_fwd(nat, f, d, sizes, False, 1, 1, table, offs, bad, w, bias, status=st1)
    assert int(st1.item()) == int(status.item())
    scale = float(pooled1.abs().max())
    assert float((pooled - pooled1).abs().max()) / scale < (2e-5 if precision == 2 else 2e-2)
