"""The fused CIN backward (csrc/cin_wgmma.cu) across its shape envelope, against the any-shape backward (precision 1) on
the same saved activations: the embedding gradient, each layer's filter gradient and, with a bias, each layer's bias
gradient, within 5e-5 of the reference's max |value|.  Both backwards run as training runs them, in two launches:
phase 1 the embedding gradient, phase 2 the weight gradients.

The data-gradient kernel writes dC_k as the bf16 hi/lo images the weight-gradient kernel reads, and sums d_bias; the
weight-gradient kernel streams row blocks through a ring of shared-memory stages filled by a producer warpgroup and
serves groups of x0 fields from one copy of each block, over many row splits.  Each case's comment names the branches
of those kernels it reaches."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import layers_ref as L

pytestmark = pytest.mark.gpu

BOTH = (False, True)

CASES = [
    # (fields, D, cross_layer_size, batch, vocab per field, seed, use_bias values)
    # The headline shape at 64 944 GEMM rows: several tiles per data-gradient CTA, dozens of row blocks per
    # weight-gradient CTA through its ring, and a last block of 48 rows.  (At the full 65 536-row batch the two
    # backward formulations, both reducing over a million rows in fp32 in different orders, differ by ~1e-4 of
    # max |dW|; this batch keeps the 5e-5 bound meaningful.)
    (26, 16, (128, 128, 128), 4096 - 37, 1000, 51, BOTH),

    # The data gradient's weight chunks: the NPJ = 16 / 32 / 64 instances; two x0 fields per weight chunk in layer 0
    # (with an odd field count, so the last chunk has one field), in a layer k >= 1 only, and at NPJ = 32 and 16; an
    # odd tile count and a ragged last tile; a batch shorter than one 64-row tile; and more tiles than CTAs.
    # NPJ 64, the headline layers; layer 0 paired; 375 tiles, more than the CTAs
    (26, 16, (128, 128, 128), 1500, 97, 1000 * 26 + 16 + 1500, BOTH),
    # NPJ 64; layer 0 paired with odd F (13th chunk has one field); ragged last tile
    (25, 8, (128, 64), 333, 97, 1000 * 25 + 8 + 333, BOTH),
    # NPJ 64; H = 40, 32: layer 1 paired only; L = 100 (LP 112, NPdc 128)
    (40, 4, (64, 100), 700, 97, 1000 * 40 + 4 + 700, BOTH),
    # NPJ 32; H = 30, 16: layer 1 paired; 3 tiles, the last one ragged
    (30, 8, (32, 32), 17, 97, 1000 * 30 + 8 + 17, BOTH),
    # NPJ 16; H = 12, 8: layer 1 paired; 2 tiles, the second one half
    (12, 32, (16, 16), 3, 97, 1000 * 12 + 32 + 3, BOTH),
    # NPJ 16; both layers paired; 40 GEMM rows: one tile, shorter than 64 rows
    (6, 4, (16, 16), 10, 97, 1000 * 6 + 4 + 10, BOTH),
    # NPJ 64; 48 GEMM rows, less than one tile
    (26, 16, (128, 128), 3, 97, 1000 * 26 + 16 + 3, BOTH),

    # The weight gradient's ring of row blocks: the NP = 16 / 32 / 64 / 128 instances, one and two x0 fields per A tile
    # with absent tiles past the last field, the whole-block h copy (ldh % 4 != 0), fewer row blocks than ring stages,
    # a ragged last block, a row split count that does not divide the blocks, and a batch shorter than one 64-row block
    # (rows past its end are never written by any copy).  Its 96-row case, NP 16 (12, 32, (16, 16), 3), and its 48-row
    # case, NP 128 (26, 16, (128, 128), 3), are the runs without bias of the two data-gradient cases of those shapes.
    # NP 128; layer 0: two fields per tile, 13 tiles in 16 slots; layer 1: one field
    (26, 4, (100, 64), 1000, 97, 1000 * 26 + 4 + 1000, (False,)),
    # NP 32; 136 GEMM rows: 3 blocks, fewer than the ring's stages; ragged last block
    (10, 8, (32, 32), 17, 97, 1000 * 10 + 8 + 17, (False,)),
    # NP 64; h of layer 1 copied as whole blocks (ldh = 34); 375 blocks over 33 splits
    (13, 16, (34, 34), 1500, 97, 1000 * 13 + 16 + 1500, (False,)),
    # the headline layers, 5 328 rows in 84 blocks, ragged
    (26, 16, (128, 128, 128), 333, 97, 1000 * 26 + 16 + 333, (False,)),

    # The weight gradient's producer warpgroup: both ways an h block (T_{k-1}, layers k >= 1) arrives -- one 2-D tensor
    # copy of its first hpitch columns when ldh % 4 == 0 (including a box wider than ldh, and rows past the batch end),
    # one bulk copy of whole rows otherwise -- and the row splits: a half-full last field group whose two warpgroups
    # take alternate blocks (with its own, longer, split), the same group run by one warpgroup when the ring has only
    # two stages, a batch shorter than one 64-row block and a ragged last block.
    # NP 128, the headline layers: h by tensor copy (ldh 128, box 68 of 128 columns); 1 250 blocks, last group of
    # each layer (one tile of two fields in layer 0, two one-field tiles in layers 1-2) on alternate blocks
    (26, 16, (128, 128, 128), 5000, 89, 7000 * 26 + 16 + 5000, (False,)),
    # NP 128; layer 0 two fields per tile; layer 1 (H 50, ldh 100) by tensor copy, box 52 columns
    (26, 4, (100, 64), 700, 89, 7000 * 26 + 4 + 700, (False,)),
    # NP 64; layer 1 h as whole rows (ldh 34); the last group's one tile shared by both warpgroups; 375 blocks
    (9, 16, (34, 34), 1500, 89, 7000 * 9 + 16 + 1500, (False,)),
    # NP 32; layer 1 by tensor copy (H 16, box 20 of 32 columns); 136 rows: 3 blocks, the last ragged
    (10, 8, (32, 32), 17, 89, 7000 * 10 + 8 + 17, (False,)),
    # NP 16; layer 1 (H 8, ldh 16): a box of 20 columns, wider than the rows (zero-filled); 96 rows, a half block
    (12, 32, (16, 16), 3, 89, 7000 * 12 + 32 + 3, (False,)),
    # NP 128; 48 rows, less than one block: the box reaches past the last row
    (26, 16, (128, 128), 3, 89, 7000 * 26 + 16 + 3, (False,)),
    # NP 128; layer 1 h as whole rows (ldh 126): 2-stage ring, so the last group's two tiles run on one warpgroup
    (62, 16, (126, 128), 40, 89, 7000 * 62 + 16 + 40, (False,)),
]


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize('f,d,sizes,b,vocab,seed,use_bias',
                         [(*row[:6], use_bias) for row in CASES for use_bias in row[6]])
def test_cin_fused_backward_matches_any_shape(nat, f, d, sizes, b, vocab, seed, use_bias):
    act, n = 1, len(sizes)
    sizes_c = nat.int_array(sizes)
    assert nat.lib.dtb_cin_tc_supported(f, d, sizes_c, n, 0)
    g = np.random.default_rng(seed)
    vocab = [vocab] * f
    table = torch.tensor(g.uniform(-0.5, 0.5, size=(sum(vocab), d)).astype(np.float32), device='cuda')
    offs = torch.tensor(np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64), device='cuda')
    idx = torch.tensor(np.stack([g.integers(0, v, size=b) for v in vocab], axis=1).astype(np.int32), device='cuda')
    fns = L.cin_field_nums(f, sizes, False)
    w = torch.tensor(np.concatenate([(g.normal(size=(f * fns[k], s)) / np.sqrt(f * fns[k])).astype(np.float32).reshape(-1)
                                     for k, s in enumerate(sizes)]), device='cuda')
    bias = torch.tensor(g.normal(size=sum(sizes)).astype(np.float32) * 0.1, device='cuda') if use_bias else None
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=False))
    pooled = torch.empty(b, pw, device='cuda')
    d_pooled = torch.tensor(g.normal(size=(b, pw)).astype(np.float32), device='cuda')
    ws_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, 0, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    saved = torch.empty(nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, 0), dtype=torch.uint8, device='cuda')
    nat.check(nat.lib.dtb_cin_fwd(P(idx), P(table), P(offs), P(w), P(bias), P(pooled), P(saved), P(ws), ws_bytes, b,
                                  f, d, sizes_c, n, 0, act, 2, None, None))

    def bwd(precision):
        gt = torch.zeros_like(table)
        dw = torch.zeros_like(w)
        db = torch.zeros(sum(sizes), device='cuda') if use_bias else None
        for phase in (1, 2):
            nat.check(nat.lib.dtb_cin_bwd_phase(P(idx), P(table), P(offs), P(w), P(d_pooled), P(saved), P(gt), P(dw),
                                                P(db), P(ws), ws_bytes, b, f, d, sizes_c, n, 0, act, precision, phase,
                                                None))
        torch.cuda.synchronize()
        return gt, dw, db

    gt, dw, db = bwd(2)
    gt2, dw2, db2 = bwd(1)

    def close(got, want, what):
        assert torch.isfinite(got).all(), f'{what}: not finite'
        scale = float(want.abs().max())
        assert scale > 0, f'{what}: empty reference gradient'
        e = float((got - want).abs().max()) / scale
        print(f'{what}: max err / max |reference| {e:.2e}')
        assert e < 5e-5, f'{what}: {e:.2e}'

    close(gt, gt2, 'embedding grad')
    o = 0
    for k, s in enumerate(sizes):
        m = f * fns[k] * s
        close(dw[o:o + m], dw2[o:o + m], f'filter grad of layer {k}')
        o += m
    if use_bias:
        o = 0
        for k, s in enumerate(sizes):
            close(db[o:o + s], db2[o:o + s], f'bias grad of layer {k}')
            o += s
