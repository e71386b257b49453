"""The fused CIN weight gradient with its producer warpgroup: per-layer filter gradients of the fused backward against
the any-shape backward on the same saved activations, within 5e-5 of max |dW|.  The cases reach both ways an h block
(T_{k-1}, layers k >= 1) arrives -- one 2-D tensor copy of its first hpitch columns when ldh % 4 == 0 (including a box
wider than ldh, and rows past the batch end), one bulk copy of whole rows otherwise -- the NP = 16 / 32 / 64 / 128
instances with one and two x0 fields per A tile, and the row splits: a half-full last field group whose two
warpgroups take alternate blocks (with its own, longer, split), the same group run by one warpgroup when the ring has
only two stages, a batch shorter than one 64-row block and a ragged last block."""
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


CASES = [
    # (fields, D, cross_layer_size, batch)
    # NP 128, the headline layers: h by tensor copy (ldh 128, box 68 of 128 columns); 1 250 blocks, last group of
    # each layer (one tile of two fields in layer 0, two one-field tiles in layers 1-2) on alternate blocks
    (26, 16, (128, 128, 128), 5000),
    # NP 128; layer 0 two fields per tile; layer 1 (H 50, ldh 100) by tensor copy, box 52 columns
    (26, 4, (100, 64), 700),
    # NP 64; layer 1 h as whole rows (ldh 34); the last group's one tile shared by both warpgroups; 375 blocks
    (9, 16, (34, 34), 1500),
    # NP 32; layer 1 by tensor copy (H 16, box 20 of 32 columns); 136 rows: 3 blocks, the last ragged
    (10, 8, (32, 32), 17),
    # NP 16; layer 1 (H 8, ldh 16): a box of 20 columns, wider than the rows (zero-filled); 96 rows, a half block
    (12, 32, (16, 16), 3),
    # NP 128; 48 rows, less than one block: the box reaches past the last row
    (26, 16, (128, 128), 3),
    # NP 128; layer 1 h as whole rows (ldh 126): 2-stage ring, so the last group's two tiles run on one warpgroup
    (62, 16, (126, 128), 40),
]


@pytest.mark.parametrize('f,d,sizes,b', CASES)
def test_cin_wgrad_producer_matches_any_shape(nat, f, d, sizes, b):
    act, n = 1, len(sizes)
    sizes_c = nat.int_array(sizes)
    assert nat.lib.dtb_cin_tc_supported(f, d, sizes_c, n, 0)
    g = np.random.default_rng(7000 * f + d + b)
    vocab = [89] * f
    table = torch.tensor(g.uniform(-0.5, 0.5, size=(sum(vocab), d)).astype(np.float32), device='cuda')
    offs = torch.tensor(np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64), device='cuda')
    idx = torch.tensor(np.stack([g.integers(0, v, size=b) for v in vocab], axis=1).astype(np.int32), device='cuda')
    fns = L.cin_field_nums(f, sizes, False)
    w = torch.tensor(np.concatenate([(g.normal(size=(f * fns[k], s)) / np.sqrt(f * fns[k])).astype(np.float32).reshape(-1)
                                     for k, s in enumerate(sizes)]), device='cuda')
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=False))
    pooled = torch.empty(b, pw, device='cuda')
    d_pooled = torch.tensor(g.normal(size=(b, pw)).astype(np.float32), device='cuda')
    ws_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, 0, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    saved = torch.empty(nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, 0), dtype=torch.uint8, device='cuda')
    nat.check(nat.lib.dtb_cin_fwd(P(idx), P(table), P(offs), P(w), None, P(pooled), P(saved), P(ws), ws_bytes, b, f, d,
                                  sizes_c, n, 0, act, 2, None, None))

    def bwd():
        gt = torch.zeros_like(table)
        dw = torch.zeros_like(w)
        for phase in (1, 2):
            nat.check(nat.lib.dtb_cin_bwd_phase(P(idx), P(table), P(offs), P(w), P(d_pooled), P(saved), P(gt), P(dw),
                                                None, P(ws), ws_bytes, b, f, d, sizes_c, n, 0, act, 2, phase, None))
        torch.cuda.synchronize()
        return dw

    dw = bwd()
    nat.lib.dtb_cin_tc_set_variant(1 | (1 << 16))       # the any-shape backward on the same saved activations
    try:
        dw2 = bwd()
    finally:
        nat.lib.dtb_cin_tc_set_variant(1)
    assert torch.isfinite(dw).all()
    o = 0
    for k, s in enumerate(sizes):
        m = f * fns[k] * s
        want = dw2[o:o + m]
        scale = float(want.abs().max())
        assert scale > 0, f'layer {k}: empty reference gradient'
        e = float((dw[o:o + m] - want).abs().max()) / scale
        assert e < 5e-5, f'filter grad of layer {k}: {e:.2e}'
        o += m
