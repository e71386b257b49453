"""The fused CIN weight gradient's ring of row blocks across its shape envelope: per-layer filter gradients of the fused
backward against the any-shape backward on the same saved activations.  The shapes reach the NP = 16 / 32 / 64 / 128
instances, one and two x0 fields per A tile with absent tiles past the last field, the whole-block h copy
(ldh % 4 != 0), fewer row blocks than ring stages, a ragged last block, a row split count that does not divide the
blocks, and a batch shorter than one 64-row block (rows past its end are never written by any copy)."""
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
    (26, 4, (100, 64), 1000),        # NP 128; layer 0: two fields per tile, 13 tiles in 16 slots; layer 1: one field
    (10, 8, (32, 32), 17),           # NP 32; 136 GEMM rows: 3 blocks, fewer than the ring's stages; ragged last block
    (12, 32, (16, 16), 3),           # NP 16; 96 GEMM rows: one full block and a half one
    (13, 16, (34, 34), 1500),        # NP 64; h of layer 1 copied as whole blocks (ldh = 34); 375 blocks over 33 splits
    (26, 16, (128, 128), 3),         # NP 128; 48 GEMM rows: less than one block
    (26, 16, (128, 128, 128), 333),  # the headline layers, 5 328 rows in 84 blocks, ragged
]


@pytest.mark.parametrize('f,d,sizes,b', CASES)
def test_cin_wgrad_ring_matches_any_shape(nat, f, d, sizes, b):
    act, n = 1, len(sizes)
    sizes_c = nat.int_array(sizes)
    assert nat.lib.dtb_cin_tc_supported(f, d, sizes_c, n, 0)
    g = np.random.default_rng(1000 * f + d + b)
    vocab = [97] * f
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
