"""The fused CIN data gradient's weight chunks across its shape envelope: the embedding gradient, each layer's filter
gradient and each layer's bias gradient of the fused backward against the any-shape backward on the same saved
activations, with and without bias.  The shapes reach the NPJ = 16 / 32 / 64 instances; two x0 fields per weight
chunk in layer 0 (with an odd field count, so the last chunk has one field), in a layer k >= 1 only, and at NPJ = 32
and 16; an odd tile count and a ragged last tile; a batch shorter than one 64-row tile; and more tiles than CTAs."""
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
    (26, 16, (128, 128, 128), 1500),  # NPJ 64, the headline layers; layer 0 paired; 375 tiles, more than the CTAs
    (25, 8, (128, 64), 333),          # NPJ 64; layer 0 paired with odd F (13th chunk has one field); ragged last tile
    (40, 4, (64, 100), 700),          # NPJ 64; H = 40, 32: layer 1 paired only; L = 100 (LP 112, NPdc 128)
    (30, 8, (32, 32), 17),            # NPJ 32; H = 30, 16: layer 1 paired; 3 tiles, the last one ragged
    (12, 32, (16, 16), 3),            # NPJ 16; H = 12, 8: layer 1 paired; 2 tiles, the second one half
    (6, 4, (16, 16), 10),             # NPJ 16; both layers paired; 40 GEMM rows: one tile, shorter than 64 rows
    (26, 16, (128, 128), 3),          # NPJ 64; 48 GEMM rows, less than one tile
]


@pytest.mark.parametrize('use_bias', [False, True])
@pytest.mark.parametrize('f,d,sizes,b', CASES)
def test_cin_dgrad_chunks_match_any_shape(nat, f, d, sizes, b, use_bias):
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
    bias = torch.tensor(g.normal(size=sum(sizes)).astype(np.float32) * 0.1, device='cuda') if use_bias else None
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=False))
    pooled = torch.empty(b, pw, device='cuda')
    d_pooled = torch.tensor(g.normal(size=(b, pw)).astype(np.float32), device='cuda')
    ws_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, 0, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    saved = torch.empty(nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, 0), dtype=torch.uint8, device='cuda')
    nat.check(nat.lib.dtb_cin_fwd(P(idx), P(table), P(offs), P(w), P(bias), P(pooled), P(saved), P(ws), ws_bytes, b,
                                  f, d, sizes_c, n, 0, act, 2, None, None))

    def bwd():
        gt = torch.zeros_like(table)
        dw = torch.zeros_like(w)
        db = torch.zeros(sum(sizes), device='cuda') if use_bias else None
        for phase in (1, 2):
            nat.check(nat.lib.dtb_cin_bwd_phase(P(idx), P(table), P(offs), P(w), P(d_pooled), P(saved), P(gt), P(dw),
                                                P(db), P(ws), ws_bytes, b, f, d, sizes_c, n, 0, act, 2, phase, None))
        torch.cuda.synchronize()
        return gt, dw, db

    gt, dw, db = bwd()
    nat.lib.dtb_cin_tc_set_variant(1 | (1 << 16))       # the any-shape backward on the same saved activations
    try:
        gt2, dw2, db2 = bwd()
    finally:
        nat.lib.dtb_cin_tc_set_variant(1)

    def close(got, want, what):
        assert torch.isfinite(got).all(), f'{what}: not finite'
        scale = float(want.abs().max())
        assert scale > 0, f'{what}: empty reference gradient'
        e = float((got - want).abs().max()) / scale
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
