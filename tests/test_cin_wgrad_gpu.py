"""The fused CIN backward at the headline shape with a multi-tile, ragged batch: the data-gradient kernel writes dC_k as the
bf16 hi/lo images the weight-gradient kernel reads, and sums d_bias; the weight-gradient kernel serves groups of x0
fields from one copy of each row block, over many row splits.  Checked against the any-shape backward."""
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


@pytest.mark.parametrize('use_bias', [True, False])
def test_cin_fused_backward_full_ragged_batch(nat, use_bias):
    f, d, sizes, act = 26, 16, (128, 128, 128), 1
    # 64 944 GEMM rows: several tiles per data-gradient CTA, dozens of row blocks per weight-gradient CTA through its
    # two-stage ring, and a last block of 48 rows.  (At the full 65 536-row batch the two backward formulations, both
    # reducing over a million rows in fp32 in different orders, differ by ~1e-4 of max |dW|, for the earlier weight-
    # gradient kernel as well; this batch keeps the 5e-5 bound of the small-batch tests meaningful.)
    b = 4096 - 37
    n = len(sizes)
    sizes_c = nat.int_array(sizes)
    assert nat.lib.dtb_cin_tc_supported(f, d, sizes_c, n, 0)
    g = np.random.default_rng(51)
    vocab = [1000] * f
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
    nat.check(nat.lib.dtb_cin_fwd(P(idx), P(table), P(offs), P(w), P(bias), P(pooled), P(saved), P(ws), ws_bytes, b, f, d,
                                  sizes_c, n, 0, act, 2, None, None))

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
    for got, want, what in ((gt, gt2, 'embedding grad'), (dw, dw2, 'filter grad'), (db, db2, 'bias grad')):
        if want is None:
            continue
        assert torch.isfinite(got).all(), what
        e = float((got - want).abs().max() / want.abs().max())
        assert e < 5e-5, f'fused vs any-shape backward, {what}: {e:.2e}'
    # every layer's filter gradient is covered, not just the largest one
    o = 0
    for k, s in enumerate(sizes):
        m = f * fns[k] * s
        e = float((dw[o:o + m] - dw2[o:o + m]).abs().max() / dw2[o:o + m].abs().max())
        assert e < 5e-5, f'filter grad of layer {k}: {e:.2e}'
        o += m
