"""The kernels outside CIN past their first pass over the batch.

A persistent or capped grid covers the batch in passes of gridDim rows, tiles or chunks, and several kernels carry state
from one pass to the next: shared-memory buffers refilled each pass, register accumulators that live across passes,
prefetches of the next pass and mbarrier rings whose phase wraps.  The float64 checks of tests/test_native_gpu.py run
every op inside its first pass; this file runs the same ops at production batch sizes.

One case table drives three checks:
  - the premise: the named kernels ran, and the work splits into at least 3 passes of the grid each one was launched
    with (the Dense weight gradient: at least 3 x kDtStages chunks per split, so its stage ring wraps twice); the last
    pass is ragged where the shape allows;
  - per-row outputs of the full batch equal, bit for bit and for every row, those of uneven consecutive slices that each
    fit in one pass (the calls tests/test_native_gpu.py validates against float64), with the same kernels launched;
  - reductions over rows (weight, bias and table gradients, batch-norm statistics) against a float64 reference computed
    on the device in row chunks.  Each bar is relative to a scale that batch-size cancellation does not shrink (the same
    float64 reduction on absolute values for multilinear contractions, else max |reference|), and each case asserts that
    its bar rejects the reference with one work unit's rows left out.
The pass counts below assume an H100 SXM (132 SMs); a card with fewer SMs runs more passes.

The launches (kernel, grid, block) come from torch.profiler in a child process (`recorded`).  Profiling in this process
would leave the profiler on the CUDA activity of everything the later test files run, and after that volume of
kernels its next sessions record none of them: tests/test_kernel_paths_gpu.py, which profiles every call it checks, then
sees empty sessions.
"""
import ctypes
import json
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from kernel_profile import launches
from oracle import layers_ref as L

pytestmark = pytest.mark.gpu

kDtStages = 4          # dense_tc.cu: stages of the weight-gradient ring


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


@pytest.fixture(autouse=True)
def _release():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def sm_count(nat):
    n = ctypes.c_int(0)
    nat.check(nat.lib.dtb_device_sm_count(ctypes.byref(n)))
    return n.value


def cdiv(a, b):
    return -(-a // b)


def rnd(*shape, seed):
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    return torch.randn(*shape, generator=g, device='cuda')


def ids(vocab, b, seed):
    g = torch.Generator(device='cuda')
    g.manual_seed(seed)
    return torch.stack([torch.randint(0, v, (b,), generator=g, device='cuda') for v in vocab], 1).to(torch.int32).contiguous()


def table(vocab, d, seed):
    flat = (torch.rand(sum(vocab), d, generator=torch.Generator(device='cuda').manual_seed(seed), device='cuda') - 0.5)
    offs = torch.tensor(np.concatenate([[0], np.cumsum(vocab)]), dtype=torch.int64, device='cuda')
    return flat.contiguous(), offs


def zeros(*shape):
    return torch.zeros(*shape, device='cuda')


def empty(*shape):
    return torch.empty(*shape, device='cuda')


# ---------------------------------------------------------------------------------------------
# the loops a case's launches run: Loop(kernel, work(grid, block) -> (units, units per pass), unit, ragged)
# ---------------------------------------------------------------------------------------------
def Loop(kernel, work, unit, ragged=True):
    return SimpleNamespace(kernel=kernel, work=work, unit=unit, ragged=ragged)


def stride(kernel, total, per_cta, unit, ragged=True, axis=0):
    """a grid-stride loop over `total` units, `per_cta(block)` of them per CTA and pass, CTAs along grid axis `axis`"""
    return Loop(kernel, lambda g, b: (total, g[axis] * per_cta(b)), unit, ragged)


def serial(kernel, rows, rows_per_iter, unit, axis=1):
    """each CTA walks its own ceil(rows / grid[axis]) rows, `rows_per_iter` per iteration (the column reductions)"""
    return Loop(kernel, lambda g, b: (cdiv(rows, g[axis]), rows_per_iter), unit, ragged=False)


def passes_of(case_id, kernels, loops):
    """Checks the premise; returns [(kernel, passes)] in launch order."""
    names = [k for k, _, _ in kernels]
    seen, out = {}, []
    for lp in loops:
        hits = [(g, b) for k, g, b in kernels if k == lp.kernel or k.startswith(lp.kernel + '<')]
        i = seen.get(lp.kernel, 0)
        seen[lp.kernel] = i + 1
        assert i < len(hits), f'{case_id}: launch {i} of {lp.kernel} did not happen; launched {names}'
        total, per = lp.work(*hits[i])
        n = total / per
        assert n >= 3, f'{case_id}: {lp.kernel} covers {total} {lp.unit}s in {n:.2f} passes of {per} (grid {hits[i][0]})'
        if lp.ragged:
            assert total % per, f'{case_id}: {lp.kernel}: {total} {lp.unit}s are a whole number of passes of {per}'
        out.append((lp.kernel, round(n, 2)))
    return out


# ---------------------------------------------------------------------------------------------
# cases.  build(nat) returns SimpleNamespace(B, run(lo, hi) -> (per-row outputs, reductions) of rows [lo, hi),
# loops (of run(0, B)), one_pass (rows a slice may hold to stay in one pass of every loop that has per-row outputs)),
# and, for the reduction cases, ref(lo, hi, absolute, keep=None) -> the float64 reductions of rows [lo, hi) (with
# `absolute`, the same contraction of absolute values; keep: a [hi - lo] row mask), unit (rows of one work unit),
# scale ('abs' or 'max') and rtol.
# ---------------------------------------------------------------------------------------------
def dt_nt(n):
    n16 = cdiv(n, 16) * 16
    return 16 if n16 <= 16 else 32 if n16 <= 32 else 64 if n16 <= 64 else 128


def dense_case(nat, M, i, o, act):
    sm = sm_count(nat)
    X, W = rnd(M, i, seed=1), rnd(i, o, seed=2) / math.sqrt(i)
    bias, dY = rnd(o, seed=3), rnd(M, o, seed=4) + 2     # mostly positive: a dropped chunk moves every bias sum
    wsb = nat.lib.dtb_dense_workspace_bytes(i, o)
    ws = torch.empty(max(wsb, 16), dtype=torch.uint8, device='cuda')
    st = {}

    def run(lo, hi):
        n = hi - lo
        Y, dX, dW, dB = empty(n, o), empty(n, i), zeros(i, o), zeros(o)
        nat.check(nat.lib.dtb_dense_fwd(P(X[lo:hi]), P(W), P(bias), P(Y), P(ws), wsb, n, i, o, act, None))
        dz = dY[lo:hi].clone()
        nat.check(nat.lib.dtb_dense_bwd(P(X[lo:hi]), P(W), P(Y), P(dz), P(dX), P(dW), P(dB), P(ws), wsb, n, i, o, act, None))
        if (lo, hi) == (0, M):
            st['Y'] = Y
        return [Y, dX], [dW, dB]

    def ref(lo, hi, absolute, keep=None):
        x, dz = X[lo:hi].double(), dY[lo:hi].double()
        if act:
            dz = dz * (st['Y'][lo:hi] > 0)
        if keep is not None:
            dz = dz * keep[:, None]
        if absolute:
            x, dz = x.abs(), dz.abs()
        return [x.T @ dz, dz.sum(0)]

    if o > 8:
        tiles_o, tiles_i = cdiv(o, dt_nt(o)), cdiv(i, dt_nt(i))
        loops = [stride('dense_tc_rows_kernel', cdiv(M, 128) * tiles_o, lambda b: 1, '128-row tile'),
                 Loop('dense_tc_wgrad_kernel', lambda g, b: (cdiv(cdiv(M, 32), g[1]), kDtStages), '32-row chunk', False),
                 stride('dense_tc_rows_kernel', cdiv(M, 128) * tiles_i, lambda b: 1, '128-row tile')]
        if act:
            loops.insert(1, stride('act_bwd_kernel', M * o, lambda b: b[0], 'element'))
        one_pass = min(sm // tiles_o, sm // tiles_i) * 128
        unit = 32
    else:
        loops = [stride('dense_narrow_fwd', M, lambda b: b[0] // 32, 'row'),
                 serial('col_sum_float_kernel', M, 8, 'row'),
                 serial('dense_narrow_bwd_dw', M, 8, 'row'),
                 stride('dense_narrow_bwd_dx', M * i, lambda b: b[0], 'element')]
        one_pass = min(sm * 8 * 8, sm * 16 * 256 // i)
        unit = 8
    return SimpleNamespace(B=M, run=run, loops=loops, one_pass=one_pass, ref=ref, unit=unit, scale='abs', rtol=1e-5)


def att_plan(hf, row_bytes, stat_bytes):
    """pnn_attention.cu att_plan: rows per CTA and buffers of the (head, field) attention kernels"""
    nbuf = 2 if 2 * row_bytes + stat_bytes <= 200 * 1024 else 1
    R = 1 if hf >= 128 else 128 // hf
    while R > 1 and R * (nbuf * row_bytes + stat_bytes) > 96 * 1024:
        R -= 1
    return R, nbuf


def attention_case(nat, B, F, D, heads, nbuf_want=None):
    sm = sm_count(nat)
    x = torch.relu(rnd(B, F, 4 * D, seed=11))
    dY = rnd(B, F, D, seed=12)
    hf = heads * F
    generic = hf > 256
    rf, nf = att_plan(hf, F * (4 * D + 4) * 4, 0)
    rb, nb = att_plan(hf, (F * (4 * D + 4) + 2 * F * (D + 4)) * 4, hf * 16)
    if nbuf_want is not None:
        assert nf == nbuf_want and nb == nbuf_want, (nf, nb)

    def run(lo, hi):
        n = hi - lo
        y, dq0, dq1 = empty(n, F, D), empty(n, F, 4 * D), empty(n, F, 4 * D)
        nat.check(nat.lib.dtb_attention_core_fwd(P(x[lo:hi]), P(y), n, F, D, heads, 1, None))
        nat.check(nat.lib.dtb_attention_core_bwd(P(x[lo:hi]), P(y), P(dY[lo:hi]), P(dq0), n, F, D, heads, 1, 0, None))
        nat.check(nat.lib.dtb_attention_core_bwd(P(x[lo:hi]), P(y), P(dY[lo:hi]), P(dq1), n, F, D, heads, 1, 1, None))
        return [y, dq0, dq1], []

    def group(R):
        def per(b):
            assert generic or b[0] == max(64, cdiv(R * hf, 32) * 32), f'block {b} does not hold {R} rows of {hf} threads'
            return R
        return per

    if generic:
        loops = [stride('attention_core_fwd_kernel', B, lambda b: 1, 'row')] + \
                [stride('attention_core_bwd_kernel', B, lambda b: 1, 'row')] * 2
        one_pass = sm * 8
    else:
        loops = [stride('attention_core_fwd_t_kernel', B, group(rf), 'row')] + \
                [stride('attention_core_bwd_t_kernel', B, group(rb), 'row')] * 2
        one_pass = sm * 8 * min(rf, rb)
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=one_pass)


def cross_case(nat, B, W, n):
    sm = sm_count(nat)
    X, K = rnd(B, W, seed=21), rnd(n, W, seed=22) / math.sqrt(W)
    Bs, dY = rnd(n, W, seed=23) * 0.1, rnd(B, W, seed=24)
    reg_f, reg_b = W <= 1024, W <= 1024 and n <= 8

    def run(lo, hi):
        m = hi - lo
        Y, xw, dX, dK, dB = empty(m, W), empty(m, n), empty(m, W), zeros(n, W), zeros(n, W)
        nat.check(nat.lib.dtb_cross_fwd(P(X[lo:hi]), P(K), P(Bs), P(Y), P(xw), m, W, n, None))
        wsb = nat.lib.dtb_cross_bwd_workspace_bytes(m, W, n)
        ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
        nat.check(nat.lib.dtb_cross_bwd(P(X[lo:hi]), P(K), P(Bs), P(xw), P(dY[lo:hi]), P(dX), P(dK), P(dB), P(ws), wsb, m, W,
                                        n, None))
        return [Y, xw, dX], [dK, dB]

    k64 = [K[l].double().reshape(W, 1).requires_grad_(True) for l in range(n)]
    b64 = [Bs[l].double().reshape(W, 1).requires_grad_(True) for l in range(n)]

    def ref(lo, hi, absolute, keep=None):
        dy = dY[lo:hi].double()
        if keep is not None:
            dy = dy * keep[:, None]
        y = L.cross(X[lo:hi].double(), k64, b64)
        g = torch.autograd.grad((y * dy).sum(), k64 + b64)
        return [torch.stack([t[:, 0] for t in g[:n]]), torch.stack([t[:, 0] for t in g[n:]])]

    warp_rows = lambda b: b[0] // 32
    loops = [stride('cross_fwd_reg_kernel' if reg_f else 'cross_fwd_kernel', B, warp_rows, 'row'),
             stride('cross_bwd_reg_kernel' if reg_b else 'cross_bwd_smem_kernel', B, warp_rows, 'row')]
    for _ in range(cdiv(n, 8)):
        loops += [serial('cross_colreduce_kernel', B, 8, 'row'), stride('cross_gsum_kernel', B, lambda b: b[0], 'row')]
    rows_f = sm * 8 * (8 if reg_f else min(4, 200 * 1024 // (8 * W)))
    rows_b = sm * 8 * (8 if reg_b else min(4, 200 * 1024 // (12 * W)))
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=min(rows_f, rows_b), ref=ref, unit=8, scale='max', rtol=5e-5)


def afm_case(nat, B, F, D=16, H=16):
    sm = sm_count(nat)
    vocab = [11 + i for i in range(F)]
    tab, offs = table(vocab, D, seed=31)
    idx = ids(vocab, B, seed=32)
    wa, ba, ph = rnd(D, H, seed=33) * 3 / math.sqrt(D), rnd(H, seed=34) * 0.1, rnd(H, 1, seed=35)
    gp = rnd(B, D, seed=36)
    P_ = F * (F - 1) // 2
    nb = nat.lib.dtb_afm_workspace_bytes(B, F, D, H)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')

    def run(lo, hi):
        n = hi - lo
        pooled, gt, dwa, dba, dph = empty(n, D), zeros(*tab.shape), zeros(D, H), zeros(H), zeros(H, 1)
        nat.check(nat.lib.dtb_afm_fwd(P(idx[lo:hi]), P(tab), P(offs), P(wa), P(ba), P(ph), P(pooled), n, F, D, H, 1, None,
                                      None))
        nat.check(nat.lib.dtb_afm_bwd(P(idx[lo:hi]), P(tab), P(offs), P(wa), P(ba), P(ph), P(gp[lo:hi]), P(gt), P(dwa),
                                      P(dba), P(dph), P(ws), nb, n, F, D, H, 1, None))
        return [pooled], [gt, dwa, dba, dph]

    t64 = tab.double().requires_grad_(True)
    w64 = [a.double().requires_grad_(True) for a in (wa, ba, ph)]

    def ref(lo, hi, absolute, keep=None):
        g = gp[lo:hi].double()
        if keep is not None:
            g = g * keep[:, None]
        rows = offs[:-1][None, :] + idx[lo:hi].long()
        emb = [t64[rows[:, f]].unsqueeze(1) for f in range(F)]
        pooled = L.afm_pooled(emb, *w64, 'relu')
        return list(torch.autograd.grad((pooled * g).sum(), [t64] + w64))

    nw = 4 if F < 99 else 2 if F < 136 else 1
    loops = [stride('afm_rows_kernel', B, lambda b: b[0] // 32, 'row'),
             stride('afm_rows_kernel', B, lambda b: b[0] // 32, 'row'),
             stride('afm_bwd_gather_kernel', cdiv(B, 128), lambda b: 1, '128-row chunk', axis=1),
             stride('afm_bwd_dw_kernel', B, lambda b: b[0] // 32, 'row')]
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=sm * 4 * nw, ref=ref, unit=1, scale='max', rtol=1e-4,
                           chunk=4096)


def pnn_case(nat, B, kt, F=26, D=16):
    sm = sm_count(nat)
    vocab = [11 + i for i in range(F)]
    tab, offs = table(vocab, D, seed=41)
    idx = ids(vocab, B, seed=42)
    pairs = F * (F - 1) // 2
    kern = rnd(*{0: (D, pairs, D), 1: (pairs, D), 2: (pairs, 1)}[kt], seed=43) / math.sqrt(D)
    g_ip, g_op = rnd(B, pairs, seed=44), rnd(B, pairs, seed=45)

    def run(lo, hi):
        n = hi - lo
        ip, op, gt, dk = empty(n, pairs), empty(n, pairs), zeros(*tab.shape), zeros(*kern.shape)
        nat.check(nat.lib.dtb_pnn_fwd(P(idx[lo:hi]), P(tab), P(offs), P(kern), P(ip), P(op), n, F, D, kt, None, None))
        nat.check(nat.lib.dtb_pnn_bwd(P(idx[lo:hi]), P(tab), P(offs), P(kern), P(g_ip[lo:hi]), P(g_op[lo:hi]), P(gt), P(dk),
                                      n, F, D, kt, None))
        return [ip, op], [gt, dk]

    def ref(lo, hi, absolute, keep=None):
        t64, k64 = tab.double(), kern.double()
        gi, go = g_ip[lo:hi].double(), g_op[lo:hi].double()
        if keep is not None:
            gi, go = gi * keep[:, None], go * keep[:, None]
        if absolute:
            t64, k64, gi, go = t64.abs(), k64.abs(), gi.abs(), go.abs()
        t64, k64 = t64.requires_grad_(True), k64.requires_grad_(True)
        rows = offs[:-1][None, :] + idx[lo:hi].long()
        emb = [t64[rows[:, f]].unsqueeze(1) for f in range(F)]
        loss = (L.inner_product(emb) * gi).sum() + (L.outer_product(emb, k64, ['mat', 'vec', 'num'][kt]) * go).sum()
        return list(torch.autograd.grad(loss, [t64, k64]))

    loops = [stride('pnn_fwd_t_kernel', cdiv(B, 128), lambda b: 1, '128-row chunk', axis=1),
             stride('pnn_bwd_de_t_kernel', cdiv(B, 128), lambda b: 1, '128-row chunk', axis=1)]
    if kt == 0:
        loops.append(serial('pnn_bwd_dk_t_kernel', B, 32, 'row'))
    else:
        loops.append(serial('pnn_bwd_dk_kernel', B, 1, 'row', axis=0))
    one_pass = min(cdiv(sm * 8, F - 1), cdiv(sm * 8, F)) * 128
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=one_pass, ref=ref, unit=128, scale='abs', rtol=2e-5,
                           chunk=1024)


def bilinear_case(nat, B, code, F=26, D=16):
    sm = sm_count(nat)
    pairs = F * (F - 1) // 2
    n_w = {0: 1, 1: F - 1, 2: pairs}[code]
    X, W = rnd(B, F, D, seed=51), rnd(n_w, D, D, seed=52) / math.sqrt(D)
    go = rnd(B, pairs, D, seed=53)

    def run(lo, hi):
        n = hi - lo
        out, dx, dw = empty(n, pairs, D), empty(n, F, D), zeros(n_w, D, D)
        nat.check(nat.lib.dtb_bilinear_fwd(P(X[lo:hi]), P(W), P(out), n, F, D, code, None))
        nat.check(nat.lib.dtb_bilinear_bwd(P(X[lo:hi]), P(W), P(go[lo:hi]), P(dx), P(dw), n, F, D, code, None))
        return [out, dx], [dw]

    bt = ['field_all', 'field_each', 'field_interaction'][code]

    def ref(lo, hi, absolute, keep=None):
        x, g = X[lo:hi].double(), go[lo:hi].double()
        if keep is not None:
            g = g * keep[:, None, None]
        if absolute:
            x, g = x.abs(), g.abs()
        w64 = W.double().requires_grad_(True)
        return list(torch.autograd.grad((L.bilinear_interaction(x, list(w64), bt) * g).sum(), [w64]))

    loops = [stride('bilinear_fwd_kernel', cdiv(B, 128), lambda b: 1, '128-row chunk', axis=1),
             stride('bilinear_bwd_dx_kernel', cdiv(B, 128), lambda b: 1, '128-row chunk', axis=1),
             serial('bilinear_bwd_dw_kernel', B, 32, 'row')]
    one_pass = min(cdiv(sm * 8, F - 1), cdiv(sm * 8, F)) * 128
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=one_pass, ref=ref, unit=128, scale='abs', rtol=2e-5,
                           chunk=2048)


def fgcnn_case(nat, B, H=26, W=16, cin=1, cout=14, kh=7, pool=2):
    sm = sm_count(nat)
    X, K = rnd(B, H, W, cin, seed=61), rnd(kh, 1, cin, cout, seed=62) / math.sqrt(kh * cin)
    bias, gp = rnd(cout, seed=63) * 0.1, rnd(B, cdiv(H, pool), W, cout, seed=64)
    st = {}
    ho = cdiv(H, pool)

    def run(lo, hi):
        n = hi - lo
        y, pooled, dy, dx, dk, db = empty(n, H, W, cout), empty(n, ho, W, cout), empty(n, H, W, cout), empty(n, H, W, cin), \
            zeros(*K.shape), zeros(cout)
        nat.check(nat.lib.dtb_conv_fields_fwd(P(X[lo:hi]), P(K), P(bias), P(y), n, H, W, cin, cout, kh, 2, None))
        nat.check(nat.lib.dtb_maxpool_fields_fwd(P(y), P(pooled), n, H, W * cout, pool, None))
        nat.check(nat.lib.dtb_maxpool_fields_bwd(P(y), P(gp[lo:hi]), P(dy), n, H, W * cout, pool, None))
        nat.check(nat.lib.dtb_conv_fields_bwd(P(X[lo:hi]), P(K), P(y), P(dy), P(dx), P(dk), P(db), n, H, W, cin, cout, kh, 2,
                                              None))
        if (lo, hi) == (0, B):
            st['y'], st['dy'] = y, dy
        return [y, pooled, dy, dx], [dk, db]

    def ref(lo, hi, absolute, keep=None):
        # the filter gradient with dZ = dY tanh'(Y) taken as given (the kernel's own Y and dY): a bilinear form in X, dZ
        y = st['y'][lo:hi].double()
        dz = st['dy'][lo:hi].double() * (1 - y * y)
        x = X[lo:hi].double()
        if keep is not None:
            dz = dz * keep.reshape(hi - lo, H, W, 1)
        if absolute:
            x, dz = x.abs(), dz.abs()
        k64, b64 = K.double().requires_grad_(True), bias.double().requires_grad_(True)
        return list(torch.autograd.grad((L.conv_fields(x, k64, b64, 'linear') * dz).sum(), [k64, b64]))

    n_pos = B * H * W
    loops = [stride('conv_fields_fwd_kernel', n_pos, lambda b: b[0], 'position'),
             stride('maxpool_fields_fwd_kernel', B * ho * W * cout, lambda b: b[0], 'element'),
             stride('maxpool_fields_bwd_kernel', B * ho * W * cout, lambda b: b[0], 'element'),
             stride('conv_fields_bwd_dx_kernel', n_pos, lambda b: b[0], 'position'),
             stride('conv_fields_bwd_dw_tiled_kernel', cdiv(n_pos, 128), lambda b: 1, '128-position tile')]
    one_pass = min(sm * 8 * 256 // (H * W), sm * 8 * 256 // (ho * W * cout))
    # a work unit of the filter gradient is one tile of 128 positions: `unit` rows (mask) below select it
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=one_pass, ref=ref, unit=('positions', H * W, 128),
                           scale='abs', rtol=5e-6)


def fm_gather_case(nat, B, vocab, D=16, C=13):
    sm = sm_count(nat)
    F = len(vocab)
    tab, offs = table(vocab, D, seed=71)
    idx = ids(vocab, B, seed=72)
    dense = rnd(B, C, seed=73)
    wl, g_lin, g_fm = rnd(F + C, seed=74), rnd(B, seed=75), rnd(B, seed=76)
    dout = rnd(B, F, D, seed=77)
    dims = [4 * (1 + f % 4) for f in range(F)]                   # widths 4..16 of a [sum V, 16] table
    dims_c = nat.int_array(dims)
    sd = sum(dims)
    dxr = rnd(B, sd + C, seed=78)

    def run(lo, hi):
        n = hi - lo
        lin, fm, emb, xr = empty(n), empty(n), empty(n, F, D), empty(n, sd + C)
        gt_s, gt_f, gw, gt_r = zeros(*tab.shape), zeros(*tab.shape), zeros(F + C), zeros(*tab.shape)
        i_ = idx[lo:hi]
        nat.check(nat.lib.dtb_fm_linear_fwd(P(i_), P(tab), P(offs), P(dense[lo:hi]), P(wl), P(lin), P(fm), n, F, D, C, None,
                                            None))
        nat.check(nat.lib.dtb_embedding_gather(P(i_), P(tab), P(offs), P(emb), n, F, D, None, None))
        nat.check(nat.lib.dtb_ragged_concat_emb_dense_fwd(P(i_), P(tab), P(offs), dims_c, P(dense[lo:hi]), P(xr), n, F, D, C,
                                                          None, None))
        nat.check(nat.lib.dtb_embedding_scatter_add(P(i_), P(offs), P(dout[lo:hi]), P(gt_s), n, F, D, None))
        nat.check(nat.lib.dtb_fm_linear_bwd(P(i_), P(tab), P(offs), P(dense[lo:hi]), P(wl), P(g_lin[lo:hi]), P(g_fm[lo:hi]),
                                            P(gt_f), P(gw), n, F, D, C, None))
        nat.check(nat.lib.dtb_ragged_concat_emb_dense_bwd(P(i_), P(offs), dims_c, P(dxr[lo:hi]), P(gt_r), n, F, D, C, None))
        return [lin, fm, emb, xr], [gt_s, gt_f, gw, gt_r]

    def ref(lo, hi, absolute, keep=None):
        rows = (offs[:-1][None, :] + idx[lo:hi].long())             # [n, F] table rows
        e = tab.double()[rows]                                      # [n, F, D]
        d_, g1, g2, dx_ = dout[lo:hi].double(), g_lin[lo:hi].double(), g_fm[lo:hi].double(), dxr[lo:hi].double()
        dn, w = dense[lo:hi].double(), wl.double()
        if keep is not None:
            d_, g1, g2, dx_ = d_ * keep[:, None, None], g1 * keep, g2 * keep, dx_ * keep[:, None]
        if absolute:
            e, d_, g1, g2, dx_, dn, w = e.abs(), d_.abs(), g1.abs(), g2.abs(), dx_.abs(), dn.abs(), w.abs()
            fm_g = g2[:, None, None] * (e.sum(1, keepdim=True) + e)
        else:
            fm_g = g2[:, None, None] * (e.sum(1, keepdim=True) - e)
        ge = g1[:, None, None] * w[None, :F, None] + fm_g           # d out / d e[b, f, :]
        scat = lambda vals: torch.zeros(tab.shape, dtype=torch.float64, device='cuda').index_add_(
            0, rows.reshape(-1), vals.reshape(-1, D))
        gw = torch.cat([(g1[:, None] * e.sum(2)).sum(0), (g1[:, None] * dn).sum(0)])
        rag = torch.zeros(rows.shape[0], F, D, dtype=torch.float64, device='cuda')
        c0 = 0
        for f, dd in enumerate(dims):
            rag[:, f, :dd] = dx_[:, c0:c0 + dd]
            c0 += dd
        return [scat(d_), scat(ge), gw, scat(rag)]

    loops = [stride('fm_linear_fwd_vec', cdiv(B, 2), lambda b: b[0] // 32, '2-row warp step'),
             stride('concat_fwd_kernel', B * F * D, lambda b: b[0], 'element'),
             stride('ragged_concat_fwd_kernel', B, lambda b: b[0] // 32, 'row'),
             stride('concat_bwd_kernel', B * F * D // 4, lambda b: b[0], 'float4'),
             stride('fm_linear_bwd_vec', B, lambda b: b[0] // 32, 'row'),
             stride('ragged_concat_bwd_kernel', B, lambda b: b[0] // 32, 'row')]
    one_pass = min(sm * 8 * 8 * 2, sm * 16 * 256 // (F * D), sm * 8 * 8)
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=one_pass, ref=ref, unit=1, scale='abs', rtol=1e-5)


HOT_VOCAB = [1, 2, 3, 1, 2, 3] + [50, 1000, 20000, 7] * 5       # 26 columns, six of them with 1-3 ids


def bn_case(nat, B, W):
    X = rnd(B, W, seed=81) * 3 + torch.linspace(-2, 2, W, device='cuda')
    dY = rnd(B, W, seed=82)
    gamma, beta = rnd(W, seed=83) + 2, rnd(W, seed=84)

    def run(lo, hi):
        n = hi - lo
        Y, dX = empty(n, W), empty(n, W)
        mm, mv, sm_, sv = zeros(W), torch.ones(W, device='cuda'), empty(W), empty(W)
        dg, db = zeros(W), zeros(W)
        ws = torch.empty(2 * W, dtype=torch.float64, device='cuda')
        nat.check(nat.lib.dtb_batchnorm_train_fwd(P(X[lo:hi]), P(Y), P(gamma), P(beta), P(mm), P(mv), P(sm_), P(sv), P(ws), n,
                                                  W, 1e-3, 0.99, None))
        nat.check(nat.lib.dtb_batchnorm_bwd(P(X[lo:hi]), P(dY[lo:hi]), P(dX), P(gamma), P(sm_), P(sv), P(dg), P(db), P(ws), n,
                                            W, 1e-3, None))
        return [], [sm_, sv, mm, mv, dg, db]

    def ref(lo, hi, absolute, keep=None):
        # the statistics of rows [lo, hi) over the whole batch's count: a dropped unit changes the sums, not the count
        x, dy = X[lo:hi].double(), dY[lo:hi].double()
        k = torch.ones(hi - lo, dtype=torch.float64, device='cuda') if keep is None else keep
        mean = (x * k[:, None]).sum(0) / B
        var = (x * x * k[:, None]).sum(0) / B - mean * mean
        inv = 1 / torch.sqrt(var + 1e-3)
        xhat = (x - mean) * inv
        return [mean, var, 0.01 * mean, 0.99 + 0.01 * var, (dy * xhat * k[:, None]).sum(0), (dy * k[:, None]).sum(0)]

    loops = [serial('col_reduce_kernel', B, 8, 'row'), stride('bn_apply_kernel', B * W, lambda b: b[0], 'element'),
             serial('col_reduce_kernel', B, 8, 'row'), stride('bn_bwd_apply_kernel', B * W, lambda b: b[0], 'element')]
    return SimpleNamespace(B=B, run=run, loops=loops, one_pass=None, ref=ref, unit=8, scale='max', rtol=1e-5,
                           whole=True)


# (id, builder, arguments)
CASES = [
    ('dense_429x128_relu', dense_case, (65536, 429, 128, 1)),
    ('dense_128x64_relu', dense_case, (65536, 128, 64, 1)),
    ('dense_32x128_relu_autoint', dense_case, (65536 * 26, 32, 128, 1)),
    # the weight gradient's fp32 wgmma accumulation drifts with the rows of one split (3e-5 of the absolute-value scale
    # at the 12 900 rows per split of 1.7 M rows, on an H100 SXM): its float64 check runs at a quarter of the rows,
    # where a bar that passes it still sees one 32-row chunk left out
    ('dense_32x128_relu_wgrad', dense_case, (16384 * 26, 32, 128, 1)),
    ('dense_64x1_narrow', dense_case, (65536, 64, 1, 0)),
    ('attention_26x32_h4', attention_case, (65536, 26, 32, 4, 2)),
    ('attention_5x16_h2', attention_case, (40000, 5, 16, 2, 2)),
    ('attention_100x64_h1_one_buffer', attention_case, (3500, 100, 64, 1, 1)),
    ('attention_39x16_h8_generic', attention_case, (3500, 39, 16, 8)),
    ('cross_845x6', cross_case, (65500, 845, 6)),
    ('cross_429x6', cross_case, (30000, 429, 6)),
    ('cross_1500x3_smem', cross_case, (15000, 1500, 3)),
    ('cross_300x10_smem_bwd', cross_case, (30000, 300, 10)),
    ('afm_26', afm_case, (16411, 26)),
    ('afm_99', afm_case, (4500, 99)),
    ('pnn_mat', pnn_case, (20011, 0)),
    ('pnn_vec', pnn_case, (20011, 1)),
    ('pnn_num', pnn_case, (20011, 2)),
    ('bilinear_all', bilinear_case, (20011, 0)),
    ('bilinear_each', bilinear_case, (20011, 1)),
    ('bilinear_interaction', bilinear_case, (20011, 2)),
    ('fgcnn', fgcnn_case, (2100,)),
    ('fm_gathers_hot_ids', fm_gather_case, (65536, HOT_VOCAB)),
    ('batchnorm_429', bn_case, (65500, 429)),
]
REDUCTIONS = ['dense_429x128_relu', 'dense_32x128_relu_wgrad', 'dense_64x1_narrow', 'cross_845x6', 'cross_429x6',
              'cross_1500x3_smem', 'cross_300x10_smem_bwd', 'afm_26', 'pnn_mat', 'pnn_vec', 'pnn_num', 'bilinear_all',
              'bilinear_each', 'bilinear_interaction', 'fgcnn', 'fm_gathers_hot_ids', 'batchnorm_429']
ROWS = [c[0] for c in CASES if c[0] not in ('batchnorm_429', 'dense_32x128_relu_wgrad')]
BY_ID = {c[0]: c for c in CASES}


def build(nat, case_id):
    _, fn, args = BY_ID[case_id]
    return fn(nat, *args)


def uneven_slices(B, m):
    sizes = [m, m * 5 // 7 + 3, m * 3 // 5 + 1]
    out, lo, i = [], 0, 0
    while lo < B:
        hi = min(B, lo + min(m, sizes[i % 3]))
        out.append((lo, hi))
        lo, i = hi, i + 1
    return out


# ---------------------------------------------------------------------------------------------
# the launches of every case, recorded in a child process (see the module docstring)
# ---------------------------------------------------------------------------------------------
def _record(path):
    """Child process: for every case, the launches of the full batch and of its first and last one-pass slice."""
    from deeptables_b200 import _native as nat
    rec = {}
    for case_id, _, _ in CASES:
        c = build(nat, case_id)
        big, _ = launches(lambda: c.run(0, c.B))
        ends = []
        if c.one_pass is not None:
            parts = uneven_slices(c.B, c.one_pass)
            ends, _ = launches(lambda: [c.run(lo, hi) for lo, hi in (parts[0], parts[-1])])
        rec[case_id] = {'big': big, 'ends': ends}
        del c
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    with open(path, 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def recorded(tmp_path_factory):
    path = str(tmp_path_factory.mktemp('launches') / 'launches.json')
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f'import sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]; import test_batch_passes_gpu as t; '
            f't._record({path!r})')
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ['-c', code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f'recording the launches failed:\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'
    with open(path) as f:
        return json.load(f)


# ---------------------------------------------------------------------------------------------
# 1. the premise: every loop of the case runs at least 3 passes
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case_id', [c[0] for c in CASES])
def test_loops_run_several_passes(nat, recorded, case_id):
    c = build(nat, case_id)
    print(f'{case_id}: B = {c.B}, passes {passes_of(case_id, recorded[case_id]["big"], c.loops)}')


# ---------------------------------------------------------------------------------------------
# 2. per-row outputs: the full batch against single-pass slices, bit for bit
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case_id', ROWS)
def test_rows_match_single_pass_slices(nat, recorded, case_id):
    c = build(nat, case_id)
    big, _ = c.run(0, c.B)
    parts = uneven_slices(c.B, c.one_pass)
    assert len(parts) >= 3
    res = [c.run(lo, hi)[0] for lo, hi in parts]
    # the kernels of the full batch against those of the first (full) and the last (ragged) slice
    names_big = sorted({k for k, _, _ in recorded[case_id]['big']})
    names_sl = sorted({k for k, _, _ in recorded[case_id]['ends']})
    assert names_big == names_sl, f'{case_id}: the full batch ran {names_big}, the slices {names_sl}'
    for j, got in enumerate(big):
        want = torch.cat([r[j] for r in res])
        if not torch.equal(got, want):
            bad = (got != want).reshape(got.shape[0], -1).any(1).nonzero()[:, 0]
            pytest.fail(f'{case_id}: output {j} differs from the one-pass slices in {len(bad)} of {c.B} rows, first rows '
                        f'{bad[:8].tolist()}, max |diff| {float((got - want).abs().max()):.3e}')


# ---------------------------------------------------------------------------------------------
# 3. reductions over rows against float64
# ---------------------------------------------------------------------------------------------
def _f64(c, lo, hi, absolute, keep=None):
    if getattr(c, 'whole', False):
        return c.ref(lo, hi, absolute, keep)
    step = getattr(c, 'chunk', 16384)
    acc = None
    for a in range(lo, hi, step):
        b = min(hi, a + step)
        part = c.ref(a, b, absolute, None if keep is None else keep[a - lo:b - lo])
        acc = [p.detach() for p in part] if acc is None else [s + p.detach() for s, p in zip(acc, part)]
    return acc


def _left_out(c):
    """rows [lo, hi) and a keep mask over them that drop one work unit from the middle of the batch"""
    if isinstance(c.unit, tuple):                      # positions of a flattened (row, position) index
        _, per_row, n = c.unit
        p0 = (c.B * per_row // 2) // n * n
        lo, hi = p0 // per_row, cdiv(p0 + n, per_row)
        keep = torch.ones((hi - lo) * per_row, dtype=torch.float64, device='cuda')
        keep[p0 - lo * per_row:p0 - lo * per_row + n] = 0
        return lo, hi, keep.reshape(hi - lo, per_row)
    u = c.unit
    lo = (c.B // u // 2) * u
    return lo, lo + u, torch.zeros(u, dtype=torch.float64, device='cuda')


@pytest.mark.parametrize('case_id', REDUCTIONS)
def test_reductions_match_float64(nat, case_id):
    c = build(nat, case_id)
    _, got = c.run(0, c.B)
    want = _f64(c, 0, c.B, False)
    scale = _f64(c, 0, c.B, True) if c.scale == 'abs' else None
    lo, hi, keep = _left_out(c)
    if getattr(c, 'whole', False):
        k = torch.ones(c.B, dtype=torch.float64, device='cuda')
        k[lo:hi] = keep
        short = c.ref(0, c.B, False, k)
    else:
        drop = [a - b for a, b in zip(_f64(c, lo, hi, False), _f64(c, lo, hi, False, keep))]
        short = [w - d for w, d in zip(want, drop)]
    worst, seen = [], []
    for j, (g, w) in enumerate(zip(got, want)):
        s = scale[j] if scale is not None else w.abs().max().expand_as(w)
        bar = c.rtol * s + 1e-30
        err = float(((g.double() - w).abs() / bar).max())
        sees = float(((short[j] - w).abs() / bar).max())
        worst.append(round(err, 4))
        seen.append(round(sees, 1))
        assert err <= 1, f'{case_id}: reduction {j} is off by {err:.2f} of its bar ({c.rtol:g} x {c.scale} scale)'
        assert sees > 1, (f'{case_id}: reduction {j}: the bar does not see one work unit left out ({sees:.2f} of the bar)')
    print(f'{case_id}: worst error / bar {worst}; one unit left out moves the reference by {seen} bars')
