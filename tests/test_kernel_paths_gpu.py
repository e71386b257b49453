"""Which kernel each shape-selected C-ABI op runs, and the inputs its dispatch has to get right.

Most ops pick one of several kernels from the shape, the pointer alignment and a shared-memory budget.  The float64
checks of tests/test_native_gpu.py run the same shapes as the path table below; this file records which kernel each
of those calls reaches (torch.profiler), so a moved threshold cannot silently take a case off its path.  It also
checks weights handed over as unaligned views (what DeepModel.freeze makes of every parameter), out-of-range ids
inside the fused gathers, the first refused shape of each envelope, and the dense Adam tail and device-step variant.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import cin_ref
from kernel_profile import launches as _launched, ran
from oracle import layers_ref as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


_KEEP = []     # ctypes only sees raw pointers: keep every device tensor of a test alive until it ends


@pytest.fixture(autouse=True)
def _keepalive():
    _KEEP.clear()
    yield
    torch.cuda.synchronize()
    _KEEP.clear()


def dev(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    t = t.cuda()
    _KEEP.append(t)
    return t


def shifted(a, off):
    """`a` as a device view `off` floats into a larger (256-byte aligned) buffer, the way a parameter sits inside
    DeepModel's flat parameter buffer."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    buf = torch.zeros(a.size + off + 4, device='cuda')
    v = buf[off:off + a.size]
    v.copy_(torch.from_numpy(a.reshape(-1)))
    _KEEP.append(buf)
    assert v.data_ptr() % 16 == 4 * off
    return v.view(a.shape)


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def make_table(vocab, d, seed=0):
    g = np.random.default_rng(seed)
    tabs = [g.uniform(-0.5, 0.5, size=(v, d)).astype(np.float32) for v in vocab]
    offs = np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64)
    return tabs, np.concatenate(tabs, axis=0), offs


def make_idx(vocab, b, seed=1):
    g = np.random.default_rng(seed)
    return np.stack([g.integers(0, v, size=b) for v in vocab], axis=1).astype(np.int32)


def emb64(tabs, idx):
    """The oracle's (B, 1, D) embeddings in float64, zero where an id is out of range (what the kernels read there)."""
    out = []
    for f, t in enumerate(tabs):
        col = idx[:, f]
        bad = (col < 0) | (col >= len(t))
        e = t[np.where(bad, 0, col)].astype(np.float64)
        e[bad] = 0.0
        out.append(torch.tensor(e[:, None, :]))
    return out


# ---------------------------------------------------------------------------------------------
# which kernels a call launched (tests/kernel_profile.py)
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def launched(nat):
    """_launched, once it has been seen to record one of this library's kernels."""
    _, flat, offs = make_table([5, 6], 4)
    idx = torch.zeros(3, 2, dtype=torch.int32, device='cuda')
    out = torch.empty(3, 2, 4, device='cuda')
    tab, off = torch.tensor(flat).cuda(), torch.tensor(offs).cuda()
    seen, _ = _launched(lambda: nat.check(nat.lib.dtb_embedding_gather(P(idx), P(tab), P(off), P(out), 3, 2, 4, None,
                                                                       None)))
    if not ran(seen, 'concat_fwd_kernel'):
        pytest.fail(f'torch.profiler did not record concat_fwd_kernel for dtb_embedding_gather (it saw {seen}): '
                    f'the kernel-path checks cannot run')
    return _launched


# ---------------------------------------------------------------------------------------------
# one builder per op: seeded inputs (shapes as in tests/test_native_gpu.py), the op's weights, launches of its forward
# and backward on given weight tensors, and its float64 forward
# ---------------------------------------------------------------------------------------------
def make_op(weights, fwd, bwd, want=None, tol=None, bits=0):
    """weights: host arrays of the op's parameters.  fwd(ws) / bwd(ws) launch the op with device tensors `ws` holding
    them and return its outputs / gradients (bwd after a fwd); the fused-gather forwards also take a status word.
    want() is the float64 forward, tol(want) the (rtol, atol) of the op's float64 check in tests/test_native_gpu.py,
    bits the status bits its ids must set."""
    return SimpleNamespace(weights=weights, fwd=fwd, bwd=bwd, want=want, tol=tol, bits=bits)


def _ids(vocab, b, seed, bad_ids):
    """Seeded ids; with bad_ids, one id one past its column's vocabulary and one id of -1 (the status bits they set)."""
    idx = make_idx(vocab, b, seed)
    if not bad_ids:
        return idx, 0
    f1, f2 = 1, len(vocab) - 1
    idx[2, f1] = vocab[f1]
    idx[b - 1, f2] = -1
    return idx, (1 << f1) | (1 << f2)


def zeros(*shape):
    return dev(np.zeros(shape, np.float32))


def fm_op(nat, vocab, d, c, b, bad_ids=False):
    tabs, flat, offs = make_table(vocab, d)
    idx, bits = _ids(vocab, b, 1, bad_ids)
    f = len(vocab)
    g = np.random.default_rng(5)
    dense = g.normal(size=(b, c)).astype(np.float32)
    wl = g.normal(size=(f + c,)).astype(np.float32)
    d_idx, d_tab, d_offs, d_dense = dev(idx), dev(flat), dev(offs), dev(dense) if c else None
    g_lin, g_fm = dev(g.normal(size=b).astype(np.float32)), dev(g.normal(size=b).astype(np.float32))

    def fwd(ws, status=None):
        out_lin, out_fm = zeros(b), zeros(b)
        nat.check(nat.lib.dtb_fm_linear_fwd(P(d_idx), P(d_tab), P(d_offs), P(d_dense), P(ws[0]), P(out_lin), P(out_fm),
                                            b, f, d, c, P(status), None))
        return [out_lin, out_fm]

    def bwd(ws):
        gt, gw = zeros(*flat.shape), zeros(f + c)
        nat.check(nat.lib.dtb_fm_linear_bwd(P(d_idx), P(d_tab), P(d_offs), P(d_dense), P(ws[0]), P(g_lin), P(g_fm), P(gt),
                                            P(gw), b, f, d, c, None))
        return [gt, gw]

    def want():
        emb = emb64(tabs, idx)
        lin = L.linear(emb, torch.tensor(dense, dtype=torch.float64) if c else None,
                       torch.tensor(wl, dtype=torch.float64).reshape(-1, 1))
        return [lin.numpy()[:, 0], L.fm(L.concat_embeddings(emb)).numpy()[:, 0]]
    return make_op([wl], fwd, bwd, want, lambda w: (1e-4, 1e-5), bits)


def att_op(nat, b, f, d, heads):
    g = np.random.default_rng(54)
    d_in = dev(np.maximum(g.normal(size=(b, f, 4 * d)), 0).astype(np.float32))
    dy = dev(g.normal(size=(b, f, d)).astype(np.float32))
    y = zeros(b, f, d)

    def fwd(ws):
        nat.check(nat.lib.dtb_attention_core_fwd(P(d_in), P(y), b, f, d, heads, 1, None))
        return [y]

    def bwd(ws):
        dq = zeros(b, f, 4 * d)
        nat.check(nat.lib.dtb_attention_core_bwd(P(d_in), P(y), P(dy), P(dq), b, f, d, heads, 1, 0, None))
        return [dq]
    return make_op([], fwd, bwd)


def pnn_op(nat, f, d, b, kt, bad_ids=False):
    vocab = [11 + i for i in range(f)]
    tabs, flat, offs = make_table(vocab, d, seed=51)
    idx, bits = _ids(vocab, b, 52, bad_ids)
    g = np.random.default_rng(53)
    pairs = f * (f - 1) // 2
    kern = (g.normal(size={0: (d, pairs, d), 1: (pairs, d), 2: (pairs, 1)}[kt]) / np.sqrt(d)).astype(np.float32)
    d_idx, d_tab, d_offs = dev(idx), dev(flat), dev(offs)
    g_ip, g_op = dev(g.normal(size=(b, pairs)).astype(np.float32)), dev(g.normal(size=(b, pairs)).astype(np.float32))

    def fwd(ws, status=None):
        ip, op = zeros(b, pairs), zeros(b, pairs)
        nat.check(nat.lib.dtb_pnn_fwd(P(d_idx), P(d_tab), P(d_offs), P(ws[0]), P(ip), P(op), b, f, d, kt, P(status), None))
        return [ip, op]

    def bwd(ws):
        gt, dk = zeros(*flat.shape), zeros(*kern.shape)
        nat.check(nat.lib.dtb_pnn_bwd(P(d_idx), P(d_tab), P(d_offs), P(ws[0]), P(g_ip), P(g_op), P(gt), P(dk), b, f, d, kt,
                                      None))
        return [gt, dk]

    def want():
        emb = emb64(tabs, idx)
        k64 = torch.tensor(kern, dtype=torch.float64)
        return [L.inner_product(emb).numpy(), L.outer_product(emb, k64, ['mat', 'vec', 'num'][kt]).numpy()]
    return make_op([kern], fwd, bwd, want, lambda w: (1e-4, 1e-5), bits)


def afm_op(nat, f, d, h, b, bad_ids=False):
    vocab = [11 + i for i in range(f)]
    tabs, flat, offs = make_table(vocab, d, seed=61)
    idx, bits = _ids(vocab, b, 62, bad_ids)
    g = np.random.default_rng(63)
    wa = (g.normal(size=(d, h)) / np.sqrt(d)).astype(np.float32) * 3
    ba = (g.normal(size=(h,)) * 0.1).astype(np.float32)
    ph = g.normal(size=(h, 1)).astype(np.float32)
    d_idx, d_tab, d_offs = dev(idx), dev(flat), dev(offs)
    gp = dev(g.normal(size=(b, d)).astype(np.float32))
    nb = nat.lib.dtb_afm_workspace_bytes(b, f, d, h)
    ws_ = dev(np.zeros(nb, np.uint8))

    def fwd(ws, status=None):
        pooled = zeros(b, d)
        nat.check(nat.lib.dtb_afm_fwd(P(d_idx), P(d_tab), P(d_offs), P(ws[0]), P(ws[1]), P(ws[2]), P(pooled), b, f, d, h, 1,
                                      P(status), None))
        return [pooled]

    def bwd(ws):
        gt, dwa, dba, dph = zeros(*flat.shape), zeros(d, h), zeros(h), zeros(h, 1)
        nat.check(nat.lib.dtb_afm_bwd(P(d_idx), P(d_tab), P(d_offs), P(ws[0]), P(ws[1]), P(ws[2]), P(gp), P(gt), P(dwa),
                                      P(dba), P(dph), P(ws_), nb, b, f, d, h, 1, None))
        return [gt, dwa, dba, dph]

    def want():
        return [L.afm_pooled(emb64(tabs, idx), *(torch.tensor(a, dtype=torch.float64) for a in (wa, ba, ph)), 'relu').numpy()]
    return make_op([wa, ba, ph], fwd, bwd, want, lambda w: (1e-4, 1e-5 * float(np.abs(w[0]).max())), bits)


def bilinear_op(nat, f, d, b, code):
    g = np.random.default_rng(71)
    pairs = f * (f - 1) // 2
    n_w = {0: 1, 1: f - 1, 2: pairs}[code]
    x = g.normal(size=(b, f, d)).astype(np.float32)
    w = (g.normal(size=(n_w, d, d)) / np.sqrt(d)).astype(np.float32)
    d_x, go = dev(x), dev(g.normal(size=(b, pairs, d)).astype(np.float32))

    def fwd(ws):
        out = zeros(b, pairs, d)
        nat.check(nat.lib.dtb_bilinear_fwd(P(d_x), P(ws[0]), P(out), b, f, d, code, None))
        return [out]

    def bwd(ws):
        dx, dw = zeros(b, f, d), zeros(n_w, d, d)
        nat.check(nat.lib.dtb_bilinear_bwd(P(d_x), P(ws[0]), P(go), P(dx), P(dw), b, f, d, code, None))
        return [dx, dw]

    def want():
        bt = ['field_all', 'field_each', 'field_interaction'][code]
        return [L.bilinear_interaction(torch.tensor(x, dtype=torch.float64), list(torch.tensor(w, dtype=torch.float64)),
                                       bt).numpy()]
    return make_op([w], fwd, bwd, want, lambda w_: (1e-4, 1e-5 * float(np.abs(w_[0]).max())))


def dense_op(nat, rows, i, o, act):
    g = np.random.default_rng(7)
    x = g.normal(size=(rows, i)).astype(np.float32)
    w = (g.normal(size=(i, o)) / np.sqrt(i)).astype(np.float32)
    bias = g.normal(size=o).astype(np.float32)
    dy = g.normal(size=(rows, o)).astype(np.float32)
    X = dev(x)
    wsb = nat.lib.dtb_dense_workspace_bytes(i, o)
    ws_ = dev(np.zeros(max(wsb, 16), np.uint8))
    st = {}

    def fwd(ws):
        st['Y'] = Y = zeros(rows, o)
        nat.check(nat.lib.dtb_dense_fwd(P(X), P(ws[0]), P(ws[1]), P(Y), P(ws_), wsb, rows, i, o, act, None))
        return [Y]

    def bwd(ws):
        dX, dW, dB = zeros(rows, i), zeros(i, o), zeros(o)
        nat.check(nat.lib.dtb_dense_bwd(P(X), P(ws[0]), P(st['Y']), P(dev(dy)), P(dX), P(dW), P(dB), P(ws_), wsb, rows, i, o,
                                        act, None))
        return [dX, dW, dB]

    def want():
        x64, w64, b64 = (torch.tensor(a, dtype=torch.float64) for a in (x, w, bias))
        return [torch.tanh(x64 @ w64 + b64).numpy() if act == 2 else L.dense(x64, w64, b64, 'relu' if act else None).numpy()]
    return make_op([w, bias], fwd, bwd, want, lambda w_: (1e-4, 1e-4 if o > 8 else 1e-5))


def cross_op(nat, b, w, n):
    g = np.random.default_rng(14)
    x = g.normal(size=(b, w)).astype(np.float32)
    ks = (g.normal(size=(n, w)) / np.sqrt(w)).astype(np.float32)
    bs = (g.normal(size=(n, w)) * 0.1).astype(np.float32)
    X, dY = dev(x), dev(g.normal(size=(b, w)).astype(np.float32))
    wsb = nat.lib.dtb_cross_bwd_workspace_bytes(b, w, n)
    ws_ = dev(np.zeros(max(wsb, 16), np.uint8))
    st = {}

    def fwd(ws):
        Y, st['xw'] = zeros(b, w), zeros(b, n)
        nat.check(nat.lib.dtb_cross_fwd(P(X), P(ws[0]), P(ws[1]), P(Y), P(st['xw']), b, w, n, None))
        return [Y]

    def bwd(ws):
        dX, dK, dB = zeros(b, w), zeros(n, w), zeros(n, w)
        nat.check(nat.lib.dtb_cross_bwd(P(X), P(ws[0]), P(ws[1]), P(st['xw']), P(dY), P(dX), P(dK), P(dB), P(ws_), wsb, b, w,
                                        n, None))
        return [dX, dK, dB]

    def want():
        return [L.cross(torch.tensor(x, dtype=torch.float64),
                        [torch.tensor(ks[i].reshape(w, 1), dtype=torch.float64) for i in range(n)],
                        [torch.tensor(bs[i].reshape(w, 1), dtype=torch.float64) for i in range(n)]).numpy()]
    return make_op([ks, bs], fwd, bwd, want, lambda w_: (1e-4, 1e-4))


def conv_op(nat, b, h, w, cin, cout, kh, act):
    g = np.random.default_rng(81)
    x = g.normal(size=(b, h, w, cin)).astype(np.float32)
    k = (g.normal(size=(kh, 1, cin, cout)) / np.sqrt(kh * cin)).astype(np.float32)
    bias = (g.normal(size=(cout,)) * 0.1).astype(np.float32)
    code = {'linear': 0, 'relu': 1, 'tanh': 2}[act]
    d_x, dy = dev(x), dev(g.normal(size=(b, h, w, cout)).astype(np.float32))
    st = {}

    def fwd(ws):
        st['y'] = y = zeros(b, h, w, cout)
        nat.check(nat.lib.dtb_conv_fields_fwd(P(d_x), P(ws[0]), P(ws[1]), P(y), b, h, w, cin, cout, kh, code, None))
        return [y]

    def bwd(ws):
        dx, dk, db = zeros(*x.shape), zeros(*k.shape), zeros(cout)
        nat.check(nat.lib.dtb_conv_fields_bwd(P(d_x), P(ws[0]), P(st['y']), P(dy), P(dx), P(dk), P(db), b, h, w, cin, cout,
                                              kh, code, None))
        return [dx, dk, db]

    def want():
        return [L.conv_fields(*(torch.tensor(a, dtype=torch.float64) for a in (x, k, bias)), act).numpy()]
    return make_op([k, bias], fwd, bwd, want, lambda w_: (1e-4, 1e-5))


def cin_op(nat, f, d, sizes, b, precision):
    vocab = [9 + i for i in range(f)]
    tabs, flat, offs = make_table(vocab, d, seed=11)
    idx = make_idx(vocab, b, seed=12)
    g = np.random.default_rng(13)
    fns = L.cin_field_nums(f, sizes, False)
    filt = [(g.normal(size=(f * fns[k], s)) / np.sqrt(f * fns[k])).astype(np.float32) for k, s in enumerate(sizes)]
    bias = np.concatenate([g.normal(size=s).astype(np.float32) * 0.1 for s in sizes])
    wcat = np.concatenate([x.reshape(-1) for x in filt])
    sizes_c, n = nat.int_array(sizes), len(sizes)
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=False))
    ws_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, 0, 1)
    ws_ = dev(np.zeros(ws_bytes, np.uint8))
    saved = dev(np.zeros(nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, 0), np.uint8))
    d_idx, d_tab, d_offs = dev(idx), dev(flat), dev(offs)
    dp = dev(g.normal(size=(b, pw)).astype(np.float32))

    def fwd(ws):
        pooled = zeros(b, pw)
        nat.check(nat.lib.dtb_cin_fwd(P(d_idx), P(d_tab), P(d_offs), P(ws[0]), P(ws[1]), P(pooled), P(saved), P(ws_), ws_bytes,
                                      b, f, d, sizes_c, n, 0, 1, precision, None, None))
        return [pooled]

    def bwd(ws):
        gt, dw, db = zeros(*flat.shape), zeros(*wcat.shape), zeros(*bias.shape)
        nat.check(nat.lib.dtb_cin_bwd(P(d_idx), P(d_tab), P(d_offs), P(ws[0]), P(dp), P(saved), P(gt), P(dw), P(db), P(ws_),
                                      ws_bytes, b, f, d, sizes_c, n, 0, 1, precision, None))
        return [gt, dw, db]

    def want():
        x = torch.cat(emb64(tabs, idx), dim=1)
        return [cin_ref.cin_pooled_f64(x, sizes, False, [torch.tensor(w_, dtype=torch.float64) for w_ in filt],
                                       [torch.tensor(b_, dtype=torch.float64)
                                        for b_ in np.split(bias, np.cumsum(sizes)[:-1])], 1).numpy()]
    tol = 1e-4 if precision == 1 else 1e-3                 # test_cin_fwd_bwd: fp32 path vs the bf16x3 tensor-core path
    return make_op([wcat, bias], fwd, bwd, want, lambda w_: (tol, tol * float(np.abs(w_[0]).max())))


def adam_call(nat, n, off):
    g = np.random.default_rng(9)
    p, m, v, gr = (shifted(a, off) for a in (g.normal(size=n), np.zeros(n), np.zeros(n), g.normal(size=n)))
    return lambda: nat.check(nat.lib.dtb_adam_dense(P(p), P(m), P(v), P(gr), n, 1e-3, 0.9, 0.999, 1e-7, 1, None))


def profile_op(launched, op, backward, ws=None):
    """Kernels of op's forward (or of its backward, after an unprofiled forward) on `ws` (default: aligned weights),
    and what the profiled call returned."""
    ws = [dev(w) for w in op.weights] if ws is None else ws
    if backward:
        op.fwd(ws)
    return launched(lambda: op.bwd(ws) if backward else op.fwd(ws))


FWD, BWD = False, True
# (op, arguments, direction, kernel that must run, kernel that must not run).  The shapes are those of the float64 checks
# in tests/test_native_gpu.py (SHAPES, test_attention_core_fwd_bwd, test_pnn_fwd_bwd, test_bilinear_fwd_bwd,
# test_dense_fwd_bwd, test_dense_tanh_activation), so both files cover the same calls.
PATHS = [
    (fm_op, ([50] * 26, 16, 13, 257), FWD, 'fm_linear_fwd_vec<1>', 'fm_linear_fwd_vec_loop'),
    (fm_op, ([30] * 26, 32, 13, 77), FWD, 'fm_linear_fwd_vec<2>', 'fm_linear_fwd_vec_loop'),
    (fm_op, ([20] * 39, 16, 5, 50), FWD, 'fm_linear_fwd_vec<2>', 'fm_linear_fwd_generic'),
    (fm_op, ([30] * 26, 64, 4, 45), FWD, 'fm_linear_fwd_vec_loop', 'fm_linear_fwd_vec'),
    (fm_op, ([10] * 26, 128, 0, 19), FWD, 'fm_linear_fwd_vec_loop', 'fm_linear_fwd_vec'),
    (fm_op, ([7, 9, 5], 10, 2, 31), FWD, 'fm_linear_fwd_generic', 'fm_linear_fwd_vec'),
    (fm_op, ([7, 9, 5, 6], 12, 3, 21), FWD, 'fm_linear_fwd_generic', 'fm_linear_fwd_vec'),
    (fm_op, ([30] * 26, 64, 4, 45), BWD, 'fm_linear_bwd_vec', 'fm_linear_bwd_generic'),
    (fm_op, ([10] * 26, 128, 0, 19), BWD, 'fm_linear_bwd_vec', 'fm_linear_bwd_generic'),
    (fm_op, ([7, 9, 5], 10, 2, 31), BWD, 'fm_linear_bwd_generic', 'fm_linear_bwd_vec'),
    (fm_op, ([7, 9, 5, 6], 12, 3, 21), BWD, 'fm_linear_bwd_generic', 'fm_linear_bwd_vec'),
    (att_op, (13, 5, 10, 2), FWD, 'attention_core_fwd_kernel', 'attention_core_fwd_t_kernel'),
    (att_op, (13, 5, 10, 2), BWD, 'attention_core_bwd_kernel', 'attention_core_bwd_t_kernel'),
    (att_op, (21, 6, 24, 2), FWD, 'attention_core_fwd_kernel', 'attention_core_fwd_t_kernel'),
    (att_op, (21, 6, 24, 2), BWD, 'attention_core_bwd_kernel', 'attention_core_bwd_t_kernel'),
    (att_op, (9, 39, 16, 8), FWD, 'attention_core_fwd_kernel', 'attention_core_fwd_t_kernel'),
    (att_op, (9, 39, 16, 8), BWD, 'attention_core_bwd_kernel', 'attention_core_bwd_t_kernel'),
    (att_op, (2, 128, 64, 8), FWD, 'attention_core_fwd_kernel', 'attention_core_fwd_t_kernel'),
    (att_op, (2, 128, 64, 8), BWD, 'attention_core_bwd_kernel', 'attention_core_bwd_t_kernel'),
    (att_op, (5, 150, 64, 1), FWD, 'attention_core_fwd_t_kernel<64>', 'attention_core_fwd_kernel'),
    (att_op, (5, 150, 64, 1), BWD, 'attention_core_bwd_kernel', 'attention_core_bwd_t_kernel'),
    (att_op, (33, 26, 32, 1), FWD, 'attention_core_fwd_t_kernel<32>', 'attention_core_fwd_kernel'),
    (att_op, (33, 26, 32, 1), BWD, 'attention_core_bwd_t_kernel<32>', 'attention_core_bwd_kernel'),
    (att_op, (19, 13, 16, 8), FWD, 'attention_core_fwd_t_kernel<2>', 'attention_core_fwd_kernel'),
    (att_op, (19, 13, 16, 8), BWD, 'attention_core_bwd_t_kernel<2>', 'attention_core_bwd_kernel'),
    (att_op, (7, 5, 128, 2), FWD, 'attention_core_fwd_t_kernel<64>', 'attention_core_fwd_kernel'),
    (att_op, (7, 5, 128, 2), BWD, 'attention_core_bwd_t_kernel<64>', 'attention_core_bwd_kernel'),
    (pnn_op, (26, 32, 40, 0), FWD, 'pnn_fwd_t_kernel<32>', 'pnn_fwd_kernel'),
    (pnn_op, (26, 32, 40, 0), BWD, 'pnn_bwd_dk_t_kernel<32>', 'pnn_bwd_dk_kernel'),
    (pnn_op, (45, 4, 9, 0), FWD, 'pnn_fwd_t_kernel<4>', 'pnn_fwd_kernel'),
    (pnn_op, (45, 4, 9, 0), BWD, 'pnn_bwd_de_t_kernel<4>', 'pnn_bwd_de_kernel'),
    (pnn_op, (7, 3, 20, 0), FWD, 'pnn_fwd_kernel', 'pnn_fwd_t_kernel'),
    (pnn_op, (7, 3, 20, 0), BWD, 'pnn_bwd_dk_kernel', 'pnn_bwd_dk_t_kernel'),
    (bilinear_op, (26, 32, 70, 2), BWD, 'bilinear_bwd_dw_kernel<32>', None),
    (bilinear_op, (51, 32, 9, 2), BWD, 'bilinear_bwd_dw_kernel<32>', None),
    (dense_op, (300, 64, 10, 1), FWD, 'dense_tc_rows_kernel<16>', 'dense_narrow_fwd'),
    (dense_op, (300, 64, 10, 1), BWD, 'dense_tc_wgrad_kernel<16>', 'dense_narrow_bwd_dw'),
    (dense_op, (130, 50, 16, 0), BWD, 'dense_tc_wgrad_kernel<16>', 'dense_narrow_bwd_dw'),
    (dense_op, (257, 37, 33, 1), FWD, 'dense_tc_rows_kernel<64>', 'dense_narrow_fwd'),
    (dense_op, (129, 40, 10, 2), FWD, 'dense_tc_rows_kernel<16>', 'dense_narrow_fwd'),
    (dense_op, (200, 48, 5, 2), FWD, 'dense_narrow_fwd', 'dense_tc_rows_kernel'),
]


def _path_id(op, args, backward, must):
    parts = [f'{len(a)}x{a[0]}' if isinstance(a, list) else str(a) for a in args]
    return '-'.join([op.__name__[:-len('_op')]] + parts + ['bwd' if backward else 'fwd', must])


@pytest.mark.parametrize('op,args,backward,must,must_not', PATHS, ids=[_path_id(*p[:4]) for p in PATHS])
def test_kernel_path(nat, launched, op, args, backward, must, must_not):
    kernels, _ = profile_op(launched, op(nat, *args), backward)
    names = [k for k, _, _ in kernels]
    assert ran(kernels, must), f'{must} did not run; launched: {names}'
    assert must_not is None or not ran(kernels, must_not), f'{must_not} ran; launched: {names}'


@pytest.mark.parametrize('off,must,must_not', [(0, 'adam_dense_vec4_kernel', None),
                                               (0, 'adam_dense_kernel', None),           # the n % 4 tail
                                               (1, 'adam_dense_kernel', 'adam_dense_vec4_kernel')])
def test_adam_kernel_path(nat, launched, off, must, must_not):
    kernels, _ = launched(adam_call(nat, 1003, off))
    names = [k for k, _, _ in kernels]
    assert ran(kernels, must), f'{must} did not run; launched: {names}'
    assert must_not is None or not ran(kernels, must_not), f'{must_not} ran; launched: {names}'


# rows per CTA of the AFM warp-per-row kernels at D = H = 16: shared memory halves them at F = 99 and again at F = 136
@pytest.mark.parametrize('f,b,warps', [(26, 70, 4), (98, 17, 4), (99, 9, 2), (135, 10, 2), (136, 11, 1), (178, 9, 1)])
def test_afm_warps_per_cta(nat, launched, f, b, warps):
    op = afm_op(nat, f, 16, 16, b)
    for backward in (FWD, BWD):
        kernels, _ = profile_op(launched, op, backward)
        rows_kernels = [(k, blk) for k, _, blk in kernels if k.startswith('afm_rows_kernel<')]
        assert rows_kernels, f'afm_rows_kernel did not run; launched: {kernels}'
        for k, blk in rows_kernels:
            assert tuple(blk) == (32 * warps, 1, 1), f'{k} ran with block {blk}, expected {warps} warps'


# ---------------------------------------------------------------------------------------------
# weights as unaligned views (DeepModel.freeze places every parameter at any 4-byte offset of one buffer)
# ---------------------------------------------------------------------------------------------
MISALIGNED = [   # (id, op, arguments, the forward kernel the shape selects)
    ('fm', fm_op, ([30] * 26, 32, 13, 77), 'fm_linear_fwd_vec<2>'),
    ('dense_wide', dense_op, (300, 64, 10, 1), 'dense_tc_rows_kernel<16>'),
    ('dense_narrow', dense_op, (77, 64, 1, 0), 'dense_narrow_fwd'),
    ('cross_reg', cross_op, (50, 429, 6), 'cross_fwd_reg_kernel<16>'),
    ('cross_smem', cross_op, (21, 1500, 3), 'cross_fwd_kernel'),
    ('pnn_t', pnn_op, (26, 16, 70, 0), 'pnn_fwd_t_kernel<16>'),
    ('pnn_generic', pnn_op, (7, 3, 20, 0), 'pnn_fwd_kernel'),
    ('afm', afm_op, (26, 16, 16, 70), 'afm_rows_kernel'),
    ('bilinear_all', bilinear_op, (26, 16, 150, 0), 'bilinear_fwd_kernel<16>'),
    ('bilinear_interaction', bilinear_op, (12, 8, 300, 2), 'bilinear_fwd_kernel<8>'),
    ('conv', conv_op, (9, 26, 16, 1, 14, 7, 'tanh'), 'conv_fields_fwd_kernel'),
    ('cin_fused', cin_op, (10, 8, (64, 32), 50, 2), 'cin_wg_fwd_kernel'),
    ('cin_any_shape', cin_op, (10, 8, (64, 32), 50, 1), 'cin_build_z_kernel'),
]


@pytest.mark.parametrize('op,args,kernel', [m[1:] for m in MISALIGNED], ids=[m[0] for m in MISALIGNED])
def test_misaligned_weights(nat, launched, op, args, kernel):
    """Weights at +1, +2 and +3 floats.  No op chooses its kernels by the alignment of its weights, so the shifted runs
    must launch the same kernels as the aligned one, and produce a bit-identical forward, which also matches the float64
    oracle within the op's tolerance.  The backward (float64-checked with aligned weights in tests/test_native_gpu.py)
    must match the aligned backward up to the order of its fp32 atomics (two runs of the fused CIN backward differ by up
    to 2e-6 of the largest gradient, test_cin_tensor_core_backward)."""
    o = op(nat, *args)
    want = o.want()
    rtol, atol = o.tol(want)
    ws0 = [dev(w) for w in o.weights]
    kf0, fwd0 = launched(lambda: o.fwd(ws0))
    kb0, bwd0 = launched(lambda: o.bwd(ws0))
    assert ran(kf0, kernel), f'{kernel} did not run; launched: {kf0}'
    for got, w_ in zip(fwd0, want):
        np.testing.assert_allclose(got.cpu().numpy(), w_, rtol=rtol, atol=atol, err_msg='aligned weights')
    for off in (1, 2, 3):
        ws = [shifted(w, off) for w in o.weights]
        kf, fwd = launched(lambda: o.fwd(ws))
        kb, bwd = launched(lambda: o.bwd(ws))
        assert [k for k, _, _ in kf] == [k for k, _, _ in kf0], f'weights at +{off} floats: forward ran {kf}, aligned {kf0}'
        assert [k for k, _, _ in kb] == [k for k, _, _ in kb0], f'weights at +{off} floats: backward ran {kb}, aligned {kb0}'
        for got, got0, w_ in zip(fwd, fwd0, want):
            assert torch.equal(got, got0), f'weights at +{off} floats: the forward differs from the aligned run'
            np.testing.assert_allclose(got.cpu().numpy(), w_, rtol=rtol, atol=atol, err_msg=f'weights at +{off} floats')
        for got, got0 in zip(bwd, bwd0):
            sc = max(float(got0.abs().max()), 1e-30)
            np.testing.assert_allclose(got.cpu().numpy(), got0.cpu().numpy(), rtol=1e-5, atol=2e-6 * sc,
                                       err_msg=f'backward, weights at +{off} floats')


# ---------------------------------------------------------------------------------------------
# out-of-range ids inside the fused gathers: status bit of the field, the embedding reads as zero
# ---------------------------------------------------------------------------------------------
OUT_OF_RANGE = [   # (id, op, arguments): the fused-gather forward paths, shapes of the path table
    ('fm_vec1', fm_op, ([50] * 26, 16, 13, 64)),
    ('fm_vec2', fm_op, ([30] * 26, 32, 13, 77)),
    ('fm_vec_loop', fm_op, ([30] * 26, 64, 4, 45)),
    ('fm_generic', fm_op, ([7, 9, 5], 10, 2, 31)),
    ('pnn_t', pnn_op, (26, 16, 70, 0)),
    ('pnn_generic', pnn_op, (7, 3, 20, 0)),
    ('afm', afm_op, (26, 16, 16, 70)),
]


@pytest.mark.parametrize('op,args', [m[1:] for m in OUT_OF_RANGE], ids=[m[0] for m in OUT_OF_RANGE])
def test_out_of_range_ids(nat, op, args):
    """One id past its column's vocabulary and one of -1: the status bits of both fields (as for dtb_embedding_gather)
    and outputs equal to the float64 oracle with those two embeddings zero."""
    o = op(nat, *args, bad_ids=True)
    status = torch.zeros(1, dtype=torch.int32, device='cuda')
    got = o.fwd([dev(w) for w in o.weights], status)
    assert int(status.item()) == o.bits
    want = o.want()
    rtol, atol = o.tol(want)
    for g_, w_ in zip(got, want):
        np.testing.assert_allclose(g_.cpu().numpy(), w_, rtol=rtol, atol=atol)


# ---------------------------------------------------------------------------------------------
# envelope edges: the first refused shape returns an error and a message, and launches nothing.  The last accepted shape
# of each is in the float64 checks of tests/test_native_gpu.py (PNN F = 45, bilinear F = 51 at D = 32, AFM F = 178 at
# D = H = 16, attention heads * F = 1024 and head width 64).
# ---------------------------------------------------------------------------------------------
def _refused(nat, call, message):
    before = nat.lib.dtb_launch_count()
    rc = call()
    torch.cuda.synchronize()
    assert rc != 0, 'accepted a shape outside the envelope'
    assert message in nat.last_error(), nat.last_error()
    assert nat.lib.dtb_launch_count() == before, 'a refused call launched a kernel'


@pytest.mark.parametrize('d', [4, 3])
def test_pnn_refuses_more_than_1024_pairs(nat, d):
    f, b = 46, 4
    vocab = [11] * f
    _, flat, offs = make_table(vocab, d)
    d_idx, d_tab, d_offs = dev(make_idx(vocab, b)), dev(flat), dev(offs)
    pairs = f * (f - 1) // 2
    k, ip, op = dev(np.zeros((d, pairs, d), np.float32)), dev(np.zeros((b, pairs), np.float32)), dev(np.zeros((b, pairs), np.float32))
    gt, dk = dev(np.zeros(flat.shape, np.float32)), dev(np.zeros((d, pairs, d), np.float32))
    _refused(nat, lambda: nat.lib.dtb_pnn_fwd(P(d_idx), P(d_tab), P(d_offs), P(k), P(ip), P(op), b, f, d, 0, None, None),
             '1035 pairs exceed one CTA')
    _refused(nat, lambda: nat.lib.dtb_pnn_bwd(P(d_idx), P(d_tab), P(d_offs), P(k), P(ip), P(op), P(gt), P(dk), b, f, d, 0,
                                              None), '1035 pairs exceed one CTA')


def test_bilinear_refuses_52_fields_at_d32(nat):
    f, d, b = 52, 32, 4
    pairs = f * (f - 1) // 2
    x, w = dev(np.zeros((b, f, d), np.float32)), dev(np.zeros((pairs, d, d), np.float32))
    out, dx, dw = dev(np.zeros((b, pairs, d), np.float32)), dev(np.zeros((b, f, d), np.float32)), dev(np.zeros((pairs, d, d), np.float32))
    _refused(nat, lambda: nat.lib.dtb_bilinear_fwd(P(x), P(w), P(out), b, f, d, 2, None), 'F = 52, D = 32')
    _refused(nat, lambda: nat.lib.dtb_bilinear_bwd(P(x), P(w), P(out), P(dx), P(dw), b, f, d, 2, None), 'F = 52, D = 32')


def test_afm_refuses_past_one_warp(nat):
    f, d, h, b = 179, 16, 16, 4
    vocab = [11] * f
    _, flat, offs = make_table(vocab, d)
    d_idx, d_tab, d_offs = dev(make_idx(vocab, b)), dev(flat), dev(offs)
    wa, ba, ph = dev(np.zeros((d, h), np.float32)), dev(np.zeros(h, np.float32)), dev(np.zeros((h, 1), np.float32))
    pooled, gt = dev(np.zeros((b, d), np.float32)), dev(np.zeros(flat.shape, np.float32))
    dwa, dba, dph = dev(np.zeros((d, h), np.float32)), dev(np.zeros(h, np.float32)), dev(np.zeros((h, 1), np.float32))
    nb = nat.lib.dtb_afm_workspace_bytes(b, f, d, h)
    ws = dev(np.zeros(nb, np.uint8))
    _refused(nat, lambda: nat.lib.dtb_afm_fwd(P(d_idx), P(d_tab), P(d_offs), P(wa), P(ba), P(ph), P(pooled), b, f, d, h, 1,
                                              None, None), '179 fields need')
    _refused(nat, lambda: nat.lib.dtb_afm_bwd(P(d_idx), P(d_tab), P(d_offs), P(wa), P(ba), P(ph), P(pooled), P(gt), P(dwa),
                                              P(dba), P(dph), P(ws), nb, b, f, d, h, 1, None), '179 fields need')


@pytest.mark.parametrize('f,d,heads', [(41, 25, 25), (5, 130, 2)], ids=['heads_x_fields_1025', 'head_width_65'])
def test_attention_refuses_outside_envelope(nat, f, d, heads):
    b = 2
    x, y = dev(np.zeros((b, f, 4 * d), np.float32)), dev(np.zeros((b, f, d), np.float32))
    dy, dx = dev(np.zeros((b, f, d), np.float32)), dev(np.zeros((b, f, 4 * d), np.float32))
    msg = 'head width <= 64 and heads*fields <= 1024'
    _refused(nat, lambda: nat.lib.dtb_attention_core_fwd(P(x), P(y), b, f, d, heads, 1, None), msg)
    _refused(nat, lambda: nat.lib.dtb_attention_core_bwd(P(x), P(y), P(dy), P(dx), b, f, d, heads, 1, 0, None), msg)


# ---------------------------------------------------------------------------------------------
# dense Adam: the scalar tail (n % 4 != 0), the all-scalar path (unaligned buffers), the device-step variant
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('off', [0, 1])
def test_adam_dense_tail_and_unaligned(nat, off):
    from deeptables_b200.engine import adam_alpha
    g = np.random.default_rng(9)
    n = 1003
    p0 = g.normal(size=n).astype(np.float32)
    pt, m, v = shifted(p0, off), shifted(np.zeros(n), off), shifted(np.zeros(n), off)
    po, mo, vo = torch.tensor(p0.copy()), torch.zeros(n), torch.zeros(n)
    for step in range(1, 6):
        grad = g.normal(size=n).astype(np.float32)
        gd = shifted(grad, off)
        nat.check(nat.lib.dtb_adam_dense(P(pt), P(m), P(v), P(gd), n, adam_alpha(step), 0.9, 0.999, 1e-7, 1, None))
        assert float(gd.abs().sum()) == 0.0                   # zero_grad, the tail included
        L.adam_step(po, torch.tensor(grad), mo, vo, step)
    # the tolerances of test_adam_dense_matches_oracle (fused multiply-adds against torch-CPU's double rounding)
    np.testing.assert_allclose(pt.cpu().numpy(), po.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(m.cpu().numpy(), mo.numpy(), rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(v.cpu().numpy(), vo.numpy(), rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize('off', [0, 1])
def test_adam_dense_dev_matches_host_step(nat, off):
    """dtb_adam_dense_dev (step size read from alpha_table[*step + 1], as a captured graph replays it) is bit-identical
    to dtb_adam_dense given that step size."""
    from deeptables_b200.engine import adam_alpha
    g = np.random.default_rng(19)
    n, steps = 1003, 4
    p0 = g.normal(size=n).astype(np.float32)
    alpha = dev(np.array([0.0] + [adam_alpha(s) for s in range(1, steps + 2)], dtype=np.float32))
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    ph, mh, vh = shifted(p0, off), shifted(np.zeros(n), off), shifted(np.zeros(n), off)
    pd, md, vd = shifted(p0, off), shifted(np.zeros(n), off), shifted(np.zeros(n), off)
    for step in range(1, steps + 1):
        grad = g.normal(size=n).astype(np.float32)
        gh, gd = shifted(grad, off), shifted(grad, off)
        nat.check(nat.lib.dtb_adam_dense(P(ph), P(mh), P(vh), P(gh), n, float(alpha[step].item()), 0.9, 0.999, 1e-7, 1,
                                         None))
        step_dev.fill_(step - 1)                              # steps completed before this one
        nat.check(nat.lib.dtb_adam_dense_dev(P(pd), P(md), P(vd), P(gd), n, P(alpha), P(step_dev), 0.9, 0.999, 1e-7, 1,
                                             None))
        assert float(gd.abs().sum()) == 0.0
    assert not torch.equal(pd, torch.tensor(p0, device='cuda'))
    for name, a_, b_ in (('weights', pd, ph), ('m', md, mh), ('v', vd, vh)):
        assert torch.equal(a_, b_), f'{name}: device-step Adam differs from the host-step kernel'
