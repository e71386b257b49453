"""The any-shape CIN formulation (csrc/cin_fp32.cu) against a float64 CIN.

dtb_cin_fwd / dtb_cin_bwd run the fused wgmma kernels only inside their envelope (D in {4, 8, 16, 32}, F <= 64, <= 64
hidden fields and <= 128 feature maps per layer); everything else runs the any-shape formulation, which also serves
as the yardstick of the fused backward's own tests.  This file runs that path at each edge just outside the envelope
and across several batch chunks of its outer product, through the same forward -> backward phase 1 -> phase 2
sequence as CINFn, and checks every output against float64.  It also checks the dispatch and the refusals at those
shapes, and out-of-range ids on both CIN paths.

The float64 CIN below takes its relu masks from the kernel's saved activations: a pre-activation within rounding of
zero may flip its mask between fp32 and float64, which would move that batch row's whole gradient.  Both the saved
activations and every mask disagreement are checked against float64 before the masks are used.
"""
import ctypes

import numpy as np
import pytest
import torch

import cin_ref
from oracle import layers_ref as L

pytestmark = pytest.mark.gpu

ACT_NONE, ACT_RELU = 0, 1
ERR_INVALID_ARG, ERR_UNSUPPORTED = -1, -2
TOL = 1e-4            # any-shape path (bf16x3 GEMMs, fp32 accumulation): max error per tensor / max |float64|
TOL_FUSED = 1e-3      # fused bf16x3 path: the precision-2 tolerance of test_native_gpu.py::test_cin_fwd_bwd


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


# ---------------------------------------------------------------------------------------------
# shapes
# ---------------------------------------------------------------------------------------------
def field_nums(f, sizes, direct):
    return L.cin_field_nums(f, sizes, direct)[:len(sizes)]      # H_k of each layer's input


def kmax(f, sizes, direct):
    return max(f * h for h in field_nums(f, sizes, direct))


def chunk_rows(b, d, k_max):
    """fp32_chunk_rows of cin_fp32.cu: batch rows per chunk so that one fp32 Z = [rows * D, Kmax] fits 384 MiB."""
    rows = (384 << 20) // (d * k_max * 4)
    return int(min(max(rows, 1), b))


def n_chunks(b, d, k_max):
    return -(-b // chunk_rows(b, d, k_max))


# (id, F, D, sizes, direct, use_bias, act, B, the same shape moved just inside the fused envelope)
OUTSIDE = [
    ('F65', 65, 4, (16, 9), False, True, ACT_RELU, 41, (64, 4, (16, 9), False)),
    ('D64', 7, 64, (16, 8), False, False, ACT_RELU, 37, (7, 32, (16, 8), False)),
    ('D5', 9, 5, (12, 7), False, True, ACT_NONE, 33, (9, 4, (12, 7), False)),
    ('D2', 6, 2, (10, 4), False, False, ACT_RELU, 50, (6, 4, (10, 4), False)),
    ('D12', 11, 12, (20, 10), False, True, ACT_RELU, 29, (11, 16, (20, 10), False)),
    ('L129', 10, 8, (16, 129), False, True, ACT_RELU, 35, (10, 8, (16, 128), False)),
    ('direct72', 6, 8, (72, 16), True, False, ACT_RELU, 31, (6, 8, (64, 16), True)),
    ('layers8', 5, 3, (8, 8, 8, 8, 8, 8, 8, 6), False, True, ACT_RELU, 23, (5, 4, (8, 8, 8, 8, 8, 8, 8, 6), False)),
    ('F1_D64', 1, 64, (4, 3), False, False, ACT_NONE, 40, (1, 32, (4, 3), False)),
]

# several chunks of Z: Kmax = F^2 = 9216 at D = 64 gives 170 rows per chunk; the narrow first layer keeps float64 cheap
MC_F, MC_D = 96, 64
MULTI_CHUNK = [
    ('chunks3_ragged', MC_F, MC_D, (8, 6, 4), False, True, ACT_RELU, 347, (64, 32, (8, 6, 4), False)),   # 170+170+7
    ('chunks2_exact', MC_F, MC_D, (8, 6), False, True, ACT_NONE, 340, (64, 32, (8, 6), False)),          # 170+170
    ('chunks2_last1', MC_F, MC_D, (8, 6), True, True, ACT_RELU, 171, (64, 32, (8, 6), True)),            # 170+1
]


def test_multi_chunk_cases_cover_the_chunk_edges():
    rows = chunk_rows(347, MC_D, MC_F * MC_F)
    assert rows == 170
    nb = {c[0]: (n_chunks(c[7], c[2], kmax(c[1], c[3], c[4])), c[7] % rows) for c in MULTI_CHUNK}
    assert nb['chunks3_ragged'][0] == 3 and nb['chunks3_ragged'][1] != 0
    assert nb['chunks2_exact'] == (2, 0)
    assert nb['chunks2_last1'] == (2, 1)


# ---------------------------------------------------------------------------------------------
# float64 CIN
# ---------------------------------------------------------------------------------------------
def gather64(tabs, idx):
    """x0 [B, F, D] in float64; zero where an id is outside its table (what the kernels read there)."""
    out = np.zeros((idx.shape[0], len(tabs), tabs[0].shape[1]))
    for i, t in enumerate(tabs):
        ok = (idx[:, i] >= 0) & (idx[:, i] < len(t))
        out[ok, i] = t[idx[ok, i]]
    return out


def scatter64(dx0, idx, tabs):
    """Table gradient of the gather: dx0 [B, F, D] added into the rows the in-range ids name."""
    want = [np.zeros(t.shape) for t in tabs]
    for i, t in enumerate(tabs):
        ok = (idx[:, i] >= 0) & (idx[:, i] < len(t))
        np.add.at(want[i], idx[ok, i], dx0[ok, i])
    return np.concatenate(want, axis=0)


def cin64(x0, filt, bias, sizes, direct, act, d_pooled, masks=None, block_rows=None):
    """Float64 CIN on x0 [B, F, D] and the gradients of sum(pooled * d_pooled).

    Layout of cin_fp32.cu: rows (b, d); Z_k[(b,d), i*H_k + j] = x0[b,i,d] * h_k[(b,d), j]; T_k = act(Z_k W_k + bias_k);
    h_{k+1} = T_k (direct) or its first half; pooled = the sum over d of the rest (all of the last layer).  Under relu,
    masks[k] ([B, D, L_k] bool) replaces pre_k > 0 when given.  Batch rows are independent, so they are evaluated in
    blocks that keep one float64 Z near 100 MB, and the weight gradients of the blocks are added up."""
    b_all, f, d = x0.shape
    n = len(sizes)
    if block_rows is None:
        block_rows = max(1, int(100e6 // (8 * d * kmax(f, sizes, direct))))
    w64 = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in filt]
    b64 = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in bias] if bias is not None else []
    pooled, dx0 = [], []
    pre = [[] for _ in sizes]
    post = [[] for _ in sizes]
    dw = [np.zeros(w.shape) for w in filt]
    db = [np.zeros(v.shape) for v in bias] if bias is not None else None
    for b0 in range(0, b_all, block_rows):
        rows = slice(b0, b0 + block_rows)
        x = torch.tensor(x0[rows], dtype=torch.float64, requires_grad=True)
        xt = x.transpose(1, 2)                                       # x0t [b, D, F]
        h, pools = xt, []
        for k, size in enumerate(sizes):
            z = (xt.unsqueeze(-1) * h.unsqueeze(-2)).reshape(xt.shape[0], d, -1)
            p = z @ w64[k]
            if bias is not None:
                p = p + b64[k]
            if act == ACT_RELU:
                t = p * torch.as_tensor(masks[k][rows], dtype=torch.float64) if masks is not None else torch.relu(p)
            else:
                t = p
            pre[k].append(p.detach().numpy())
            post[k].append(t.detach().numpy())
            if direct:
                h, pool = t, t
            elif k < n - 1:
                h, pool = t[..., :size // 2], t[..., size // 2:]
            else:
                pool = t
            pools.append(pool.sum(1))
        out = torch.cat(pools, dim=1)
        grads = torch.autograd.grad((out * torch.as_tensor(d_pooled[rows], dtype=torch.float64)).sum(), [x] + w64 + b64)
        pooled.append(out.detach().numpy())
        dx0.append(grads[0].numpy())
        for k in range(n):
            dw[k] += grads[1 + k].numpy()
            if bias is not None:
                db[k] += grads[1 + n + k].numpy()
    return dict(pooled=np.concatenate(pooled), pre=[np.concatenate(v) for v in pre],
                T=[np.concatenate(v) for v in post], dx0=np.concatenate(dx0), dw=dw, db=db)


def make_weights(f, sizes, direct, use_bias, seed):
    """Filters scaled by 1 / (sqrt(K_k) * rms of the embeddings), which keeps every layer's activations near 1, so that
    the pooled columns of the last of 8 layers weigh as much in the check as those of the first."""
    g = np.random.default_rng(seed)
    filt = [(g.normal(size=(f * h, s)) / (np.sqrt(f * h) * np.sqrt(1 / 12))).astype(np.float32)
            for h, s in zip(field_nums(f, sizes, direct), sizes)]
    bias = [(g.normal(size=s) * 0.1).astype(np.float32) for s in sizes] if use_bias else None
    return filt, bias


@pytest.mark.parametrize('direct', [False, True])
def test_float64_cin_matches_the_oracle(direct):
    """The float64 CIN of this file, in row blocks of 4, against oracle.layers_ref.cin at act=linear."""
    f, d, b = 4, 3, 9
    sizes = (6, 5) if not direct else (5, 3)
    vocab = [7, 8, 9, 10]
    tabs, _, _ = make_table(vocab, d, seed=2)
    idx = make_idx(vocab, b, seed=3)
    filt, bias = make_weights(f, sizes, direct, True, seed=4)
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=direct))
    dp = np.random.default_rng(5).normal(size=(b, pw))
    ref = cin64(gather64(tabs, idx), filt, bias, sizes, direct, ACT_NONE, dp, block_rows=4)
    t64 = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in tabs]
    x = torch.cat(L.embedding_lookup(t64, torch.tensor(idx)), dim=1)
    f64 = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in filt]
    b64 = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in bias]
    want = cin_ref.cin_pooled_f64(x, sizes, direct, f64, b64, ACT_NONE)
    grads = torch.autograd.grad((want * torch.tensor(dp)).sum(), t64 + f64 + b64)
    pairs = [('pooled', ref['pooled'], want.detach().numpy()),
             ('table grad', scatter64(ref['dx0'], idx, tabs), torch.cat(grads[:f]).numpy())]
    pairs += [(f'filter {k} grad', ref['dw'][k], grads[f + k].numpy()) for k in range(len(sizes))]
    pairs += [(f'bias {k} grad', ref['db'][k], grads[f + len(sizes) + k].numpy()) for k in range(len(sizes))]
    for what, got, exp in pairs:
        np.testing.assert_allclose(got, exp, rtol=0, atol=1e-12 * np.abs(exp).max(), err_msg=what)


# ---------------------------------------------------------------------------------------------
# one shape through forward, backward phase 1, backward phase 2
# ---------------------------------------------------------------------------------------------
def _rel(got, want):
    return float(np.abs(np.asarray(got, dtype=np.float64) - want).max() / np.abs(want).max())


def launches(nat, fn):
    """How many kernels of this library fn() launched (dtb_launch_count)."""
    before = nat.lib.dtb_launch_count()
    fn()
    return nat.lib.dtb_launch_count() - before


def run_case(nat, name, f, d, sizes, direct, use_bias, act, b, bad_ids=False):
    n = len(sizes)
    sizes_c = nat.int_array(sizes)
    fused = nat.lib.dtb_cin_resolved_precision(f, d, sizes_c, n, int(direct), 0) != 1
    tol = TOL_FUSED if fused else TOL
    vocab = [b // 3 + 5 + i for i in range(f)]
    tabs, flat, offs = make_table([v + 2 for v in vocab], d, seed=61)    # the last two rows of every table: no id
    idx = make_idx(vocab, b, seed=62)
    bits = 0
    if bad_ids:                       # one id one past its table, one id of -1; nothing valid names their neighbours
        fa, fb = 1, f - 1
        idx[idx[:, fa + 1] == 0, fa + 1] = 1
        idx[b // 2, fa] = len(tabs[fa])
        idx[b - 1, fb] = -1
        bits = (1 << fa) | (1 << fb)
    filt, bias = make_weights(f, sizes, direct, use_bias, seed=63)
    wcat = np.concatenate([w.reshape(-1) for w in filt])
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=direct))
    dp = np.random.default_rng(64).normal(size=(b, pw)).astype(np.float32)
    d_idx, d_tab, d_offs, d_w, d_dp = dev(idx), dev(flat), dev(offs), dev(wcat), dev(dp)
    d_b = dev(np.concatenate(bias)) if use_bias else None
    ws_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, int(direct), 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    saved = torch.empty(nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, int(direct)), dtype=torch.uint8, device='cuda')
    pooled = torch.full((b, pw), float('nan'), device='cuda')
    status = torch.zeros(1, dtype=torch.int32, device='cuda')
    shape = (b, f, d, sizes_c, n, int(direct), act, 0)

    def fwd(out, sv, w_, nbytes):
        nat.check(nat.lib.dtb_cin_fwd(P(d_idx), P(d_tab), P(d_offs), P(d_w), P(d_b), P(out), P(sv), P(w_), nbytes,
                                      *shape, P(status), None))

    def bwd(phase, gt_, dw_, db_):
        args = (P(d_idx), P(d_tab), P(d_offs), P(d_w), P(d_dp), P(saved), P(gt_), P(dw_), P(db_), P(ws), ws_bytes,
                *shape)
        if phase == 0:
            nat.check(nat.lib.dtb_cin_bwd(*args, None))
        else:
            nat.check(nat.lib.dtb_cin_bwd_phase(*args, phase, None))

    n_fwd = launches(nat, lambda: fwd(pooled, saved, ws, ws_bytes))
    assert int(status.item()) == bits
    got_pooled = pooled.cpu().numpy()

    # the saved activations: x0t [B, D, F], then T_k [B, D, L_k] after bias and activation
    sv = saved.view(torch.float32).cpu().numpy()
    x0 = gather64(tabs, idx)
    assert np.array_equal(sv[:b * d * f].reshape(b, d, f), x0.transpose(0, 2, 1).astype(np.float32)), 'saved x0t'
    t_saved, at = [], b * d * f
    for s in sizes:
        t_saved.append(sv[at:at + b * d * s].reshape(b, d, s))
        at += b * d * s
    masks = [t > 0 for t in t_saved] if act == ACT_RELU else None
    ref = cin64(x0, filt, bias, sizes, direct, act, dp.astype(np.float64), masks)
    err = {'pooled': _rel(got_pooled, ref['pooled'])}
    for k in range(n):
        e = _rel(t_saved[k], ref['T'][k])
        assert e <= tol, f'saved T_{k}: max error {e:.2e} of max |float64|'
        if act == ACT_RELU:
            flip = masks[k] != (ref['pre'][k] > 0)
            worst = float(np.abs(ref['pre'][k][flip]).max()) if flip.any() else 0.0
            assert worst < 1e-5 * np.abs(ref['pre'][k]).max(), \
                f'layer {k}: {int(flip.sum())} relu masks differ from float64, at pre-activations up to {worst:.2e}'

    # backward as CINFn runs it: phase 1 (table gradient), then phase 2 (filter and bias gradients)
    gt = torch.zeros(flat.shape, device='cuda')
    dw = torch.zeros(wcat.shape, device='cuda')
    db = torch.zeros(sum(sizes), device='cuda') if use_bias else None
    n_p1 = launches(nat, lambda: bwd(1, gt, dw, db))
    torch.cuda.synchronize()
    assert float(dw.abs().max()) == 0.0, 'phase 1 wrote filter gradients'
    # the fused dgrad kernel adds the bias gradient in phase 1 already; the any-shape backward leaves it to phase 2
    assert fused or db is None or float(db.abs().max()) == 0.0, 'phase 1 wrote bias gradients'
    n_p2 = launches(nat, lambda: bwd(2, gt, dw, db))
    want_t = scatter64(ref['dx0'], idx, tabs)
    got_t, got_w = gt.cpu().numpy(), dw.cpu().numpy()
    err['table grad'] = _rel(got_t, want_t)
    touched = scatter64(np.ones_like(ref['dx0']), idx, tabs)[:, 0] > 0
    assert (~touched).sum() >= 2 * f
    assert not np.any(got_t[~touched]), 'gradient in table rows no id names'
    w_at = np.cumsum([0] + [w.size for w in filt])
    for k in range(n):
        err[f'filter {k} grad'] = _rel(got_w[w_at[k]:w_at[k + 1]], ref['dw'][k].reshape(-1))
    if use_bias:
        got_b = db.cpu().numpy()
        b_at = np.cumsum([0] + list(sizes))
        for k in range(n):
            err[f'bias {k} grad'] = _rel(got_b[b_at[k]:b_at[k + 1]], ref['db'][k])
    print(f'\n{name} ({"fused" if fused else "any-shape"}, {n_chunks(b, d, kmax(f, sizes, direct))} chunk(s)): '
          + ', '.join(f'{k} {v:.2e}' for k, v in err.items()) + f'  [bound {tol:.0e}]')
    bad = {k: v for k, v in err.items() if not v <= tol}
    assert not bad, f'max error / max |float64| above {tol:.0e}: {bad}'
    if fused:
        return

    # the kernels cin_fp32.cu launches per chunk of batch rows, so that a moved Z budget is a visible failure.  Forward:
    # the gather, then per layer and chunk the outer product Z, the weight pack and the GEMM of dense_tc.cu, the bias /
    # relu epilogue (when there is one), and per layer the pooling.  Phase 1, per chunk: per layer dC, the weight pack,
    # the GEMM dZ = dC W^T and its reduction, then the scatter into the table.  Phase 2, per layer and chunk: the bias
    # column sums (with a bias), Z rebuilt, the weight-gradient GEMM.
    nc = n_chunks(b, d, kmax(f, sizes, direct))
    epilogue = int(use_bias or act == ACT_RELU)
    assert n_fwd == 1 + n * (nc * (3 + epilogue) + 1), f'forward: {n_fwd} launches at {nc} chunk(s)'
    assert n_p1 == nc * (4 * n + 1), f'backward phase 1: {n_p1} launches at {nc} chunk(s)'
    assert n_p2 == nc * n * (2 + int(use_bias)), f'backward phase 2: {n_p2} launches at {nc} chunk(s)'

    # the one-call backward (phase 0) equals phases 1 + 2 up to the order of the fp32 atomics
    gt0 = torch.zeros(flat.shape, device='cuda')
    dw0 = torch.zeros(wcat.shape, device='cuda')
    db0 = torch.zeros(sum(sizes), device='cuda') if use_bias else None
    bwd(0, gt0, dw0, db0)
    for what, a_, b_ in (('table grad', gt0, gt), ('filter grad', dw0, dw), ('bias grad', db0, db)):
        if b_ is not None:
            e = float((a_ - b_).abs().max() / b_.abs().max())
            assert e < 2e-6, f'phase 0 vs phases 1 + 2, {what}: {e:.2e}'

    # inference: no saved buffer, the activations live in a training=0 workspace behind Z; same bits as training
    ws_inf_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, int(direct), 0)
    ws_inf = torch.empty(ws_inf_bytes, dtype=torch.uint8, device='cuda')
    pooled_inf = torch.full((b, pw), float('nan'), device='cuda')
    fwd(pooled_inf, None, ws_inf, ws_inf_bytes)
    assert torch.equal(pooled_inf, pooled), 'inference forward differs from the training forward'


@pytest.mark.parametrize('name,f,d,sizes,direct,use_bias,act,b', [c[:8] for c in OUTSIDE + MULTI_CHUNK],
                         ids=[c[0] for c in OUTSIDE + MULTI_CHUNK])
def test_any_shape_cin_matches_float64(nat, name, f, d, sizes, direct, use_bias, act, b):
    assert nat.lib.dtb_cin_resolved_precision(f, d, nat.int_array(sizes), len(sizes), int(direct), 0) == 1
    run_case(nat, name, f, d, sizes, direct, use_bias, act, b)


# ---------------------------------------------------------------------------------------------
# out-of-range ids on both CIN paths
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('f,d,sizes,use_bias,b,path', [(10, 8, (16, 8), True, 50, 2), (9, 5, (12, 7), True, 33, 1)],
                         ids=['fused', 'any_shape'])
def test_out_of_range_ids(nat, f, d, sizes, use_bias, b, path):
    """One id one past its table and one id of -1: the status bits of exactly those two fields, pooled equal to float64
    with the two embeddings zero, and no gradient from them in any table row (the rows they would name if they were
    taken as offsets are named by no valid id, so they must stay exactly zero)."""
    assert nat.lib.dtb_cin_resolved_precision(f, d, nat.int_array(sizes), len(sizes), 0, 0) == path
    run_case(nat, f'out_of_range_{"fused" if path == 2 else "any_shape"}', f, d, sizes, False, use_bias,
             ACT_RELU, b, bad_ids=True)


# ---------------------------------------------------------------------------------------------
# dispatch and refusals
# ---------------------------------------------------------------------------------------------
def _refused(nat, call, rc_want, message):
    before = nat.lib.dtb_launch_count()
    rc = call()
    torch.cuda.synchronize()
    assert rc == rc_want, f'returned {rc}, expected {rc_want} ({nat.last_error()})'
    assert message in nat.last_error(), nat.last_error()
    assert nat.lib.dtb_launch_count() == before, 'a refused call launched a kernel'


def _buffers(nat, f, d, sizes, direct, b):
    """Device buffers of their full sizes for a CIN call (so that nothing could be read past them)."""
    sizes_c = nat.int_array(sizes)
    n = len(sizes)
    vocab = [5] * f
    _, flat, offs = make_table(vocab, d)
    fns = field_nums(f, sizes, direct)
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=direct))
    nw = sum(f * h * s for h, s in zip(fns, sizes))
    z = lambda *shape: dev(np.zeros(shape, np.float32))
    return dict(idx=dev(make_idx(vocab, b)), tab=dev(flat), offs=dev(offs), w=z(nw), bias=z(sum(sizes)),
                pooled=z(b, pw), dp=z(b, pw), gt=z(*flat.shape), dw=z(nw), db=z(sum(sizes)),
                saved=dev(np.zeros(nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, int(direct)), np.uint8)),
                ws=dev(np.zeros(nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, int(direct), 1), np.uint8)))


@pytest.mark.parametrize('f,d,sizes,direct,inside', [(c[1], c[2], c[3], c[4], c[8]) for c in OUTSIDE + MULTI_CHUNK],
                         ids=[c[0] for c in OUTSIDE + MULTI_CHUNK])
def test_outside_shapes_dispatch_and_refusals(nat, f, d, sizes, direct, inside):
    """Auto runs the any-shape path here and the fused path one step inside; the fused codes 2-4 are refused by the
    forward and the backward; a workspace one byte short is refused.  None of the refusals launches a kernel."""
    b = 4
    sizes_c = nat.int_array(sizes)
    n = len(sizes)
    assert not nat.lib.dtb_cin_tc_supported(f, d, sizes_c, n, int(direct))
    assert nat.lib.dtb_cin_resolved_precision(f, d, sizes_c, n, int(direct), 0) == 1
    fi, di, si, diri = inside
    assert nat.lib.dtb_cin_resolved_precision(fi, di, nat.int_array(si), len(si), int(diri), 0) == 2
    m = _buffers(nat, f, d, sizes, direct, b)
    ws_bytes = m['ws'].numel()
    assert ws_bytes == nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, int(direct), 1)

    def fwd(precision, saved, nbytes):
        return nat.lib.dtb_cin_fwd(P(m['idx']), P(m['tab']), P(m['offs']), P(m['w']), P(m['bias']), P(m['pooled']),
                                   P(saved), P(m['ws']), nbytes, b, f, d, sizes_c, n, int(direct), ACT_RELU, precision,
                                   None, None)

    def bwd(precision, nbytes, phase=0):
        args = (P(m['idx']), P(m['tab']), P(m['offs']), P(m['w']), P(m['dp']), P(m['saved']), P(m['gt']), P(m['dw']),
                P(m['db']), P(m['ws']), nbytes, b, f, d, sizes_c, n, int(direct), ACT_RELU, precision)
        if phase == 0:
            return nat.lib.dtb_cin_bwd(*args, None)
        return nat.lib.dtb_cin_bwd_phase(*args, phase, None)

    for precision in (2, 3, 4):
        assert nat.lib.dtb_cin_resolved_precision(f, d, sizes_c, n, int(direct), precision) == precision
        _refused(nat, lambda: fwd(precision, m['saved'], ws_bytes), ERR_UNSUPPORTED,
                 'dtb_cin_fwd: tensor-core path requested but shape unsupported')
        for phase in (0, 1, 2):
            _refused(nat, lambda: bwd(precision, ws_bytes, phase), ERR_UNSUPPORTED,
                     'dtb_cin_bwd: tensor-core path requested but shape unsupported')
    for precision in (0, 1):
        _refused(nat, lambda: fwd(precision, m['saved'], ws_bytes - 1), ERR_INVALID_ARG,
                 'dtb_cin_fwd: workspace too small')
        for phase in (0, 1, 2):
            _refused(nat, lambda: bwd(precision, ws_bytes - 1, phase), ERR_INVALID_ARG,
                     'dtb_cin_bwd: workspace too small')
        inf_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, int(direct), 0)
        _refused(nat, lambda: fwd(precision, None, inf_bytes - 1), ERR_INVALID_ARG, 'dtb_cin_fwd: workspace too small')


def test_nine_layers_refused(nat):
    f, d, b = 3, 4, 4
    nine, eight = (4,) * 9, (4,) * 8
    c9 = nat.int_array(nine)
    assert nat.lib.dtb_cin_workspace_bytes(b, f, d, c9, 9, 0, 1) == 0
    assert nat.lib.dtb_cin_saved_bytes(b, f, d, c9, 9, 0) == 0
    assert nat.lib.dtb_cin_resolved_precision(f, d, c9, 9, 0, 0) == ERR_INVALID_ARG
    assert not nat.lib.dtb_cin_tc_supported(f, d, c9, 9, 0)
    m = _buffers(nat, f, d, eight, False, b)              # buffers of the 8-layer shape, larger than 9 layers could use
    ws_bytes = m['ws'].numel()
    for precision in (0, 1, 2):
        _refused(nat, lambda: nat.lib.dtb_cin_fwd(P(m['idx']), P(m['tab']), P(m['offs']), P(m['w']), None,
                                                  P(m['pooled']), P(m['saved']), P(m['ws']), ws_bytes, b, f, d, c9, 9,
                                                  0, ACT_RELU, precision, None, None),
                 ERR_INVALID_ARG, 'dtb_cin_fwd: invalid CIN configuration')
        args = (P(m['idx']), P(m['tab']), P(m['offs']), P(m['w']), P(m['dp']), P(m['saved']), P(m['gt']), P(m['dw']),
                None, P(m['ws']), ws_bytes, b, f, d, c9, 9, 0, ACT_RELU, precision)
        _refused(nat, lambda: nat.lib.dtb_cin_bwd(*args, None), ERR_INVALID_ARG, 'dtb_cin_bwd: invalid CIN configuration')
        for phase in (1, 2):
            _refused(nat, lambda: nat.lib.dtb_cin_bwd_phase(*args, phase, None), ERR_INVALID_ARG,
                     'dtb_cin_bwd: invalid CIN configuration')
