"""The kernels that write embedding-table gradients or updates, at the production batch (65 536 rows) with long-tailed ids.

Collisions in the table are handled with fp32 atomics (scatter-add, concat / ragged concat backward, FM + linear
backward, PNN backward) or with an ownership claim (atomicMax on last_step / claim) that lets exactly one reference of a
row update or pack it (the row-wise optimisers, the data-parallel gradient pack).  Uniform ids over small vocabularies
never stress either: here one id can own a whole column, a Zipf column puts thousands of references on its hottest row
and spreads them over thousands of CTAs, and out-of-range ids sit among them.

Exact checks: every operand is a small integer (table values in {-1, 0, 1}, upstream gradients in [-3, 3]), so each
product is exact and fp32 addition is exact in any order while every partial sum stays below 2^24.  Each case computes
that worst case from its own operands (the float64 reference run on |operands|: the sum of the magnitudes of every term
that reaches a table element) and asserts it, and then the kernel must equal the float64 index_add_ reference bit for
bit.  The row-wise optimisers must be bit-identical to the dense sweep fed the same gradient bits.

Bounded checks (AFM and the CIN embedding gradient, whose per-reference arithmetic is not integer-closed): the kernel's
own per-reference gradients from an identity-remapped run, summed in float64, bound each hot row of a capped run.

The kernel each case names is confirmed once per distinct shape by test_case_kernels_are_the_named_ones."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BATCH = 65536
BATCH_RAGGED = 65536 - 37
EXACT = 2 ** 24                       # fp32 adds integers exactly while every partial sum stays below this

# 26 and 39 fields: vocabularies of 10^3 .. 10^5 with vocab-1 fields among them
VOCAB26 = [100000, 1000, 1, 30000, 5000, 1, 2000, 70000, 10000, 1000, 3000, 1, 50000, 1500, 20000, 1000, 8000, 1,
           40000, 2500, 1000, 15000, 6000, 1000, 1, 90000]
VOCAB39 = VOCAB26 + [1000, 1, 4000, 25000, 1000, 12000, 1, 3000, 60000, 1000, 7000, 1, 2000]
VOCAB_OPT = [20000, 1000, 1, 5000, 2000, 1, 1000, 8000, 3000, 1000, 1500, 1, 10000, 1000, 4000, 1000, 2500, 1,
             6000, 1000, 1000, 3000, 2000, 1000, 1, 12000]
# capped_zipf needs V * cap >= B in every field: no vocab-1 fields
VOCAB_CAPPED = [v for v in VOCAB26 if v > 1]
CAP = 512


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


@pytest.fixture(autouse=True)
def _release_device_memory():
    """The cases hold up to several GB each: hand the cached blocks back to the device between them."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


# ---- 1. id distributions ----------------------------------------------------------------------------------------------
def _zipf_col(g, v, b, target, a=1.1):
    """Zipf(a) ranks over v ids; rank 0 (the hottest) is id `target`, the other ranks land on a random permutation."""
    w = np.arange(1, v + 1, dtype=np.float64) ** -a
    cdf = np.cumsum(w)
    ranks = np.minimum(np.searchsorted(cdf / cdf[-1], g.random(b), side='right'), v - 1)
    perm = g.permutation(v)
    k = int(np.nonzero(perm == target)[0][0])
    perm[0], perm[k] = perm[k], perm[0]
    return perm[ranks]


def make_ids(kind, vocab, b, seed):
    """[b, F] int32 ids.  Even fields centre on id 0 and odd fields on id V_f - 1, so the hot rows sit on both edges of
    the row_offsets boundaries.
      one_id        every row of a field uses that one id
      zipf          Zipf(1.1): the hot row takes a large share of the batch, with a long tail of singletons
      capped_zipf   the same, with the references beyond the CAP-th of any row moved to uniform ids
      mixed_invalid zipf with about 1% of -1 and 1% of V_f (out of range: no contribution)
    vocab-1 fields are always id 0 (and the out-of-range ids of mixed_invalid)."""
    g = np.random.default_rng(seed)
    cols = []
    for f, v in enumerate(vocab):
        target = 0 if f % 2 == 0 else v - 1
        if kind == 'one_id' or v == 1:
            col = np.full(b, target, dtype=np.int64)
        else:
            col = _zipf_col(g, v, b, target)
        if kind == 'capped_zipf':
            assert v * CAP >= b
            for _ in range(20):
                order = np.argsort(col, kind='stable')
                s = col[order]
                first = np.searchsorted(s, s, side='left')
                over = order[np.arange(b) - first >= CAP]
                if over.size == 0:
                    break
                col[over] = g.integers(0, v, size=over.size)
            assert np.bincount(col, minlength=v).max() <= CAP
        if kind == 'mixed_invalid':
            u = g.random(b)
            col[u < 0.01] = -1
            col[(u >= 0.01) & (u < 0.02)] = v
        cols.append(col)
    return np.stack(cols, axis=1).astype(np.int32)


def test_id_distributions_reach_the_regime():
    """The generators produce what the kernel tests rely on: a hot row with thousands of references spread over the
    whole batch, a tail of singletons, the cap, and invalid ids in every field."""
    z = make_ids('zipf', VOCAB26, BATCH, seed=1)
    big = [f for f, v in enumerate(VOCAB26) if v >= 50000]
    for f in big:
        counts = np.bincount(z[:, f], minlength=VOCAB26[f])
        assert counts.max() > 0.08 * BATCH and (counts == 1).sum() > 1000, f
        hot = int(counts.argmax())
        assert hot == (0 if f % 2 == 0 else VOCAB26[f] - 1)
        where = np.nonzero(z[:, f] == hot)[0]
        assert where[0] < 256 and where[-1] > BATCH - 256         # spread over the first and the last CTAs
    c = make_ids('capped_zipf', VOCAB_CAPPED, BATCH, seed=1)
    assert max(np.bincount(c[:, f]).max() for f in range(len(VOCAB_CAPPED))) == CAP
    m = make_ids('mixed_invalid', VOCAB26, BATCH, seed=1)
    v = np.array(VOCAB26)
    for f in range(len(VOCAB26)):
        if VOCAB26[f] > 1:
            assert (m[:, f] == -1).any() and (m[:, f] == v[f]).any()
    o = make_ids('one_id', VOCAB26, BATCH, seed=1)
    assert (o[:, 0] == 0).all() and (o[:, 1] == VOCAB26[1] - 1).all()


# ---- float64 references on the device ---------------------------------------------------------------------------------
class Refs:
    """Flat table rows of a batch of ids and the float64 scatter of per-reference gradients."""

    def __init__(self, ids, vocab):
        self.idx = torch.as_tensor(ids).cuda()
        self.b, self.f = ids.shape
        self.vocab = vocab
        offs = np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64)
        self.n_rows = int(offs[-1])
        self.offs = torch.as_tensor(offs).cuda()
        v = torch.as_tensor(np.asarray(vocab, dtype=np.int64)).cuda()
        i64 = self.idx.long()
        self.valid = (i64 >= 0) & (i64 < v)
        self.rows = torch.where(self.valid, self.offs[:-1] + i64.clamp(min=0), torch.zeros_like(i64))

    def emb(self, table):
        """[B, F, D] float64 embeddings, zero for out-of-range ids (what the kernels read for them)."""
        return table.double()[self.rows] * self.valid.unsqueeze(-1)

    def scatter(self, d):
        """float64 sum of the per-reference gradients d [B, F, D] into their table rows: one index_add_."""
        out = torch.zeros(self.n_rows, d.shape[-1], dtype=torch.float64, device='cuda')
        return out.index_add_(0, self.rows[self.valid], d[self.valid])

    def distinct_rows(self):
        return torch.unique(self.rows[self.valid])


def int_tensor(shape, lo, hi, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g, device='cuda').float()


def assert_exact(got, refs, d, d_abs, what):
    """got (fp32, [rows, D]) == the float64 scatter of d, after checking that no partial sum can reach 2^24."""
    bound = float(refs.scatter(d_abs).max())
    assert bound < EXACT, f'{what}: worst-case partial sum {bound:.0f} >= 2^24, the case is not exact'
    want = refs.scatter(d)
    bad = got.double() != want
    assert not bool(bad.any()), (f'{what}: {int(bad.sum())} table elements differ from the exact sum; first at '
                                 f'{bad.nonzero()[0].tolist()}: got {float(got[bad][0])}, want {float(want[bad][0])}')


# ---- 2. exact checks ---------------------------------------------------------------------------------------------------
# concat_bwd_kernel<4> (D % 4 == 0: one 16-byte RED per 4 floats) and concat_bwd_kernel<1> (scalar atomics)
SCATTER_CASES = [  # (dist, vocab, D, B, kernel)
    ('one_id', VOCAB26, 16, BATCH, 'concat_bwd_kernel<4>'),
    ('zipf', VOCAB26, 16, BATCH, 'concat_bwd_kernel<4>'),
    ('mixed_invalid', VOCAB39, 16, BATCH_RAGGED, 'concat_bwd_kernel<4>'),
    ('one_id', VOCAB39, 10, BATCH, 'concat_bwd_kernel<1>'),
    ('zipf', VOCAB26, 10, BATCH_RAGGED, 'concat_bwd_kernel<1>'),
    ('mixed_invalid', VOCAB26, 12, BATCH, 'concat_bwd_kernel<4>'),
]


def _case_id(c):
    return '-'.join(str(len(x)) + 'f' if isinstance(x, list) else str(x) for x in c)


@pytest.mark.parametrize('dist,vocab,d,b,kernel', SCATTER_CASES, ids=[_case_id(c) for c in SCATTER_CASES])
@pytest.mark.parametrize('c', [0, 13])
def test_scatter_and_concat_bwd_exact(nat, dist, vocab, d, b, kernel, c):
    """c = 0: dtb_embedding_scatter_add; c = 13: dtb_concat_emb_dense_bwd (the dense columns are skipped).
    Per reference |d| <= 3: worst case 3 * B < 2^24 on any row."""
    ids = make_ids(dist, vocab, b, seed=11)
    refs = Refs(ids, vocab)
    f = len(vocab)
    dX = int_tensor((b, f * d + c), -3, 3, seed=12)

    def run():
        gt = torch.zeros(refs.n_rows, d, device='cuda')
        if c == 0:
            nat.check(nat.lib.dtb_embedding_scatter_add(P(refs.idx), P(refs.offs), P(dX), P(gt), b, f, d, None))
        else:
            nat.check(nat.lib.dtb_concat_emb_dense_bwd(P(refs.idx), P(refs.offs), P(dX), P(gt), b, f, d, c, None))
        return gt

    gt = run()
    per_ref = dX[:, :f * d].reshape(b, f, d).double()
    assert_exact(gt, refs, per_ref, per_ref.abs(), f'{dist} D={d} C={c}')
    if dist == 'mixed_invalid':
        # the forward reports the out-of-range ids: bit f % 32 for every field that has one, and reads zeros for them
        status = torch.zeros(1, dtype=torch.int32, device='cuda')
        table = int_tensor((refs.n_rows, d), -1, 1, seed=13) + 2.0          # no zero entries
        out = torch.empty(b, f, d, device='cuda')
        nat.check(nat.lib.dtb_embedding_gather(P(refs.idx), P(table), P(refs.offs), P(out), b, f, d, P(status), None))
        want_status = 0
        for ff in torch.nonzero((~refs.valid).any(dim=0)).flatten().tolist():
            want_status |= 1 << (ff % 32)
        assert int(status.item()) == np.int32(np.uint32(want_status))
        assert torch.equal(out == 0, (~refs.valid).unsqueeze(-1).expand(b, f, d))


RAGGED_CASES = [  # (dist, widths cycle, Dmax, B, kernel)
    ('one_id', [4, 8, 16, 12], 16, BATCH, 'ragged_concat_bwd_kernel<4>'),
    ('zipf', [16, 4, 8, 16, 12], 16, BATCH_RAGGED, 'ragged_concat_bwd_kernel<4>'),
    ('mixed_invalid', [3, 16, 7, 10, 1], 16, BATCH, 'ragged_concat_bwd_kernel<1>'),
    ('one_id', [5, 12, 2, 9], 12, BATCH_RAGGED, 'ragged_concat_bwd_kernel<1>'),
]


@pytest.mark.parametrize('dist,widths,dmax,b,kernel', RAGGED_CASES, ids=[_case_id(c) for c in RAGGED_CASES])
def test_ragged_concat_bwd_exact(nat, dist, widths, dmax, b, kernel):
    """Per-column widths: field f adds into columns [0, D_f) of its rows; the padding columns [D_f, Dmax) of every row
    stay exactly zero (the exact reference has zeros there).  |d| <= 3: worst case 3 * B < 2^24."""
    vocab = VOCAB26
    f = len(vocab)
    dims = [widths[i % len(widths)] for i in range(f)]
    ids = make_ids(dist, vocab, b, seed=21)
    refs = Refs(ids, vocab)
    c = 5
    sd = sum(dims)
    dX = int_tensor((b, sd + c), -3, 3, seed=22)
    dims_c = nat.int_array(dims)

    def run():
        gt = torch.zeros(refs.n_rows, dmax, device='cuda')
        nat.check(nat.lib.dtb_ragged_concat_emb_dense_bwd(P(refs.idx), P(refs.offs), dims_c, P(dX), P(gt), b, f, dmax,
                                                          c, None))
        return gt

    gt = run()
    per_ref = torch.zeros(b, f, dmax, dtype=torch.float64, device='cuda')
    col0 = np.concatenate([[0], np.cumsum(dims)])
    for ff in range(f):
        per_ref[:, ff, :dims[ff]] = dX[:, col0[ff]:col0[ff + 1]].double()
    assert_exact(gt, refs, per_ref, per_ref.abs(), f'{dist} ragged')


# fm_linear_bwd_vec: one warp per batch row, lanes over F * D/4 float4 slots (Q = D/4 lanes per field: 1, 4, 8, 16, 32),
# grad_wlin partials in shared memory (s_gw) then one global atomic per CTA; fm_linear_bwd_generic for D % 4 != 0 or
# D = 12 (Q = 3 not a power of two)
FM_CASES = [  # (dist, vocab, D, B, kernel)
    ('one_id', VOCAB26, 4, BATCH, 'fm_linear_bwd_vec'),
    ('zipf', VOCAB26, 16, BATCH, 'fm_linear_bwd_vec'),
    ('mixed_invalid', VOCAB39, 16, BATCH_RAGGED, 'fm_linear_bwd_vec'),
    ('zipf', VOCAB26, 32, BATCH_RAGGED, 'fm_linear_bwd_vec'),
    ('one_id', VOCAB26, 64, BATCH, 'fm_linear_bwd_vec'),
    ('zipf', VOCAB39, 128, BATCH, 'fm_linear_bwd_vec'),
    ('one_id', VOCAB39, 128, BATCH_RAGGED, 'fm_linear_bwd_vec'),
    ('zipf', VOCAB26, 12, BATCH, 'fm_linear_bwd_generic'),
    ('mixed_invalid', VOCAB26, 10, BATCH, 'fm_linear_bwd_generic'),
]


@pytest.mark.parametrize('dist,vocab,d,b,kernel', FM_CASES, ids=[_case_id(c) for c in FM_CASES])
@pytest.mark.parametrize('branches', ['lin_fm', 'fm', 'lin'])
def test_fm_linear_bwd_exact(nat, dist, vocab, d, b, kernel, branches):
    """grad_table and grad_wlin of FM + linear with g_lin / g_fm each present or absent.
    Per reference d = g_fm * (sum_f' e_f' - e_f) + g_lin * w_f.  grad_wlin[f] = sum_b g_lin * sum_d e[b, f, d] takes
    the whole batch on every field: |g_lin| <= 3 while 3 * D * B < 2^24, else |g_lin| <= 1 (D = 128)."""
    f = len(vocab)
    c = 13
    ids = make_ids(dist, vocab, b, seed=31)
    refs = Refs(ids, vocab)
    table = int_tensor((refs.n_rows, d), -1, 1, seed=32)
    dense = int_tensor((b, c), -3, 3, seed=33)
    w_lin = int_tensor((f + c,), -1, 1, seed=34)
    gl_max = 3 if 3 * d * b < EXACT else 1
    g_lin = int_tensor((b,), -gl_max, gl_max, seed=35) if 'lin' in branches else None
    g_fm = int_tensor((b,), -3, 3, seed=36) if 'fm' in branches else None

    def run():
        gt = torch.zeros(refs.n_rows, d, device='cuda')
        gw = torch.zeros(f + c, device='cuda')
        nat.check(nat.lib.dtb_fm_linear_bwd(P(refs.idx), P(table), P(refs.offs), P(dense), P(w_lin), P(g_lin), P(g_fm),
                                            P(gt), P(gw), b, f, d, c, None))
        return gt, gw

    (gt, gw) = run()
    e = refs.emb(table)
    d_ref = torch.zeros_like(e)
    if g_fm is not None:
        d_ref += g_fm.double()[:, None, None] * (e.sum(dim=1, keepdim=True) - e)
    if g_lin is not None:
        d_ref += g_lin.double()[:, None, None] * w_lin.double()[None, :f, None]
    # |g_fm| * (sum_f' |e_f'| + |e_f|) + |g_lin w_f| bounds every term that reaches the element
    d_abs = torch.zeros_like(e)
    if g_fm is not None:
        ea = e.abs()
        d_abs += g_fm.double().abs()[:, None, None] * (ea.sum(dim=1, keepdim=True) + ea)
    if g_lin is not None:
        d_abs += (g_lin.double().abs()[:, None, None] * w_lin.double().abs()[None, :f, None]).expand_as(e)
    assert_exact(gt, refs, d_ref, d_abs, f'{dist} D={d} {branches} grad_table')
    if g_lin is None:
        assert not bool(gw.any()), 'grad_wlin written without g_lin'
        return
    gl64 = g_lin.double()
    want_w = torch.cat([(gl64[:, None] * e.sum(dim=2)).sum(dim=0), (gl64[:, None] * dense.double()).sum(dim=0)])
    bound_w = torch.cat([(gl64.abs()[:, None] * e.abs().sum(dim=2)).sum(dim=0),
                         (gl64.abs()[:, None] * dense.double().abs()).sum(dim=0)])
    assert float(bound_w.max()) < EXACT, f'grad_wlin worst case {float(bound_w.max()):.0f} >= 2^24'
    assert torch.equal(gw.double(), want_w), (f'grad_wlin differs from the exact sum at '
                                              f'{(gw.double() != want_w).nonzero().flatten().tolist()}')


def _pnn_per_ref(e, g_ip, g_op, kern, ktype, row, col, chunk=4096):
    """[B, F, D] float64 gradient of sum(g_ip * ip + g_op * op) with respect to each embedding (OuterProduct /
    InnerProduct, oracle/layers_ref.py), in batch chunks."""
    b, f, d = e.shape
    out = torch.zeros_like(e)
    ri = torch.as_tensor(row, device=e.device)
    ci = torch.as_tensor(col, device=e.device)
    k = kern.double()
    for s in range(0, b, chunk):
        ei, ej = e[s:s + chunk, ri], e[s:s + chunk, ci]               # [n, P, D]
        gi, go = g_ip[s:s + chunk].double().unsqueeze(-1), g_op[s:s + chunk].double().unsqueeze(-1)
        di, dj = gi * ej, gi * ei
        if ktype == 'mat':                                             # op = sum_k (sum_d ei[d] K[k,p,d]) ej[k]
            di = di + go * torch.einsum('npk,kpd->npd', ej, k)
            dj = dj + go * torch.einsum('npd,kpd->npk', ei, k)
        else:                                                          # vec K [P, D], num K [P, 1]
            di = di + go * k.unsqueeze(0) * ej
            dj = dj + go * k.unsqueeze(0) * ei
        o = out[s:s + chunk]
        o.index_add_(1, ri, di)
        o.index_add_(1, ci, dj)
    return out


# pnn_bwd_de_t_kernel<DT>: thread = (row, field), D in {4, 8, 16, 32}, one float4 RED per 4 floats (skipped when all
# four lanes are zero); pnn_bwd_de_kernel (per-row): D outside that set, shared-memory partials then scalar atomics
PNN_CASES = [  # (dist, F, D, B, kernel)
    ('one_id', 26, 16, BATCH, 'pnn_bwd_de_t_kernel<16>'),
    ('zipf', 26, 16, BATCH_RAGGED, 'pnn_bwd_de_t_kernel<16>'),
    ('mixed_invalid', 39, 4, BATCH, 'pnn_bwd_de_t_kernel<4>'),
    ('one_id', 26, 12, BATCH, 'pnn_bwd_de_kernel'),
    ('mixed_invalid', 26, 10, BATCH_RAGGED, 'pnn_bwd_de_kernel'),
]


@pytest.mark.parametrize('dist,f,d,b,kernel', PNN_CASES, ids=[_case_id(c) for c in PNN_CASES])
@pytest.mark.parametrize('ktype', ['mat', 'vec', 'num'])
def test_pnn_bwd_exact(nat, dist, f, d, b, kernel, ktype):
    """Embedding gradient of the PNN inner and outer products; kernels in {-1, 0, 1}.  A reference takes F-1 pairs of
    up to 3 (inner) + 3 (vec / num) or 3 * D (mat) per element: for mat at 65 536 references on one row that passes
    2^24, so the mat cases give the outer product an upstream gradient on one batch row in 8 only (sparse g_op)."""
    vocab = (VOCAB39 if f == 39 else VOCAB26)
    ids = make_ids(dist, vocab, b, seed=41)
    refs = Refs(ids, vocab)
    table = int_tensor((refs.n_rows, d), -1, 1, seed=42)
    pairs = f * (f - 1) // 2
    shape = {'mat': (d, pairs, d), 'vec': (pairs, d), 'num': (pairs, 1)}[ktype]
    kern = int_tensor(shape, -1, 1, seed=43)
    g_ip = int_tensor((b, pairs), -3, 3, seed=44)
    g_op = int_tensor((b, pairs), -3, 3, seed=45)
    if ktype == 'mat':
        g_op[torch.arange(b, device='cuda') % 8 != 0] = 0
    kt = {'mat': 0, 'vec': 1, 'num': 2}[ktype]

    def run():
        gt = torch.zeros(refs.n_rows, d, device='cuda')
        dk = torch.zeros(shape, device='cuda')
        nat.check(nat.lib.dtb_pnn_bwd(P(refs.idx), P(table), P(refs.offs), P(kern), P(g_ip), P(g_op), P(gt), P(dk),
                                      b, f, d, kt, None))
        return gt

    gt = run()
    from oracle.layers_ref import pair_lists
    row, col = pair_lists(f)
    e = refs.emb(table)
    d_ref = _pnn_per_ref(e, g_ip, g_op, kern, ktype, row, col)
    d_abs = _pnn_per_ref(e.abs(), g_ip.abs(), g_op.abs(), kern.abs(), ktype, row, col)
    assert_exact(gt, refs, d_ref, d_abs, f'{dist} F={f} D={d} {ktype}')


# grad_rows_pack_kernel: atomicMax claim per row on `claim`, the winner moves the row into packed and zeroes it, the
# other references write zeros; grad_rows_unpack_kernel: plain read-modify-write of the non-zero packed references
PACK_CASES = [  # (ranks, D, B)
    (1, 16, BATCH), (2, 4, BATCH), (3, 128, BATCH_RAGGED), (4, 16, BATCH), (4, 32, BATCH_RAGGED),
]


@pytest.mark.parametrize('world,d,b', PACK_CASES)
def test_grad_rows_pack_unpack_exact(nat, world, d, b):
    """1-4 ranks simulated in one process, each with its own skewed ids over one shared vocabulary, two steps (the
    claim array carries over).  Integer gradients, |d| <= 3: every sum is exact (3 * B * world < 2^24)."""
    vocab = VOCAB26
    f = len(vocab)
    assert 3 * b * world < EXACT
    claims = None
    for step in (1, 2):
        ranks = []
        for r in range(world):
            dist = 'one_id' if (step == 2 and r == world - 1) else ('mixed_invalid' if r % 2 else 'zipf')
            refs = Refs(make_ids(dist, vocab, b, seed=100 * step + r), vocab)
            gout = int_tensor((b, f, d), -3, 3, seed=1000 * step + r)
            grad = torch.zeros(refs.n_rows, d, device='cuda')
            nat.check(nat.lib.dtb_embedding_scatter_add(P(refs.idx), P(refs.offs), P(gout), P(grad), b, f, d, None))
            ranks.append((refs, gout, grad))
        if claims is None:
            claims = [torch.zeros(ranks[0][0].n_rows, dtype=torch.int32, device='cuda') for _ in range(world)]
        packed = []
        for r, (refs, gout, grad) in enumerate(ranks):
            want_r = refs.scatter(gout.double())
            assert torch.equal(grad.double(), want_r)                         # the scatter itself (exact)
            pk = torch.full((b, f, d), float('nan'), device='cuda')
            nat.check(nat.lib.dtb_grad_rows_pack(P(refs.idx), P(refs.offs), P(grad), P(claims[r]), P(pk), step, b, f,
                                                 d, None))
            assert not bool(grad.any()), f'rank {r}: {int((grad != 0).any(dim=1).sum())} claimed rows not zeroed'
            assert not bool(pk.isnan().any()), f'rank {r}: packed references left unwritten'
            # exactly one reference per distinct valid row carries the row (none for a row whose sum is zero)
            carries = (pk != 0).any(dim=-1) & refs.valid
            per_row = torch.bincount(refs.rows[carries], minlength=refs.n_rows)
            want_rows = (want_r != 0).any(dim=1)
            assert int(per_row.max()) <= 1, f'rank {r}: a row is carried by {int(per_row.max())} references'
            assert torch.equal(per_row.bool(), want_rows), f'rank {r}: carried rows differ from the non-zero rows'
            assert not bool((pk != 0).any(dim=-1)[~refs.valid].any()), f'rank {r}: an invalid reference carries data'
            assert torch.equal(claims[r][refs.distinct_rows()], torch.full_like(refs.distinct_rows(), step,
                                                                                dtype=torch.int32))
            packed.append(pk)
        want = sum(refs.scatter(gout.double()) for refs, gout, _ in ranks)
        outs = []
        for _ in range(2):
            acc = torch.zeros(ranks[0][0].n_rows, d, device='cuda')
            for (refs, _, _), pk in zip(ranks, packed):
                nat.check(nat.lib.dtb_grad_rows_unpack(P(refs.idx), P(refs.offs), P(pk), P(acc), b, f, d, None))
            outs.append(acc)
        assert torch.equal(outs[0], outs[1]), 'unpacking ranks 0..W-1 in order twice gave different bits'
        bad = outs[0].double() != want
        assert not bool(bad.any()), f'step {step}: {int(bad.sum())} elements of the unpacked sum differ from the exact sum'


# ---- 4. row-wise optimisers under contention ----------------------------------------------------------------------------
# six steps of fresh ids; step 4 puts one id on the whole batch in every field: every CTA races for the same claims
OPT_STEPS = ['zipf', 'zipf', 'mixed_invalid', 'one_id', 'zipf', 'zipf']


def _opt_step_ids(step, b):
    return Refs(make_ids(OPT_STEPS[step - 1], VOCAB_OPT, b, seed=500 + step), VOCAB_OPT)


def _scattered_grad(nat, refs, d, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    gout = torch.randn(refs.b, refs.f, d, generator=g, device='cuda')
    gd = torch.zeros(refs.n_rows, d, device='cuda')
    nat.check(nat.lib.dtb_embedding_scatter_add(P(refs.idx), P(refs.offs), P(gout), P(gd), refs.b, refs.f, d, None))
    return gd


def _assert_touched_current(refs, step, lasts, what):
    rows = refs.distinct_rows()
    for name, last in lasts:
        got = last[rows]
        assert bool((got == step).all()), (f'{what} {name}: {int((got != step).sum())} of {rows.numel()} rows read '
                                           f'at step {step} have last_step != {step}')


def _assert_same(a, b_, what):
    bad = a != b_
    assert not bool(bad.any()), (f'{what}: {int(bad.sum())} of {bad.numel()} entries differ, max |diff| '
                                 f'{float((a - b_).abs().max()):.3e}, first at {bad.nonzero()[0].tolist()}')


@pytest.mark.parametrize('d,b', [(4, BATCH), (16, BATCH), (128, BATCH), (16, BATCH_RAGGED)])
def test_adam_rows_hot_ids_bit_identical_to_dense(nat, d, b):
    """adam_rows_kernel<0> (catch-up) / <1> (apply) with host and device step counters, and the flush, against
    dtb_adam_dense on the same gradient bits (scattered once, then copied).  D = 4, 16, 128: Q = 1, 4, 32 lanes per
    row."""
    from deeptables_b200.engine import adam_alpha
    steps = len(OPT_STEPS)
    n_rows = sum(VOCAB_OPT)
    g = torch.Generator(device='cuda').manual_seed(d)
    w0 = (torch.rand(n_rows, d, generator=g, device='cuda') - 0.5) * 0.1
    alpha = torch.tensor([0.0] + [adam_alpha(s) for s in range(1, steps + 2)], dtype=torch.float32, device='cuda')
    b1, b2, eps = 0.9, 0.999, 1e-7

    def state():
        return w0.clone(), torch.zeros(n_rows, d, device='cuda'), torch.zeros(n_rows, d, device='cuda')

    (wd, md, vd), (wh, mh, vh), (wv, mv, vv) = state(), state(), state()
    last_h = torch.zeros(n_rows, dtype=torch.int32, device='cuda')
    last_v = torch.zeros(n_rows, dtype=torch.int32, device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    for step in range(1, steps + 1):
        refs = _opt_step_ids(step, b)
        ix, of = P(refs.idx), P(refs.offs)
        gd = _scattered_grad(nat, refs, d, seed=700 + step)
        gh, gv = gd.clone(), gd.clone()
        nat.check(nat.lib.dtb_adam_rows_catchup(ix, of, P(wh), P(mh), P(vh), P(last_h), P(alpha), step - 1, b1, b2, eps,
                                                b, refs.f, d, None))
        step_dev.fill_(step - 1)
        nat.check(nat.lib.dtb_adam_rows_catchup_dev(ix, of, P(wv), P(mv), P(vv), P(last_v), P(alpha), P(step_dev), b1, b2,
                                                    eps, b, refs.f, d, None))
        rows = refs.distinct_rows()
        for label, w in (('host', wh), ('dev', wv)):
            _assert_same(w[rows], wd[rows], f'step {step} {label}: rows read by the step after the catch-up')
        nat.check(nat.lib.dtb_adam_dense(P(wd), P(md), P(vd), P(gd), n_rows * d, float(alpha[step].item()), b1, b2, eps,
                                         1, None))
        nat.check(nat.lib.dtb_adam_rows_apply(ix, of, P(wh), P(mh), P(vh), P(gh), P(last_h), P(alpha), step, b1, b2, eps,
                                              b, refs.f, d, None))
        nat.check(nat.lib.dtb_adam_rows_apply_dev(ix, of, P(wv), P(mv), P(vv), P(gv), P(last_v), P(alpha), P(step_dev),
                                                  b1, b2, eps, b, refs.f, d, None))
        assert not bool(gh.any()) and not bool(gv.any()), f'step {step}: gradient rows left after the apply'
        _assert_touched_current(refs, step, (('host', last_h), ('dev', last_v)), f'step {step}')
        for label, w, m, v in (('host', wh, mh, vh), ('dev', wv, mv, vv)):
            for name, a_, b_ in (('weights', w, wd), ('m', m, md), ('v', v, vd)):
                _assert_same(a_[rows], b_[rows], f'step {step} {label} {name}: rows the step applied')
    for w, m, v, last in ((wh, mh, vh, last_h), (wv, mv, vv, last_v)):
        nat.check(nat.lib.dtb_adam_rows_flush(P(w), P(m), P(v), P(last), P(alpha), steps, b1, b2, eps, n_rows, d, None))
    torch.cuda.synchronize()
    for label, w, m, v in (('host', wh, mh, vh), ('dev', wv, mv, vv)):
        for name, a_, b_ in (('weights', w, wd), ('m', m, md), ('v', v, vd)):
            _assert_same(a_, b_, f'after the flush, {label} {name}')
    assert int(last_h.min().item()) == steps and int(last_v.min().item()) == steps


def _optim_variants():
    from deeptables_b200 import optimizers as O
    return {
        'sgd': O.SGD(learning_rate=0.05),
        'sgd_momentum': O.SGD(learning_rate=0.05, momentum=0.9),
        'sgd_nesterov': O.SGD(learning_rate=0.05, momentum=0.9, nesterov=True),
        'rmsprop': O.RMSprop(learning_rate=0.01),
        'rmsprop_centered_momentum': O.RMSprop(learning_rate=0.01, momentum=0.9, centered=True),
        'adagrad': O.Adagrad(learning_rate=0.1),
    }


@pytest.mark.parametrize('d', [4, 16, 128])
@pytest.mark.parametrize('name', ['sgd', 'sgd_momentum', 'sgd_nesterov', 'rmsprop', 'rmsprop_centered_momentum',
                                  'adagrad'])
def test_optim_rows_hot_ids_bit_identical_to_dense(nat, name, d):
    """optim_rows_kernel<0> / <1> and the flush for SGD (plain, momentum, Nesterov), RMSprop (plain, centered with
    momentum) and Adagrad, host and device step counters, against dtb_optim_dense on the same gradient bits."""
    from deeptables_b200 import optimizers as O
    from deeptables_b200.deepmodel import _native_optim_params
    spec = O.resolve(_optim_variants()[name])
    hp = _native_optim_params(spec)
    inits = O.slot_inits(spec)
    steps = len(OPT_STEPS)
    b = BATCH
    n_rows = sum(VOCAB_OPT)
    g = torch.Generator(device='cuda').manual_seed(d + 1)
    w0 = (torch.rand(n_rows, d, generator=g, device='cuda') - 0.5) * 0.1

    def state():
        return w0.clone(), [None if s is None else torch.full((n_rows, d), s, device='cuda') for s in inits]

    (wd, sd), (wh, sh), (wv, sv) = state(), state(), state()
    last_h = torch.zeros(n_rows, dtype=torch.int32, device='cuda')
    last_v = torch.zeros(n_rows, dtype=torch.int32, device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    for step in range(1, steps + 1):
        refs = _opt_step_ids(step, b)
        ix, of = P(refs.idx), P(refs.offs)
        gd = _scattered_grad(nat, refs, d, seed=900 + step)
        gh, gv = gd.clone(), gd.clone()
        nat.check(nat.lib.dtb_optim_rows_catchup(ix, of, P(wh), *map(P, sh), P(last_h), step - 1, hp, b, refs.f, d, None))
        step_dev.fill_(step - 1)
        nat.check(nat.lib.dtb_optim_rows_catchup_dev(ix, of, P(wv), *map(P, sv), P(last_v), P(step_dev), hp, b, refs.f, d,
                                                     None))
        nat.check(nat.lib.dtb_optim_dense(P(wd), P(gd), *map(P, sd), n_rows * d, hp, 1, None))
        nat.check(nat.lib.dtb_optim_rows_apply(ix, of, P(wh), *map(P, sh), P(gh), P(last_h), step, hp, b, refs.f, d,
                                               None))
        nat.check(nat.lib.dtb_optim_rows_apply_dev(ix, of, P(wv), *map(P, sv), P(gv), P(last_v), P(step_dev), hp, b,
                                                   refs.f, d, None))
        assert not bool(gh.any()) and not bool(gv.any()), f'step {step}: gradient rows left after the apply'
        _assert_touched_current(refs, step, (('host', last_h), ('dev', last_v)), f'step {step}')
        rows = refs.distinct_rows()
        for label, w, sl in (('host', wh, sh), ('dev', wv, sv)):
            _assert_same(w[rows], wd[rows], f'step {step} {label} weights: rows the step applied')
            for k, (a_, b_) in enumerate(zip(sl, sd)):
                if a_ is not None:
                    _assert_same(a_[rows], b_[rows], f'step {step} {label} slot {k}: rows the step applied')
    nat.check(nat.lib.dtb_optim_rows_flush(P(wh), *map(P, sh), P(last_h), steps, hp, n_rows, d, None))
    step_dev.fill_(steps)
    nat.check(nat.lib.dtb_optim_rows_flush_dev(P(wv), *map(P, sv), P(last_v), P(step_dev), hp, n_rows, d, None))
    torch.cuda.synchronize()
    assert not torch.equal(wd, w0)
    for label, w, sl in (('host', wh, sh), ('dev', wv, sv)):
        _assert_same(w, wd, f'after the flush, {label} weights')
        for k, (a_, b_) in enumerate(zip(sl, sd)):
            if a_ is not None:
                _assert_same(a_, b_, f'after the flush, {label} slot {k}')


# ---- 3. bounded checks: AFM and CIN, whose per-reference gradients are not integer-closed ----------------------------
def _identity_remap(refs, table):
    """Ids, row offsets and table of the identity-remapped batch: field f owns rows [f * B, (f + 1) * B) and reference
    (b, f) reads row f * B + b, a copy of the row the skewed batch reads."""
    b, f = refs.b, refs.f
    idx_id = torch.arange(b, dtype=torch.int32, device='cuda').unsqueeze(1).expand(b, f).contiguous()
    offs_id = torch.arange(f + 1, dtype=torch.int64, device='cuda') * b
    return idx_id, offs_id, table[refs.rows.t().reshape(-1)].contiguous()


def assert_bounded(refs, run, table, what):
    """run(idx, offs, table) -> the op's fp32 table gradient.  Two identity-remapped runs give the kernel's own
    per-reference gradients d_{b,f} (one reference per row: no sum) and their run-to-run spread; on the skewed ids
    every table row must equal the float64 sum of its d_{b,f} within tol = n_row * 2^-24 * sum |d| + the summed
    spread.  A lost or doubled reference moves its row by d_{b,f}, and rounding of up to tol can hide up to tol of
    that: on every row with at least 64 references, the largest element of every d_{b,f} must exceed 2 * tol there."""
    b, f = refs.b, refs.f
    idx_id, offs_id, tab_id = _identity_remap(refs, table)
    d1 = run(idx_id, offs_id, tab_id).view(f, b, -1).transpose(0, 1).double()
    d2 = run(idx_id, offs_id, tab_id).view(f, b, -1).transpose(0, 1).double()
    got = run(refs.idx, refs.offs, table)
    n_row = torch.bincount(refs.rows[refs.valid], minlength=refs.n_rows).double()
    assert int(n_row.max()) == CAP, f'{what}: no row reaches the cap, the case does not test the hot-row regime'
    want = refs.scatter(d1)
    tol = n_row[:, None] * 2.0 ** -24 * refs.scatter(d1.abs()) + refs.scatter((d1 - d2).abs())
    err = (got.double() - want).abs()
    bad = err > tol
    assert not bool(bad.any()), (f'{what}: {int(bad.any(dim=1).sum())} table rows off their float64 sum by more than '
                                 f'the bound; worst err / bound {float((err / tol.clamp(min=1e-30)).max()):.3g}')
    sel = refs.valid & (n_row[refs.rows] >= 64)
    margin = (d1.abs() - 2 * tol[refs.rows]).amax(dim=-1)[sel]
    assert int(sel.sum()) > 0
    assert bool((margin > 0).all()), (f'{what}: {int((margin <= 0).sum())} of {int(sel.sum())} references of hot rows '
                                      f'are within twice the bound: a lost contribution could pass')


def _capped_vocab(f):
    return [v if v > 1 else 1000 for v in VOCAB26] if f == 26 else [1000 + 37 * i for i in range(f)]


# afm_rows_kernel<.., 2> (the backward's row pass) at 4 warps per CTA (26 fields) and at 2 (99 fields: shared memory),
# then afm_bwd_gather_kernel<16>: thread = (row, field), one float4 RED per 4 floats, skipped when all four are zero.
# 99 fields at 4 096 rows: the workspace holds [B, P, H + D] floats, 4 096 * 4 851 * 32 * 4 B = 2.5 GB there.
AFM_CASES = [(26, 16, 16, BATCH, 4), (99, 16, 16, 4096, 2)]


@pytest.mark.parametrize('f,d,h,b,warps', AFM_CASES)
def test_afm_bwd_hot_rows_bounded(nat, f, d, h, b, warps):
    """dtb_afm_bwd's table gradient on capped_zipf ids, bounded as assert_bounded says."""
    vocab = _capped_vocab(f)
    refs = Refs(make_ids('capped_zipf', vocab, b, seed=61), vocab)
    g = torch.Generator(device='cuda').manual_seed(62)
    table = torch.rand(refs.n_rows, d, generator=g, device='cuda') * 2 - 1
    wa = torch.randn(d, h, generator=g, device='cuda') * (3 / d ** 0.5)
    ba = torch.randn(h, generator=g, device='cuda') * 0.1
    ph = torch.randn(h, 1, generator=g, device='cuda')
    gp = torch.randn(b, d, generator=g, device='cuda')
    nb = nat.lib.dtb_afm_workspace_bytes(b, f, d, h)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')

    def bwd(idx, offs, tab):
        gt = torch.zeros(tab.shape, device='cuda')
        dwa, dba, dph = torch.zeros(d, h, device='cuda'), torch.zeros(h, device='cuda'), torch.zeros(h, 1, device='cuda')
        nat.check(nat.lib.dtb_afm_bwd(P(idx), P(tab), P(offs), P(wa), P(ba), P(ph), P(gp), P(gt), P(dwa), P(dba), P(dph),
                                      P(ws), nb, b, f, d, h, 1, None))
        return gt

    assert_bounded(refs, bwd, table, f'AFM F={f}')


# dtb_cin_bwd_phase phase 1 (the embedding gradient).  Precision 1: the any-shape fp32 formulation, whose
# cin_scatter_t_kernel adds every (row, field, d) into the table with a scalar atomic; precision 2: the fused wgmma data
# gradient cin_wg_dgrad_kernel.  The headline shape takes both; D = 10 lies outside the fused kernels (any shape only).
CIN_CASES = [  # (F, D, layer sizes, precision, kernel)
    (26, 16, (128, 128, 128), 1, 'cin_scatter_t_kernel'),
    (26, 16, (128, 128, 128), 2, 'cin_wg_dgrad_kernel'),
    (26, 10, (64, 32), 1, 'cin_scatter_t_kernel'),
]


def _cin_setup(nat, f, d, sizes, b, seed):
    from oracle import layers_ref as L
    sizes_c = nat.int_array(sizes)
    n = len(sizes)
    g = torch.Generator(device='cuda').manual_seed(seed)
    fns = L.cin_field_nums(f, sizes, False)
    w = torch.cat([(torch.randn(f * fns[k] * s, generator=g, device='cuda') / (f * fns[k]) ** 0.5)
                   for k, s in enumerate(sizes)])
    pw = L.cin_pooled_width(f, dict(cross_layer_size=sizes, direct=False))
    dp = torch.randn(b, pw, generator=g, device='cuda')
    ws_bytes = nat.lib.dtb_cin_workspace_bytes(b, f, d, sizes_c, n, 0, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    saved = torch.empty(nat.lib.dtb_cin_saved_bytes(b, f, d, sizes_c, n, 0), dtype=torch.uint8, device='cuda')
    pooled = torch.empty(b, pw, device='cuda')
    dw = torch.zeros_like(w)

    def bwd(idx, offs, tab, precision):
        """forward (saving the activations), then phase 1 of the backward; returns the table gradient"""
        nat.check(nat.lib.dtb_cin_fwd(P(idx), P(tab), P(offs), P(w), None, P(pooled), P(saved), P(ws), ws_bytes, b, f,
                                      d, sizes_c, n, 0, 1, precision, None, None))
        gt = torch.zeros(tab.shape, device='cuda')
        nat.check(nat.lib.dtb_cin_bwd_phase(P(idx), P(tab), P(offs), P(w), P(dp), P(saved), P(gt), P(dw), None, P(ws),
                                            ws_bytes, b, f, d, sizes_c, n, 0, 1, precision, 1, None))
        return gt

    return bwd


@pytest.mark.parametrize('f,d,sizes,precision,kernel', CIN_CASES, ids=[_case_id(c) for c in CIN_CASES])
def test_cin_bwd_phase1_hot_rows_bounded(nat, f, d, sizes, precision, kernel):
    """The CIN embedding gradient on capped_zipf ids at the production batch, bounded as assert_bounded says."""
    sizes_c = nat.int_array(sizes)
    assert bool(nat.lib.dtb_cin_tc_supported(f, d, sizes_c, len(sizes), 0)) == (d == 16)
    assert nat.lib.dtb_cin_resolved_precision(f, d, sizes_c, len(sizes), 0, precision) == precision
    vocab = _capped_vocab(f)
    refs = Refs(make_ids('capped_zipf', vocab, BATCH, seed=71), vocab)
    g = torch.Generator(device='cuda').manual_seed(72)
    table = torch.rand(refs.n_rows, d, generator=g, device='cuda') - 0.5
    bwd = _cin_setup(nat, f, d, sizes, BATCH, seed=73)
    assert_bounded(refs, lambda idx, offs, tab: bwd(idx, offs, tab, precision), table, f'CIN {sizes} precision {precision}')


# ---- the kernel each case names ----------------------------------------------------------------------------------------
# The hot-id cases run unprofiled.  The kernel a shape selects depends on F, D, the layer sizes, the precision code and
# the alignment of the buffers, not on the batch or the ids, so each distinct (op, shape, kernel) of the tables above is
# profiled once here on a 256-row batch of uniform ids, with every buffer allocated before the profiled call.
PROFILE_B = 256


def _profiled_calls(nat):
    calls = []
    small = lambda f: [50] * f                                                       # noqa: E731

    def ids_offs(f):
        vocab = small(f)
        ids = torch.as_tensor(make_ids('zipf', vocab, PROFILE_B, seed=3)).cuda()
        return ids, torch.as_tensor(np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64)).cuda(), sum(vocab)

    for (_, vocab, d, _, kernel) in {(len(c[1]), c[2]): c for c in SCATTER_CASES}.values():
        f = len(vocab)
        ids, offs, rows = ids_offs(f)
        dX, gt = torch.ones(PROFILE_B, f * d, device='cuda'), torch.zeros(rows, d, device='cuda')
        calls.append((f'scatter-{f}f-{d}', kernel, lambda ids=ids, offs=offs, dX=dX, gt=gt, f=f, d=d: nat.check(
            nat.lib.dtb_embedding_scatter_add(P(ids), P(offs), P(dX), P(gt), PROFILE_B, f, d, None))))
    for (_, widths, dmax, _, kernel) in RAGGED_CASES:
        f = 26
        dims = [widths[i % len(widths)] for i in range(f)]
        ids, offs, rows = ids_offs(f)
        dX, gt = torch.ones(PROFILE_B, sum(dims) + 5, device='cuda'), torch.zeros(rows, dmax, device='cuda')
        dims_c = nat.int_array(dims)
        calls.append((f'ragged-{widths}', kernel, lambda ids=ids, offs=offs, dX=dX, gt=gt, dims_c=dims_c, dmax=dmax: nat.check(
            nat.lib.dtb_ragged_concat_emb_dense_bwd(P(ids), P(offs), dims_c, P(dX), P(gt), PROFILE_B, 26, dmax, 5, None))))
    for (_, vocab, d, _, kernel) in {(len(c[1]), c[2]): c for c in FM_CASES}.values():
        f, c = len(vocab), 13
        ids, offs, rows = ids_offs(f)
        tab, gt = torch.ones(rows, d, device='cuda'), torch.zeros(rows, d, device='cuda')
        dense, wl = torch.ones(PROFILE_B, c, device='cuda'), torch.ones(f + c, device='cuda')
        gl, gf, gw = torch.ones(PROFILE_B, device='cuda'), torch.ones(PROFILE_B, device='cuda'), torch.zeros(f + c, device='cuda')
        calls.append((f'fm-{f}f-{d}', kernel, lambda ids=ids, offs=offs, tab=tab, gt=gt, dense=dense, wl=wl, gl=gl, gf=gf,
                      gw=gw, f=f, d=d, c=c: nat.check(nat.lib.dtb_fm_linear_bwd(
                          P(ids), P(tab), P(offs), P(dense), P(wl), P(gl), P(gf), P(gt), P(gw), PROFILE_B, f, d, c, None))))
    for (_, f, d, _, kernel) in {(c[1], c[2]): c for c in PNN_CASES}.values():
        ids, offs, rows = ids_offs(f)
        pairs = f * (f - 1) // 2
        for ktype, kt, shape in (('mat', 0, (d, pairs, d)), ('vec', 1, (pairs, d)), ('num', 2, (pairs, 1))):
            tab, gt = torch.ones(rows, d, device='cuda'), torch.zeros(rows, d, device='cuda')
            kern, dk = torch.ones(shape, device='cuda'), torch.zeros(shape, device='cuda')
            gi, go = torch.ones(PROFILE_B, pairs, device='cuda'), torch.ones(PROFILE_B, pairs, device='cuda')
            calls.append((f'pnn-{f}f-{d}-{ktype}', kernel, lambda ids=ids, offs=offs, tab=tab, gt=gt, kern=kern, dk=dk,
                          gi=gi, go=go, f=f, d=d, kt=kt: nat.check(nat.lib.dtb_pnn_bwd(
                              P(ids), P(tab), P(offs), P(kern), P(gi), P(go), P(gt), P(dk), PROFILE_B, f, d, kt, None))))
    for (f, d, h, _, warps) in AFM_CASES:
        ids, offs, rows = ids_offs(f)
        tab, gt = torch.ones(rows, d, device='cuda'), torch.zeros(rows, d, device='cuda')
        wa, ba, ph = torch.ones(d, h, device='cuda'), torch.zeros(h, device='cuda'), torch.ones(h, 1, device='cuda')
        gp, dwa, dba, dph = (torch.ones(PROFILE_B, d, device='cuda'), torch.zeros(d, h, device='cuda'),
                             torch.zeros(h, device='cuda'), torch.zeros(h, 1, device='cuda'))
        nb = nat.lib.dtb_afm_workspace_bytes(PROFILE_B, f, d, h)
        ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
        calls.append((f'afm-{f}f', (f'afm_bwd_gather_kernel<{d}>', ('afm_rows_kernel<', (32 * warps, 1, 1))),
                      lambda ids=ids, offs=offs, tab=tab, gt=gt, wa=wa, ba=ba, ph=ph, gp=gp, dwa=dwa, dba=dba, dph=dph,
                      ws=ws, nb=nb, f=f, d=d, h=h: nat.check(nat.lib.dtb_afm_bwd(
                          P(ids), P(tab), P(offs), P(wa), P(ba), P(ph), P(gp), P(gt), P(dwa), P(dba), P(dph), P(ws), nb,
                          PROFILE_B, f, d, h, 1, None))))
    for (f, d, sizes, precision, kernel) in CIN_CASES:
        ids, offs, rows = ids_offs(f)
        tab = torch.full((rows, d), 0.1, device='cuda')
        bwd = _cin_setup(nat, f, d, sizes, PROFILE_B, seed=5)
        calls.append((f'cin-{d}-{sizes}-{precision}', kernel,
                      lambda bwd=bwd, ids=ids, offs=offs, tab=tab, precision=precision: bwd(ids, offs, tab, precision)))
    return calls


def test_case_kernels_are_the_named_ones(nat):
    """One profiled call per distinct shape of the cases above: the kernel each case names is the one that runs."""
    from kernel_profile import launches, ran
    wrong = []
    for name, want, call in _profiled_calls(nat):
        kernels, _ = launches(call)
        if isinstance(want, tuple):                          # AFM: the gather kernel and the row pass's warps per CTA
            gather, (prefix, block) = want
            rows_blocks = [tuple(blk) for k, _, blk in kernels if k.startswith(prefix)]
            ok = ran(kernels, gather) and rows_blocks and all(blk == block for blk in rows_blocks)
        else:
            ok = ran(kernels, want)
        if not ok:
            wrong.append(f'{name}: expected {want}, launched {[k for k, _, _ in kernels]}')
    assert not wrong, '\n'.join(wrong)
