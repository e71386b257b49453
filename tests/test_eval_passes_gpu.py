"""The loss, streaming-metric, permutation-importance, SHAP and boosting kernels past their first pass over the rows.

These kernels run grid-stride loops over a capped grid, and several carry batch-wide state from one pass to the next:
the hinge losses' "not binary" flag, the per-block shared-memory counters and R2 sums of the streaming metrics (global
64-bit atomics past 8 192 counters), the tie range the AUC count caches per thread, the atomic max of |g| and h that
sets the boosting gradients' fixed-point shift, and the tree stages gbdt_leaves_kernel walks outside its row loop.
Their own tests run inside one pass; production runs them over whole prediction arrays, held-out sets, coalition
frames and training frames.  This file runs them at a million rows and more, in the manner of
tests/test_batch_passes_gpu.py:
  - the premise: the named kernels ran, and each loop covers its work in at least 3 passes of the grid it was
    launched with, the last one ragged;
  - exactness where the arithmetic is exact: counters, gathers, permutations, leaf ids and fixed-point values equal the
    numpy reference bit for bit, and per-row float outputs that do not depend on the row count equal uneven
    single-pass slices bit for bit;
  - float64 reductions against a float64 reference, with a bar that rejects the reference with one 32-row warp left
    out.  The importance sums and the SHAP means add in a fixed order, restated here in numpy (checked against
    math.fsum in tests/test_eval_passes_cpu.py): those must be the same bits.
The pass counts assume an H100 SXM (132 SMs); a card with fewer SMs runs more passes.

The launches come from torch.profiler in a child process, for the reason tests/test_batch_passes_gpu.py gives.
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

import gbm_ref as R
import importance_ref as IR
import loss_ref
import metrics_state_ref as SR
from deeptables_b200 import losses as LS
from kernel_profile import launches
from test_batch_passes_gpu import Loop, cdiv, passes_of, stride, uneven_slices
from test_losses_gpu import CODE, TASKS, _labels
from test_metrics_gpu import _binary_data, _binary_entries, _plan

pytestmark = pytest.mark.gpu

ROWS = 1_000_003
HINGE_ROWS = 2_000_003     # the hinge losses' label check: 3+ passes over one label column
WARP = 32
THREADS = 256          # the block of every kernel here


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


@pytest.fixture(autouse=True)
def _release():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def P(t, offset_bytes=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + offset_bytes)


def sm_count(nat):
    n = ctypes.c_int(0)
    nat.check(nat.lib.dtb_device_sm_count(ctypes.byref(n)))
    return n.value


def dev(a):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def rows_loop(kernel, rows, per_sm_cap, sm, unit='row'):
    """a grid-stride loop over `rows`, one per thread, launched on min(ceil(rows / 256), sm * per_sm_cap) CTAs"""
    want = min(cdiv(rows, THREADS), sm * per_sm_cap)

    def per(b):
        assert b[0] == THREADS, f'{kernel}: block {b}'
        return b[0]
    lp = stride(kernel, rows, per, unit)
    work = lp.work
    lp.work = lambda g, b: (work(g, b) if g[0] == want else pytest.fail(f'{kernel}: grid {g}, expected {want} CTAs'))
    return lp


def left_out(rows):
    """the rows of one warp in the middle of the batch"""
    lo = rows // WARP // 2 * WARP
    return lo, lo + WARP


def check_bar(what, got, want, scale, drop, rtol):
    """float64 `got` against `want` within rtol x scale, and the bar rejects `want - drop` (one warp left out).
    Returns (worst error / bar, bars the left-out warp moves the reference)."""
    bar = rtol * np.asarray(scale, np.float64) + 1e-300
    err = float(np.max(np.abs(np.asarray(got, np.float64) - want) / bar))
    sees = float(np.min(np.abs(np.asarray(drop, np.float64)) / bar))
    assert err <= 1, f'{what}: off by {err:.3g} of its bar ({rtol:g} relative)'
    assert sees > 1, f'{what}: the bar does not see one warp left out ({sees:.3g} of the bar)'
    return round(err, 4), round(sees, 1)


# ---------------------------------------------------------------------------------------------
# losses: dtb_loss_fwd_bwd ('auto'), dtb_focal_loss_fwd_bwd and dtb_keras_loss_fwd_bwd (every Keras class)
# ---------------------------------------------------------------------------------------------
AUTO = {'binary': 'BinaryCrossentropy', 'multilabel': 'BinaryCrossentropy', 'regression': 'MeanSquaredError',
        'multiclass': 'CategoricalCrossentropy'}
FOCAL_GAMMA, FOCAL_ALPHA = 2.0, 0.25
# The loss sum adds float32 per-row losses in float64.  Against float64 per-row losses the float32 evaluation leaves a
# systematic gap: the rows where the probability saturates and clips all carry the same float32 value, log(2^-23) or
# similar, with the same rounding error.  A float32 restatement on the CPU at these shapes and sigma = 8 is up to 6e-8
# of the absolute loss sum away from float64, so the bar is 1e-6; one 32-row warp of a million rows is ~3e-5 of it.
LOSS_RTOL = 1e-6


def loss_inputs(kind, task, weighted, rows=ROWS, sigma=8.0):
    seed = sum(map(ord, f'{kind}/{task}/{weighted}/{rows}'))
    g = np.random.default_rng(seed)
    cols = TASKS[task]
    z = (g.normal(size=(rows, cols)) * sigma).astype(np.float32)
    y = _labels(g, task, rows, cols)
    if task == 'regression' and kind == 'Poisson':              # log(p + eps) of the identity output needs p > 0
        z, y = np.abs(z) + 0.1, np.abs(y)
    w = g.uniform(0.5, 2.0, size=rows).astype(np.float32) if weighted else None
    return z, y, w


def loss_call(nat, kind, task, z, y, w, want_grad=True):
    """one launch over device rows z, y (w): (prob, dz or None, float64 loss sum)"""
    rows, cols = z.shape
    prob = torch.empty(rows, cols, device='cuda')
    dz = torch.empty(rows, cols, device='cuda') if want_grad else None
    acc = torch.zeros(1, dtype=torch.float64, device='cuda')
    if kind == 'auto':
        nat.check(nat.lib.dtb_loss_fwd_bwd(P(z), P(y), P(w), P(prob), P(dz), P(acc), rows, cols, CODE[task], None))
    elif kind == 'focal':
        nat.check(nat.lib.dtb_focal_loss_fwd_bwd(P(z), P(y), P(prob), P(dz), P(acc), rows, cols,
                                                 2 if task == 'multiclass' else 0, FOCAL_GAMMA, FOCAL_ALPHA, None))
    else:
        spec = LS.resolve(getattr(LS, kind)(), task)
        scratch = torch.empty(1, dtype=torch.int32, device='cuda')
        lp = nat.LossParams(loss=spec.code, delta=spec.delta, label_smoothing=spec.label_smoothing,
                            scratch=scratch.data_ptr())
        nat.check(nat.lib.dtb_keras_loss_fwd_bwd(P(z), P(y), P(w), P(prob), P(dz), P(acc), rows, cols, CODE[task], lp,
                                                 None))
    return prob, dz, acc


def loss_per_row(kind, task, y, p):
    """float64 per-row loss of probabilities p (the task output) and labels y, both [rows, cols]"""
    if kind == 'focal':
        eps, hi = loss_ref.EPS, loss_ref.ONE_MINUS_EPS           # the kernel's float32 clip bounds
        if task == 'multiclass':                               # CategoricalFocalLoss: renormalise, clip, sum
            q = torch.clamp(p / p.sum(-1, keepdim=True), eps, hi)
            return (FOCAL_ALPHA * torch.pow(1.0 - q, FOCAL_GAMMA) * (-y * torch.log(q))).sum(-1)
        pt1 = torch.where(y == 1, p, torch.ones_like(p)).clamp(eps, hi)
        pt0 = torch.where(y == 0, p, torch.zeros_like(p)).clamp(eps, hi)
        e = -FOCAL_ALPHA * torch.pow(1.0 - pt1, FOCAL_GAMMA) * torch.log(pt1) \
            - (1.0 - FOCAL_ALPHA) * torch.pow(pt0, FOCAL_GAMMA) * torch.log(1.0 - pt0)
        return e.mean(-1)                                      # BinaryFocalLoss: the mean over every element
    spec = LS.resolve(getattr(LS, AUTO[task] if kind == 'auto' else kind)(), task)
    k, delta, s = loss_ref.spec_args(spec)
    return loss_ref.per_row(k, y, p, delta, s)


def loss_float64(kind, task, prob, y, w):
    """(dz, weighted per-row losses, sum_c |p_c dLoss/dp_c| per row) in float64, from the kernel's own float32
    probabilities: where a probability clips, float32 and float64 would otherwise clip different rows."""
    rows = prob.shape[0]
    p = torch.tensor(prob, dtype=torch.float64, requires_grad=True)
    per = loss_per_row(kind, task, torch.tensor(y, dtype=torch.float64), p)
    if w is not None:
        per = per * torch.tensor(w, dtype=torch.float64)
    (gp,) = torch.autograd.grad(per.sum() / rows, [p])
    p = p.detach()
    if task == 'regression':
        gz = gp
    elif task == 'multiclass':
        gz = p * (gp - (gp * p).sum(-1, keepdim=True))
    else:
        gz = gp * p * (1.0 - p)
    return gz.numpy(), per.detach().numpy(), (p * gp).abs().sum(-1, keepdim=True).numpy()


def loss_case(nat, kind, task, weighted, rows=ROWS):
    """The premise holds the loss kernel to 3 passes; the hinge losses' label check over rows x cols labels gets its 3
    passes in the cases of hinge_case, at 2 000 003 rows."""
    sm = sm_count(nat)
    z, y, w = loss_inputs(kind, task, weighted, rows)
    zd, yd, wd = dev(z), dev(y), dev(w)
    name = {'auto': 'loss_kernel', 'focal': 'focal_loss_kernel'}.get(kind, 'keras_loss_kernel')
    loops = [rows_loop(name, rows, 8, sm)]
    if kind in ('Hinge', 'SquaredHinge') and rows == HINGE_ROWS:
        loops.insert(0, rows_loop('hinge_labels_kernel', rows * TASKS[task], 16, sm, 'label'))

    def run(lo=0, hi=rows, want_grad=True):
        return loss_call(nat, kind, task, zd[lo:hi], yd[lo:hi], None if wd is None else wd[lo:hi], want_grad)
    return SimpleNamespace(run=run, loops=loops, one_pass=sm * 8 * THREADS, z=z, y=y, w=w, rows=rows)


def _loss_ids():
    out = []
    for kind in list(LS._CLASSES) + ['auto']:
        for task in TASKS:
            out.append((f'loss-{kind}-{task}', kind, task, len(out) % 2 == 1))
    for task in ('binary', 'multilabel', 'multiclass'):
        out.append((f'loss-focal-{task}', 'focal', task, False))      # the focal losses take no sample weights
    return out


LOSS_CASES = _loss_ids()


def check_loss(c, kind, task, what):
    """the full batch: prob against single-pass slices (bits) and float64; dz and the loss sum against float64"""
    prob_d, dz_d, acc_d = c.run()
    prob, dz, acc = host(prob_d), host(dz_d), float(acc_d.item())
    parts = uneven_slices(c.rows, c.one_pass)
    assert len(parts) >= 3
    sliced = torch.cat([c.run(lo, hi, want_grad=False)[0] for lo, hi in parts])
    if not torch.equal(prob_d, sliced):
        bad = (prob_d != sliced).any(1).nonzero()[:, 0]
        pytest.fail(f'{what}: prob differs from the single-pass slices in {len(bad)} rows, first {bad[:8].tolist()}')
    np.testing.assert_allclose(prob, host(loss_ref_output(c.z, task)), rtol=1e-4, atol=1e-6, err_msg=f'{what}: prob')
    gz, per, terms = loss_float64(kind, task, prob, c.y, c.w)
    # test_losses_gpu.py's bar; its floor 1e-7 was set at 257 rows, and dz scales with 1 / rows
    bar = 1e-7 * 257 / c.rows + 2e-6 * terms + 2e-4 * np.abs(gz)
    ratio = np.abs(dz - gz) / bar
    if kind == 'CategoricalHinge':
        # a row whose margin is 0 within float32 rounding may take either side of max(margin, 0)
        p64, y64 = prob.astype(np.float64), c.y.astype(np.float64)
        pos, neg = (y64 * p64).sum(-1), ((1.0 - y64) * p64).max(-1)
        kink = np.abs(neg - pos + 1.0) <= 1e-6 * (1.0 + np.abs(pos) + np.abs(neg))
        ratio[kink] = 0.0
        print(f'{what}: {int(kink.sum())} rows on the hinge\'s kink')
    bad = ratio > 1
    assert not bad.any(), (f'{what}: dz differs in {int(bad.any(1).sum())} rows, first '
                           f'{np.argwhere(bad)[:5].tolist()}: {dz[bad][:5]} vs {gz[bad][:5]}')
    lo, hi = left_out(c.rows)
    err, sees = check_bar(f'{what}: loss sum', acc, per.sum(), np.abs(per).sum(), per[lo:hi].sum(), LOSS_RTOL)
    return float(ratio.max()), err, sees


def loss_ref_output(z, task):
    return loss_ref.output(torch.tensor(z, dtype=torch.float64), task)


@pytest.mark.parametrize('case_id,kind,task,weighted', LOSS_CASES, ids=[c[0] for c in LOSS_CASES])
def test_losses_past_the_first_pass(nat, case_id, kind, task, weighted):
    c = loss_case(nat, kind, task, weighted)
    worst_dz, err, sees = check_loss(c, kind, task, case_id)
    print(f'{case_id}: dz worst error / bar {worst_dz:.3g}; loss sum error / bar {err}, one warp left out moves it '
          f'{sees} bars')


def hinge_case(nat, kind, where):
    """regression-task hinge over 2 000 003 labels: the labels' check runs 3+ passes.  `where` puts the only label
    outside {0, 1} in the last row, the first, or nowhere."""
    c = loss_case(nat, kind, 'regression', where == 'first', HINGE_ROWS)
    g = np.random.default_rng(5)
    c.z[:] = (g.normal(size=c.z.shape) * 2).astype(np.float32)
    c.y[:] = (g.random(c.y.shape) < 0.5).astype(np.float32)
    if where != 'none':
        c.y[-1 if where == 'last' else 0, 0] = 0.5
    zd, yd, wd = dev(c.z), dev(c.y), dev(c.w)
    c.run = lambda lo=0, hi=c.rows, want_grad=True: loss_call(nat, kind, 'regression', zd[lo:hi], yd[lo:hi],
                                                              None if wd is None else wd[lo:hi], want_grad)
    return c


HINGE_CASES = [(f'hinge-{kind}-{where}', kind, where) for kind in ('Hinge', 'SquaredHinge')
               for where in ('last', 'first', 'none')]


@pytest.mark.parametrize('case_id,kind,where', HINGE_CASES, ids=[c[0] for c in HINGE_CASES])
def test_hinge_label_check_covers_every_pass(nat, case_id, kind, where):
    c = hinge_case(nat, kind, where)
    worst_dz, err, sees = check_loss(c, kind, 'regression', case_id)
    _, dz, _ = c.run()
    dz, y = host(dz)[:, 0], c.y[:, 0]
    zero = y == 0
    if where == 'none':
        # labels 0 / 1 become -1 / 1: a y = 0 row inside the margin has a gradient
        assert np.count_nonzero(dz[zero]), f'{case_id}: no y = 0 row was converted to -1'
    else:
        # one label outside {0, 1} turns the conversion off for every row: y' = 0 has no gradient
        first_pass = np.arange(c.rows) < c.one_pass
        assert not np.any(dz[zero & first_pass]), f'{case_id}: rows of the first pass used the converted label'
        assert not np.any(dz[zero]), f'{case_id}: {np.count_nonzero(dz[zero])} rows used the converted label'
    print(f'{case_id}: dz worst error / bar {worst_dz:.3g}; loss sum error / bar {err}, one warp left out moves it '
          f'{sees} bars')


# ---------------------------------------------------------------------------------------------
# streaming metrics: dtb_metrics_update over one call of a million rows
# ---------------------------------------------------------------------------------------------
def metric_plan(name):
    from deeptables_b200 import metrics as M
    if name in _binary_entries():
        return _plan(_binary_entries()[name], 'binary', 2, 1)
    if name == 'multiclass_topk':
        return _plan(['categorical_accuracy', M.TopKCategoricalAccuracy(k=2), 'f1_score', 'categorical_crossentropy',
                      'precision', M.AUC()], 'multiclass', 6, 6)
    if name == 'global_atomics':            # 12 033 counters: past the 8 192 a block keeps in shared memory
        return _plan([M.AUC(num_thresholds=1000), 'categorical_accuracy'], 'multiclass', 6, 6)
    assert name == 'every_sum'              # all eight sums, R2 over three columns
    specs = [M.resolve(e, 'regression') for e in ('r2_score', M.MeanSquaredError(), M.MeanAbsoluteError(), 'mape',
                                                  'msle', 'logcosh')]
    specs += [M.resolve('bce', 'binary', 2), M.resolve('categorical_crossentropy', 'multiclass', 3)]
    plan = M.Plan(specs, 3)
    assert plan.sums == 255
    return plan


def metric_data(name, kind, rows=ROWS):
    g = np.random.default_rng(17)
    if name in _binary_entries():
        return _binary_data(rows, kind, seed=rows)
    if name == 'every_sum':
        y = g.random((rows, 3)).astype(np.float32)
        y[::7] = 0.0                                            # MAPE's eps, MSLE's clip, BCE's 0 label
        return y, g.random((rows, 3)).astype(np.float32)
    labels = g.integers(0, 6, size=rows)
    y = np.eye(6, dtype=np.float32)[labels]
    z = g.normal(size=(rows, 6)) + y
    p = (np.exp(z) / np.exp(z).sum(-1, keepdims=True)).astype(np.float32)
    p[: rows // 4] = p[: rows // 4].round(1)                    # ties, and rows of zeros and ones
    return y, p


METRIC_CASES = [(f'metrics-{n}-{k}', n, k) for n in _binary_entries() for k in ('random', 'equal', 'on_thresholds')] + \
               [(f'metrics-{n}', n, None) for n in ('multiclass_topk', 'every_sum', 'global_atomics')]


def metric_case(nat, name, kind):
    from deeptables_b200 import engine as E
    sm = sm_count(nat)
    plan = metric_plan(name)
    y, p = metric_data(name, kind)
    yd, pd_ = dev(y), dev(p)
    st = E.MetricsState(plan, torch.device('cuda', 0))

    def run(lo=0, hi=ROWS):
        st.reset()
        st.update(pd_[lo:hi], yd[lo:hi])
        return st.read().copy()
    return SimpleNamespace(run=run, loops=[rows_loop('metrics_update_kernel', ROWS, 8, sm)], plan=plan, y=y, p=p,
                           one_pass=sm * 8 * THREADS)


def sum_words(plan):
    """indices of the float64 words the plan fills: the row sums, then R2's three per column"""
    return [k for k in range(7) if plan.sums & (1 << k)] + (list(range(8, 8 + 3 * plan.cols)) if plan.sums & 128 else [])


@pytest.mark.parametrize('case_id,name,kind', METRIC_CASES, ids=[c[0] for c in METRIC_CASES])
def test_metrics_past_the_first_pass(nat, case_id, name, kind):
    c = metric_case(nat, name, kind)
    plan, cnt = c.plan, c.plan.counters
    if name == 'global_atomics':
        assert plan.words - cnt > 8192
    got = c.run()
    want = SR.state_of(plan, c.y, c.p)
    assert np.array_equal(got[cnt:], want[cnt:]), \
        f'{case_id}: counters differ at {np.flatnonzero(got[cnt:] != want[cnt:])[:10].tolist()}'
    words = sum_words(plan)
    report = ''
    if words:
        lo, hi = left_out(ROWS)
        scale = SR.state_of(plan, np.abs(c.y), c.p)[:cnt].view(np.float64)    # R2's sum y: sum |y|; the rest are >= 0
        drop = SR.state_of(plan, c.y[lo:hi], c.p[lo:hi])[:cnt].view(np.float64)
        w = want[:cnt].view(np.float64)
        err, sees = check_bar(f'{case_id}: float64 sums', got[:cnt].view(np.float64)[words], w[words],
                              np.maximum(np.abs(w[words]), scale[words]), drop[words], 1e-12)
        report = f'; float64 sums error / bar {err}, one warp left out moves them {sees} bars'
    # the full batch against the sum of single-pass slices
    parts = uneven_slices(ROWS, c.one_pass)
    assert len(parts) >= 3
    states = [c.run(lo, hi) for lo, hi in parts]
    total = np.sum([s[cnt:] for s in states], axis=0, dtype=np.uint64)
    assert np.array_equal(got[cnt:], total), f'{case_id}: counters differ from the sum of single-pass slices'
    if words:
        sl = np.sum([s[:cnt].view(np.float64) for s in states], axis=0)
        gw = got[:cnt].view(np.float64)
        scale = np.maximum(np.abs(gw[words]), SR.state_of(plan, np.abs(c.y), c.p)[:cnt].view(np.float64)[words])
        assert np.all(np.abs(gw[words] - sl[words]) <= 1e-12 * scale), f'{case_id}: sums differ from the slices'
    print(f'{case_id}: {plan.words - cnt} counters equal{report}')


# ---------------------------------------------------------------------------------------------
# permutation importance: permutation keys and shuffle, AUC counts, label counts, fixed-order float64 sums
# ---------------------------------------------------------------------------------------------
IMP_ACCURACY, IMP_F1, IMP_F1_MACRO = 3, 4, 5
IMP_LOG_LOSS, IMP_MSE, IMP_RMSE, IMP_MAE, IMP_R2 = 2, 6, 7, 8, 9
SUM_BLOCKS = 256                # importance.cu kSumBlocks: the fixed grid of sum_partials_kernel


def block_tree(v):
    """importance.cu block_tree_sum over the last axis (256 wide): sh[i] += sh[i + s] for s = 128, 64, ..., 1"""
    v = np.array(v, np.float64)
    s = v.shape[-1] // 2
    while s:
        v[..., :s] = v[..., :s] + v[..., s:2 * s]
        s //= 2
    return v[..., 0]


def sum_partials_order(terms, blocks=SUM_BLOCKS, threads=THREADS):
    """the float64 sum dtb_importance_sums forms: thread t of block b adds rows b * 256 + t + k * 65 536 in order from
    0.0, each block reduces its threads with block_tree, and the finishing block reduces the 256 partials the same way"""
    terms = np.asarray(terms, np.float64)
    per = blocks * threads
    acc = np.zeros((blocks, threads))
    for base in range(0, len(terms), per):
        chunk = np.zeros(per)                               # x + 0.0 == x: the rows past the end add nothing
        part = terms[base:base + per]
        chunk[:len(part)] = part
        acc = acc + chunk.reshape(blocks, threads)
    return block_tree(block_tree(acc))


def shap_means_order(values):
    """dtb_shap_means of float64 values [groups, n]: lane l adds rows l, l + 32, ... in order from 0.0, then the
    warp_sum butterfly (dtb_common.cuh: v += shfl_xor(v, o) for o = 16, 8, 4, 2, 1); lane 0's sum over n"""
    values = np.asarray(values, np.float64)
    groups, n = values.shape
    acc = np.zeros((groups, WARP))
    for j in range(0, n, WARP):
        chunk = np.zeros((groups, WARP))
        part = values[:, j:j + WARP]
        chunk[:, :part.shape[1]] = part
        acc = acc + chunk
    lanes = np.arange(WARP)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[:, lanes ^ o]
    return acc[:, 0] / n


def importance_case(nat, what, arg=None):
    sm = sm_count(nat)
    g = np.random.default_rng(23)
    rows = ROWS
    if what == 'perm':
        width, column, seed, it = 5, 3, 0x9e3779b9, 4
        src = dev(g.integers(-2 ** 31, 2 ** 31, size=(rows, width), dtype=np.int64).astype(np.int32))

        def run():
            keys = torch.empty(rows, dtype=torch.int64, device='cuda')
            nat.check(nat.lib.dtb_perm_keys(P(keys), rows, seed, it, column, None))
            sk = torch.sort(keys).values
            dst = torch.full_like(src, -7)
            nat.check(nat.lib.dtb_shuffle_column(P(src), P(dst), P(sk), rows, width, column, None))
            back = dst.clone()
            nat.check(nat.lib.dtb_shuffle_column(P(src), P(back), None, rows, width, column, None))
            return keys, dst, back
        loops = [rows_loop('perm_keys_kernel', rows, 8, sm), rows_loop('shuffle_column_kernel', rows, 8, sm),
                 rows_loop('shuffle_column_kernel', rows, 8, sm)]
        return SimpleNamespace(run=run, loops=loops, src=src, width=width, column=column, seed=seed, it=it)
    if what == 'auc':
        p = (np.floor(g.random(rows) * 64) / 64).astype(np.float32)      # 64 values: tie runs across pass boundaries
        pos = {'mixed': g.random(rows) < 0.3, 'all_positive': np.ones(rows, bool),
               'all_negative': np.zeros(rows, bool)}[arg].astype(np.int32)
        pd_, posd = dev(p), dev(pos)

        def run():
            sp, order = torch.sort(pd_)
            scratch = torch.zeros(2, dtype=torch.int64, device='cuda')
            out = torch.empty(1, dtype=torch.float64, device='cuda')
            nat.check(nat.lib.dtb_importance_auc(P(sp), P(order), P(posd), rows, P(scratch), P(out), None))
            return sp, order, scratch, out
        return SimpleNamespace(run=run, loops=[rows_loop('auc_count_kernel', rows, 8, sm)], pos=pos)
    if what == 'labels':
        metric, cols = arg
        if cols == 1:
            p = g.random((rows, 1)).astype(np.float32)
            p[::9] = 0.5                                                  # p > 1 - p decides: class 0
            label = (g.random(rows) < 0.4).astype(np.int32)
            pd_ = dev(p)
        else:                                                             # quantised: ties go to the first maximum
            gen = torch.Generator(device='cuda').manual_seed(29)
            pd_ = torch.randint(0, 40, (rows, cols), generator=gen, device='cuda').float() / 40
            label = g.integers(0, cols, size=rows).astype(np.int32)
        labeld = dev(label)
        classes = 2 if cols == 1 else cols
        pos = 1 if cols == 1 else 7

        def run():
            scratch = torch.zeros(nat.lib.dtb_importance_scratch_bytes(cols) // 8, dtype=torch.int64, device='cuda')
            out = torch.empty(1, dtype=torch.float64, device='cuda')
            nat.check(nat.lib.dtb_importance_labels(metric, P(pd_), P(labeld), rows, cols, pos, P(scratch), P(out),
                                                    None))
            return scratch, out
        return SimpleNamespace(run=run, loops=[rows_loop('label_count_kernel', rows, 8, sm)], prob=pd_, label=label,
                               classes=classes, pos=pos, cols=cols, metric=metric)
    assert what == 'sums'
    metric, cols = arg
    prob = g.random((rows, cols)).astype(np.float32)
    if metric == IMP_LOG_LOSS:
        if cols > 1:
            prob /= prob.sum(1, keepdims=True)
        prob[::11] = np.float32(1e-9)                                     # clipped at float32's eps
        label = g.integers(0, max(cols, 2), size=rows).astype(np.int32)
        target = None
    else:
        label = None
        target = prob[:, 0].astype(np.float64) + g.normal(size=rows) * 0.3
    aux = float(np.sum((target - target.mean()) ** 2)) if metric == IMP_R2 else 0.0
    pd_, labeld, targetd = dev(prob), dev(label), dev(target)

    def run():
        scratch = torch.empty(nat.lib.dtb_importance_scratch_bytes(cols) // 8, dtype=torch.float64, device='cuda')
        out = torch.empty(1, dtype=torch.float64, device='cuda')
        nat.check(nat.lib.dtb_importance_sums(metric, P(pd_), P(labeld), P(targetd), rows, cols, aux, P(scratch),
                                              P(out), None))
        return out
    loops = [Loop('sum_partials_kernel', lambda gr, b: (rows, gr[0] * b[0]) if gr[0] == SUM_BLOCKS else
                  pytest.fail(f'sum_partials_kernel: grid {gr}'), 'row')]
    return SimpleNamespace(run=run, loops=loops, prob=prob, label=label, target=target, aux=aux, metric=metric,
                           cols=cols)


def test_permutation_keys_and_shuffle(nat):
    c = importance_case(nat, 'perm')
    keys, dst, back = c.run()
    rows = ROWS
    want_keys = IR.perm_keys(c.seed, c.it, c.column, rows)
    assert np.array_equal(host(keys), want_keys), 'dtb_perm_keys differs from the restated keys'
    perm = IR.permutation(c.seed, c.it, c.column, rows)
    src, got = host(c.src), host(dst)
    assert np.array_equal(got[:, c.column], src[perm, c.column]), 'the shuffled column is not the permutation'
    others = [j for j in range(c.width) if j != c.column]
    assert np.all(got[:, others] == -7), 'dtb_shuffle_column wrote outside its column'
    b = host(back)
    assert np.array_equal(b[:, c.column], src[:, c.column]) and np.array_equal(b[:, others], got[:, others])


AUC_CASES = ['mixed', 'all_positive', 'all_negative']


@pytest.mark.parametrize('kind', AUC_CASES)
def test_importance_auc_counts(nat, kind):
    c = importance_case(nat, 'auc', kind)
    sp, order, scratch, out = c.run()
    s, o = host(sp), host(order)
    assert np.all(s[1:] >= s[:-1])
    lo, hi = np.searchsorted(s, s, 'left'), np.searchsorted(s, s, 'right')
    positive = c.pos[o] != 0
    rank2 = int((lo + 1 + hi)[positive].sum())
    npos = int(positive.sum())
    nneg = ROWS - npos
    got = host(scratch).view(np.uint64)
    assert got.tolist() == [rank2, npos], f'rank sum / positives {got.tolist()}, numpy {[rank2, npos]}'
    value = float(out.item())
    if npos == 0 or nneg == 0:
        assert math.isnan(value)
    else:
        want = (float(rank2) - npos * (npos + 1.0)) / (2.0 * npos * nneg)
        assert value == want, f'AUC {value!r}, numpy {want!r}'
    ties = np.diff(np.flatnonzero(np.diff(s) != 0))
    print(f'{kind}: AUC {value}, 2 x rank sum {rank2}, {npos} positives, tie runs up to {ties.max() if len(ties) else ROWS}')


LABEL_CASES = [(m, cols) for cols in (1, 200) for m in (IMP_ACCURACY, IMP_F1, IMP_F1_MACRO)]


@pytest.mark.parametrize('metric,cols', LABEL_CASES, ids=[f'{m}-{c}' for m, c in LABEL_CASES])
def test_importance_label_counts(nat, metric, cols):
    c = importance_case(nat, 'labels', (metric, cols))
    scratch, out = c.run()
    if cols == 1:
        p = host(c.prob)[:, 0]
        pred = (p > np.float32(1) - p).astype(np.int64)
    else:
        pred = host(torch.argmax(c.prob, 1))                 # torch.argmax: the first maximal index
    label, K = c.label.astype(np.int64), c.classes
    hit = pred == label
    want = np.concatenate([[hit.sum()], np.bincount(label[hit], minlength=K), np.bincount(pred, minlength=K),
                           np.bincount(label, minlength=K)]).astype(np.uint64)
    got = host(scratch).view(np.uint64)[:1 + 3 * K]
    assert np.array_equal(got, want), f'counters differ at {np.flatnonzero(got != want)[:10].tolist()}'
    tp, npred, ntrue = want[1:1 + K].astype(np.float64), want[1 + K:1 + 2 * K].astype(np.float64), \
        want[1 + 2 * K:].astype(np.float64)
    den = ntrue + npred
    f1 = np.where(den == 0, 0.0, 2.0 * tp / np.where(den == 0, 1.0, den))
    if metric == IMP_ACCURACY:
        value = float(want[0]) / ROWS
    elif metric == IMP_F1:
        value = f1[c.pos]
    else:
        value = np.mean(f1[den > 0])
    assert float(out.item()) == value, f'{out.item()!r} vs {value!r}'


SUM_CASES = [(IMP_MSE, 1), (IMP_RMSE, 1), (IMP_MAE, 1), (IMP_R2, 1), (IMP_LOG_LOSS, 1), (IMP_LOG_LOSS, 5)]


def importance_terms(c):
    """float64 per-row terms of dtb_importance_sums"""
    if c.metric == IMP_LOG_LOSS:
        eps = np.float32(np.finfo(np.float32).eps)
        if c.cols == 1:
            p = c.prob[:, 0]
            q = np.where(c.label != 0, p, np.float32(1) - p)
        else:
            q = c.prob[np.arange(ROWS), c.label]
        q = np.minimum(np.maximum(q, eps), np.float32(1) - eps).astype(np.float32)
        return -np.log(q.astype(np.float64))
    d = c.target - c.prob[:, 0].astype(np.float64)
    return np.abs(d) if c.metric == IMP_MAE else d * d


def importance_finish(c, s):
    if c.metric == IMP_R2:
        return 1.0 - s / c.aux
    if c.metric == IMP_RMSE:
        return math.sqrt(s / ROWS)
    return s / ROWS


@pytest.mark.parametrize('metric,cols', SUM_CASES, ids=[f'{m}-{c}' for m, c in SUM_CASES])
def test_importance_sums_in_their_fixed_order(nat, metric, cols):
    c = importance_case(nat, 'sums', (metric, cols))
    got = float(c.run().item())
    terms = importance_terms(c)
    want = importance_finish(c, sum_partials_order(terms))
    lo, hi = left_out(ROWS)
    short_terms = terms.copy()
    short_terms[lo:hi] = 0.0
    short = importance_finish(c, sum_partials_order(short_terms))
    if metric == IMP_LOG_LOSS:
        # the device's log and numpy's differ in the last bit of some rows
        err, sees = check_bar(f'log loss {cols}', got, want, abs(want), want - short, 1e-13)
        print(f'log loss, {cols} column(s): error / bar {err}, one warp left out moves it {sees} bars')
    else:
        assert got == want, f'metric {metric}: {got!r}, the restated order gives {want!r} (fsum {math.fsum(terms)!r})'
        assert short != want
        print(f'metric {metric}: the same bits as the restated order; one warp left out changes it by '
              f'{abs(want - short) / abs(want):.2e} relative')


# ---------------------------------------------------------------------------------------------
# SHAP: coalition frames and the per-coalition means
# ---------------------------------------------------------------------------------------------
SHAP_K, SHAP_BG, SHAP_F, SHAP_C, SHAP_X = 2048, 100, 26, 13, 16


def shap_compose_inputs():
    g = np.random.default_rng(31)
    F, C = SHAP_F, SHAP_C
    inp = SimpleNamespace(
        x_cat=g.integers(0, 1000, (SHAP_X, F)).astype(np.int32), x_cont=g.normal(size=(SHAP_X, C)).astype(np.float32),
        bg_cat=g.integers(0, 1000, (SHAP_BG, F)).astype(np.int32),
        bg_cont=g.normal(size=(SHAP_BG, C)).astype(np.float32),
        masks=g.integers(0, 2 ** 32, (SHAP_K, 2), dtype=np.uint64).astype(np.uint32),
        x_index=g.integers(0, SHAP_X, SHAP_K).astype(np.int32))
    bits = np.full(F + C, -1, np.int32)
    bits[g.permutation(F + C)[:34]] = np.arange(34)         # 34 columns vary (bits 0..33, two mask words), 5 never do
    inp.cat_bit, inp.cont_bit = bits[:F], bits[F:]
    return inp


def shap_compose_ref(inp):
    rows = SHAP_K * SHAP_BG
    k, j = np.arange(rows) // SHAP_BG, np.arange(rows) % SHAP_BG

    def takes(bit):
        b = np.maximum(bit, 0)
        return (bit[None, :] >= 0) & (((inp.masks[:, b >> 5] >> (b & 31).astype(np.uint32)) & 1) != 0)
    tc, tn = takes(inp.cat_bit)[k], takes(inp.cont_bit)[k]
    xi = inp.x_index[k]
    return np.where(tc, inp.x_cat[xi], inp.bg_cat[j]), np.where(tn, inp.x_cont[xi], inp.bg_cont[j])


def shap_compose_case(nat):
    sm = sm_count(nat)
    inp = shap_compose_inputs()
    d = {k: dev(v.view(np.int32) if v.dtype == np.uint32 else v) for k, v in vars(inp).items()}
    rows = SHAP_K * SHAP_BG

    def run():
        out_cat = torch.empty(rows, SHAP_F, dtype=torch.int32, device='cuda')
        out_cont = torch.empty(rows, SHAP_C, device='cuda')
        nat.check(nat.lib.dtb_shap_compose(P(d['x_cat']), P(d['x_cont']), P(d['bg_cat']), P(d['bg_cont']),
                                           P(d['masks']), 2, P(d['x_index']), P(d['cat_bit']), P(d['cont_bit']),
                                           SHAP_K, SHAP_BG, SHAP_F, SHAP_C, P(out_cat), P(out_cont), None))
        return out_cat, out_cont
    return SimpleNamespace(run=run, inp=inp,
                           loops=[rows_loop('shap_compose_kernel', rows * (SHAP_F + SHAP_C), 16, sm, 'element')])


def test_shap_compose_is_the_numpy_composition(nat):
    c = shap_compose_case(nat)
    out_cat, out_cont = c.run()
    want_cat, want_cont = shap_compose_ref(c.inp)
    assert np.array_equal(host(out_cat), want_cat), 'categorical columns differ'
    assert np.array_equal(host(out_cont).view(np.uint32), want_cont.view(np.uint32)), 'continuous columns differ'


SHAP_GROUPS, SHAP_N = 60_001, 100
SHAP_MEANS = [('value', 0, 1), ('class_1col', 1, 1), ('class_3col', 1, 3)]


def shap_means_case(nat, kind, cols):
    sm = sm_count(nat)
    g = np.random.default_rng(37)
    rows = SHAP_GROUPS * SHAP_N
    prob = g.random((rows, cols)).astype(np.float32)
    if kind == 1:
        prob = (np.floor(prob * 8) / 8).astype(np.float32)       # ties: the first maximum, and p = 0.5 -> class 0
    pd_ = dev(prob)

    def run():
        out = torch.full((SHAP_GROUPS,), float('nan'), dtype=torch.float64, device='cuda')
        nat.check(nat.lib.dtb_shap_means(P(pd_), SHAP_GROUPS, SHAP_N, cols, kind, P(out), None))
        return out

    def per(b):
        assert b[0] == THREADS
        return b[0] // WARP
    return SimpleNamespace(run=run, prob=prob, loops=[stride('shap_means_kernel', SHAP_GROUPS, per, 'group')])


@pytest.mark.parametrize('case_id,kind,cols', SHAP_MEANS, ids=[c[0] for c in SHAP_MEANS])
def test_shap_means_in_their_fixed_order(nat, case_id, kind, cols):
    c = shap_means_case(nat, kind, cols)
    got = host(c.run())
    p = c.prob
    if kind == 0:
        v = p[:, 0].astype(np.float64)
    elif cols == 1:
        v = (p[:, 0] > np.float32(1) - p[:, 0]).astype(np.float64)
    else:
        v = p.argmax(1).astype(np.float64)
    v = v.reshape(SHAP_GROUPS, SHAP_N)
    want = shap_means_order(v)
    bad = np.flatnonzero(got.view(np.uint64) != want.view(np.uint64))
    assert not len(bad), (f'{case_id}: {len(bad)} groups differ from the restated order, first {bad[:5].tolist()}: '
                          f'{got[bad[:3]].tolist()} vs {want[bad[:3]].tolist()}')
    print(f'{case_id}: {SHAP_GROUPS} means, the same bits as the restated order')


# ---------------------------------------------------------------------------------------------
# boosting: gradients and their batch-wide max, fixed point, score update, tree traversal
# ---------------------------------------------------------------------------------------------
GBDT_OBJ = {'binary': (0, 1), 'regression': (1, 1), 'multiclass': (2, 3)}     # objective code, score columns
GRAD_CASES = [(f'gbdt_grad-{o}-{w}', o, w) for o in GBDT_OBJ for w in ('last_row', 'last_cta')]


def spike_rows(nat, rows, where):
    """two rows in the last pass: the batch's last two, or the first two of the last CTA's last pass"""
    if where == 'last_row':
        return rows - 1, rows - 2
    grid = min(cdiv(rows, THREADS), sm_count(nat) * 8)
    base = (grid - 1) * THREADS
    r = base + (rows - 1 - base) // (grid * THREADS) * grid * THREADS
    assert r + 1 < rows
    return r, r + 1


def gbdt_grad_case(nat, objective, where, rows=ROWS):
    sm = sm_count(nat)
    code, K = GBDT_OBJ[objective]
    k = 1 if K > 1 else 0
    g = np.random.default_rng(41 + code)
    rg, rh = spike_rows(nat, rows, where)
    if objective == 'binary':        # |s| >= 0.5: h < 0.235; |s| <= 5: |g| < 0.994
        scores = (g.choice([-1.0, 1.0], rows) * g.uniform(0.5, 5.0, rows))[:, None]
        label = (g.random(rows) < 0.5).astype(np.float32)
        scores[rg], label[rg] = -40.0, 1.0                      # g = -1
        scores[rh] = 0.0                                        # h = 0.25
    elif objective == 'regression':
        scores = g.normal(size=(rows, 1)) * 3
        label = g.normal(size=rows).astype(np.float32)
        scores[rg], label[rg] = 100.0, 0.0                      # g = 100; h = 1 everywhere
    else:                            # p_k <= 0.16: h < 0.2 and |g| < 0.9996
        scores = g.uniform(0.0, 1.0, (rows, K))
        scores[:, k] = g.uniform(-6.0, -1.0, rows)
        label = g.integers(0, K, rows).astype(np.float32)
        scores[rg], label[rg] = [0.0, -40.0, 0.0], k            # g = -1
        scores[rh] = [0.0, math.log(2.0), 0.0]                  # p_k = 1 / 2: h = 3 / 8
    sd, ld = dev(scores), dev(label)

    def run():
        gd, hd = torch.empty(rows, device='cuda'), torch.empty(rows, device='cuda')
        mx = torch.zeros(2, device='cuda')
        nat.check(nat.lib.dtb_gbdt_grad(P(sd), P(ld), rows, K, k, code, P(gd), P(hd), P(mx), None))
        m = host(mx)
        sg, sh = R.shift(m[0], rows), R.shift(m[1], rows)
        gq, hq = torch.empty(rows, dtype=torch.int64, device='cuda'), torch.empty(rows, dtype=torch.int64, device='cuda')
        nat.check(nat.lib.dtb_gbdt_fixed(P(gd), P(hd), rows, sg, sh, P(gq), P(hq), None))
        return gd, hd, m, (sg, sh), gq, hq
    return SimpleNamespace(run=run, scores=scores, label=label, K=K, k=k, spikes=(rg, rh), rows=rows,
                           loops=[rows_loop('gbdt_grad_kernel', rows, 8, sm), rows_loop('gbdt_fixed_kernel', rows, 8, sm)])


def ulps32(a, b):
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia)
    ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


@pytest.mark.parametrize('case_id,objective,where', GRAD_CASES, ids=[c[0] for c in GRAD_CASES])
def test_gbdt_gradients_max_and_fixed_point(nat, case_id, objective, where):
    c = gbdt_grad_case(nat, objective, where)
    gd, hd, m, (sg, sh), gq, hq = c.run()
    g, h = host(gd), host(hd)
    name = {'binary': 'binary', 'regression': 'regression', 'multiclass': 'softmax'}[objective]
    wg, wh = R.grad_hess(c.scores, c.label, name, c.K)
    # float64 exp on the device and in numpy can differ in the last bit before the rounding to float32
    ug, uh = ulps32(g, wg[c.k]), ulps32(h, wh[c.k])
    assert ug.max() <= 1 and uh.max() <= 1, f'{case_id}: g / h differ by {ug.max()} / {uh.max()} float32 ulps'
    # the batch-wide max: exactly the largest |g| and h, which the two spike rows hold
    assert m[0] == np.abs(g).max() and m[1] == h.max(), f'{case_id}: max_gh {m}, rows give {np.abs(g).max()}, {h.max()}'
    rg, rh = c.spikes
    assert m[0] == abs(g[rg]) and np.sum(np.abs(g) == m[0]) == 1, f'{case_id}: the largest |g| is not row {rg} alone'
    if objective != 'regression':
        assert m[1] == h[rh] and np.sum(h == m[1]) == 1, f'{case_id}: the largest h is not row {rh} alone'
    assert (sg, sh) == (R.shift(np.abs(wg[c.k]).max(), c.rows), R.shift(wh[c.k].max(), c.rows))
    assert np.array_equal(host(gq), R.fixed(g, sg)) and np.array_equal(host(hq), R.fixed(h, sh)), \
        f'{case_id}: fixed point differs'
    print(f'{case_id}: max |g| {m[0]} (row {rg}), max h {m[1]} (row {rh}); shifts {sg}, {sh}; '
          f'{int((ug > 0).sum())} / {int((uh > 0).sum())} rows 1 ulp off numpy exp')


UPDATE_COUNTS, UPDATE_BEGINS, UPDATE_ROWS = [600_001, 900_001, 550_001], [900_001, 0, 1_500_002], 2_100_000


def gbdt_update_case(nat):
    sm = sm_count(nat)
    g = np.random.default_rng(43)
    rows, K, k, stride_ = UPDATE_ROWS, 2, 1, 4
    index = g.permutation(rows).astype(np.int32)
    values = g.normal(size=len(UPDATE_COUNTS)).astype(np.float32)
    scores = g.normal(size=(rows, K))
    idx_d, vals_d = dev(index), dev(values)
    seg_b, seg_c = dev(np.asarray(UPDATE_BEGINS, np.int64)), dev(np.asarray(UPDATE_COUNTS, np.int64))

    def run():
        s = dev(scores)
        log = torch.full((rows, stride_), -1, dtype=torch.int32, device='cuda')
        nat.check(nat.lib.dtb_gbdt_update(P(idx_d), P(seg_b), P(seg_c), len(values), max(UPDATE_COUNTS), P(vals_d),
                                          P(s), K, k, P(log, 2 * 4), stride_, None))
        return s, log

    def work(gr, b):
        assert gr[1] == len(values) and b[0] == THREADS, (gr, b)
        return min(UPDATE_COUNTS), gr[0] * b[0]
    return SimpleNamespace(run=run, index=index, values=values, scores=scores, k=k,
                           loops=[Loop('gbdt_update_kernel', work, 'row of the smallest leaf')])


def test_gbdt_update_scores_and_leaf_log(nat):
    c = gbdt_update_case(nat)
    s, log = c.run()
    leaf = np.full(UPDATE_ROWS, -1, np.int64)
    for l, (b, n) in enumerate(zip(UPDATE_BEGINS, UPDATE_COUNTS)):
        leaf[c.index[b:b + n]] = l
    m = leaf >= 0
    want = c.scores.copy()
    want[m, c.k] = c.scores[m, c.k] + c.values[leaf[m]].astype(np.float64)
    got = host(s)
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), \
        f'scores differ in {int((got != want).any(1).sum())} rows'
    want_log = np.full((UPDATE_ROWS, 4), -1, np.int32)
    want_log[m, 2] = leaf[m]
    assert np.array_equal(host(log), want_log), 'leaf log differs'


LEAF_TREES, LEAF_LEAVES, LEAF_NF = 60, 255, 12


def random_trees(g, edges, n_trees, n_leaves):
    """leaf-wise trees in gbm_ref's node lists: each split takes a random leaf, feature and bin"""
    trees = []
    for _ in range(n_trees):
        t = {'feature': [], 'bin': [], 'left': [], 'right': []}
        parent = [None]
        for new in range(1, n_leaves):
            leaf = int(g.integers(0, new))
            f = int(g.integers(0, len(edges)))
            node = len(t['feature'])
            t['feature'].append(f)
            t['bin'].append(int(g.integers(0, len(edges[f]))))
            t['left'].append(~leaf)
            t['right'].append(~new)
            if parent[leaf] is not None:
                pn, side = parent[leaf]
                t['left' if side == 0 else 'right'][pn] = node
            parent[leaf] = (node, 0)
            parent.append((node, 1))
        trees.append(t)
    return trees


def traverse_fast(tree, X, edges):
    """gbm_ref.traverse with the node thresholds looked up once (it is checked against gbm_ref.traverse below)"""
    feat = np.asarray(tree['feature'])
    thr = np.array([edges[f][b] for f, b in zip(tree['feature'], tree['bin'])], np.float32)
    left, right = np.asarray(tree['left']), np.asarray(tree['right'])
    node = np.zeros(len(X), np.int64)
    out = np.empty(len(X), np.int32)
    live = np.arange(len(X))
    while len(live):
        n = node[live]
        nxt = np.where(X[live, feat[n]] <= thr[n], left[n], right[n])
        done = nxt < 0
        out[live[done]] = ~nxt[done]
        node[live[~done]] = nxt[~done]
        live = live[~done]
    return out


def gbdt_leaves_case(nat):
    sm = sm_count(nat)
    g = np.random.default_rng(47)
    rows = ROWS
    X = np.empty((rows, LEAF_NF), np.float32)
    edges = []
    for j in range(LEAF_NF):
        if j % 3 == 0:                                           # integer codes, integer thresholds: x == t goes left
            X[:, j] = g.integers(0, 50, rows)
            edges.append(np.arange(49, dtype=np.float32))
        else:
            X[:, j] = g.normal(size=rows)
            X[g.random(rows) < 0.1, j] = np.nan                  # NaN goes right
            edges.append(np.sort(g.normal(size=63)).astype(np.float32))
    trees = random_trees(g, edges, LEAF_TREES, LEAF_LEAVES)
    cat_cols = [j for j in range(LEAF_NF) if j % 3 == 0]
    cont_cols = [j for j in range(LEAF_NF) if j % 3]
    feat_col = [cat_cols.index(j) if j in cat_cols else -1 - cont_cols.index(j) for j in range(LEAF_NF)]
    cat, cont = dev(X[:, cat_cols].astype(np.int32)), dev(X[:, cont_cols])
    nodes = [len(t['feature']) for t in trees]
    arr = lambda key, dt: dev(np.concatenate([np.asarray(t[key], dt) for t in trees]))
    thr = dev(np.concatenate([[edges[f][b] for f, b in zip(t['feature'], t['bin'])] for t in trees]).astype(np.float32))
    d = dict(feature=arr('feature', np.int32), left=arr('left', np.int32), right=arr('right', np.int32), thr=thr,
             off=dev(np.concatenate([[0], np.cumsum(nodes)]).astype(np.int32)), fc=dev(np.asarray(feat_col, np.int32)))
    out_stride, out_col = LEAF_TREES + 2, 1

    def run():
        out = torch.full((rows, out_stride), -1, dtype=torch.int32, device='cuda')
        nat.check(nat.lib.dtb_gbdt_leaves(P(cat), cat.shape[1], P(cont), cont.shape[1], P(d['fc']), P(d['feature']),
                                          P(d['thr']), P(d['left']), P(d['right']), P(d['off']), LEAF_TREES, max(nodes),
                                          rows, P(out), None, out_stride, out_col, None))
        return out
    stages, t0 = 0, 0
    off = np.concatenate([[0], np.cumsum(nodes)])
    while t0 < LEAF_TREES:
        t1 = t0
        while t1 < LEAF_TREES and off[t1 + 1] - off[t0] <= nat.GBDT_STAGE_NODES:
            t1 += 1
        stages, t0 = stages + 1, t1
    return SimpleNamespace(run=run, X=X, edges=edges, trees=trees, stages=stages, out_col=out_col,
                           loops=[rows_loop('gbdt_leaves_kernel', rows, 6, sm)])


def test_gbdt_leaves_equal_the_traversal(nat):
    c = gbdt_leaves_case(nat)
    out = host(c.run())
    assert np.all(out[:, 0] == -1) and np.all(out[:, -1] == -1), 'dtb_gbdt_leaves wrote outside its columns'
    for t, tree in enumerate(c.trees):
        want = traverse_fast(tree, c.X, c.edges)
        if t == 0:
            assert np.array_equal(want[:3000], R.traverse(tree, c.X[:3000], c.edges))
        got = out[:, c.out_col + t]
        assert np.array_equal(got, want), f'tree {t} (stage of {t}): {int((got != want).sum())} rows differ'
    print(f'{LEAF_TREES} trees of {LEAF_LEAVES} leaves in {c.stages} stages over {ROWS} rows: every leaf equal')


# ---------------------------------------------------------------------------------------------
# 1. the premise, from launches recorded in a child process
# ---------------------------------------------------------------------------------------------
def _premise_cases():
    out = [(cid, loss_case, (kind, task, weighted)) for cid, kind, task, weighted in LOSS_CASES]
    out += [(cid, hinge_case, (kind, where)) for cid, kind, where in HINGE_CASES]
    out += [(cid, metric_case, (name, kind)) for cid, name, kind in METRIC_CASES]
    out += [('importance-perm', importance_case, ('perm',))]
    out += [(f'importance-auc-{k}', importance_case, ('auc', k)) for k in AUC_CASES]
    out += [(f'importance-labels-{m}-{c}', importance_case, ('labels', (m, c))) for m, c in LABEL_CASES]
    out += [(f'importance-sums-{m}-{c}', importance_case, ('sums', (m, c))) for m, c in SUM_CASES]
    out += [('shap-compose', shap_compose_case, ()), *[(f'shap-means-{i}', shap_means_case, (k, c))
                                                         for i, k, c in SHAP_MEANS]]
    out += [(cid, gbdt_grad_case, (o, w)) for cid, o, w in GRAD_CASES]
    out += [('gbdt-update', gbdt_update_case, ()), ('gbdt-leaves', gbdt_leaves_case, ())]
    return out


CASES = _premise_cases()
BY_ID = {c[0]: c for c in CASES}


def build(nat, case_id):
    _, fn, args = BY_ID[case_id]
    return fn(nat, *args)


def _record(path):
    """Child process: the launches of every case's full call."""
    from deeptables_b200 import _native as nat
    rec = {}
    for case_id, _, _ in CASES:
        c = build(nat, case_id)
        rec[case_id], _ = launches(c.run)
        del c
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    with open(path, 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def recorded(tmp_path_factory):
    path = str(tmp_path_factory.mktemp('launches') / 'launches.json')
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f'import sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]; import test_eval_passes_gpu as t; '
            f't._record({path!r})')
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ['-c', code], capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f'recording the launches failed:\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'
    with open(path) as f:
        return json.load(f)


@pytest.mark.parametrize('case_id', [c[0] for c in CASES])
def test_loops_run_several_passes(nat, recorded, case_id):
    c = build(nat, case_id)
    print(f'{case_id}: passes {passes_of(case_id, recorded[case_id], c.loops)}')
