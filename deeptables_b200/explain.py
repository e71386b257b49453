"""Kernel SHAP on the device (the work behind ``utils.shap.DeepTablesExplainer``).

shap's KernelExplainer with the identity link and no L1 feature selection.  For each explained row x, the columns whose
background values differ from x's vary; the coalitions over them are chosen on the host by shap's scheme (every subset
of the sizes the budget covers, the rest drawn by size weight), and the value of a coalition is the mean, over the
background rows, of the model function on the background row with the coalition's columns taken from x.  Those values
are computed here: the frames are encoded and uploaded once, ``dtb_shap_compose`` writes the synthetic rows of a range
of coalitions (of several explained rows at once), the inference forward runs over them in batches and
``dtb_shap_means`` reduces each coalition's rows into one float64.  The host reads the values once per group of
explained rows and solves shap's constrained weighted least squares in float64.  DefaultPreprocessor encodes each cell
on its own, so composing encoded columns is composing raw ones.  Quantile-bin columns (``auto_discrete``) and
gradient-boosted leaf columns are not columns of X: they get mask bit -1 and no SHAP column, and are recomputed from
each composed row on the device, the bin columns first.

The model function is ``DeepTable.predict(X, encode_to_label=False)``: the prediction on regression, the class code
otherwise.  The draws of row i come from ``np.random.RandomState([seed, i])``, so a given seed gives the same bits for
any batch size or number of ranks.  Data parallel: every rank calls with the same frames, row i is explained on rank
``i % world`` and the results are all-gathered, so every rank returns what one process would.
"""
import collections
import itertools
import time
from math import comb

import numpy as np
import torch

from . import _native as N, consts, discrete
from ._native import check, ptr, stream_ptr
from .analysis import Stages, check_positive_int, fitted_model, forward_rows, gather_strided, is_int, model_columns, \
    rank_share

SHAP_VALUE, SHAP_CLASS = 0, 1             # DTB_SHAP_* (deeptables_b200.h)
_NUMBER_TYPES = (int, float, np.number)
_GROUP_ROWS = 32              # explained rows whose coalition values the host reads at once
_DRAW_CHUNK = 1024            # random coalitions drawn per numpy call

Row = collections.namedtuple('Row', 'varying masks weights values fx')


def budget(M, nsamples):
    """shap's number of coalitions for M varying columns: 2M + 2048 for 'auto', capped at 2^M - 2 when M <= 30."""
    n = 2 * M + 2 ** 11 if nsamples == 'auto' else int(nsamples)
    return min(n, 2 ** M - 2) if M <= 30 else n


def check_nsamples(nsamples):
    if isinstance(nsamples, str) and nsamples == 'auto':
        return
    if not is_int(nsamples) or nsamples < 1:
        raise ValueError(f"nsamples must be 'auto' or a positive integer, got {nsamples!r}")


def _not_equal(a, b):
    """shap's test of one value against one background value: numbers by np.isclose (NaN equal to NaN), else ==."""
    if isinstance(a, _NUMBER_TYPES) and isinstance(b, _NUMBER_TYPES):
        return not np.isclose(a, b, equal_nan=True)
    return not a == b


_not_equal_u = np.frompyfunc(_not_equal, 2, 1)


def varying_columns(x, background):
    """Positions of the columns where some background value differs from x's.  ``x``: one row of values;
    ``background``: a list of per-column value arrays."""
    out = []
    for j, (v, col) in enumerate(zip(x, background)):
        if col.dtype.kind in 'iuf' and isinstance(v, _NUMBER_TYPES) and not isinstance(v, (bool, np.bool_)):
            differs = not np.all(np.isclose(v, col, equal_nan=True))
        else:
            differs = bool(np.any(_not_equal_u(v, col).astype(bool)))
        if differs:
            out.append(j)
    return np.array(out, np.int64)


def sample_coalitions(M, nsamples, rng):
    """shap KernelExplainer's coalitions for M >= 2 varying columns: (masks bool [K, M], weights float64 [K]).

    Sizes are enumerated in order while the remaining budget covers all their subsets (paired sizes: with their
    complements); the rest of the budget is drawn from ``rng`` by the remaining size weights, a drawn mask being the
    ``size`` columns with the smallest of M uniform keys, its complement added for a paired size, and a repeated mask
    adding 1 to its weight instead of taking a slot.  The drawn weights are then rescaled to the weight left over."""
    n = budget(M, nsamples)
    n_sizes, n_paired = M // 2, (M - 1) // 2            # ceil((M-1)/2), floor((M-1)/2)
    wv = np.array([(M - 1.0) / (s * (M - s)) for s in range(1, n_sizes + 1)])
    wv[:n_paired] *= 2
    wv /= np.sum(wv)
    masks, weights = [], []
    left, full, rem = n, 0, wv.copy()
    for s in range(1, n_sizes + 1):
        paired = s <= n_paired
        nsub = comb(M, s) * (2 if paired else 1)
        if left * rem[s - 1] / nsub < 1.0 - 1e-8:
            break
        full += 1
        left -= nsub
        if rem[s - 1] < 1.0:
            rem /= 1 - rem[s - 1]
        w = wv[s - 1] / comb(M, s) / (2.0 if paired else 1.0)
        idx = np.array(list(itertools.combinations(range(M), s)), np.int64)
        m = np.zeros((len(idx), M), bool)
        m[np.arange(len(idx))[:, None], idx] = True
        if paired:
            m = np.stack([m, ~m], axis=1).reshape(-1, M)
        masks.append(m)
        weights.append(np.full(len(m), w))
    fixed = sum(len(m) for m in masks)
    left = n - fixed
    if full != n_sizes and left > 0:
        rw = wv.copy()
        rw[:n_paired] /= 2
        rw = rw[full:]
        rw /= np.sum(rw)
        sizes = rng.choice(len(rw), 4 * left, p=rw) + full + 1
        drawn, w_drawn, seen = [], [], {}
        pos = 0
        while left > 0 and pos < len(sizes):
            size = sizes[pos:pos + _DRAW_CHUNK]
            keys = rng.random_sample((len(size), M))
            chunk = keys.argsort(axis=1).argsort(axis=1) < size[:, None]
            packed = np.packbits(chunk, axis=1)
            for i in range(len(size)):
                if left <= 0:
                    break
                key = packed[i].tobytes()
                paired = size[i] <= n_paired
                at = seen.get(key)
                if at is None:
                    seen[key] = len(drawn)
                    drawn.append(chunk[i])
                    w_drawn.append(1.0)
                    left -= 1
                    if left > 0 and paired:
                        drawn.append(~chunk[i])
                        w_drawn.append(1.0)
                        left -= 1
                else:
                    w_drawn[at] += 1.0
                    if paired:
                        w_drawn[at + 1] += 1.0
            pos += len(size)
        w_drawn = np.array(w_drawn)
        w_drawn *= np.sum(wv[full:]) / w_drawn.sum()
        masks.append(np.array(drawn, bool).reshape(-1, M))
        weights.append(w_drawn)
    return np.concatenate(masks), np.concatenate(weights)


def solve(masks, weights, values, fx, expected):
    """shap's solve with the identity link: weighted least squares of the coalition values minus E on the masks, with
    the sum of the values held at f(x) - E by eliminating the last column, in float64."""
    Z = masks.astype(np.float64)
    total = fx - expected
    y = values - expected - Z[:, -1] * total
    Zt = Z[:, :-1] - Z[:, -1:]
    wZ = Zt * weights[:, None]
    A, b = wZ.T @ Zt, wZ.T @ y
    try:
        phi = np.linalg.solve(A, b)
    except np.linalg.LinAlgError:
        phi = np.linalg.pinv(A) @ b
    return np.append(phi, total - np.sum(phi))


class Background:
    """The background rows, encoded and uploaded once, and E, the mean of the model function over them."""

    def __init__(self, dt_model, frame, batch_size):
        model = fitted_model(dt_model)
        if len(frame) < 1:
            raise ValueError('the background has no rows')
        self.dt_model, self.model = dt_model, model
        self.columns = frame.columns.to_list()
        self.values = [frame[c].to_numpy() for c in self.columns]
        self.rows = len(frame)
        self.cols = model._output_dim()
        self.kind = SHAP_VALUE if model.task == consts.TASK_REGRESSION else SHAP_CLASS
        model.flush_optimizer_state()           # every embedding row current: the forward needs no per-batch catch-up
        self.cat, self.cont = self.encode(frame)
        cat_names, cont_names = model_columns(model)
        pos = {str(c): j for j, c in enumerate(self.columns)}
        dev = model.device
        # the bit of each encoded column in a coalition mask is its column's position in the frame
        self.cat_bit = torch.tensor([pos.get(n, -1) for n in cat_names], dtype=torch.int32, device=dev)
        self.cont_bit = torch.tensor([pos.get(n, -1) for n in cont_names], dtype=torch.int32, device=dev)
        self.words = (len(self.columns) + 31) // 32
        self.expected = float(self.means(self.cat, self.cont, self.rows, self.rows, batch_size).cpu()[0])

    def encode(self, frame):
        return self.model._to_device_inputs(self.dt_model.preprocessor.transform_X(frame))

    def means(self, cat, cont, rows, n, batch_size):
        """float64 [rows // n] device tensor: the mean of the model function over each n consecutive input rows."""
        pred = torch.empty(rows, self.cols, dtype=torch.float32, device=self.model.device)
        forward_rows(self.model, cat, cont, pred, batch_size)
        out = torch.empty(rows // n, dtype=torch.float64, device=self.model.device)
        check(N.lib.dtb_shap_means(ptr(pred), rows // n, n, self.cols, self.kind, ptr(out), stream_ptr()),
              'shap_means')
        return out


def shap_values(bg, X, nsamples='auto', seed=0, batch_size=65536, stages=None, trace=None):
    """float64 [len(X), columns] Kernel SHAP values of the model function at each row of X against ``bg``.

    ``stages``: a dict that receives the seconds spent in host sampling, compose, forward, means and solve (device
    stages timed with CUDA events).  ``trace``: a dict that receives, per explained row, its Row(varying columns,
    masks, weights, coalition values, f(x))."""
    check_nsamples(nsamples)
    check_positive_int(batch_size, 'batch_size')
    if X.columns.to_list() != bg.columns:
        raise ValueError(f'X has columns {X.columns.to_list()}, the explainer {bg.columns}')
    model, dev = bg.model, bg.model.device
    n_rows, n_cols, N_bg = len(X), len(bg.columns), bg.rows
    if n_rows == 0:
        return np.zeros((0, n_cols), np.float64)
    timer = Stages(stages)
    model.flush_optimizer_state()
    x_cat, x_cont = bg.encode(X)
    fx = bg.means(x_cat, x_cont, n_rows, 1, batch_size).cpu().numpy()
    x_values = X.to_numpy(dtype=object)
    phi = np.zeros((n_rows, n_cols), np.float64)

    mine = rank_share(n_rows)
    per_chunk = max(1, batch_size // N_bg)          # coalitions per compose launch
    F = x_cat.shape[1] if x_cat is not None else 0
    C = x_cont.shape[1] if x_cont is not None else 0
    out_cat = torch.empty(per_chunk * N_bg, F, dtype=torch.int32, device=dev) if F else None
    out_cont = torch.empty(per_chunk * N_bg, C, dtype=torch.float32, device=dev) if C else None
    pred = torch.empty(per_chunk * N_bg, bg.cols, dtype=torch.float32, device=dev)

    def sample(i):
        vary = varying_columns(x_values[i], bg.values)
        M = len(vary)
        if M < 2:
            return vary, None, None
        masks, weights = sample_coalitions(M, nsamples, np.random.RandomState([seed, i]))
        return vary, masks, weights

    def enqueue(group):
        """Launch the coalition values of every row in ``group``; returns (plans, host tensor, event) or None."""
        t0 = time.perf_counter()
        plans = [(i,) + sample(i) for i in group]
        full, x_index = [], []
        for i, vary, masks, _ in plans:
            if masks is not None:
                m = np.zeros((len(masks), n_cols), bool)
                m[:, vary] = masks
                full.append(m)
                x_index.append(np.full(len(m), i, np.int32))
        timer.host('sampling', t0)
        if not full:
            return plans, None, None
        packed = np.packbits(np.concatenate(full), axis=1, bitorder='little')
        packed = np.pad(packed, ((0, 0), (0, 4 * bg.words - packed.shape[1])))
        masks_dev = torch.as_tensor(packed.view(np.uint32)).to(dev)
        index_dev = torch.as_tensor(np.concatenate(x_index)).to(dev)
        K = len(index_dev)
        values = torch.empty(K, dtype=torch.float64, device=dev)
        for k0 in range(0, K, per_chunk):
            k = min(per_chunk, K - k0)
            rows = k * N_bg
            with timer.device('compose'):
                check(N.lib.dtb_shap_compose(ptr(x_cat), ptr(x_cont), ptr(bg.cat), ptr(bg.cont), ptr(masks_dev[k0:]),
                                             bg.words, ptr(index_dev[k0:]), ptr(bg.cat_bit), ptr(bg.cont_bit), k,
                                             N_bg, F, C, ptr(out_cat), ptr(out_cont), stream_ptr()), 'shap_compose')
                discrete.rewrite_derived(bg.dt_model.preprocessor, out_cat[:rows] if F else None,
                                         out_cont[:rows] if C else None)
            with timer.device('forward'):
                forward_rows(model, out_cat, out_cont, pred[:rows], batch_size)
            with timer.device('means'):
                check(N.lib.dtb_shap_means(ptr(pred), k, N_bg, bg.cols, bg.kind, ptr(values[k0:]), stream_ptr()),
                      'shap_means')
        host = torch.empty(K, dtype=torch.float64, pin_memory=True)
        host.copy_(values, non_blocking=True)
        event = torch.cuda.Event()
        event.record()
        return plans, host, event

    def finish(pending):
        plans, host, event = pending
        if event is not None:
            event.synchronize()
        values = host.numpy() if host is not None else None
        t0 = time.perf_counter()
        at = 0
        for i, vary, masks, weights in plans:
            total = fx[i] - bg.expected
            y = None
            if masks is not None:
                y = values[at:at + len(masks)].copy()
                at += len(masks)
                phi[i, vary] = solve(masks, weights, y, fx[i], bg.expected)
            elif len(vary) == 1:
                phi[i, vary[0]] = total
            if trace is not None:
                trace[i] = Row(vary, masks, weights, y, fx[i])
        timer.host('solve', t0)

    pending = None
    for g0 in range(0, len(mine), _GROUP_ROWS):
        current = enqueue(mine[g0:g0 + _GROUP_ROWS])     # host sampling of this group overlaps the previous one's GPU work
        if pending is not None:
            finish(pending)
        pending = current
    if pending is not None:
        finish(pending)

    timer.finish()
    return gather_strided(phi[mine], n_rows)


# ---------------------------------------------------------------------------------------------------------------------
# expected gradients (utils.shap.DeepTablesGradientExplainer)
# ---------------------------------------------------------------------------------------------------------------------
GRAD_IDENTITY, GRAD_SIGMOID, GRAD_SOFTMAX = 0, 1, 2      # DTB_GRADSHAP_* (deeptables_b200.h)
_ALPHA_BITS = 24                                          # alpha is a multiple of 2^-24: exact in float32, below 1


def check_gradient_options(dt_model):
    """The derived columns of ``apply_gbm_features`` and ``auto_discrete`` are step functions of the continuous inputs:
    a gradient cannot attribute their jumps."""
    cfg = getattr(dt_model, 'config', None)
    for option in ('apply_gbm_features', 'auto_discrete'):
        if cfg is not None and getattr(cfg, option, False):
            raise NotImplementedError(f'{option}=True: expected gradients cannot attribute the jumps of its derived '
                                      f'columns')


def gradient_draws(seed, i, nsamples, bg_rows, rng=None):
    """The samples of explained row i: background rows j (int32 [nsamples], uniform with replacement) then the
    interpolation points alpha (float32 [nsamples], uniform on [0, 1) in steps of 2^-24), both from
    ``np.random.RandomState([seed, i])``.  ``rng``: a RandomState to reseed instead of building one (the same draws,
    at a sixth of the host time)."""
    if rng is None:
        rng = np.random.RandomState()
    rng.seed([seed, i])
    j = rng.randint(0, bg_rows, size=nsamples).astype(np.int32)
    alpha = (np.floor(rng.random_sample(nsamples) * 2.0 ** _ALPHA_BITS) / 2.0 ** _ALPHA_BITS).astype(np.float32)
    return j, alpha


def output_kind(task):
    return {consts.TASK_REGRESSION: GRAD_IDENTITY, consts.TASK_MULTICLASS: GRAD_SOFTMAX}.get(task, GRAD_SIGMOID)


def output_means(bg, cat, cont, rows, batch_size):
    """float64 [outputs]: the mean of the explained output (the output layer) over ``rows`` input rows."""
    pred = torch.empty(rows, bg.cols, dtype=torch.float32, device=bg.model.device)
    forward_rows(bg.model, cat, cont, pred, batch_size)
    return pred.cpu().numpy().astype(np.float64).mean(axis=0)


class _Embeddings:
    """What the gradient kernels read of the model's embedding table: the table, its row offsets and the column offset
    of each field in a flat row (device int32 [F + 1])."""

    def __init__(self, model):
        t = model.table
        self.table, self.row_offsets, self.dim, self.ragged = t.weight, t.row_offsets, t.dim, t.ragged
        self.fields = t.n_fields
        self.col_offsets = torch.tensor(np.concatenate([[0], np.cumsum(t.field_dims)]), dtype=torch.int32,
                                        device=model.device)
        self.width = int(sum(t.field_dims))


def gradient_values(bg, X, nsamples=200, seed=0, batch_size=65536, stages=None):
    """float64 [len(X), columns, outputs] expected gradients of the output layer at each row of X against ``bg``.

    Pair (i, s) interpolates between row i and background row j_s at alpha_s (``gradient_draws``); its value in an
    encoded column is the gradient of the output there times the column's difference x - b (summed over the
    embedding coordinates of a categorical field); a row's value is the mean over its samples.  Each frame column
    takes the value of the encoded column read from it, 0 when the model reads none.  ``stages``: a dict that receives
    the seconds spent in compose, forward, backward, reduce and means (CUDA events) and on the host in encode (the
    preprocessor and the upload) and draws."""
    check_positive_int(nsamples, 'nsamples')
    check_positive_int(batch_size, 'batch_size')
    if X.columns.to_list() != bg.columns:
        raise ValueError(f'X has columns {X.columns.to_list()}, the explainer {bg.columns}')
    model, dev = bg.model, bg.model.device
    n_rows, n_cols, K, N_bg = len(X), len(bg.columns), bg.cols, bg.rows
    phi = np.zeros((n_rows, n_cols, K), np.float64)
    if n_rows == 0:
        return phi
    timer = Stages(stages)
    model.flush_optimizer_state()
    t0 = time.perf_counter()
    x_cat, x_cont = bg.encode(X)
    timer.host('encode', t0)
    F = x_cat.shape[1] if x_cat is not None else 0
    C = x_cont.shape[1] if x_cont is not None else 0
    emb = _Embeddings(model) if F else None
    kind = output_kind(model.task)
    bits = np.concatenate([bg.cat_bit.cpu().numpy(), bg.cont_bit.cpu().numpy()])     # frame column of each encoded one
    cols = F + C

    mine = rank_share(n_rows)
    group_rows = max(1, batch_size // nsamples)
    rng = np.random.RandomState()

    def tables():
        return (ptr(x_cat), ptr(x_cont), ptr(bg.cat), ptr(bg.cont), ptr(emb.table) if F else None,
                ptr(emb.row_offsets) if F else None, ptr(emb.col_offsets) if F else None, emb.dim if F else 0)

    for g0 in range(0, len(mine), group_rows):
        group = mine[g0:g0 + group_rows]
        t0 = time.perf_counter()
        draws = [gradient_draws(seed, i, nsamples, N_bg, rng) for i in group]
        timer.host('draws', t0)
        x_index = torch.as_tensor(np.repeat(np.array(group, np.int32), nsamples)).to(dev)
        bg_index = torch.as_tensor(np.concatenate([d[0] for d in draws])).to(dev)
        alpha = torch.as_tensor(np.concatenate([d[1] for d in draws])).to(dev)
        P = len(group) * nsamples
        values = torch.empty(K, P, cols, dtype=torch.float64, device=dev)
        for p0 in range(0, P, batch_size):
            m = min(batch_size, P - p0)
            with timer.device('compose'):
                out_emb = torch.empty((F, m, emb.dim) if not emb.ragged else (m, emb.width), dtype=torch.float32,
                                      device=dev) if F else None
                out_cont = torch.empty(m, C, dtype=torch.float32, device=dev) if C else None
                check(N.lib.dtb_gradshap_compose(*tables(), ptr(x_index[p0:]), ptr(bg_index[p0:]), ptr(alpha[p0:]),
                                                 m, F, C, 0 if F and emb.ragged else 1, ptr(out_emb), ptr(out_cont),
                                                 stream_ptr()), 'gradshap_compose')
            inputs = []
            if F:       # the tensor-backed field block reads [F, m, D] in place; its gradient comes back as (m, F, D)
                out_emb = (out_emb if emb.ragged else out_emb.permute(1, 0, 2)).detach().requires_grad_(True)
                inputs.append(out_emb)
            if C:
                out_cont = out_cont.requires_grad_(True)
                inputs.append(out_cont)
            with timer.device('forward'):
                z = model.input_forward(out_emb, out_cont)
            dz = torch.empty(m, K, dtype=torch.float32, device=dev)
            for k in range(K):
                with timer.device('backward'):
                    check(N.lib.dtb_gradshap_output_grad(ptr(z.detach()), m, K, k, kind, ptr(dz), stream_ptr()),
                          'gradshap_output_grad')
                    grads = torch.autograd.grad(z, inputs, grad_outputs=dz, retain_graph=k < K - 1,
                                                allow_unused=True)
                    grads = [torch.zeros_like(t) if g is None else g.contiguous() for t, g in zip(inputs, grads)]
                g_emb = grads[0] if F else None
                g_cont = grads[-1] if C else None
                with timer.device('reduce'):
                    check(N.lib.dtb_gradshap_reduce(*tables(), ptr(x_index[p0:]), ptr(bg_index[p0:]), m, F, C,
                                                    ptr(g_emb), ptr(g_cont), ptr(values[k, p0:]), stream_ptr()),
                          'gradshap_reduce')
            del z, inputs
        with timer.device('means'):
            means = torch.empty(K, len(group), cols, dtype=torch.float64, device=dev)
            for k in range(K):
                check(N.lib.dtb_gradshap_means(ptr(values[k]), len(group), nsamples, cols, ptr(means[k]),
                                               stream_ptr()), 'gradshap_means')
        host = means.cpu().numpy()
        rows = np.array(group)
        for e in range(cols):
            if bits[e] >= 0:
                phi[rows, bits[e], :] += host[:, :, e].T
    timer.finish()
    return gather_strided(phi[mine], n_rows)
