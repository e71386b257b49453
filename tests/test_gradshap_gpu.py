"""Expected gradients on the GPU: the kernels against the numpy restatement bit for bit, the input gradients of every
net against float64 autograd of the oracle model, the closed form of a linear model, completeness, multi-output
layouts, determinism across batch sizes and ranks, and the model left exactly as it was.

Input gradients: tests/test_model_grads_gpu.py's cases (every net and preset, at toy shapes and at the shapes that
pick the production kernels), with each batch's embedding rows moved off the table by a small random step so that no
two rows are copies.  Bar: max |g - g64| <= RTOL * max |g64| over the block and over the continuous inputs.  An fp32
forward may take a relu or max decision the other way where the float64 input lies within rounding of the threshold;
the gradient of an input belongs to its own row only, so such a decision moves that row alone.  Cases the train-step
test marks as having such decisions (``widen``) may have up to WIDEN_ROWS of their rows over the bar; every other row,
and every row of the other cases, meets it."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import gradshap_ref
from oracle import model_ref as M
from test_model_grads_gpu import ALL, RTOL, build, make_batch, snapshot, state64

pytestmark = pytest.mark.gpu

WIDEN_ROWS = 0.05
ROWS, TEST_ROWS = 3000, 300


def _c(t):
    from deeptables_b200._native import ptr
    return ptr(t)


# ---------------------------------------------------------------------------------------------------------------------
# the kernels, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dims', [[8, 8, 8, 8, 8], [4, 16, 8, 3, 12]], ids=['uniform', 'ragged'])
@pytest.mark.parametrize('conts', [0, 5])
def test_kernels_equal_the_restatement(dims, conts):
    from deeptables_b200 import _native as N
    from deeptables_b200._native import check, stream_ptr
    g = np.random.default_rng(len(dims) + conts + dims[1])
    vocab = [7, 30, 5, 11, 2]
    F, dmax = len(vocab), max(dims)
    offs = np.concatenate([[0], np.cumsum(vocab)]).astype(np.int64)
    table = g.normal(size=(offs[-1], dmax)).astype(np.float32)
    for f, d in enumerate(dims):
        table[offs[f]:offs[f + 1], d:] = 0
    nx, nb, P = 40, 9, 70_001
    x_cat = np.stack([g.integers(0, v, nx) for v in vocab], 1).astype(np.int32)
    bg_cat = np.stack([g.integers(0, v, nb) for v in vocab], 1).astype(np.int32)
    bg_cat[3] = x_cat[0]                                   # equal ids: zero differences
    x_cat[5, 2] = 77                                       # out of range: zeros
    x_cont = g.normal(size=(nx, conts)).astype(np.float32) if conts else None
    bg_cont = g.normal(size=(nb, conts)).astype(np.float32) if conts else None
    if conts:
        bg_cont[3, :2] = x_cont[0, :2]
    xi = g.integers(0, nx, P).astype(np.int32)
    bi = g.integers(0, nb, P).astype(np.int32)
    xi[:50], bi[:50] = 0, 3
    alpha = (np.floor(g.random(P) * 2 ** 24) / 2 ** 24).astype(np.float32)
    ragged = len(set(dims)) > 1
    col = np.concatenate([[0], np.cumsum(dims)]).astype(np.int32)
    dev = lambda a: None if a is None else torch.as_tensor(a).cuda()
    t = {k: dev(v) for k, v in dict(x_cat=x_cat, x_cont=x_cont, bg_cat=bg_cat, bg_cont=bg_cont, table=table,
                                     offs=offs, col=col, xi=xi, bi=bi, alpha=alpha).items()}
    common = (_c(t['x_cat']), _c(t['x_cont']), _c(t['bg_cat']), _c(t['bg_cont']), _c(t['table']), _c(t['offs']),
              _c(t['col']), dmax)
    out_emb = torch.full((P, int(col[-1])) if ragged else (F, P, dmax), 7.0, device='cuda')
    out_cont = torch.empty(P, conts, device='cuda') if conts else None
    check(N.lib.dtb_gradshap_compose(*common, _c(t['xi']), _c(t['bi']), _c(t['alpha']), P, F, conts,
                                     0 if ragged else 1, _c(out_emb), _c(out_cont), stream_ptr()))
    want_emb, want_cont = gradshap_ref.compose(x_cat, x_cont, bg_cat, bg_cont, table, offs, dims, xi, bi, alpha)
    got = out_emb.cpu().numpy()
    if ragged:
        flat = np.concatenate([want_emb[:, f, :d] for f, d in enumerate(dims)], axis=1)
        assert got.tobytes() == flat.tobytes()
    else:
        assert got.tobytes() == np.ascontiguousarray(want_emb.transpose(1, 0, 2)).tobytes()
    if conts:
        assert out_cont.cpu().numpy().tobytes() == want_cont.tobytes()

    g_emb = g.normal(size=(P, F, dmax)).astype(np.float32)
    for f, d in enumerate(dims):
        g_emb[:, f, d:] = 0
    g_flat = np.concatenate([g_emb[:, f, :d] for f, d in enumerate(dims)], axis=1)
    g_cont = g.normal(size=(P, conts)).astype(np.float32) if conts else None
    vals = torch.empty(P, F + conts, dtype=torch.float64, device='cuda')
    g_flat_d, g_cont_d = dev(g_flat), dev(g_cont)          # held: a freed temporary's memory is handed out again
    check(N.lib.dtb_gradshap_reduce(*common, _c(t['xi']), _c(t['bi']), P, F, conts, _c(g_flat_d), _c(g_cont_d),
                                    _c(vals), stream_ptr()))
    want = gradshap_ref.reduce(x_cat, x_cont, bg_cat, bg_cont, table, offs, dims, xi, bi, g_emb, g_cont)
    assert vals.cpu().numpy().tobytes() == want.tobytes()
    assert np.all(want[:50, [0, 1, 3, 4]] == 0)

    rows, n = 7, 10_000
    out = torch.empty(rows, F + conts, dtype=torch.float64, device='cuda')
    check(N.lib.dtb_gradshap_means(_c(vals), rows, n, F + conts, _c(out), stream_ptr()))
    assert out.cpu().numpy().tobytes() == gradshap_ref.means(want[:rows * n], rows, n).tobytes()


@pytest.mark.parametrize('kind,cols', [(0, 1), (1, 1), (1, 3), (2, 4)])
def test_output_grad_matches_float64(kind, cols):
    from deeptables_b200 import _native as N
    from deeptables_b200._native import check, stream_ptr
    z = torch.randn(5000, cols, device='cuda') * 4
    z64 = z.double().requires_grad_(True)
    out = {0: lambda v: v, 1: torch.sigmoid, 2: lambda v: torch.softmax(v, -1)}[kind](z64)
    for k in range(cols):
        dz = torch.empty_like(z)
        check(N.lib.dtb_gradshap_output_grad(_c(z), 5000, cols, k, kind, _c(dz), stream_ptr()))
        (want,) = torch.autograd.grad(out[:, k].sum(), z64, retain_graph=True)
        torch.testing.assert_close(dz.double(), want, rtol=1e-5, atol=1e-6)      # float32 against float64


# ---------------------------------------------------------------------------------------------------------------------
# input gradients against float64
# ---------------------------------------------------------------------------------------------------------------------
def _gpu_input_grads(model, emb, cont, ragged):
    """Per output column: (block gradient [B, F, D] or [B, sum D], continuous gradient [B, C])."""
    from deeptables_b200 import _native as N, explain
    from deeptables_b200._native import check, stream_ptr
    inputs = []
    if emb is not None:
        x = emb if ragged else emb.permute(1, 0, 2).contiguous().permute(1, 0, 2)     # the field-major layout
        x = x.detach().requires_grad_(True)
        inputs.append(x)
    else:
        x = None
    c = cont.detach().requires_grad_(True) if cont is not None else None
    if c is not None:
        inputs.append(c)
    z = model.input_forward(x, c)
    K = z.shape[1]
    out = []
    for k in range(K):
        dz = torch.empty_like(z)
        check(N.lib.dtb_gradshap_output_grad(_c(z.detach()), z.shape[0], K, k, explain.output_kind(model.task),
                                             _c(dz), stream_ptr()))
        gs = torch.autograd.grad(z, inputs, dz, retain_graph=True, allow_unused=True)
        gs = [torch.zeros_like(i) if g is None else g for i, g in zip(inputs, gs)]
        out.append((gs[0] if x is not None else None, gs[-1] if c is not None else None))
    return out


def _ref_input_grads(snap, conf, c, emb64, cont64):
    st = state64(snap)
    F = len(c['vocab'])
    B = (emb64 if emb64 is not None else cont64).shape[0]
    leaves = []
    if F:
        cols = np.concatenate([[0], np.cumsum(c['dims'])])
        for f in range(F):
            leaf = emb64[:, f, :c['dims'][f]].clone().requires_grad_(True) if emb64.dim() == 3 else \
                emb64[:, cols[f]:cols[f + 1]].clone().requires_grad_(True)
            st[f'emb_categorical_vars_all/embeddings_{f}'] = leaf
            leaves.append(leaf)
    idx = torch.arange(B, device='cuda').unsqueeze(1).expand(B, F).contiguous() if F else None
    cont = cont64.clone().requires_grad_(True) if cont64 is not None else None
    out, _ = M.forward(st, conf, idx, cont, F, False, c['task'])
    res = []
    for k in range(out.shape[1]):
        targets = leaves + ([cont] if cont is not None else [])
        gs = torch.autograd.grad(out[:, k].sum(), targets, retain_graph=True, allow_unused=True)
        gs = [torch.zeros_like(t) if g is None else g for t, g in zip(targets, gs)]
        ge = torch.cat(gs[:F], dim=1) if F else None
        res.append((ge, gs[-1] if cont is not None else None))
    return res


@pytest.mark.parametrize('name', sorted(ALL))
def test_input_gradients_match_float64(name):
    c = ALL[name]
    model, conf = build(c, c['table_mode'])
    snap = snapshot(model)
    if c['tweak'] is not None:
        c['tweak'](snap)
        model.load_state_dict(snap)
        snap = snapshot(model)
    idx, cont, _, _ = make_batch(c, 0)
    g = np.random.default_rng(11)
    ragged = len(set(c['dims'])) > 1
    emb = emb_flat = None
    if c['vocab']:
        offs = model.table.row_offsets_host
        rows = model.table.weight[torch.as_tensor(np.array(offs[:-1]) + idx, dtype=torch.long).cuda()]   # [B, F, Dmax]
        rows = rows + 0.01 * torch.as_tensor(g.normal(size=rows.shape), dtype=torch.float32).cuda()
        for f, d in enumerate(c['dims']):
            rows[:, f, d:] = 0
        emb = rows
        emb_flat = torch.cat([rows[:, f, :d] for f, d in enumerate(c['dims'])], dim=1) if ragged else None
    cont_t = torch.as_tensor(cont).cuda() if cont is not None else None
    got = _gpu_input_grads(model, emb_flat if ragged else emb, cont_t, ragged)
    want = _ref_input_grads(snap, conf, c, (emb_flat if ragged else emb).double() if emb is not None else None,
                            cont_t.double() if cont_t is not None else None)
    assert len(got) == len(want) == model._output_dim()
    B = c['b']
    for (ge, gc), (we, wc) in zip(got, want):
        for g32, g64 in ((ge, we), (gc, wc)):
            if g64 is None:
                continue
            g32 = g32.reshape(B, -1).double()
            g64 = g64.reshape(B, -1)
            bar = RTOL * float(g64.abs().max())
            over = int(((g32 - g64).abs().max(dim=1).values > bar).sum())
            allowed = int(WIDEN_ROWS * B) if c['widen'] else 0
            assert over <= allowed, f'{name}: {over} rows over the bar {bar:.3g}, ' \
                                    f'max err {float((g32 - g64).abs().max()):.3g}'
        if we is not None:
            assert float(we.abs().max()) > 0          # (nets that do not read the continuous inputs give them 0)


# ---------------------------------------------------------------------------------------------------------------------
# the explainer end to end
# ---------------------------------------------------------------------------------------------------------------------
def _frame(rows, seed, n_cat=3, n_cont=3):
    """tests/test_shap_gpu.py's frame: plus a constant column auto_discard_unique drops and an excluded one."""
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'c{i}': g.choice(['a', 'b', 'c', 'd', 'e', 'f'][:3 + i % 4], rows) for i in range(n_cat)})
    for i in range(n_cont):
        X[f'n{i}'] = g.normal(size=rows)
    X['const'] = 'k'
    X['skip'] = g.normal(size=rows)
    lead = (X['c0'] == 'a').astype(float) * 2 + X['n0'] + 0.5 * X['n1'] * (X['c1'] == 'b')
    return X, lead + 0.3 * g.normal(size=rows)


_CACHE = {}


def _fitted(task, nets='DeepFM', **kw):
    key = (task, tuple(nets) if isinstance(nets, list) else nets, tuple(sorted(kw.items())))
    if key not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        X, lead = _frame(ROWS + TEST_ROWS, 5)
        nets = getattr(deepnets, nets) if isinstance(nets, str) else nets
        cin = {'cross_layer_size': (16, 16), 'activation': 'relu', 'use_residual': False, 'use_bias': False,
               'direct': False, 'reduce_D': False}
        if task == 'multilabel':         # tests/test_pdp_gpu.py's construction: DeepTable.fit takes no 2-D labels
            from deeptables_b200.deepmodel import DeepModel
            y = np.stack([lead > 0.8, X['n2'] > 0, X['c2'] == 'a'], 1).astype(np.float32)
            conf = deeptable.ModelConfig(nets=nets, task='multilabel', metrics=['binary_accuracy'],
                                         exclude_columns=['skip'], embeddings_output_dim=4, **kw)
            pre = deeptable.DefaultPreprocessor(conf)
            Xt, _ = pre.fit_transform(X.iloc[:ROWS], y[:ROWS])
            model = DeepModel('multilabel', 3, conf, pre.categorical_columns, pre.continuous_columns)
            model.fit(Xt, y[:ROWS], epochs=2, batch_size=128, verbose=0)
            dt = deeptable.DeepTable(conf, preprocessor=pre)
            dt._DeepTable__current_model = model
        else:
            if task == 'binary':
                y = pd.Series(np.where(lead > 0.8, 'yes', 'no'))
            elif task == 'multiclass':
                y = pd.Series(np.digitize(lead, [0.5, 1.5]).astype(str))
            else:
                y = pd.Series(3.0 * lead)
            conf = deeptable.ModelConfig(nets=nets, metrics=['mse' if task == 'regression' else 'AUC'],
                                         exclude_columns=['skip'], embeddings_output_dim=4, earlystopping_patience=1,
                                         cin_params=cin, **kw)
            dt = deeptable.DeepTable(config=conf)
            dt.fit(X.iloc[:ROWS], y.iloc[:ROWS], epochs=2, batch_size=128, verbose=0)
        _CACHE[key] = (dt, X.iloc[ROWS:].reset_index(drop=True))
    return _CACHE[key]


def _outputs(dt, frame):
    """The explained output of each row on the host: [rows, outputs] float64."""
    from deeptables_b200 import analysis, explain
    bg = explain.Background(dt, frame, 65536)
    pred = torch.empty(len(frame), bg.cols, dtype=torch.float32, device='cuda')
    analysis.forward_rows(bg.model, bg.cat, bg.cont, pred, 65536)
    return pred.cpu().numpy().astype(np.float64)


def test_linear_regression_has_the_closed_form():
    from deeptables_b200 import explain
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    dt, X = _fitted('regression', ['linear'])
    ex = DeepTablesGradientExplainer(dt, X.iloc[40:], num_samples=30, random_state=3)
    x = X.iloc[:12]
    phi = ex.get_shap_values(x, nsamples=64)
    assert phi.shape == (12, X.shape[1]) and phi.dtype == np.float64
    bg = ex._background
    model = bg.model
    sd = model.state_dict()
    w = sd['linear_logit/kernel'].double().cpu().numpy().reshape(-1) * float(sd['task_output/kernel'].reshape(-1)[0])
    x_cat, x_cont = bg.encode(x)
    table = model.table.weight.double().cpu().numpy()
    offs = model.table.row_offsets_host
    F = x_cat.shape[1]
    xc, bc = x_cat.cpu().numpy(), bg.cat.cpu().numpy()
    xn, bn = x_cont.cpu().numpy().astype(np.float64), bg.cont.cpu().numpy().astype(np.float64)
    bits = np.concatenate([bg.cat_bit.cpu().numpy(), bg.cont_bit.cpu().numpy()])
    for i in range(12):
        j, _ = explain.gradient_draws(3, i, 64, bg.rows)
        want = np.zeros(X.shape[1])
        for f in range(F):
            d = table[offs[f] + xc[i, f]].sum() - table[offs[f] + bc[j, f]].sum(axis=1)
            want[bits[f]] += w[f] * d.mean()
        for cc in range(xn.shape[1]):
            want[bits[F + cc]] += w[F + cc] * (xn[i, cc] - bn[j, cc]).mean()
        np.testing.assert_allclose(phi[i], want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
    # columns the model does not read get exactly 0
    for name in ('const', 'skip'):
        assert np.all(phi[:, X.columns.get_loc(name)] == 0)


@pytest.mark.parametrize('nets', ['DeepFM', 'xDeepFM'])
def test_completeness(nets):
    """One background row, 4096 samples: sum_c phi_c is f(x) - f(b) up to the Monte Carlo error of the path integral,
    bounded here by 2% of |f(x) - f(b)| plus 2e-3 (the sampling error of 4096 uniform points is about 1/64 of the
    spread of the path's gradient, which on these models stays within a few times |f(x) - f(b)|)."""
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    dt, X = _fitted('binary', nets)
    b = X.iloc[[100]]
    ex = DeepTablesGradientExplainer(dt, b, num_samples=None, random_state=11)
    x = X.iloc[:16]
    phi = ex.get_shap_values(x, nsamples=4096)
    f = _outputs(dt, x)[:, 0]
    fb = _outputs(dt, b)[0, 0]
    assert abs(ex.expected_value - fb) < 1e-12
    gap = phi.sum(axis=1) - (f - fb)
    assert np.all(np.abs(gap) <= 0.02 * np.abs(f - fb) + 2e-3), (gap, f - fb)


@pytest.mark.parametrize('task', ['multiclass', 'multilabel'])
def test_multi_output_layout(task):
    from deeptables_b200.utils import shap as S
    dt, X = _fitted(task, ['linear', 'fm_nets', 'dnn_nets'])
    ex = S.DeepTablesGradientExplainer(dt, X.iloc[50:], num_samples=20, random_state=1)
    phi = ex.get_shap_values(X.iloc[:9], nsamples=100)
    K = ex._background.cols
    assert K == 3 and phi.shape == (9, X.shape[1], K)
    assert ex.expected_value.shape == (K,) and ex.expected_value.dtype == np.float64
    np.testing.assert_array_equal(ex.expected_value, _outputs(dt, S._background_rows(X.iloc[50:], 20)).mean(0))
    if task == 'multiclass':
        np.testing.assert_allclose(phi.sum(axis=2), 0.0, atol=1e-6)      # the softmax outputs sum to 1
    assert np.any(phi != 0)


def test_identical_bits_for_any_batch_size_and_the_model_untouched():
    """Batch sizes 65536 and 37 (fewer rows than one explained row's 50 samples) give the same bits: every kernel on
    the DeepFM path computes a row from that row alone."""
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    dt, X = _fitted('binary', 'DeepFM')
    dm = dt.get_model()
    before = {k: v.detach().clone() for k, v in dm.state_dict().items()}
    step, seeds = dm._step, dm._scope._seed_counter
    grad = None if dm.table.grad is None else dm.table.grad.clone()
    a = DeepTablesGradientExplainer(dt, X.iloc[30:], num_samples=25, random_state=5).get_shap_values(X.iloc[:20], 50)
    b = DeepTablesGradientExplainer(dt, X.iloc[30:], num_samples=25, random_state=5,
                                    batch_size=37).get_shap_values(X.iloc[:20], 50)
    assert a.tobytes() == b.tobytes()
    after = dm.state_dict()
    for k, v in before.items():
        assert v.cpu().numpy().tobytes() == after[k].cpu().numpy().tobytes(), k
    assert dm._step == step and dm._scope._seed_counter == seeds
    if grad is not None:
        assert dm.table.grad.cpu().numpy().tobytes() == grad.cpu().numpy().tobytes()


def _train_state(dm):
    """Everything a train step reads besides its batch: parameters and buffers, their gradients and optimiser slots,
    the table's gradient, slots and row stamps, the step counter and the dropout seed counter."""
    t, sc = dm.table, dm._scope
    out = {f'sd/{k}': v for k, v in dm.state_dict().items()}
    for name in ('flat_p', 'flat_g', 'flat_m', 'flat_v'):
        if getattr(sc, name, None) is not None:
            out[name] = getattr(sc, name)
    for i, slot in enumerate(getattr(sc, 'flat_slots', None) or []):
        if slot is not None:
            out[f'flat_slot{i}'] = slot
    for name in ('weight', 'grad', 'm', 'v', 'last_step'):
        if getattr(t, name, None) is not None:
            out[f'table.{name}'] = getattr(t, name)
    out = {k: v.detach().cpu().numpy().tobytes() for k, v in out.items()}
    out['step'], out['seeds'] = dm._step, sc._seed_counter
    return out


@pytest.mark.parametrize('nets', ['DeepFM', 'xDeepFM'])
def test_the_state_a_train_step_reads_is_untouched(tmp_path, nets):
    """The train step of a loaded model is not bit-reproducible by itself (its scatter-adds are atomic), so instead of
    comparing a step taken after a call with one taken without it, everything the step reads is compared bit for bit,
    after a train step has created the gradient and optimiser state."""
    from deeptables_b200 import deeptable
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    dt, X = _fitted('binary', nets)
    dt.save(str(tmp_path / 'm'))
    d = deeptable.DeepTable.load(str(tmp_path / 'm'))
    m = d.get_model()
    Xf, lead = _frame(600, 9)
    y = pd.Series(np.where(lead > 0.8, 'yes', 'no'))
    cat, cont = m._to_device_inputs(d.preprocessor.transform_X(Xf.iloc[:256]))
    m.train_on_batch(cat.cpu().numpy(), cont.cpu().numpy(),
                     np.asarray(d.preprocessor.transform_y(y.iloc[:256]), np.float32))
    m.flush_optimizer_state()            # what the explainer does first: brings the lazily updated rows current
    before = _train_state(m)
    DeepTablesGradientExplainer(d, X.iloc[30:], num_samples=10, random_state=0).get_shap_values(X.iloc[:8], 20)
    after = _train_state(m)
    assert before.keys() == after.keys() and 'table.grad' in before and 'flat_g' in before
    assert [k for k in before if before[k] != after[k]] == []


def test_unread_columns_and_refusals():
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    dt, X = _fitted('binary', 'DeepFM')
    ex = DeepTablesGradientExplainer(dt, X.iloc[5:], num_samples=10, random_state=0)
    phi = ex.get_shap_values(X.iloc[:4].to_numpy(dtype=object), nsamples=8)       # an array of the columns works too
    assert np.all(phi[:, X.columns.get_loc('skip')] == 0) and np.all(phi[:, X.columns.get_loc('const')] == 0)
    with pytest.raises(ValueError, match='X_to_explain'):
        ex.get_shap_values(X.iloc[:1, ::-1])
    with pytest.raises(ValueError, match='nsamples'):
        ex.get_shap_values(X.iloc[:1], nsamples=0)


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, backend, model_dir, data, out_dir):
    import torch.distributed as dist
    from deeptables_b200 import deeptable
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    kw = {'device_id': torch.device('cuda', rank)} if backend == 'nccl' else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    try:
        dt = deeptable.DeepTable.load(model_dir)
        X, x = pd.read_pickle(data)
        np.random.seed(rank)                         # rank 0's seed is the one every rank uses
        phi = DeepTablesGradientExplainer(dt, X, num_samples=20).get_shap_values(x, nsamples=64)
        np.save(os.path.join(out_dir, f'phi{rank}.npy'), phi)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('backend', ['nccl', 'gloo'])
def test_data_parallel_ranks_return_the_single_process_array(tmp_path, backend):
    """World size 2; over gloo both ranks may share one GPU."""
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import torch.multiprocessing as mp
    from deeptables_b200.utils.shap import DeepTablesGradientExplainer
    dt, X = _fitted('regression')
    x = X.iloc[:11]
    dt.save(str(tmp_path / 'm'))
    pd.to_pickle((X, x), str(tmp_path / 'data.pkl'))
    np.random.seed(0)
    single = DeepTablesGradientExplainer(dt, X, num_samples=20).get_shap_values(x, nsamples=64)
    mp.spawn(_dp_worker, args=(2, _free_port(), backend, str(tmp_path / 'm'), str(tmp_path / 'data.pkl'),
                               str(tmp_path)), nprocs=2, join=True)
    for rank in range(2):
        assert np.array_equal(np.load(tmp_path / f'phi{rank}.npy'), single)
