"""Learning-rate schedules and callbacks on the GPU: the rate-table kernels against float64 step by step and the row
form bit-identical to the dense sweep under a rate that rises and falls, the constant-rate bits unchanged, DeepModel
training against the oracle trainer, CUDA-graph replay, checkpoints, DeepTable.fit with ReduceLROnPlateau and data
parallel."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import lr_ref
import optim_ref as R
from deeptables_b200 import callbacks as C
from deeptables_b200 import optimizers as O
from deeptables_b200 import schedules as S

pytestmark = pytest.mark.gpu

VARIANTS = {
    'sgd': O.SGD(learning_rate=0.05),
    'sgd_momentum': O.SGD(learning_rate=0.05, momentum=0.9),
    'sgd_nesterov': O.SGD(learning_rate=0.05, momentum=0.9, nesterov=True),
    'rmsprop': O.RMSprop(learning_rate=0.01),
    'rmsprop_momentum': O.RMSprop(learning_rate=0.01, momentum=0.9),
    'rmsprop_centered': O.RMSprop(learning_rate=0.01, centered=True),
    'rmsprop_centered_momentum': O.RMSprop(learning_rate=0.01, momentum=0.9, centered=True),
    'adagrad': O.Adagrad(learning_rate=0.1),
    'adam': O.Adam(learning_rate=0.01),
}


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


def _hp(spec):
    from deeptables_b200.deepmodel import _native_optim_params
    return _native_optim_params(spec)


def _ptrs(ts):
    from deeptables_b200._native import ptr
    return [ptr(t) for t in ts]


def _rising_falling(lr0, steps):
    """float32 rates of steps 0..steps: a CosineDecay warmup from lr0 / 4 to 2 * lr0 over 40 steps and its decay, then
    from t = 3000 on a PiecewiseConstantDecay step up to 3 * lr0."""
    cos = S.resolve(S.CosineDecay(lr0 / 4, decay_steps=2000, alpha=0.1, warmup_target=2 * lr0, warmup_steps=40))
    up = S.resolve(S.PiecewiseConstantDecay([3000], [lr0, 3 * lr0]))
    t = np.arange(-1, steps)
    r = np.where(t < 3000, S.rates(cos, np.maximum(t, 0)), S.rates(up, np.maximum(t, 0)))
    r[0] = 0.0
    return r.astype(np.float32)


def _device_table(spec, rates32):
    """What the kernels read: the rate, or Adam's alpha with the rate folded in."""
    vals = lr_ref.adam_alphas(rates32, spec.beta_1, spec.beta_2) if spec.kind == 'adam' else rates32
    return vals, torch.tensor(vals, device='cuda')


def _at(spec, rate):
    return spec._replace(learning_rate=float(rate), schedule=None)


# ---- 1. kernels: dense sweep vs float64, row form vs dense sweep -----------------------------------------------------------
@pytest.mark.parametrize('name', list(VARIANTS))
@pytest.mark.parametrize('n,off', [(1003, 0), (4099, 1)])
def test_table_dense_sweep_matches_oracle(nat, name, n, off):
    spec = O.resolve(VARIANTS[name])
    gen = np.random.default_rng(n + off)
    rates = _rising_falling(spec.learning_rate, 60)
    host, table = _device_table(spec, rates)

    def buf(vals):
        t = torch.zeros(n + 4, dtype=torch.float32, device='cuda')[off:off + n]
        return t.copy_(torch.as_tensor(np.asarray(vals, dtype=np.float32)))

    p0 = gen.normal(size=n).astype(np.float32)
    arms = []
    for _ in range(2):                                   # host step, device step
        slots = [buf(np.zeros(n)), buf(np.zeros(n))] if spec.kind == 'adam' else \
            [None if s is None else buf(np.full(n, s)) for s in O.slot_inits(spec)]
        arms.append((buf(p0), buf(np.zeros(n)), slots))
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    pr = torch.tensor(p0, dtype=torch.float64)
    sr = R.new_slots(spec, pr)
    for t in range(1, 61):
        gg = gen.normal(size=n).astype(np.float32)
        gg[gen.random(n) < 0.2] = 0.0
        step_dev.fill_(t - 1)
        for k, (p, g, slots) in enumerate(arms):
            g.copy_(torch.as_tensor(gg))
            if spec.kind == 'adam':
                if k == 0:
                    nat.check(nat.lib.dtb_adam_dense(*_ptrs([p] + slots + [g]), n, float(host[t]), spec.beta_1,
                                                     spec.beta_2, spec.epsilon, 1, None))
                else:
                    nat.check(nat.lib.dtb_adam_dense_dev(*_ptrs([p] + slots + [g]), n, nat.ptr(table),
                                                         nat.ptr(step_dev), spec.beta_1, spec.beta_2, spec.epsilon, 1,
                                                         None))
            else:
                src = (t, None) if k == 0 else (0, nat.ptr(step_dev))
                nat.check(nat.lib.dtb_optim_dense_lr(*_ptrs([p, g] + slots), n, _hp(spec), nat.ptr(table), *src, 1,
                                                     None))
        R.step(_at(spec, rates[t]), pr, torch.tensor(gg, dtype=torch.float64), sr, t)
        if t in (1, 20, 41, 60):
            torch.cuda.synchronize()
            # fp32 against float64: ~1e-6 relative per step, far below one step at these rates
            np.testing.assert_allclose(arms[0][0].cpu().numpy(), pr.numpy(), rtol=1e-5, atol=1e-5,
                                       err_msg=f'{name}: p at step {t}')
    for k in range(len(arms[0][2])):
        if arms[0][2][k] is not None:
            assert torch.equal(arms[0][2][k], arms[1][2][k]), f'{name}: slot {k}, host vs device step'
    assert torch.equal(arms[0][0], arms[1][0]), f'{name}: host vs device step'


GAP_STEPS = 5060


def _rows_schedule(s):
    """as test_optimizers_gpu: rows touched every step, after gaps of 50 and 5 000 steps, duplicates, out-of-range
    ids and rows never touched (fields of 40 and 30 rows)"""
    return np.array([[0, s % 30],
                     [0, -1],
                     [5 if s in (1, 51, 5051) else 40, s % 2],
                     [7 if s in (2, GAP_STEPS) else 0, 29 - s % 30]], dtype=np.int32)


@pytest.mark.parametrize('name', list(VARIANTS))
def test_table_row_form_is_bit_identical_to_dense_sweep(nat, name):
    spec = O.resolve(VARIANTS[name])
    adam = spec.kind == 'adam'
    vocab, d = [40, 30], 8
    rows = sum(vocab)
    offs = torch.tensor([0, 40, 70], dtype=torch.int64, device='cuda')
    gen = np.random.default_rng(7)
    w0 = torch.tensor(gen.normal(scale=0.05, size=(rows, d)).astype(np.float32), device='cuda')
    w0[3] = 0.0
    inits = (0.0, 0.0, None) if adam else O.slot_inits(spec)
    host, table = _device_table(spec, _rising_falling(spec.learning_rate, GAP_STEPS + 1))
    hp = None if adam else _hp(spec)
    b1b2e = (spec.beta_1, spec.beta_2, spec.epsilon) if adam else ()

    def state():
        return w0.clone(), [None if s is None else torch.full((rows, d), s, device='cuda') for s in inits], \
            torch.zeros(rows, d, device='cuda')

    (wd, sd, gd), (wh, sh, gh), (wv, sv, gv) = state(), state(), state()
    if adam:
        sd, sh, sv = sd[:2], sh[:2], sv[:2]
    last_h = torch.zeros(rows, dtype=torch.int32, device='cuda')
    last_v = torch.zeros(rows, dtype=torch.int32, device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    lo = [0, 40]
    T = nat.ptr(table)
    for s in range(1, GAP_STEPS + 1):
        ids = _rows_schedule(s)
        gtab = np.zeros((rows, d), dtype=np.float32)
        for b in range(ids.shape[0]):
            for f in range(2):
                if 0 <= ids[b, f] < vocab[f]:
                    gtab[lo[f] + ids[b, f]] += gen.normal(size=d).astype(np.float32)
        gt = torch.as_tensor(gtab).cuda()
        gd.copy_(gt), gh.copy_(gt), gv.copy_(gt)
        idx = torch.as_tensor(ids).cuda()
        step_dev.fill_(s - 1)
        if adam:
            nat.check(nat.lib.dtb_adam_dense(*_ptrs([wd] + sd + [gd]), rows * d, float(host[s]), *b1b2e, 1, None))
            nat.check(nat.lib.dtb_adam_rows_catchup(*_ptrs([idx, offs, wh] + sh + [last_h]), T, s - 1, *b1b2e, 4, 2, d,
                                                    None))
            nat.check(nat.lib.dtb_adam_rows_apply(*_ptrs([idx, offs, wh] + sh + [gh, last_h]), T, s, *b1b2e, 4, 2, d,
                                                  None))
            nat.check(nat.lib.dtb_adam_rows_catchup_dev(*_ptrs([idx, offs, wv] + sv + [last_v]), T, nat.ptr(step_dev),
                                                        *b1b2e, 4, 2, d, None))
            nat.check(nat.lib.dtb_adam_rows_apply_dev(*_ptrs([idx, offs, wv] + sv + [gv, last_v]), T,
                                                      nat.ptr(step_dev), *b1b2e, 4, 2, d, None))
        else:
            nat.check(nat.lib.dtb_optim_dense_lr(*_ptrs([wd, gd] + sd), rows * d, hp, T, s, None, 1, None))
            nat.check(nat.lib.dtb_optim_rows_catchup(*_ptrs([idx, offs, wh] + sh + [last_h]), s - 1, hp, 4, 2, d, None))
            nat.check(nat.lib.dtb_optim_rows_apply_lr(*_ptrs([idx, offs, wh] + sh + [gh, last_h]), T, s, None, hp, 4, 2,
                                                      d, None))
            nat.check(nat.lib.dtb_optim_rows_catchup_dev(*_ptrs([idx, offs, wv] + sv + [last_v, step_dev]), hp, 4, 2, d,
                                                         None))
            nat.check(nat.lib.dtb_optim_rows_apply_lr(*_ptrs([idx, offs, wv] + sv + [gv, last_v]), T, 0,
                                                      nat.ptr(step_dev), hp, 4, 2, d, None))
        if s in (2, 52, 3001, 5051, GAP_STEPS):
            for b, f in np.ndindex(*ids.shape):
                if 0 <= ids[b, f] < vocab[f]:
                    r = lo[f] + int(ids[b, f])
                    assert torch.equal(wh[r], wd[r]) and torch.equal(wv[r], wd[r]), f'{name}: row {r} at step {s}'
    if adam:
        nat.check(nat.lib.dtb_adam_rows_flush(*_ptrs([wh] + sh + [last_h]), T, GAP_STEPS, *b1b2e, rows, d, None))
        nat.check(nat.lib.dtb_adam_rows_flush(*_ptrs([wv] + sv + [last_v]), T, GAP_STEPS, *b1b2e, rows, d, None))
    else:
        nat.check(nat.lib.dtb_optim_rows_flush(*_ptrs([wh] + sh + [last_h]), GAP_STEPS, hp, rows, d, None))
        step_dev.fill_(GAP_STEPS)
        nat.check(nat.lib.dtb_optim_rows_flush_dev(*_ptrs([wv] + sv + [last_v, step_dev]), hp, rows, d, None))
    torch.cuda.synchronize()
    assert not torch.equal(wd, w0)
    for label, w, sl in (('host', wh, sh), ('dev', wv, sv)):
        assert torch.equal(w, wd), f'{name}: {label} row form weights differ from the dense sweep'
        for k, (a, b) in enumerate(zip(sl, sd)):
            if a is not None:
                assert torch.equal(a, b), f'{name}: {label} row form slot {k} differs from the dense sweep'


# ---- 2. a constant table gives the constant-rate symbols' bits -------------------------------------------------------------
@pytest.mark.parametrize('name', [k for k in VARIANTS if k != 'adam'])
def test_constant_table_matches_constant_rate_symbols(nat, name):
    spec = O.resolve(VARIANTS[name])
    hp = _hp(spec)
    n, rows, d = 4099, 70, 8
    gen = np.random.default_rng(3)
    table = torch.full((40,), float(np.float32(spec.learning_rate)), device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    offs = torch.tensor([0, 40, 70], dtype=torch.int64, device='cuda')

    def arm(size):
        p = torch.tensor(gen.normal(size=size).astype(np.float32), device='cuda')
        return [p.clone() for _ in range(3)], [[None if s is None else torch.full(p.shape, s, device='cuda')
                                                for s in O.slot_inits(spec)] for _ in range(3)]

    (dp_, ds), (rp, rs), (gp, gs) = arm(n), arm((rows, d)), arm(n)
    last = [torch.zeros(rows, dtype=torch.int32, device='cuda') for _ in range(3)]
    acc = [torch.zeros(1, dtype=torch.float64, device='cuda') for _ in range(3)]
    for t in range(1, 12):
        step_dev.fill_(t - 1)
        g = torch.tensor(gen.normal(size=n).astype(np.float32), device='cuda')
        gr = torch.tensor(gen.normal(size=(rows, d)).astype(np.float32), device='cuda')
        ids = torch.tensor(gen.integers(0, 30, size=(5, 2)), dtype=torch.int32, device='cuda')
        lr = [(None, 0, None), (nat.ptr(table), t, None), (nat.ptr(table), 0, nat.ptr(step_dev))]
        for k in range(3):
            gk, gkr, gkg = g.clone(), gr.clone(), g.clone()
            if k == 0:
                nat.check(nat.lib.dtb_optim_dense(*_ptrs([dp_[k], gk] + ds[k]), n, hp, 1, None))
                nat.check(nat.lib.dtb_optim_rows_apply(*_ptrs([ids, offs, rp[k]] + rs[k] + [gkr, last[k]]), t, hp, 5, 2,
                                                       d, None))
                nat.check(nat.lib.dtb_optim_dense_reg(*_ptrs([gp[k], gkg] + gs[k]), n, hp, 1, 1e-3, 1e-2,
                                                      nat.ptr(acc[k]), 1.0, None))
            else:
                nat.check(nat.lib.dtb_optim_dense_lr(*_ptrs([dp_[k], gk] + ds[k]), n, hp, *lr[k], 1, None))
                nat.check(nat.lib.dtb_optim_rows_apply_lr(*_ptrs([ids, offs, rp[k]] + rs[k] + [gkr, last[k]]), *lr[k],
                                                          hp, 5, 2, d, None))
                nat.check(nat.lib.dtb_optim_dense_reg_lr(*_ptrs([gp[k], gkg] + gs[k]), n, hp, *lr[k], 1, 1e-3, 1e-2,
                                                         nat.ptr(acc[k]), 1.0, None))
    torch.cuda.synchronize()
    for k in (1, 2):
        for what, a, b, sa, sb in (('dense', dp_[k], dp_[0], ds[k], ds[0]), ('rows', rp[k], rp[0], rs[k], rs[0]),
                                   ('reg', gp[k], gp[0], gs[k], gs[0])):
            assert torch.equal(a, b), f'{name}: {what} form {k}'
            for x, y in zip(sa, sb):
                assert x is None or torch.equal(x, y), f'{name}: {what} form {k} slot'
        # the float64 loss term is summed with atomics in block order: equal to rounding, not to the bit
        assert abs(float(acc[k].item()) - float(acc[0].item())) <= 1e-12 * float(acc[0].item())


def test_table_forms_refuse_a_missing_table(nat):
    p = torch.zeros(8, device='cuda')
    hp = _hp(O.resolve('sgd'))
    assert nat.lib.dtb_optim_dense_lr(*_ptrs([p, p, None, None, None]), 8, hp, None, 1, None, 1, None) != 0
    assert nat.lib.dtb_optim_dense_lr(*_ptrs([p, p, None, None, None]), 8, hp, nat.ptr(p), 0, None, 1, None) != 0
    assert 'lr_table' in nat.last_error()


# ---- model-level helpers -----------------------------------------------------------------------------------------------------
def build(nets, vocab, dim, n_cont, seed=5, **cfg_kw):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    kw = dict(nets=nets, embeddings_output_dim=dim, embedding_dropout=0, metrics=['AUC'],
              dnn_params={'hidden_units': ((16, 0, False), (8, 0, True)), 'activation': 'relu'},
              cin_params={'cross_layer_size': (8, 6), 'activation': 'relu', 'use_residual': False,
                          'use_bias': False, 'direct': False, 'reduce_D': False})
    kw.update(cfg_kw)
    conf = deeptable.ModelConfig(**kw)
    cats = [CategoricalColumn(f'c{i}', v, dim) for i, v in enumerate(vocab)]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(n_cont)])] if n_cont else []
    model = DeepModel('binary', 2, conf, cats, conts, seed=seed)
    model._build_model()
    return model, conf


def batch(vocab, n_cont, b, seed=0):
    g = np.random.default_rng(seed)
    idx = np.stack([g.integers(0, v, size=b) for v in vocab], axis=1).astype(np.int32)
    cont = g.normal(size=(b, n_cont)).astype(np.float32)
    y = (g.random(b) < 0.35).astype(np.float32)
    return idx, cont, y


MODEL_OPTS = {
    'adam_exponential': O.Adam(learning_rate=S.ExponentialDecay(0.01, decay_steps=3, decay_rate=0.5)),
    'adam_cosine_warmup': O.Adam(learning_rate=S.CosineDecay(1e-3, 6, warmup_target=0.02, warmup_steps=3)),
    'sgd_piecewise': O.SGD(learning_rate=S.PiecewiseConstantDecay([2, 5], [0.05, 0.2, 0.02]), momentum=0.9),
    'rmsprop_polynomial': O.RMSprop(learning_rate=S.PolynomialDecay(0.01, 5, end_learning_rate=1e-3, cycle=True)),
    'adagrad_inverse': O.Adagrad(learning_rate=S.InverseTimeDecay(0.1, 2, 1.0, staircase=True)),
    'rmsprop_restarts': O.RMSprop(learning_rate=S.CosineDecayRestarts(0.01, 3, t_mul=2.0, m_mul=0.5)),
}


# ---- 3. DeepModel vs the oracle trainer at the per-step rate -----------------------------------------------------------------
@pytest.mark.parametrize('nets', [['linear', 'fm_nets', 'dnn_nets'], ['linear', 'cin_nets', 'dnn_nets']])
@pytest.mark.parametrize('name', list(MODEL_OPTS))
def test_training_follows_the_schedule(nets, name):
    vocab, dim, n_cont, b = [11, 7, 13, 5, 9], 4, 3, 48
    model, conf = build(nets, vocab, dim, n_cont, optimizer=MODEL_OPTS[name])
    spec = O.resolve(MODEL_OPTS[name])
    sname, sconf = S.to_config(spec.schedule)
    state = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    ref = R.OptimRefTrainer(state, conf, len(vocab), optimizer=spec)
    losses_g, losses_r = [], []
    for step in range(8):
        rate = float(np.float32(lr_ref.rate(sname, sconf, step)))
        assert model.optimizer.learning_rate == rate and model.optimizer.iterations == step
        ref.opt = _at(spec, rate)
        idx, cont, y = batch(vocab, n_cont, b, seed=step)
        losses_g.append(model.train_on_batch(idx, cont, y))
        losses_r.append(ref.train_step(torch.tensor(idx), torch.tensor(cont), torch.tensor(y)))
    np.testing.assert_allclose(losses_g, losses_r, rtol=2e-3, atol=1e-5)
    tol = dict(rtol=1e-3, atol=2e-5) if spec.kind in ('sgd', 'adagrad') else dict(rtol=1e-2, atol=5e-4)
    new_state = model.state_dict()
    for k, v in ref.state.items():
        np.testing.assert_allclose(new_state[k].cpu().numpy(), v.numpy(), err_msg=k, **tol)


# ---- 4. CUDA-graph replay vs eager, with a rate set after the capture ---------------------------------------------------------
SMALL = dict(nets=['linear', 'fm_nets', 'dnn_nets'], vocab=[400, 300, 500], dim=4, n_cont=2, b=2)


def _distinct_batch(vocab, n_cont, b, seed):
    g = np.random.default_rng(seed)
    idx = np.stack([g.choice(v, size=b, replace=False) for v in vocab], axis=1).astype(np.int32)
    cont = g.normal(size=(b, n_cont)).astype(np.float32)
    y = (g.random(b) < 0.35).astype(np.float32)
    return idx, cont, y


def _train(optimizer, steps, model=None, seed=9, set_at=None):
    """`steps` steps of two rows; set_at = {step: rate} sets model.optimizer.learning_rate before that step, as an
    epoch-begin callback does."""
    s = SMALL
    if model is None:
        model, _ = build(s['nets'], s['vocab'], s['dim'], s['n_cont'], seed=seed, optimizer=optimizer)
    for step in range(model._step, model._step + steps):
        if set_at and step in set_at:
            model.optimizer.learning_rate = set_at[step]
        model.train_on_batch(*_distinct_batch(s['vocab'], s['n_cont'], s['b'], seed=step))
    return model


def _states_equal(a, b, what):
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f'{what}: {k} differs'


GRAPH_CASES = {
    'adam_exponential': (MODEL_OPTS['adam_exponential'], None),
    'rmsprop_restarts': (MODEL_OPTS['rmsprop_restarts'], None),
    'sgd_piecewise': (MODEL_OPTS['sgd_piecewise'], None),
    'adam_set': ('auto', {4: 0.01, 7: 0.0005}),
    'rmsprop_set': (O.RMSprop(momentum=0.9, centered=True), {4: 0.01, 7: 0.0005}),
    'adagrad_set': ('adagrad', {5: 0.05}),
}


@pytest.mark.parametrize('name', list(GRAPH_CASES))
def test_cuda_graph_replay_is_bit_identical_to_eager(monkeypatch, name):
    opt, set_at = GRAPH_CASES[name]
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    eager = _train(opt, 10, set_at=set_at)
    assert not eager._graphs
    monkeypatch.setenv('DTB_CUDA_GRAPH', '1')
    graphed = _train(opt, 10, set_at=set_at)
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    _states_equal(graphed, eager, f'{name}: graph replay vs eager')
    if set_at:
        last = max(set_at)
        assert graphed.optimizer.learning_rate == float(np.float32(set_at[last]))
        plain = _train(opt, 10)
        assert not torch.equal(plain.state_dict()[next(iter(plain.state_dict()))],
                               graphed.state_dict()[next(iter(plain.state_dict()))]), 'the set rate was not used'


def test_learning_rate_scheduler_after_capture_matches_eager(monkeypatch):
    """DeepModel.fit with LearningRateScheduler, which sets the rate at every epoch begin: the train step is captured
    in epoch 0 and replayed at the rates of epochs 1 and 2.  Two-row batches without repeated ids (see _train)."""
    s = SMALL
    parts = [_distinct_batch(s['vocab'], s['n_cont'], 2, seed) for seed in range(10)]
    idx, cont, y = (np.concatenate([p[k] for p in parts]) for k in range(3))
    X = pd.DataFrame({**{f'c{i}': idx[:, i] for i in range(len(s['vocab']))},
                      **{f'n{i}': cont[:, i] for i in range(s['n_cont'])}})
    runs = {}
    for graphs in ('0', '1'):
        monkeypatch.setenv('DTB_CUDA_GRAPH', graphs)
        model, _ = build(s['nets'], s['vocab'], s['dim'], s['n_cont'], seed=9, optimizer=O.RMSprop(momentum=0.9))
        cb = C.LearningRateScheduler(lambda epoch, lr: 0.004 / (epoch + 1))
        history = model.fit(X, y, batch_size=2, epochs=3, verbose=0, callbacks=[cb], shuffle=False,
                            validation_data=(X.head(4), y[:4]))
        runs[graphs] = (model, history.history)
    (eager, he), (graphed, hg) = runs['0'], runs['1']
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    assert graphed._step == 30
    _states_equal(graphed, eager, 'LearningRateScheduler: graph replay vs eager')
    assert he['loss'] == hg['loss']
    want = [float(np.float32(v)) for v in (0.004, 0.002, 0.004 / 3)]
    assert hg['learning_rate'] == want
    assert graphed._rates.host[[1, 10, 11, 20, 21, 30]].tolist() == [want[0], want[0], want[1], want[1], want[2],
                                                                      want[2]]


# ---- 5. checkpoints ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('opt,set_at', [(MODEL_OPTS['adam_cosine_warmup'], None), (MODEL_OPTS['sgd_piecewise'], None),
                                        ('auto', {2: 0.0005}), (O.RMSprop(momentum=0.9), {1: 0.0001})],
                         ids=['adam_schedule', 'sgd_schedule', 'adam_reduced', 'rmsprop_reduced'])
def test_checkpoint_resume_is_bit_identical(monkeypatch, tmp_path, opt, set_at):
    from deeptables_b200.deepmodel import DeepModel
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    straight = _train(opt, 6, set_at=set_at)
    first = _train(opt, 3, set_at=set_at)
    path = str(tmp_path / 'ck.npz')
    first.save(path)
    resumed = DeepModel('binary', 2, first.config, first.categorical_columns, first.continuous_columns,
                        model_file=path, seed=123)
    assert resumed._step == 3
    assert resumed.optimizer.learning_rate == first.optimizer.learning_rate
    _train(opt, 3, model=resumed)
    _states_equal(resumed, straight, 'save after 3 steps, load, 3 more')


# ---- 6. public surface ---------------------------------------------------------------------------------------------------------
def _frame(n):
    g = np.random.default_rng(0)
    df = pd.DataFrame({
        'job': g.choice(list('abcdefghijkl'), size=n), 'marital': g.choice(['m', 's', 'd'], size=n),
        'housing': g.choice(['yes', 'no'], size=n), 'age': g.integers(18, 90, size=n).astype(float),
        'duration': g.exponential(200, size=n),
    })
    logit = (df['housing'] == 'yes') * 1.5 + (df['duration'] - 200) / 150 + (df['job'] == 'a') * 2 - 1
    y = np.where(g.random(n) < 1 / (1 + np.exp(-logit)), 'yes', 'no')
    return df, y


def test_deeptable_fit_with_reduce_lr_on_plateau():
    from deeptables_b200 import deeptable, deepnets
    df, y = _frame(2000)
    conf = deeptable.ModelConfig(nets=deepnets.DeepFM, embedding_dropout=0, metrics=['AUC'],
                                 earlystopping_patience=100, optimizer=O.Adam(learning_rate=0.004))
    dt = deeptable.DeepTable(config=conf)
    # min_delta larger than any change of the loss: every epoch after the first counts as a plateau
    cb = C.ReduceLROnPlateau(monitor='loss', patience=1, factor=0.5, min_delta=10.0)
    m, history = dt.fit(df, y, batch_size=128, epochs=4, verbose=0, callbacks=[cb])
    lrs = history.history['learning_rate']
    want = [float(np.float32(0.004)), float(np.float32(0.004)), float(np.float32(0.002)), float(np.float32(0.001))]
    assert lrs == want
    assert m.optimizer.learning_rate == float(np.float32(0.0005))
    per_epoch = m._step // 4
    # the steps of the last epoch used the rate set after the third: Adam's alpha over its bias correction
    o = m._opt
    s = m._step
    alpha = float(np.float32(np.float32(0.001) * np.sqrt(1 - o.beta_2 ** s) / (1 - o.beta_1 ** s)))
    assert abs(float(m._rates.host[s]) - alpha) <= 1e-7 * alpha and per_epoch > 0
    assert float(m._rates.host[s + 1]) < alpha


# ---- 7. data parallel ----------------------------------------------------------------------------------------------------------
DP_VOCAB, DP_DIM, DP_CONT, DP_B = [50, 40, 30, 20, 60], 8, 3, 64


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out_dir, case):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        opt = MODEL_OPTS['rmsprop_restarts'] if case == 'schedule' else O.SGD(learning_rate=0.05, momentum=0.9)
        m, _ = build(['linear', 'fm_nets', 'dnn_nets'], DP_VOCAB, DP_DIM, DP_CONT, seed=11, optimizer=opt)
        cb = C.ReduceLROnPlateau(monitor='loss', patience=1, factor=0.5, min_delta=0.0)
        cb.set_model(m)
        cb.on_train_begin()
        for epoch in range(4):
            m._loss_acc.zero_()
            for step in range(3):
                m.train_on_batch(*batch(DP_VOCAB, DP_CONT, DP_B, seed=(epoch * 3 + step) * world + rank))
            if case == 'plateau':
                # the per-rank training loss: the ranks see different values and may decide differently
                cb.on_epoch_end(epoch, {'loss': float(m._loss_acc.item()) + (0.0 if rank == 0 else -epoch)})
                m._agree_learning_rate()
        m.sync_replica_buffers()
        sd = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), **sd)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('case', ['schedule', 'plateau'])
def test_data_parallel_replicas_stay_bit_identical(tmp_path, case):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path), case), nprocs=world, join=True)
    r0 = np.load(tmp_path / 'rank0.npz')
    r1 = np.load(tmp_path / 'rank1.npz')
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]), f'replica 1 diverged from replica 0 on {k}'
