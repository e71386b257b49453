"""Keras weight regularizers on the GPU: dtb_reg_grad against float64, the fused table sweeps bit-identical to
dtb_reg_grad followed by the plain sweep (and against the float64 optimiser oracle), DeepModel training against a
float64 reference trainer with the regularized loss, and the training-loop properties that go with it (the table never
goes lazy, ragged padding stays zero, CUDA-graph replay, checkpoints, validation loss, data parallel)."""
import os
import socket

import numpy as np
import pytest
import torch

import optim_ref as OR
import reg_ref
from deeptables_b200 import optimizers as O, regularizers as R
from deeptables_b200.engine import adam_alpha
from test_optimizers_gpu import VARIANTS, _distinct_batch, _hp, _ptrs, _states_equal, batch, build

pytestmark = pytest.mark.gpu

REGS = {'l1': R.L1(0.02), 'l2': R.L2(0.05), 'l1l2': R.L1L2(0.02, 0.05)}
SHAPES = [(1003, 0), (1003, 1), (1002, 2), (4099, 3), (4096, 0)]


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


def _buf(vals, off):
    vals = np.asarray(vals, dtype=np.float32)
    t = torch.zeros(vals.size + 4, dtype=torch.float32, device='cuda')[off:off + vals.size]
    return t.copy_(torch.as_tensor(vals))


def _weights(gen, n):
    w = gen.normal(size=n).astype(np.float32)
    w[gen.random(n) < 0.1] = 0.0                      # exact zeros: zero L1 gradient
    return w


# ---- 1. dtb_reg_grad against float64 --------------------------------------------------------------------------------
@pytest.mark.parametrize('reg', list(REGS))
@pytest.mark.parametrize('n,off', SHAPES)
def test_reg_grad_matches_float64(nat, reg, n, off):
    """n % 4 != 0 runs the scalar tail behind the float4 pass; buffers at +1/+2/+3 floats run the scalar kernel."""
    spec = R.resolve(REGS[reg])
    gen = np.random.default_rng(n + off)
    w0 = _weights(gen, n)
    g0 = gen.normal(size=n).astype(np.float32)
    p, g = _buf(w0, off), _buf(g0, off)
    acc = torch.full((1,), 0.5, dtype=torch.float64, device='cuda')
    nat.check(nat.lib.dtb_reg_grad(*_ptrs([p, g]), n, spec.l1, spec.l2, nat.ptr(acc), 3.0, None), 'reg_grad')
    loss_only = torch.zeros(1, dtype=torch.float64, device='cuda')
    nat.check(nat.lib.dtb_reg_grad(nat.ptr(p), None, n, spec.l1, spec.l2, nat.ptr(loss_only), 1.0, None), 'reg_grad')
    torch.cuda.synchronize()
    w = torch.tensor(w0, dtype=torch.float64)
    l1, l2 = float(np.float32(spec.l1)), float(np.float32(spec.l2))      # the kernels' fp32 factors
    want_g = torch.tensor(g0, dtype=torch.float64) + reg_ref.reg_grad(w, l1, l2)
    np.testing.assert_allclose(g.cpu().numpy(), want_g.numpy(), rtol=1e-6, atol=1e-7)
    assert torch.equal(p.cpu(), torch.tensor(w0)), 'the weights are read only'
    if spec.l1:
        zeros = w0 == 0
        assert bool((g.cpu().numpy()[zeros] == g0[zeros]).all()), 'sign(0) = 0: no L1 gradient at exact zeros'
    want_loss = float(reg_ref.reg_loss(w, l1, l2))
    assert abs(float(acc.item()) - (0.5 + 3.0 * want_loss)) <= 1e-12 * (1 + 3.0 * want_loss)
    assert abs(float(loss_only.item()) - want_loss) <= 1e-12 * (1 + want_loss)


def test_reg_grad_refuses_negative_factors(nat):
    p = torch.zeros(8, device='cuda')
    for l1, l2 in ((-0.1, 0.0), (0.0, -1e-9), (float('inf'), 0.0), (0.0, float('nan'))):
        assert nat.lib.dtb_reg_grad(nat.ptr(p), nat.ptr(p), 8, l1, l2, None, 1.0, None) != 0
        assert 'regularization factors' in nat.last_error()


# ---- 2. fused sweeps: bit-identical to dtb_reg_grad + the plain sweep, and against the float64 oracle ---------------
def _check_oracle(p, pr, what):
    np.testing.assert_allclose(p.cpu().numpy(), pr.numpy(), rtol=1e-5, atol=1e-5, err_msg=what)


@pytest.mark.parametrize('reg', list(REGS))
@pytest.mark.parametrize('n,off', [(4099, 0), (1003, 1)])
def test_fused_adam_sweep_is_bit_identical_to_unfused(nat, reg, n, off):
    spec = R.resolve(REGS[reg])
    o = O.resolve(O.Adam(learning_rate=0.01))
    gen = np.random.default_rng(n + off + 7)
    w0 = _weights(gen, n)
    # unfused (reg_grad, adam_dense), fused host-step form, fused CUDA-graph form
    arms = [[_buf(w0, off), _buf(np.zeros(n), off), _buf(np.zeros(n), off), _buf(np.zeros(n), off)] for _ in range(3)]
    accs = [torch.zeros(1, dtype=torch.float64, device='cuda') for _ in range(3)]
    alpha = torch.tensor([0.0] + [adam_alpha(s, o.learning_rate, o.beta_1, o.beta_2) for s in range(1, 30)],
                         dtype=torch.float32, device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    pr = torch.tensor(w0, dtype=torch.float64)
    sr = OR.new_slots(o, pr)
    l1, l2 = float(np.float32(spec.l1)), float(np.float32(spec.l2))
    for t in range(1, 21):
        gg = gen.normal(size=n).astype(np.float32)
        gg[gen.random(n) < 0.3] = 0.0
        a = float(alpha[t].item())
        for p, m, v, g in arms:
            g.copy_(torch.as_tensor(gg))
        (p, m, v, g), (pf, mf, vf, gf), (pd, md, vd, gd) = arms
        nat.check(nat.lib.dtb_reg_grad(*_ptrs([p, g]), n, spec.l1, spec.l2, nat.ptr(accs[0]), 2.0, None))
        nat.check(nat.lib.dtb_adam_dense(*_ptrs([p, m, v, g]), n, a, o.beta_1, o.beta_2, o.epsilon, 1, None))
        nat.check(nat.lib.dtb_adam_dense_reg(*_ptrs([pf, mf, vf, gf]), n, a, o.beta_1, o.beta_2, o.epsilon, 1,
                                             spec.l1, spec.l2, nat.ptr(accs[1]), 2.0, None))
        step_dev.fill_(t - 1)
        nat.check(nat.lib.dtb_adam_dense_reg_dev(*_ptrs([pd, md, vd, gd]), n, nat.ptr(alpha), nat.ptr(step_dev),
                                                 o.beta_1, o.beta_2, o.epsilon, 1, spec.l1, spec.l2, nat.ptr(accs[2]),
                                                 2.0, None))
        gt = torch.tensor(gg, dtype=torch.float64) + reg_ref.reg_grad(pr, l1, l2)
        OR.step(o, pr, gt, sr, t)
    torch.cuda.synchronize()
    ref = arms[0]
    for label, arm in (('host', arms[1]), ('dev', arms[2])):
        for k, (x, y) in enumerate(zip(arm, ref)):
            assert torch.equal(x, y), f'{reg}: fused {label} form, buffer {k} differs from reg_grad + adam_dense'
    assert bool((ref[3] == 0).all())
    for acc in accs[1:]:
        assert abs(float(acc.item()) - float(accs[0].item())) <= 1e-12 * float(accs[0].item())
    _check_oracle(ref[0], pr, f'{reg}: adam p')


@pytest.mark.parametrize('name', list(VARIANTS))
@pytest.mark.parametrize('n,off', [(4099, 0), (1003, 1)])
def test_fused_optim_sweep_is_bit_identical_to_unfused(nat, name, n, off):
    spec = R.resolve(REGS['l1l2'])
    o = O.resolve(VARIANTS[name])
    hp = _hp(o)
    gen = np.random.default_rng(n + off + 11)
    w0 = _weights(gen, n)

    def arm():
        return [_buf(w0, off), _buf(np.zeros(n), off)], \
            [None if s is None else _buf(np.full(n, s), off) for s in O.slot_inits(o)]

    (pg, su), (pgf, sf) = arm(), arm()
    accs = [torch.zeros(1, dtype=torch.float64, device='cuda') for _ in range(2)]
    pr = torch.tensor(w0, dtype=torch.float64)
    sr = OR.new_slots(o, pr)
    l1, l2 = float(np.float32(spec.l1)), float(np.float32(spec.l2))
    for t in range(1, 21):
        gg = gen.normal(size=n).astype(np.float32)
        gg[gen.random(n) < 0.3] = 0.0
        pg[1].copy_(torch.as_tensor(gg))
        pgf[1].copy_(torch.as_tensor(gg))
        nat.check(nat.lib.dtb_reg_grad(*_ptrs(pg), n, spec.l1, spec.l2, nat.ptr(accs[0]), 1.0, None))
        nat.check(nat.lib.dtb_optim_dense(*_ptrs(pg + su), n, hp, 1, None))
        nat.check(nat.lib.dtb_optim_dense_reg(*_ptrs(pgf + sf), n, hp, 1, spec.l1, spec.l2, nat.ptr(accs[1]), 1.0,
                                              None))
        gt = torch.tensor(gg, dtype=torch.float64) + reg_ref.reg_grad(pr, l1, l2)
        OR.step(o, pr, gt, sr, t)
    torch.cuda.synchronize()
    assert torch.equal(pgf[0], pg[0]) and bool((pgf[1] == 0).all()), f'{name}: fused weights differ'
    for k, (a, b) in enumerate(zip(sf, su)):
        if a is not None:
            assert torch.equal(a, b), f'{name}: fused slot {k} differs'
    assert abs(float(accs[1].item()) - float(accs[0].item())) <= 1e-12 * float(accs[0].item())
    _check_oracle(pg[0], pr, f'{name}: p')


# ---- 3. DeepModel against the float64 reference trainer ------------------------------------------------------------------
EMB_REG, KERNEL_REG = R.L2(0.01), R.L1L2(l1=1e-3, l2=0.01)
TRAIN_OPTS = {'adam': 'auto', 'sgd': O.SGD(learning_rate=0.05, momentum=0.9), 'rmsprop': 'rmsprop', 'adagrad': 'adagrad'}
NETS = ['dnn_nets', 'linear', 'fm_nets', 'cin_nets']


def _reg_build(nets, vocab, dim, n_cont, emb=EMB_REG, kernel=KERNEL_REG, seed=5, dnn_extra=None, **kw):
    dnn = {'hidden_units': ((16, 0, False), (8, 0, True)), 'activation': 'relu', 'kernel_regularizer': kernel,
           **(dnn_extra or {})}
    return build(nets, vocab, dim, n_cont, seed=seed, embeddings_regularizer=emb, dnn_params=dnn, **kw)


@pytest.mark.parametrize('name', list(TRAIN_OPTS))
def test_training_matches_float64_reference(name):
    vocab, dim, n_cont, b = [11, 7, 13, 5, 9], 4, 3, 48
    model, conf = _reg_build(NETS, vocab, dim, n_cont, optimizer=TRAIN_OPTS[name])
    assert not model.table.lazy_active
    state = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    regs = reg_ref.regularized_weights(state, R.resolve(EMB_REG), R.resolve(KERNEL_REG))
    assert sorted(k for k in regs if 'dense' in k) == ['dnn_dense_1/kernel', 'dnn_dense_2/kernel']
    assert sorted(model._scope.regularizers) == ['dnn_dense_1/kernel', 'dnn_dense_2/kernel']
    assert 'regularizer: L2(l2=0.01)' in str(model.model_desc)
    assert 'dnn_dense_1/kernel: L1L2(l1=0.001, l2=0.01)' in str(model.model_desc)
    ref = reg_ref.RegRefTrainer(state, conf, len(vocab), regs, O.resolve(TRAIN_OPTS[name]))
    losses_g, losses_r = [], []
    for step in range(20):
        idx, cont, y = batch(vocab, n_cont, b, seed=step)
        losses_g.append(model.train_on_batch(idx, cont, y))
        losses_r.append(ref.train_step(torch.tensor(idx), torch.tensor(cont, dtype=torch.float64),
                                       torch.tensor(y, dtype=torch.float64)))
    assert ref.reg_term() > 0.01 * losses_r[-1], 'the regularization term is a visible part of the loss'
    np.testing.assert_allclose(losses_g, losses_r, rtol=2e-3, atol=1e-5)
    tol = dict(rtol=1e-3, atol=2e-5) if name in ('sgd', 'adagrad') else dict(rtol=1e-2, atol=2e-4)
    new_state = model.state_dict()
    for k, v in ref.state.items():
        np.testing.assert_allclose(new_state[k].cpu().numpy(), v.numpy(), err_msg=k, **tol)


def test_validation_and_evaluate_loss_include_the_term(monkeypatch):
    import pandas as pd
    vocab, dim, n_cont = [11, 7, 13, 5, 9], 4, 3
    model, _ = _reg_build(['linear', 'fm_nets', 'dnn_nets'], vocab, dim, n_cont)
    idx, cont, y = batch(vocab, n_cont, 300, seed=3)
    X = pd.DataFrame({**{f'c{i}': idx[:, i] for i in range(len(vocab))}, **{f'n{i}': cont[:, i] for i in range(n_cont)}})
    hist = model.fit(X.iloc[:200], y[:200], batch_size=50, epochs=2, verbose=0,
                     validation_data=(X.iloc[200:], y[200:]), validation_steps=2)
    state = {k: v.detach().cpu().double() for k, v in model.state_dict().items()}
    term = sum(float(reg_ref.reg_loss(state[k], *r)) for k, r in
               reg_ref.regularized_weights(state, R.resolve(EMB_REG), R.resolve(KERNEL_REG)).items())
    with_term = model.evaluate(X.iloc[200:], y[200:], batch_size=50)['loss']
    monkeypatch.setattr(model, '_reg_loss', lambda *a: None)
    data_only = model.evaluate(X.iloc[200:], y[200:], batch_size=50)['loss']
    assert term > 0.01
    assert abs(with_term - data_only - term) < 1e-5 * (1 + term)
    assert abs(hist.history['val_loss'][-1] - with_term) < 1e-6 * (1 + with_term)


def test_zero_regularizers_train_bit_identically_to_none(monkeypatch):
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    vocab, dim, n_cont = [400, 300, 500], 4, 2
    plain, _ = build(['linear', 'fm_nets', 'dnn_nets'], vocab, dim, n_cont, seed=9)
    zero, _ = _reg_build(['linear', 'fm_nets', 'dnn_nets'], vocab, dim, n_cont, emb=R.L1L2(), kernel=R.L1L2(0.0, 0.0),
                         seed=9)
    assert zero._emb_reg is None and not zero._scope.reg_segments and zero.table.lazy_active
    for step in range(8):
        args = _distinct_batch(vocab, n_cont, 2, seed=step)
        assert plain.train_on_batch(*args) == zero.train_on_batch(*args)
    _states_equal(zero, plain, 'L1L2(0, 0) vs no regularizer')


def test_unregularized_models_never_call_the_new_entry_points(monkeypatch):
    """A model without regularizers runs the kernels it ran before: none of the new entry points, in the eager step,
    the CUDA-graph capture or evaluation."""
    from deeptables_b200 import _native as N

    def boom(*a):
        raise AssertionError('a regularization kernel ran for a model without regularizers')

    for name in ('dtb_reg_grad', 'dtb_adam_dense_reg', 'dtb_adam_dense_reg_dev', 'dtb_optim_dense_reg'):
        monkeypatch.setattr(N.lib, name, boom)
    vocab, n_cont, b = [50, 40, 30, 20], 2, 64
    for opt in ('auto', 'rmsprop'):
        model, _ = build(['linear', 'cin_nets', 'dnn_nets'], vocab, 8, n_cont, optimizer=opt)
        for step in range(4):
            model.train_on_batch(*batch(vocab, n_cont, b, seed=step))
        assert model._graphs, 'the CUDA-graph form ran too'
        model._table_mode_override = 'dense'
        for step in range(2):
            model.train_on_batch(*batch(vocab, n_cont, b, seed=step))
        idx, cont, y = batch(vocab, n_cont, b, seed=9)
        model._evaluate_tensors(*[torch.as_tensor(a).cuda() for a in (idx, cont, y.reshape(-1, 1))], b, 1, {})


@pytest.mark.parametrize('opt', ['auto', 'adagrad'])
def test_regularized_table_never_goes_lazy(opt):
    vocab, n_cont, b = [400, 300, 500], 2, 8
    model, _ = _reg_build(['linear', 'fm_nets', 'dnn_nets'], vocab, 4, n_cont, optimizer=opt)
    assert model.table.lazy_adam and not model.table.lazy_active
    w0 = model.table.weight.clone()
    for step in range(3):
        model._table_mode_override = 'lazy' if step % 2 else None
        model.train_on_batch(*batch(vocab, n_cont, b, seed=step))
        assert not model.table.lazy_active
    # every row moved, touched by a batch or not
    assert bool((model.table.weight != w0).all(dim=1).all())


def test_ragged_padding_stays_zero():
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    vocab, dims, n_cont = [30, 20, 40], [8, 3, 5], 2
    conf = deeptable.ModelConfig(nets=['dnn_nets'], fixed_embedding_dim=False, embedding_dropout=0,
                                 embeddings_regularizer=R.L1L2(0.01, 0.01),
                                 dnn_params={'hidden_units': ((16, 0, False),), 'activation': 'relu'})
    cats = [CategoricalColumn(f'c{i}', v, d) for i, (v, d) in enumerate(zip(vocab, dims))]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(n_cont)])]
    for opt in ('auto', O.SGD(momentum=0.9)):
        model = DeepModel('binary', 2, conf.__class__(**{**conf._asdict(), 'optimizer': opt}), cats, conts, seed=3)
        model._build_model()
        t = model.table
        assert t.ragged
        for step in range(6):
            model.train_on_batch(*batch(vocab, n_cont, 32, seed=step))
        lo = t.row_offsets_host
        for i, d in enumerate(dims):
            assert bool((t.weight[lo[i]:lo[i + 1], d:] == 0).all()), f'{opt!r}: padding of field {i}'


@pytest.mark.parametrize('opt', ['auto', 'rmsprop'])
def test_cuda_graph_replay_is_bit_identical_to_eager(monkeypatch, opt):
    s = dict(nets=['linear', 'fm_nets', 'dnn_nets'], vocab=[400, 300, 500], dim=4, n_cont=2)

    def run():
        model, _ = _reg_build(s['nets'], s['vocab'], s['dim'], s['n_cont'], seed=9, optimizer=opt)
        losses = [model.train_on_batch(*_distinct_batch(s['vocab'], s['n_cont'], 2, seed=k)) for k in range(10)]
        return model, losses

    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    eager, le = run()
    assert not eager._graphs
    monkeypatch.setenv('DTB_CUDA_GRAPH', '1')
    graphed, lg = run()
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    _states_equal(graphed, eager, f'{opt}: graph replay vs eager')
    np.testing.assert_allclose(lg, le, rtol=1e-12)


def test_custom_dnn_D_A_D_B_applies_kernel_regularizer():
    from deeptables_b200 import deepnets
    vocab, dim, n_cont, b = [11, 7, 13], 4, 3, 32
    extra = {'custom_dnn_fn': deepnets.custom_dnn_D_A_D_B}
    reg, _ = _reg_build(['dnn_nets'], vocab, dim, n_cont, emb=None, seed=4, dnn_extra=extra)
    plain, _ = _reg_build(['dnn_nets'], vocab, dim, n_cont, emb=None, kernel=None, seed=4, dnn_extra=extra)
    names = ['dnn_custom_dense_1/kernel', 'dnn_custom_dense_2/kernel']
    assert sorted(reg._scope.regularizers) == names
    state = {k: v.detach().cpu().double() for k, v in reg.state_dict().items()}
    term = sum(float(reg_ref.reg_loss(state[k], 1e-3, 0.01)) for k in names)
    args = batch(vocab, n_cont, b, seed=0)
    # first step: same initial weights, so the losses differ by the term on them
    assert abs(reg.train_on_batch(*args) - plain.train_on_batch(*args) - term) < 1e-5 * (1 + term)


@pytest.mark.parametrize('opt', ['auto', O.SGD(momentum=0.9)], ids=['adam', 'sgd_momentum'])
def test_checkpoint_resume_is_bit_identical(monkeypatch, tmp_path, opt):
    from deeptables_b200.deepmodel import DeepModel
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    s = dict(nets=['linear', 'fm_nets', 'dnn_nets'], vocab=[400, 300, 500], dim=4, n_cont=2)

    def train(model, steps):
        for k in range(model._step, model._step + steps):
            model.train_on_batch(*_distinct_batch(s['vocab'], s['n_cont'], 2, seed=k))
        return model

    straight = train(_reg_build(s['nets'], s['vocab'], s['dim'], s['n_cont'], seed=9, optimizer=opt)[0], 6)
    first = train(_reg_build(s['nets'], s['vocab'], s['dim'], s['n_cont'], seed=9, optimizer=opt)[0], 3)
    path = str(tmp_path / 'ck.npz')
    first.save(path)
    resumed = DeepModel('binary', 2, first.config, first.categorical_columns, first.continuous_columns,
                        model_file=path, seed=123)
    assert resumed._step == 3 and not resumed.table.lazy_active
    train(resumed, 3)
    _states_equal(resumed, straight, 'save after 3 steps, load, 3 more')


# ---- 4. data parallel ------------------------------------------------------------------------------------------------------
DP_VOCAB, DP_DIM, DP_CONT, DP_B = [50, 40, 30, 20, 60], 8, 3, 64


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_build():
    return _reg_build(['linear', 'fm_nets', 'cin_nets', 'dnn_nets'], DP_VOCAB, DP_DIM, DP_CONT, seed=11,
                      cin_params={'cross_layer_size': (16, 16), 'activation': 'relu', 'use_residual': False,
                                  'use_bias': False, 'direct': False, 'reduce_D': False})[0]


def _dp_worker(rank, world, port, out_dir, same_shard):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        m = _dp_build()
        for step in range(6):
            m.train_on_batch(*batch(DP_VOCAB, DP_CONT, DP_B, seed=step if same_shard else step * world + rank))
        m.sync_replica_buffers()
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), **{k: v.detach().cpu().numpy() for k, v in m.state_dict().items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('same_shard', [True, False])
def test_data_parallel_replicas_stay_bit_identical(tmp_path, same_shard):
    """Ranks fed the same shard reproduce the single-GPU run on it: the mean of identical data gradients plus the
    regularization gradient counted once (added after the exchange, not summed over the replicas)."""
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path), same_shard), nprocs=world, join=True)
    r0, r1 = np.load(tmp_path / 'rank0.npz'), np.load(tmp_path / 'rank1.npz')
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]), f'replica 1 diverged from replica 0 on {k}'
    if same_shard:
        single = _dp_build()
        for step in range(6):
            single.train_on_batch(*batch(DP_VOCAB, DP_CONT, DP_B, seed=step))
        sd = single.state_dict()
        for k in r0.files:
            np.testing.assert_allclose(r0[k], sd[k].cpu().numpy(), rtol=1e-4, atol=1e-6, err_msg=k)
