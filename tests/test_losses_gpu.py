"""Keras 3 losses on the GPU (ModelConfig.loss): dtb_keras_loss_fwd_bwd against the float64 restatement of
tests/loss_ref.py, the losses 'auto' already computes keeping their kernel and their bits, DeepModel training,
history, validation and evaluation losses against a float64 reference trainer, CUDA-graph replay, the hinge losses'
label check, DeepTable save / load and data parallel."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import loss_ref
from deeptables_b200 import losses as LS, optimizers as O
from test_optimizers_gpu import _states_equal

pytestmark = pytest.mark.gpu

TASKS = {'binary': 1, 'multilabel': 3, 'multiclass': 5, 'regression': 1}
CODE = {'binary': 0, 'multilabel': 0, 'regression': 1, 'multiclass': 2}
LOSSES = {**{kind: getattr(LS, kind)() for kind in LS._CLASSES},
          'Huber_delta0.5': LS.Huber(delta=0.5), 'BinaryCrossentropy_s0.1': LS.BinaryCrossentropy(label_smoothing=0.1),
          'CategoricalCrossentropy_s0.2': LS.CategoricalCrossentropy(label_smoothing=0.2)}


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


def _dev(a):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _kernel(nat, spec, task, z, y, w=None, want_grad=True):
    """One dtb_keras_loss_fwd_bwd call: (prob, dz or None, summed loss)."""
    rows, cols = z.shape
    zd, yd, wd = _dev(z), _dev(y), _dev(w)
    prob = torch.empty(rows, cols, device='cuda')
    dz = torch.empty(rows, cols, device='cuda') if want_grad else None
    acc = torch.zeros(1, dtype=torch.float64, device='cuda')
    scratch = torch.empty(1, dtype=torch.int32, device='cuda')
    lp = nat.LossParams(loss=spec.code, delta=spec.delta, label_smoothing=spec.label_smoothing,
                        scratch=scratch.data_ptr())
    nat.check(nat.lib.dtb_keras_loss_fwd_bwd(nat.ptr(zd), nat.ptr(yd), nat.ptr(wd), nat.ptr(prob), nat.ptr(dz),
                                             nat.ptr(acc), rows, cols, CODE[task], lp, None), 'keras_loss_fwd_bwd')
    torch.cuda.synchronize()
    return prob.cpu().numpy(), None if dz is None else dz.cpu().numpy(), float(acc.item())


def _float64(spec, task, z, y, w=None, terms=False):
    """(p, dLoss/dz, loss) in float64; with ``terms`` also sum_c |p_c dLoss/dp_c| per row, the size of the terms the
    softmax Jacobian and the renormalisation add up (they cancel where dLoss/dp is large, as MAPE's is at y = 0)."""
    z64 = torch.tensor(z, dtype=torch.float64, requires_grad=True)
    y64 = torch.tensor(y, dtype=torch.float64)
    w64 = None if w is None else torch.tensor(w, dtype=torch.float64)
    p = loss_ref.output(z64, task)
    loss = loss_ref.batch_loss(spec, y64, p, w64)
    (gz,) = torch.autograd.grad(loss, [z64])
    out = p.detach().numpy(), gz.numpy(), float(loss.detach())
    if not terms:
        return out
    pl = p.detach().clone().requires_grad_(True)
    (gp,) = torch.autograd.grad(loss_ref.batch_loss(spec, y64, pl, w64), [pl])
    return out + ((pl.detach() * gp).abs().sum(-1, keepdim=True).numpy(),)


def _labels(g, task, rows, cols):
    if task in ('binary', 'multilabel'):
        return (g.random((rows, cols)) < 0.4).astype(np.float32)
    if task == 'multiclass':
        return np.eye(cols, dtype=np.float32)[g.integers(0, cols, size=rows)]
    return g.normal(size=(rows, cols)).astype(np.float32)


def _check(nat, spec, task, z, y, w=None):
    """The tolerances of test_native_gpu.py::test_losses, dz's widened by float32 rounding (2e-6, ~16 ulp) of the terms
    summed per row; the evaluation form (dz NULL) adds the same loss."""
    rows = z.shape[0]
    prob, dz, acc = _kernel(nat, spec, task, z, y, w)
    p, gz, loss, terms = _float64(spec, task, z, y, w, terms=True)
    np.testing.assert_allclose(prob, p, rtol=1e-4, atol=1e-6)
    bad = np.abs(dz - gz) > 1e-7 + 2e-6 * terms + 2e-4 * np.abs(gz)
    assert not bad.any(), f'{spec} on {task}: dz differs at {np.argwhere(bad)[:5].tolist()}: {dz[bad][:5]} vs {gz[bad][:5]}'
    np.testing.assert_allclose(acc / rows, loss, rtol=1e-5)
    prob2, none, acc2 = _kernel(nat, spec, task, z, y, w, want_grad=False)
    assert none is None and np.array_equal(prob2, prob)
    assert abs(acc2 - acc) <= 1e-12 * abs(acc), 'dz = NULL changed the loss'


# ---- 1. the kernel against float64 ------------------------------------------------------------------------------------
@pytest.mark.parametrize('task', list(TASKS))
@pytest.mark.parametrize('name', list(LOSSES))
def test_kernel_matches_float64(nat, name, task):
    spec = LS.resolve(LOSSES[name], task)
    rows, cols = 257, TASKS[task]
    g = np.random.default_rng(sum(map(ord, name + task)))
    z = (g.normal(size=(rows, cols)) * 2).astype(np.float32)
    y = _labels(g, task, rows, cols)
    if task == 'regression' and spec.kind == 'Poisson':         # log(p + eps) of the identity output needs p > 0
        z, y = np.abs(z) + 0.1, np.abs(y)
    w = g.uniform(0.5, 2.0, size=rows).astype(np.float32)
    for weights in (None, w):
        _check(nat, spec, task, z, y, weights)


# rows where TensorFlow's gradient conventions decide (tests/test_losses_cpu.py checks the float64 side by hand)
EDGES = {
    'huber_at_delta': (LS.Huber(delta=0.5), 'regression', [[0.75], [-0.25], [3.0], [0.25]], [[0.25], [0.25], [0.0], [0.25]]),
    'hinge_at_margin': (LS.Hinge(), 'regression', [[1.0], [-1.0], [0.3], [2.0]], [[1.0], [0.0], [1.0], [0.0]]),
    'squared_hinge_at_margin': (LS.SquaredHinge(), 'regression', [[1.0], [-1.0], [0.3]], [[1.0], [0.0], [0.0]]),
    'hinge_unconverted': (LS.Hinge(), 'regression', [[1.0], [-1.0], [0.3]], [[1.0], [0.0], [0.5]]),
    'mape_zero_label': (LS.MeanAbsolutePercentageError(), 'regression', [[0.5], [1.0], [-2.0]], [[0.0], [2.0], [0.0]]),
    'mae_zero_error': (LS.MeanAbsoluteError(), 'regression', [[0.5], [1.0]], [[0.5], [-1.0]]),
    'msle_below_eps': (LS.MeanSquaredLogarithmicError(), 'regression', [[-0.5], [1e-8], [0.5]], [[1.0], [1.0], [0.2]]),
    'kl_below_eps': (LS.KLDivergence(), 'regression', [[-0.5], [1.5], [0.5], [1e-9]], [[0.5], [0.5], [0.3], [0.0]]),
    'kl_softmax_below_eps': (LS.KLDivergence(), 'multiclass', [[-30.0, 0.0, 1.0], [0.0, 1.0, 2.0]],
                             [[1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]),
    'categorical_hinge_ties': (LS.CategoricalHinge(), 'multiclass', [[0.3, 0.3, -1.0], [1.0, 1.0, 1.0], [2.0, 0.0, 2.0]],
                               [[0.0, 0.0, 1.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]),
    'categorical_hinge_multilabel_ties': (LS.CategoricalHinge(), 'multilabel', [[0.3, 0.3, -1.0], [5.0, 5.0, 5.0]],
                                          [[0.0, 0.0, 1.0], [0.0, 0.0, 0.0]]),
}


@pytest.mark.parametrize('case', list(EDGES))
def test_edges_match_float64(nat, case):
    loss, task, z, y = EDGES[case]
    z, y = np.array(z, dtype=np.float32), np.array(y, dtype=np.float32)
    spec = LS.resolve(loss, task)
    _check(nat, spec, task, z, y)
    _check(nat, spec, task, z, y, np.linspace(0.5, 2.0, z.shape[0]).astype(np.float32))


def test_hinge_label_check_runs_on_the_device(nat):
    """One label outside {0, 1} anywhere in the batch turns the conversion off for every row."""
    spec = LS.resolve('hinge', 'binary')
    g = np.random.default_rng(4)
    z = g.normal(size=(1001, 1)).astype(np.float32)
    y = (g.random((1001, 1)) < 0.5).astype(np.float32)
    _, dz_binary, acc_binary = _kernel(nat, spec, 'regression', z, y)
    y[700, 0] = 0.5
    _, dz_other, acc_other = _kernel(nat, spec, 'regression', z, y)
    p, gz, loss = _float64(spec, 'regression', z, y)
    np.testing.assert_allclose(dz_other, gz, rtol=2e-4, atol=1e-7)
    np.testing.assert_allclose(acc_other / 1001, loss, rtol=1e-5)
    zero = y[:, 0] == 0
    assert np.all(dz_other[zero] == 0) and not np.all(dz_binary[zero] == 0), 'y = 0 rows: y\' = 0 unconverted, -1 converted'


def test_refusals_of_the_entry_point(nat):
    z = torch.zeros(4, 1, device='cuda')
    for kw in (dict(loss=0), dict(loss=14), dict(loss=LS.CODES['Huber'], delta=0.0),
               dict(loss=LS.CODES['Huber'], delta=float('inf')), dict(loss=LS.CODES['BinaryCrossentropy'], label_smoothing=1.5),
               dict(loss=LS.CODES['Hinge'])):
        lp = nat.LossParams(**{'delta': 1.0, **kw})
        rc = nat.lib.dtb_keras_loss_fwd_bwd(nat.ptr(z), nat.ptr(z), None, nat.ptr(z), None, None, 4, 1, 1, lp, None)
        assert rc != 0, kw


# ---- 2. models ----------------------------------------------------------------------------------------------------------------
VOCAB, DIM, N_CONT, N_CLASSES = [400, 300, 500], 4, 2, 4


def _build(task, loss, seed=9, nets=('linear', 'fm_nets', 'dnn_nets'), **kw):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    conf = deeptable.ModelConfig(nets=list(nets), embeddings_output_dim=DIM, embedding_dropout=0, metrics=[],
                                 dnn_params={'hidden_units': ((16, 0, False), (8, 0, True)), 'activation': 'relu'},
                                 loss=loss, **kw)
    cats = [CategoricalColumn(f'c{i}', v, DIM) for i, v in enumerate(VOCAB)]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(N_CONT)])]
    model = DeepModel(task, N_CLASSES if task == 'multiclass' else 2, conf, cats, conts, seed=seed)
    model._build_model()
    return model, conf


def _batch(task, b, seed, distinct=False):
    """(ids, continuous, labels as the model trains on them, class ids or None)."""
    g = np.random.default_rng(seed)
    idx = np.stack([g.choice(v, size=b, replace=False) if distinct else g.integers(0, v, size=b) for v in VOCAB],
                   axis=1).astype(np.int32)
    cont = g.normal(size=(b, N_CONT)).astype(np.float32)
    if task == 'multiclass':
        k = g.integers(0, N_CLASSES, size=b)
        return idx, cont, np.eye(N_CLASSES, dtype=np.float32)[k], k
    if task == 'regression':
        return idx, cont, (cont[:, 0] + 0.5 * g.normal(size=b)).astype(np.float32), None
    return idx, cont, (g.random(b) < 0.35).astype(np.float32), None


BUILTIN = [('binary', 'binary_crossentropy'), ('binary', LS.BinaryCrossentropy()), ('regression', 'mse'),
           ('regression', LS.MeanSquaredError()), ('multiclass', 'categorical_crossentropy')]


@pytest.mark.parametrize('task,loss', BUILTIN, ids=[f'{t}-{l!r}' for t, l in BUILTIN])
def test_the_auto_losses_keep_their_kernel_and_bits(monkeypatch, task, loss):
    from deeptables_b200 import _native as N

    def boom(*a):
        raise AssertionError('dtb_keras_loss_fwd_bwd ran for a loss that auto computes')

    monkeypatch.setattr(N.lib, 'dtb_keras_loss_fwd_bwd', boom)
    runs = []
    for cfg_loss in ('auto', loss):
        model, _ = _build(task, cfg_loss)
        losses = [model.train_on_batch(*_batch(task, 2, seed=k, distinct=True)[:3]) for k in range(8)]
        assert model._graphs, 'the CUDA-graph form ran too'
        idx, cont, y, _ = _batch(task, 64, seed=99)
        vloss = model._evaluate_tensors(*[torch.as_tensor(a).cuda() for a in (idx, cont, y.reshape(64, -1))], 64, 1, {})
        runs.append((model, losses, vloss))
    (auto, la, va), (named, ln, vn) = runs
    _states_equal(named, auto, f'{loss!r} vs auto')
    assert la == ln and va == vn


TRAINED = [('regression', LS.Huber(delta=0.5)), ('regression', 'mae'), ('binary', 'poisson'),
           ('multiclass', LS.KLDivergence()), ('binary', LS.BinaryCrossentropy(label_smoothing=0.1)),
           ('multiclass', LS.CategoricalCrossentropy(label_smoothing=0.1)), ('binary', 'hinge'),
           ('regression', 'log_cosh')]
TRAINED_IDS = [f'{t}-{l!r}' for t, l in TRAINED]


@pytest.mark.parametrize('task,loss', TRAINED, ids=TRAINED_IDS)
def test_training_matches_float64_reference(task, loss):
    """20 steps of SGD against the float64 trainer, at test_optimizers_gpu.py's SGD tolerances: its steps are
    proportional to the gradient, so they compare the loss gradients themselves (Adam's first steps are lr * sign(g)
    wherever g is tiny, whatever its float32 rounding)."""
    opt = O.SGD(learning_rate=0.01)
    model, conf = _build(task, loss, seed=5, optimizer=opt)
    spec = LS.resolve(loss, task)
    assert model.model_desc.loss == str(spec) and model._loss == spec
    state = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    ref = loss_ref.LossRefTrainer(state, conf, len(VOCAB), spec, task, optimizer=O.resolve(opt))
    losses_g, losses_r = [], []
    for step in range(20):
        idx, cont, y, _ = _batch(task, 48, seed=step)
        losses_g.append(model.train_on_batch(idx, cont, y))
        losses_r.append(ref.train_step(torch.tensor(idx), torch.tensor(cont, dtype=torch.float64),
                                       torch.tensor(y, dtype=torch.float64)))
    np.testing.assert_allclose(losses_g, losses_r, rtol=2e-3, atol=1e-5)
    new_state = model.state_dict()
    for k, v in ref.state.items():
        np.testing.assert_allclose(new_state[k].cpu().numpy(), v.numpy(), err_msg=k, rtol=1e-3, atol=2e-5)


def _frame(idx, cont):
    return pd.DataFrame({**{f'c{i}': idx[:, i] for i in range(len(VOCAB))}, **{f'n{i}': cont[:, i] for i in range(N_CONT)}})


@pytest.mark.parametrize('task,loss', TRAINED[:6], ids=TRAINED_IDS[:6])
def test_history_val_loss_and_evaluate_are_the_float64_loss(task, loss):
    model, conf = _build(task, loss, seed=6)
    spec = LS.resolve(loss, task)
    n, nv = 200, 120
    idx, cont, y, k = _batch(task, n + nv, seed=42)
    labels = k if task == 'multiclass' else y          # fit / evaluate take class ids and one-hot them
    X = _frame(idx, cont)
    state0 = {kk: v.detach().cpu().clone() for kk, v in model.state_dict().items()}
    before = loss_ref.LossRefTrainer(state0, conf, len(VOCAB), spec, task)
    want_train = float(before.loss_and_grads(torch.tensor(idx[:n]), torch.tensor(cont[:n], dtype=torch.float64),
                                             torch.tensor(y[:n], dtype=torch.float64))[0])
    hist = model.fit(X.iloc[:n], labels[:n], batch_size=n, epochs=1, verbose=0, shuffle=False,
                     validation_data=(X.iloc[n:], labels[n:]))
    state1 = {kk: v.detach().cpu().clone() for kk, v in model.state_dict().items()}
    after = loss_ref.LossRefTrainer(state1, conf, len(VOCAB), spec, task)
    want_val = after.loss(torch.tensor(idx[n:]), torch.tensor(cont[n:], dtype=torch.float64),
                          torch.tensor(y[n:], dtype=torch.float64))
    np.testing.assert_allclose(hist.history['loss'][0], want_train, rtol=1e-4)
    np.testing.assert_allclose(hist.history['val_loss'][0], want_val, rtol=1e-4)
    np.testing.assert_allclose(model.evaluate(X.iloc[n:], labels[n:], batch_size=50)['loss'], want_val, rtol=1e-4)


def test_sample_weights_scale_each_row(monkeypatch):
    """Keras's sum_over_batch_size: sum_r w_r l_r / rows, also with weights; weighted steps run eagerly."""
    model, conf = _build('regression', LS.Huber(delta=0.5), seed=3)
    spec = LS.resolve(LS.Huber(delta=0.5), 'regression')
    idx, cont, y, _ = _batch('regression', 64, seed=1)
    w = np.random.default_rng(1).uniform(0.0, 3.0, size=64).astype(np.float32)
    state = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    ref = loss_ref.LossRefTrainer(state, conf, len(VOCAB), spec, 'regression')
    params = {k: v.detach().clone() for k, v in ref.state.items()}
    from oracle import model_ref as M
    out, _ = M.forward(params, conf, torch.tensor(idx), torch.tensor(cont, dtype=torch.float64), len(VOCAB), True,
                       'regression')
    want = float(loss_ref.batch_loss(spec, torch.tensor(y, dtype=torch.float64).reshape(64, 1), out,
                                     torch.tensor(w, dtype=torch.float64)))
    got = model.train_on_batch(idx, cont, y, sample_weight=w)
    np.testing.assert_allclose(got, want, rtol=1e-5)


@pytest.mark.parametrize('task,loss', [('regression', LS.Huber(delta=0.5)), ('binary', 'squared_hinge'),
                                       ('multiclass', LS.CategoricalCrossentropy(label_smoothing=0.1)),
                                       ('binary', LS.BinaryCrossentropy(label_smoothing=0.1))],
                         ids=['huber', 'squared_hinge', 'cce_smoothed', 'bce_smoothed'])
def test_cuda_graph_replay_is_bit_identical_to_eager(monkeypatch, task, loss):
    def run():
        model, _ = _build(task, loss)
        losses = [model.train_on_batch(*_batch(task, 2, seed=k, distinct=True)[:3]) for k in range(10)]
        idx, cont, _, _ = _batch(task, 64, seed=77)
        pred = model.predict_step(torch.as_tensor(idx).cuda(), torch.as_tensor(cont).cuda())
        return model, losses, pred

    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    eager, le, pe = run()
    assert not eager._graphs
    monkeypatch.setenv('DTB_CUDA_GRAPH', '1')
    graphed, lg, pg = run()
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    _states_equal(graphed, eager, f'{loss!r}: graph replay vs eager')
    assert torch.equal(pg, pe)
    np.testing.assert_allclose(lg, le, rtol=1e-12)      # float64 atomics may add the rows in another order


def test_deeptable_save_and_load_keep_the_loss(tmp_path):
    from deeptables_b200 import deeptable, deepnets
    g = np.random.default_rng(0)
    n = 2000
    df = pd.DataFrame({'job': g.choice(list('abcdefgh'), size=n), 'housing': g.choice(['yes', 'no'], size=n),
                       'age': g.integers(18, 90, size=n).astype(float), 'balance': g.normal(1000, 500, size=n)})
    y = ((df['housing'] == 'yes') * 2.0 + (df['age'] - 50) / 20 + g.normal(size=n) * 0.3).values
    conf = deeptable.ModelConfig(nets=deepnets.DeepFM, embedding_dropout=0, metrics=['mse'], auto_scale=True,
                                 loss=LS.Huber(delta=0.5))
    dt = deeptable.DeepTable(config=conf)
    model, history = dt.fit(df, y, batch_size=128, epochs=2, verbose=0)
    assert model.model_desc.loss == 'huber(delta=0.5)'
    assert history.history['loss'][-1] < history.history['loss'][0]
    result = dt.evaluate(df, y, batch_size=512, verbose=0)
    dt.save(str(tmp_path / 'm'))
    dt2 = deeptable.DeepTable.load(str(tmp_path / 'm'))
    assert dt2.get_model().model_desc.loss == 'huber(delta=0.5)'
    again = dt2.evaluate(df, y, batch_size=512, verbose=0)
    assert again.keys() == result.keys()
    for k in result:              # the float64 loss sum adds the warps' partial sums in any order
        np.testing.assert_allclose(again[k], result[k], rtol=1e-9, err_msg=k)


# ---- 3. data parallel ------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        m, _ = _build('regression', LS.Huber(delta=0.5), seed=11)
        for step in range(6):
            m.train_on_batch(*_batch('regression', 64, seed=step * world + rank)[:3])
        m.sync_replica_buffers()
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), **{k: v.detach().cpu().numpy() for k, v in m.state_dict().items()})
    finally:
        dist.destroy_process_group()


def test_data_parallel_replicas_stay_bit_identical(tmp_path):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    r0, r1 = np.load(tmp_path / 'rank0.npz'), np.load(tmp_path / 'rank1.npz')
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]), f'replica 1 diverged from replica 0 on {k}'
