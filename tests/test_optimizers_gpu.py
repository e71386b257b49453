"""SGD, RMSprop and Adagrad on the GPU, and Adam at other hyperparameters: the dense sweep against the float64 oracle,
the exact-lazy row form bit-identical to the dense sweep, DeepModel training against the oracle trainer, the lazy /
dense table switch, CUDA-graph replay, checkpoints, the public DeepTable surface and data parallel."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import optim_ref as R
from deeptables_b200 import optimizers as O

pytestmark = pytest.mark.gpu

# the eight dense-sweep variants (learning rates large enough that 20 steps move the weights far beyond fp32 noise)
VARIANTS = {
    'sgd': O.SGD(learning_rate=0.05),
    'sgd_momentum': O.SGD(learning_rate=0.05, momentum=0.9),
    'sgd_nesterov': O.SGD(learning_rate=0.05, momentum=0.9, nesterov=True),
    'rmsprop': O.RMSprop(learning_rate=0.01),
    'rmsprop_momentum': O.RMSprop(learning_rate=0.01, momentum=0.9),
    'rmsprop_centered': O.RMSprop(learning_rate=0.01, centered=True),
    'rmsprop_centered_momentum': O.RMSprop(learning_rate=0.01, momentum=0.9, centered=True),
    'adagrad': O.Adagrad(learning_rate=0.1),
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


# ---- 1. dense sweep vs the float64 oracle ---------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(VARIANTS))
@pytest.mark.parametrize('n,off', [(1003, 0), (1003, 1), (1002, 2), (4099, 3)])
def test_dense_sweep_matches_oracle(nat, name, n, off):
    """n % 4 != 0 runs the scalar tail behind the float4 sweep; buffers at +1/+2/+3 floats run the scalar kernel."""
    spec = O.resolve(VARIANTS[name])
    hp = _hp(spec)
    gen = np.random.default_rng(n + off)

    def buf(vals):
        t = torch.zeros(n + 4, dtype=torch.float32, device='cuda')[off:off + n]
        return t.copy_(torch.as_tensor(np.asarray(vals, dtype=np.float32)))

    p0 = gen.normal(size=n).astype(np.float32)
    p, g = buf(p0), buf(np.zeros(n))
    slots = [None if s is None else buf(np.full(n, s)) for s in O.slot_inits(spec)]
    pr = torch.tensor(p0, dtype=torch.float64)
    sr = R.new_slots(spec, pr)
    for t in range(1, 21):
        gg = gen.normal(size=n).astype(np.float32)
        gg[gen.random(n) < 0.2] = 0.0                 # elements without a gradient this step
        if t in (6, 13):
            gg[:] = 0.0                               # whole zero-gradient steps
        g.copy_(torch.as_tensor(gg))
        nat.check(nat.lib.dtb_optim_dense(*_ptrs([p, g] + slots), n, hp, 1, None), 'optim_dense')
        R.step(spec, pr, torch.tensor(gg, dtype=torch.float64), sr, t)
    torch.cuda.synchronize()
    assert bool((g == 0).all()), 'the gradient is zeroed behind the sweep'
    # fp32 arithmetic against float64: relative error ~1e-6 per step, far below one step (>= 1e-3 here)
    np.testing.assert_allclose(p.cpu().numpy(), pr.numpy(), rtol=1e-5, atol=1e-5, err_msg=f'{name}: p')
    for k, (s, r) in enumerate(zip(slots, sr)):
        if s is not None:
            np.testing.assert_allclose(s.cpu().numpy(), r.numpy(), rtol=1e-5, atol=1e-6, err_msg=f'{name}: slot {k}')


def test_dense_sweep_refuses_missing_slots(nat):
    p = torch.zeros(8, device='cuda')
    rc = nat.lib.dtb_optim_dense(*_ptrs([p, p, None, None, None]), 8, _hp(O.resolve(O.RMSprop(momentum=0.9))), 1, None)
    assert rc != 0 and 'RMSprop needs slot s0' in nat.last_error()


# ---- 2. row form vs dense sweep: bit-identical ----------------------------------------------------------------------
GAP_STEPS = 5060


def _rows_schedule(s):
    """ids [4, 2] of step s over fields of 40 and 30 rows: row 0 every step (twice: a duplicate id), row 5 at steps 1,
    51 and 5051 (gaps of 50 and 5 000), row 7 at steps 2 and 5060, field 1 cycling through its rows, out-of-range ids
    (40 in field 0, -1 in field 1) in every step, and field-0 rows that are never touched."""
    return np.array([[0, s % 30],
                     [0, -1],
                     [5 if s in (1, 51, 5051) else 40, s % 2],
                     [7 if s in (2, GAP_STEPS) else 0, 29 - s % 30]], dtype=np.int32)


@pytest.mark.parametrize('name', list(VARIANTS))
def test_row_form_is_bit_identical_to_dense_sweep(nat, name):
    spec = O.resolve(VARIANTS[name])
    hp = _hp(spec)
    vocab, d = [40, 30], 8
    rows = sum(vocab)
    offs = torch.tensor([0, 40, 70], dtype=torch.int64, device='cuda')
    gen = np.random.default_rng(7)
    w0 = torch.tensor(gen.normal(scale=0.05, size=(rows, d)).astype(np.float32), device='cuda')
    w0[3] = 0.0                                        # a never-touched row at 0
    inits = O.slot_inits(spec)

    def state():
        return w0.clone(), [None if s is None else torch.full((rows, d), s, device='cuda') for s in inits], \
            torch.zeros(rows, d, device='cuda')

    (wd, sd, gd), (wh, sh, gh), (wv, sv, gv) = state(), state(), state()
    last_h = torch.zeros(rows, dtype=torch.int32, device='cuda')
    last_v = torch.zeros(rows, dtype=torch.int32, device='cuda')
    step_dev = torch.zeros(1, dtype=torch.int32, device='cuda')
    lo = [0, 40]
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
        nat.check(nat.lib.dtb_optim_dense(*_ptrs([wd, gd] + sd), rows * d, hp, 1, None), 'optim_dense')
        nat.check(nat.lib.dtb_optim_rows_catchup(*_ptrs([idx, offs, wh] + sh + [last_h]), s - 1, hp, 4, 2, d, None))
        nat.check(nat.lib.dtb_optim_rows_apply(*_ptrs([idx, offs, wh] + sh + [gh, last_h]), s, hp, 4, 2, d, None))
        step_dev.fill_(s - 1)
        nat.check(nat.lib.dtb_optim_rows_catchup_dev(*_ptrs([idx, offs, wv] + sv + [last_v, step_dev]), hp, 4, 2, d, None))
        nat.check(nat.lib.dtb_optim_rows_apply_dev(*_ptrs([idx, offs, wv] + sv + [gv, last_v, step_dev]), hp, 4, 2, d,
                                                   None))
        if s in (2, 52, 5051, GAP_STEPS):               # the rows a step touched are current right after it
            for b, f in np.ndindex(*ids.shape):
                if 0 <= ids[b, f] < vocab[f]:
                    r = lo[f] + int(ids[b, f])
                    assert torch.equal(wh[r], wd[r]) and torch.equal(wv[r], wd[r]), f'{name}: row {r} at step {s}'
    nat.check(nat.lib.dtb_optim_rows_flush(*_ptrs([wh] + sh + [last_h]), GAP_STEPS, hp, rows, d, None))
    step_dev.fill_(GAP_STEPS)
    nat.check(nat.lib.dtb_optim_rows_flush_dev(*_ptrs([wv] + sv + [last_v, step_dev]), hp, rows, d, None))
    torch.cuda.synchronize()
    assert not torch.equal(wd, w0)
    assert bool((gh == 0).all()) and bool((gv == 0).all())
    for label, w, sl in (('host', wh, sh), ('dev', wv, sv)):
        assert torch.equal(w, wd), f'{name}: {label} row form weights differ from the dense sweep'
        for k, (a, b) in enumerate(zip(sl, sd)):
            if a is not None:
                assert torch.equal(a, b), f'{name}: {label} row form slot {k} differs from the dense sweep'


# ---- model-level helpers ---------------------------------------------------------------------------------------------
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


MODEL_OPTS = {'sgd': 'sgd', 'sgd_nesterov': O.SGD(momentum=0.9, nesterov=True), 'rmsprop': 'rmsprop',
              'rmsprop_centered_momentum': O.RMSprop(momentum=0.9, centered=True), 'adagrad': 'adagrad'}


# ---- 3. DeepModel vs the oracle trainer -----------------------------------------------------------------------------
@pytest.mark.parametrize('nets', [['linear', 'fm_nets', 'dnn_nets'], ['linear', 'cin_nets', 'dnn_nets']])
@pytest.mark.parametrize('name', list(MODEL_OPTS))
def test_training_matches_oracle(nets, name):
    _training_matches_oracle(nets, MODEL_OPTS[name])


def _training_matches_oracle(nets, optimizer):
    vocab, dim, n_cont, b = [11, 7, 13, 5, 9], 4, 3, 48
    model, conf = build(nets, vocab, dim, n_cont, optimizer=optimizer)
    spec = O.resolve(optimizer)
    assert model.model_desc.optimizer == spec.keras_name
    state = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    ref = R.OptimRefTrainer(state, conf, len(vocab), optimizer=spec)
    losses_g, losses_r = [], []
    for step in range(8):
        idx, cont, y = batch(vocab, n_cont, b, seed=step)
        losses_g.append(model.train_on_batch(idx, cont, y))
        losses_r.append(ref.train_step(torch.tensor(idx), torch.tensor(cont), torch.tensor(y)))
    np.testing.assert_allclose(losses_g, losses_r, rtol=2e-3, atol=1e-5)
    if spec.kind in ('sgd', 'adagrad'):
        # SGD and Adagrad steps are proportional to the gradient: an fp32 gradient error of ~1e-5 relative moves a
        # weight by ~1e-5 of its (<= 1e-2) total displacement, so the weights agree far more tightly than Adam's
        tol = dict(rtol=1e-3, atol=2e-5)
    else:
        # Adam and RMSprop normalise the step (g / sqrt(v)): a tiny gradient with an fp32 error still takes an O(lr)
        # step, so compare against lr * steps, as for Adam (test_model_gpu)
        tol = dict(rtol=1e-2, atol=2e-4)
    new_state = model.state_dict()
    for k, v in ref.state.items():
        np.testing.assert_allclose(new_state[k].cpu().numpy(), v.numpy(), err_msg=k, **tol)


# ---- 4. Adam -----------------------------------------------------------------------------------------------------------
# Two rows per step for the bit-identity tests below.  The backward kernels reduce over batch rows with fp32 atomics in
# scheduling order (e.g. the linear-weight gradient of fm_linear_bwd: one warp per row, atomicAdd into shared memory),
# so two runs of the same steps on 8 rows can differ in the last bit before any optimiser runs.  With at most two
# nonzero terms per zero-initialised accumulator every order gives the same sum (a + b == b + a), so the runs compared
# here compute the same gradients and any difference would be the optimiser's or the graph's.
SMALL = dict(nets=['linear', 'fm_nets', 'dnn_nets'], vocab=[400, 300, 500], dim=4, n_cont=2, b=2)


def _distinct_batch(vocab, n_cont, b, seed):
    """Like batch(), but no id repeats within a field: the backward kernels scatter-add into the table gradient with
    fp32 atomics, and a table row that takes two contributions on top of another op's could sum them in either order.
    With one contribution per table row and op (and two rows per batch, see SMALL), two runs of the same steps give
    the same bits."""
    g = np.random.default_rng(seed)
    idx = np.stack([g.choice(v, size=b, replace=False) for v in vocab], axis=1).astype(np.int32)
    cont = g.normal(size=(b, n_cont)).astype(np.float32)
    y = (g.random(b) < 0.35).astype(np.float32)
    return idx, cont, y


def _train(optimizer, steps, model=None, seed=9, **extra):
    s = SMALL
    if model is None:
        model, _ = build(s['nets'], s['vocab'], s['dim'], s['n_cont'], seed=seed, optimizer=optimizer, **extra)
    for step in range(model._step, model._step + steps):
        model.train_on_batch(*_distinct_batch(s['vocab'], s['n_cont'], s['b'], seed=step))
    return model


def _states_equal(a, b, what):
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f'{what}: {k} differs'


def test_adam_by_name_and_instance_is_auto(monkeypatch):
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    auto = _train('auto', 8)
    for opt in ('adam', 'Adam', O.Adam()):
        _states_equal(_train(opt, 8), auto, repr(opt))


def test_adam_hyperparameters_match_oracle():
    _training_matches_oracle(['linear', 'fm_nets', 'dnn_nets'],
                             O.Adam(learning_rate=3e-3, beta_1=0.8, beta_2=0.99, epsilon=1e-6))


# ---- 5. lazy / dense table switch ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('optimizer', [O.SGD(momentum=0.9), O.RMSprop(momentum=0.9, centered=True), 'adagrad'],
                         ids=['sgd_momentum', 'rmsprop_centered_momentum', 'adagrad'])
def test_lazy_and_dense_table_switch_is_transparent(optimizer):
    vocab, n_cont, b = [400, 300, 500], 2, 32
    results = {}
    for name, schedule in (('lazy', ['lazy'] * 8), ('dense', ['dense'] * 8),
                           ('mixed', ['lazy', 'lazy', 'dense', 'dense', 'lazy', 'dense', 'lazy', 'lazy'])):
        model, conf = build(['linear', 'fm_nets', 'dnn_nets'], vocab, 4, n_cont, seed=9, optimizer=optimizer)
        modes = []
        for step, mode in enumerate(schedule):
            model._table_mode_override = mode
            model.train_on_batch(*batch(vocab, n_cont, b, seed=step))
            modes.append(model.table.lazy_active)
        assert modes == [m == 'lazy' for m in schedule]
        results[name] = {k: v.clone() for k, v in model.state_dict().items()}
    for k in results['lazy']:
        for other in ('dense', 'mixed'):
            torch.testing.assert_close(results['lazy'][k], results[other][k], rtol=1e-5, atol=1e-7, msg=f'{other}:{k}')


# ---- 6. CUDA graphs -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(MODEL_OPTS))
def test_cuda_graph_replay_is_bit_identical_to_eager(monkeypatch, name):
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    eager = _train(MODEL_OPTS[name], 10)
    assert not eager._graphs
    monkeypatch.setenv('DTB_CUDA_GRAPH', '1')
    graphed = _train(MODEL_OPTS[name], 10)
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    _states_equal(graphed, eager, f'{name}: graph replay vs eager')


# ---- 7. checkpoints ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', list(MODEL_OPTS))
def test_checkpoint_resume_is_bit_identical(monkeypatch, tmp_path, name):
    from deeptables_b200.deepmodel import DeepModel
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    opt = MODEL_OPTS[name]
    straight = _train(opt, 6)
    first = _train(opt, 3)
    path = str(tmp_path / 'ck.npz')
    first.save(path)
    resumed = DeepModel('binary', 2, first.config, first.categorical_columns, first.continuous_columns,
                        model_file=path, seed=123)
    assert resumed._step == 3
    _train(opt, 3, model=resumed)
    _states_equal(resumed, straight, f'{name}: save after 3 steps, load, 3 more')


def test_checkpoint_of_another_optimizer_restarts_at_step_zero(tmp_path):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    src = _train(O.SGD(momentum=0.9), 3)
    path = str(tmp_path / 'ck.npz')
    src.save(path)
    for other in (O.RMSprop(momentum=0.9), O.SGD(momentum=0.5), 'auto'):
        conf = deeptable.ModelConfig(**{**src.config._asdict(), 'optimizer': other})
        m = DeepModel('binary', 2, conf, src.categorical_columns, src.continuous_columns, model_file=path)
        assert m._step == 0, repr(other)
        _states_equal(m, src, f'{other!r}: weights still load')
    same = DeepModel('binary', 2, src.config, src.categorical_columns, src.continuous_columns, model_file=path)
    assert same._step == 3


# ---- 8. public API ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('optimizer', ['rmsprop', O.RMSprop()], ids=['name', 'instance'])
def test_deeptable_fit_with_rmsprop(tmp_path, optimizer):
    """The reference's example trains with optimizer=keras.optimizers.RMSprop()."""
    from deeptables_b200 import deeptable, deepnets
    g = np.random.default_rng(0)
    n = 3000
    df = pd.DataFrame({
        'job': g.choice(list('abcdefghijkl'), size=n), 'marital': g.choice(['m', 's', 'd'], size=n),
        'education': g.choice(['p', 's', 't', 'u'], size=n), 'default': g.choice(['yes', 'no'], size=n),
        'housing': g.choice(['yes', 'no'], size=n), 'contact': g.choice(['c', 't', 'u'], size=n),
        'age': g.integers(18, 90, size=n).astype(float), 'balance': g.normal(1000, 500, size=n),
        'duration': g.exponential(200, size=n), 'campaign': g.integers(1, 10, size=n).astype(float),
    })
    logit = (df['housing'] == 'yes') * 1.5 + (df['duration'] - 200) / 150 + (df['job'] == 'a') * 2 - 1
    y = np.where(g.random(n) < 1 / (1 + np.exp(-logit)), 'yes', 'no')
    conf = deeptable.ModelConfig(nets=deepnets.DeepFM, embedding_dropout=0, metrics=['AUC'], auto_scale=True,
                                 earlystopping_patience=5, optimizer=optimizer)
    dt = deeptable.DeepTable(config=conf)
    model, history = dt.fit(df, y, batch_size=128, epochs=6, verbose=0)
    assert model.model_desc.optimizer == 'RMSprop'
    result = dt.evaluate(df, y, batch_size=512, verbose=0)
    assert result['AUC'] > 0.62
    proba = dt.predict_proba(df.head(100))
    dt.save(str(tmp_path / 'm'))
    dt2 = deeptable.DeepTable.load(str(tmp_path / 'm'))
    np.testing.assert_allclose(dt2.predict_proba(df.head(100)), proba, rtol=1e-5, atol=1e-6)


# ---- 9. data parallel ------------------------------------------------------------------------------------------------------
DP_VOCAB, DP_DIM, DP_CONT, DP_B = [50, 40, 30, 20, 60], 8, 3, 64
DP_OPTS = {'rmsprop_momentum': O.RMSprop(momentum=0.9), 'sgd_momentum': O.SGD(momentum=0.9)}


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_build(optimizer):
    model, _ = build(['linear', 'fm_nets', 'cin_nets', 'dnn_nets'], DP_VOCAB, DP_DIM, DP_CONT, seed=11,
                     optimizer=optimizer, cin_params={'cross_layer_size': (16, 16), 'activation': 'relu',
                                                      'use_residual': False, 'use_bias': False, 'direct': False,
                                                      'reduce_D': False})
    return model


def _dp_worker(rank, world, port, out_dir, same_shard, table_mode, opt_name):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        m = _dp_build(DP_OPTS[opt_name])
        m._table_mode_override = table_mode          # None: adaptive; 'lazy': row-wise update of the union of ids
        for step in range(6):
            m.train_on_batch(*batch(DP_VOCAB, DP_CONT, DP_B, seed=step if same_shard else step * world + rank))
        m.sync_replica_buffers()
        sd = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), **sd)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('opt_name', list(DP_OPTS))
@pytest.mark.parametrize('table_mode', [None, 'lazy'])
@pytest.mark.parametrize('same_shard', [True, False])
def test_data_parallel_replicas_stay_bit_identical(tmp_path, opt_name, table_mode, same_shard):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path), same_shard, table_mode, opt_name), nprocs=world,
             join=True)
    r0 = np.load(tmp_path / 'rank0.npz')
    r1 = np.load(tmp_path / 'rank1.npz')
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]), f'replica 1 diverged from replica 0 on {k}'
    if same_shard:
        single = _dp_build(DP_OPTS[opt_name])
        for step in range(6):
            single.train_on_batch(*batch(DP_VOCAB, DP_CONT, DP_B, seed=step))
        sd = single.state_dict()
        for k in r0.files:
            np.testing.assert_allclose(r0[k], sd[k].cpu().numpy(), rtol=1e-4, atol=1e-6, err_msg=k)
