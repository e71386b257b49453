"""Columns of different embedding widths (fixed_embedding_dim=False) on the GPU: the
model against the reference's own vectors and the oracle trainer, the padded table's invariants, the nets that refuse
mixed widths, embedding dropout, checkpoints, the public DeepTable surface and data parallel."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import optim_ref as R
from deeptables_b200 import optimizers as O

pytestmark = pytest.mark.gpu

HIDDEN = {'hidden_units': ((16, 0, False), (8, 0, False)), 'activation': 'relu'}


# ---- 1. the model ------------------------------------------------------------------------------------------------------
def build(nets, vocab, dims, n_cont, seed=9, task='binary', num_classes=2, **cfg_kw):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    kw = dict(nets=nets, fixed_embedding_dim=False, embedding_dropout=0, dnn_params=HIDDEN,
              cross_params={'num_cross_layer': 2})
    kw.update(cfg_kw)
    conf = deeptable.ModelConfig(**kw)
    cats = [CategoricalColumn(f'c{i}', v, d) for i, (v, d) in enumerate(zip(vocab, dims))]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(n_cont)])] if n_cont else []
    model = DeepModel(task, num_classes, conf, cats, conts, seed=seed)
    model._build_model()
    return model, conf


def batch(vocab, n_cont, b, seed=0):
    g = np.random.default_rng(seed)
    idx = np.stack([g.integers(0, v, size=b) for v in vocab], axis=1).astype(np.int32)
    cont = g.normal(size=(b, n_cont)).astype(np.float32)
    y = (g.random(b) < 0.35).astype(np.float32)
    return idx, cont, y


def _golden_cases():
    import test_widths_cpu as C
    return [(C, m) for m in C.MODEL_CASES]


@pytest.mark.parametrize('cm', _golden_cases(), ids=[m['case'] for _, m in _golden_cases()])
def test_model_reproduces_reference_at_mixed_widths(cm):
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    C, meta = cm
    case, p = meta['case'], meta['params']
    conf = C.model_config(p)
    cats = [CategoricalColumn(f'c{i}', v, d) for i, (v, d) in enumerate(zip(p['vocab'], p['dims']))]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(p['n_cont'])])] if p['n_cont'] else []
    model = DeepModel(p['task'], p['num_classes'], conf, cats, conts, seed=3)
    model._build_model()
    assert model.table.ragged and model.table.dim == max(p['dims'])
    assert f"output_dims: {p['dims']}" in str(model.model_desc)
    assert f"shape: (2, {sum(p['dims']) + p['n_cont']})" in str(model.model_desc)
    model.load_state_dict({k: v.to(torch.float32) for k, v in C.weights(case).items()}, strict=True)
    for i, d in enumerate(p['dims']):
        rows = model.table.weight[model.table.row_offsets_host[i]:model.table.row_offsets_host[i + 1]]
        assert not rows[:, d:].any()
    ids = torch.tensor(C.Z[f'{case}/ids'].astype(np.int32)).cuda()
    cont = torch.tensor(C.Z[f'{case}/cont'].astype(np.float32)).cuda() if p['n_cont'] else None
    got = model.predict_step(ids, cont).cpu().double().numpy()
    np.testing.assert_allclose(got, C.Z[f'{case}/out_infer'], rtol=1e-3, atol=1e-5)
    if p['task'] in ('binary', 'regression'):
        y = torch.zeros(got.shape[0], 1, device='cuda')
        got = model.train_step(ids, cont, y).detach().cpu().double().numpy()
        np.testing.assert_allclose(got, C.Z[f'{case}/out_train'], rtol=1e-3, atol=1e-5)


OPTS = {'adam': 'auto', 'sgd_momentum': O.SGD(learning_rate=0.05, momentum=0.9), 'rmsprop': O.RMSprop(momentum=0.9),
        'adagrad': O.Adagrad(learning_rate=0.05)}
WIDTHS = {'dmax16': [4, 16, 8, 12, 4], 'dmax20': [20, 4, 8, 3, 12]}      # row-wise (lazy) table update / dense sweep
VOCAB = [11, 7, 13, 5, 9]


@pytest.mark.parametrize('widths', list(WIDTHS))
@pytest.mark.parametrize('nets', [['dnn_nets'], ['dcn_nets']], ids=['dnn', 'dcn'])
@pytest.mark.parametrize('name', list(OPTS))
def test_training_matches_oracle(name, nets, widths):
    dims, n_cont, b = WIDTHS[widths], 3, 48
    model, conf = build(nets, VOCAB, dims, n_cont, optimizer=OPTS[name])
    assert model.table.lazy_adam == (widths == 'dmax16')
    spec = O.resolve(OPTS[name])
    state = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    ref = R.OptimRefTrainer(state, conf, len(VOCAB), optimizer=spec)
    losses_g, losses_r = [], []
    for step in range(8):
        idx, cont, y = batch(VOCAB, n_cont, b, seed=step)
        losses_g.append(model.train_on_batch(idx, cont, y))
        losses_r.append(ref.train_step(torch.tensor(idx), torch.tensor(cont), torch.tensor(y)))
    np.testing.assert_allclose(losses_g, losses_r, rtol=2e-3, atol=1e-5)
    tol = dict(rtol=1e-3, atol=2e-5) if spec.kind in ('sgd', 'adagrad') else dict(rtol=1e-2, atol=2e-4)
    new_state = model.state_dict()
    for k, v in ref.state.items():
        assert tuple(new_state[k].shape) == tuple(v.shape), k
        np.testing.assert_allclose(new_state[k].cpu().numpy(), v.numpy(), err_msg=k, **tol)
    _assert_padding_intact(model)


def _assert_padding_intact(model):
    """Padding columns: +0.0 in the weights, the gradient and Adam's m, v; the initial value in the other slots."""
    t = model.table
    if t.slot_inits is None:
        bufs, wants = [t.weight, t.grad, t.m, t.v], [0.0] * 4
    else:
        live = [(s, v) for s, v in zip(t.slots, t.slot_inits) if s is not None]
        bufs, wants = [t.weight, t.grad] + [s for s, _ in live], [0.0, 0.0] + [v for _, v in live]
    for i, d in enumerate(t.field_dims):
        lo, hi = t.row_offsets_host[i], t.row_offsets_host[i + 1]
        for buf, want in zip(bufs, wants):
            pad = buf[lo:hi, d:]
            assert torch.equal(pad, torch.full_like(pad, want)) and not torch.signbit(pad).any(), (i, want)


# Two rows per step and no id repeated inside a field: every table row then takes at most one gradient contribution and
# the dense backward kernels reduce at most two terms, so two runs of the same steps give the same bits (see
# test_optimizers_gpu.py).
SMALL_VOCAB = [400, 300, 500, 200]


def _distinct_batch(vocab, n_cont, b, seed):
    g = np.random.default_rng(seed)
    idx = np.stack([g.choice(v, size=b, replace=False) for v in vocab], axis=1).astype(np.int32)
    return idx, g.normal(size=(b, n_cont)).astype(np.float32), (g.random(b) < 0.35).astype(np.float32)


def _train(optimizer, steps, model=None, dims=(4, 16, 8, 12), nets=('dnn_nets',), mode=None, **extra):
    if model is None:
        model, _ = build(list(nets), SMALL_VOCAB, list(dims), 2, optimizer=optimizer, **extra)
    model._table_mode_override = mode
    for step in range(model._step, model._step + steps):
        model.train_on_batch(*_distinct_batch(SMALL_VOCAB, 2, 2, seed=step))
    return model


def _states_equal(a, b, what):
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f'{what}: {k} differs'


@pytest.mark.parametrize('name', list(OPTS))
def test_cuda_graph_replay_is_bit_identical_to_eager(monkeypatch, name):
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    eager = _train(OPTS[name], 10, nets=('dcn_nets',))
    assert not eager._graphs
    monkeypatch.setenv('DTB_CUDA_GRAPH', '1')
    graphed = _train(OPTS[name], 10, nets=('dcn_nets',))
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    _states_equal(graphed, eager, f'{name}: graph replay vs eager')
    _assert_padding_intact(graphed)


@pytest.mark.parametrize('name', list(OPTS))
def test_lazy_and_dense_table_modes_give_identical_bits(monkeypatch, name):
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    lazy = _train(OPTS[name], 8, mode='lazy')
    dense = _train(OPTS[name], 8, mode='dense')
    assert lazy.table.lazy_active and not dense.table.lazy_active
    _states_equal(lazy, dense, f'{name}: lazy vs dense table update')
    _assert_padding_intact(lazy)
    _assert_padding_intact(dense)


# ---- 2. nets ------------------------------------------------------------------------------------------------------------
def test_equal_width_nets_are_refused_before_training():
    from deeptables_b200 import deepnets
    for nets in [[n] for n in sorted(deepnets.EQUAL_WIDTH_NETS)] + [deepnets.DeepFM, deepnets.xDeepFM, deepnets.PNN]:
        with pytest.raises(ValueError, match=r'needs one embedding width.*\[4, 16, 8, 12\]'):
            build(nets, SMALL_VOCAB, [4, 16, 8, 12], 2)
    for nets in (['dnn_nets'], ['cross_nets'], ['cross_dnn_nets'], ['dcn_nets'], deepnets.DCN):
        model, _ = build(nets, SMALL_VOCAB, [4, 16, 8, 12], 2)
        model.train_on_batch(*batch(SMALL_VOCAB, 2, 16))


def test_custom_net_sees_the_reference_shapes_and_gets_gradients():
    from deeptables_b200 import layers
    seen = {}

    def probe_nets(embeddings, flatten_emb_layer, dense_layer, concat_emb_dense, config, model_desc):
        seen['items'] = [tuple(e.shape) for e in embeddings]
        flat = flatten_emb_layer.reshape(flatten_emb_layer.shape[0], -1)
        seen['flat'] = tuple(flat.shape)
        x = layers.Concatenate(axis=-1)([e.reshape(e.shape[0], -1) for e in embeddings] + [flat])
        return layers.Dense(4, activation='relu', name='probe_dense')(x)

    dims = [4, 16, 8, 12]
    model, _ = build([probe_nets], SMALL_VOCAB, dims, 2)
    before = model.table.weight.clone()
    model.train_on_batch(*batch(SMALL_VOCAB, 2, 16))
    assert seen['items'] == [(16, 1, d) for d in dims] and seen['flat'] == (16, sum(dims))
    assert not torch.equal(before, model.table.weight)
    _assert_padding_intact(model)
    out = model.apply({**{f'c{i}': np.zeros(5, np.int32) for i in range(4)}, 'n0': np.zeros(5), 'n1': np.zeros(5)},
                      ['flatten_embeddings', 'concat_embedding_dense'])
    assert out[0].shape == (5, sum(dims)) and out[1].shape == (5, sum(dims) + 2)
    for i, d in enumerate(dims):
        c0 = sum(dims[:i])
        np.testing.assert_array_equal(out[0][:, c0:c0 + d], np.tile(model.table.field_weight(i)[0].cpu().numpy(), (5, 1)))


def test_embedding_dropout_trains_and_is_off_at_inference():
    model, conf = build(['dnn_nets'], SMALL_VOCAB, [4, 16, 8, 12], 2, embedding_dropout=0.3)
    losses = [model.train_on_batch(*batch(SMALL_VOCAB, 2, 64, seed=s)) for s in range(6)]
    assert np.isfinite(losses).all() and not model._graphs
    _assert_padding_intact(model)
    idx, cont, _ = batch(SMALL_VOCAB, 2, 32, seed=99)
    ids, xc = torch.tensor(idx, device='cuda'), torch.tensor(cont, device='cuda')
    a, b = model.predict_step(ids, xc), model.predict_step(ids, xc)
    assert torch.equal(a, b)
    same, _ = build(['dnn_nets'], SMALL_VOCAB, [4, 16, 8, 12], 2, embedding_dropout=0.0)
    same.load_state_dict(model.state_dict())
    assert torch.equal(same.predict_step(ids, xc), a)
    flat = model.apply({**{f'c{i}': idx[:, i] for i in range(4)}, 'n0': cont[:, 0], 'n1': cont[:, 1]},
                       ['flatten_embeddings'])
    assert flat.shape == (32, 40)


# ---- 3. checkpoints ------------------------------------------------------------------------------------------------------
def test_save_load_round_trips_per_column_shapes(tmp_path):
    from deeptables_b200.deepmodel import DeepModel
    src = _train('auto', 3)
    path = str(tmp_path / 'ck.npz')
    src.save(path)
    with np.load(path) as z:
        for i, (v, d) in enumerate(zip(SMALL_VOCAB, [4, 16, 8, 12])):
            assert z[f'emb_categorical_vars_all/embeddings_{i}'].shape == (v, d)
        assert z['__adam_table_m__'].shape == (sum(SMALL_VOCAB), 16)
    back = DeepModel('binary', 2, src.config, src.categorical_columns, src.continuous_columns, model_file=path, seed=77)
    _states_equal(back, src, 'reloaded')
    _assert_padding_intact(back)


@pytest.mark.parametrize('name', list(OPTS))
def test_checkpoint_resume_is_bit_identical(monkeypatch, tmp_path, name):
    from deeptables_b200.deepmodel import DeepModel
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    straight = _train(OPTS[name], 6)
    first = _train(OPTS[name], 3)
    path = str(tmp_path / 'ck.npz')
    first.save(path)
    resumed = DeepModel('binary', 2, first.config, first.categorical_columns, first.continuous_columns,
                        model_file=path, seed=123)
    assert resumed._step == 3
    _train(OPTS[name], 3, model=resumed)
    _states_equal(resumed, straight, f'{name}: save after 3 steps, load, 3 more')


# ---- 4. public API -------------------------------------------------------------------------------------------------------
def test_deeptable_fit_with_per_column_widths(tmp_path):
    from deeptables_b200 import deeptable
    g = np.random.default_rng(0)
    n = 3000
    df = pd.DataFrame({'two': g.choice(['a', 'b'], size=n), 'small': g.choice(list('abcdefgh'), size=n),
                       'mid': g.integers(0, 120, size=n).astype(str), 'big': g.integers(0, 2000, size=n).astype(str),
                       'x': g.normal(size=n), 'z': g.exponential(size=n)})
    logit = (df['two'] == 'a') * 1.5 + df['x'] - (df['small'] == 'c') * 2 + 0.2
    y = np.where(g.random(n) < 1 / (1 + np.exp(-logit)), 'yes', 'no')
    conf = deeptable.ModelConfig(fixed_embedding_dim=False, metrics=['AUC'], auto_scale=True, earlystopping_patience=5)
    dt = deeptable.DeepTable(config=conf)
    model, history = dt.fit(df, y, batch_size=128, epochs=5, verbose=0)
    dims = [c.embeddings_output_dim for c in dt.preprocessor.categorical_columns]
    assert len(set(dims)) > 1 and model.table.ragged
    result = dt.evaluate(df, y, batch_size=512, verbose=0)
    assert result['AUC'] > 0.6
    proba = dt.predict_proba(df.head(100))
    assert proba.shape[0] == 100 and np.isfinite(proba).all()
    dt.save(str(tmp_path / 'm'))
    dt2 = deeptable.DeepTable.load(str(tmp_path / 'm'))
    np.testing.assert_allclose(dt2.predict_proba(df.head(100)), proba, rtol=1e-5, atol=1e-6)


# ---- 5. data parallel ------------------------------------------------------------------------------------------------------
DP_VOCAB, DP_DIMS, DP_CONT, DP_B = [50, 40, 30, 20, 60], [4, 8, 16, 12, 4], 3, 64


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out_dir, table_mode):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        m, _ = build(['dcn_nets'], DP_VOCAB, DP_DIMS, DP_CONT, seed=11, optimizer=O.RMSprop(momentum=0.9))
        m._table_mode_override = table_mode
        for step in range(6):
            m.train_on_batch(*batch(DP_VOCAB, DP_CONT, DP_B, seed=step * world + rank))
        m.sync_replica_buffers()
        _assert_padding_intact(m)
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), **{k: v.detach().cpu().numpy() for k, v in m.state_dict().items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('table_mode', [None, 'lazy'])
def test_data_parallel_replicas_stay_bit_identical(tmp_path, table_mode):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path), table_mode), nprocs=world, join=True)
    r0, r1 = np.load(tmp_path / 'rank0.npz'), np.load(tmp_path / 'rank1.npz')
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]), f'replica 1 diverged from replica 0 on {k}'
