"""Dropout on the GPU: the attention kernels with dropout on the softmax weights against a float64 statement built
from the documented mask, the mask's statistics and its independence of batch slices, device-memory seeds against host
seeds, CUDA-graph replay of dropout train steps against eager steps, inference, DeepTable.fit and data parallel."""
import math
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import dropout_ref as D

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


def rnd(*shape, seed):
    return torch.tensor(np.random.default_rng(seed).normal(size=shape).astype(np.float32), device='cuda')


def att_fwd(nat, x, heads, res, rate, seed, seed_dev=None, row_offset=0):
    b, f, d4 = x.shape
    y = torch.empty(b, f, d4 // 4, device='cuda')
    nat.check(nat.lib.dtb_attention_core_dropout_fwd(nat.ptr(x), nat.ptr(y), b, f, d4 // 4, heads, res, rate, seed,
                                                     nat.ptr(seed_dev), row_offset, None))
    return y


def att_bwd(nat, x, y, dy, heads, res, mask_in, rate, seed, seed_dev=None, row_offset=0):
    b, f, d4 = x.shape
    dq = torch.empty_like(x)
    nat.check(nat.lib.dtb_attention_core_dropout_bwd(nat.ptr(x), nat.ptr(y), nat.ptr(dy), nat.ptr(dq), b, f, d4 // 4,
                                                     heads, res, mask_in, rate, seed, nat.ptr(seed_dev), row_offset, None))
    return dq


def att_ref(x, dy, heads, res, mask_in, keep, scale):
    """float64: softmax -> mask * scale -> . V -> + R -> relu, and autograd's gradient w.r.t. [Q|K|V|R] (mask_in: of
    the pre-relu projections, zero where the relu output is zero)"""
    b, f, d4 = x.shape
    d, dh = d4 // 4, d4 // 4 // heads
    x64 = x.double().cpu().requires_grad_(True)
    q, k, v, r = x64.split(d, dim=2)

    def per_head(t):
        return t.reshape(b, f, heads, dh).permute(0, 2, 1, 3)

    w = torch.softmax(per_head(q) @ per_head(k).transpose(-1, -2) / math.sqrt(dh), dim=-1)
    w = w * torch.tensor(keep, dtype=torch.float64) * float(scale)
    out = (w @ per_head(v)).permute(0, 2, 1, 3).reshape(b, f, d)
    if res:
        out = out + r
    y = torch.relu(out)
    y.backward(dy.double().cpu())
    g = x64.grad
    if mask_in:
        g = g * (x64.detach() > 0)
    return y.detach().numpy(), g.numpy()


# ---- 1. the attention kernels against float64 --------------------------------------------------------------------------------
# heads * F <= 256 threads and D % 4 == 0: the kernels with the head width as a template parameter (D / heads = 2 .. 32)
T_SHAPES = [(d, h, f) for d in (8, 16, 32) for h in (1, 2, 4) for f in (3, 26)]
# the any-shape kernels: D % 4 != 0; more than 256 (head, field) threads; heads of 64 (template forward, any-shape backward)
G_SHAPES = [(6, 3, 5), (16, 8, 39), (64, 1, 4)]


@pytest.mark.parametrize('rate', [0.1, 0.5])
@pytest.mark.parametrize('res', [0, 1])
@pytest.mark.parametrize('d,heads,f', T_SHAPES + G_SHAPES)
def test_attention_dropout_matches_float64(nat, d, heads, f, res, rate):
    b, seed = 37, 0x5EED00000000 + d * 1000 + heads * 100 + f
    for mask_in in (0, 1):
        x = rnd(b, f, 4 * d, seed=d + heads + f + mask_in)
        if mask_in:
            x = torch.relu(x)
        dy = rnd(b, f, d, seed=99)
        keep = D.attention_keep(seed, rate, b, heads, f)
        y_ref, g_ref = att_ref(x, dy, heads, res, mask_in, keep, D.scale(rate))
        y = att_fwd(nat, x, heads, res, rate, seed)
        g = att_bwd(nat, x, y, dy, heads, res, mask_in, rate, seed)
        np.testing.assert_allclose(y.cpu().numpy(), y_ref, rtol=2e-4, atol=2e-5)
        np.testing.assert_allclose(g.cpu().numpy(), g_ref, rtol=2e-4, atol=5e-5)
        assert 0 < keep.mean() < 1


@pytest.mark.parametrize('d,heads,f', [(32, 4, 26), (16, 2, 3), (6, 3, 5), (64, 1, 4)])
def test_rate_zero_is_bit_identical_to_the_entry_points_without_dropout(nat, d, heads, f):
    b = 300
    x, dy = torch.relu(rnd(b, f, 4 * d, seed=1)), rnd(b, f, d, seed=2)
    y0, g0 = torch.empty(b, f, d, device='cuda'), torch.empty_like(x)
    nat.check(nat.lib.dtb_attention_core_fwd(nat.ptr(x), nat.ptr(y0), b, f, d, heads, 1, None))
    nat.check(nat.lib.dtb_attention_core_bwd(nat.ptr(x), nat.ptr(y0), nat.ptr(dy), nat.ptr(g0), b, f, d, heads, 1, 1, None))
    y = att_fwd(nat, x, heads, 1, 0.0, 123)
    g = att_bwd(nat, x, y, dy, heads, 1, 1, 0.0, 123)
    assert torch.equal(y, y0) and torch.equal(g, g0)


def test_attention_dropout_refuses_a_bad_rate(nat):
    x = rnd(2, 3, 32, seed=1)
    y = torch.empty(2, 3, 8, device='cuda')
    for rate in (-0.5, 1.0):
        assert nat.lib.dtb_attention_core_dropout_fwd(nat.ptr(x), nat.ptr(y), 2, 3, 8, 2, 1, rate, 1, None, 0, None) != 0
        assert 'rate' in nat.last_error()


# ---- 2. a batch and its slices draw the same bits ----------------------------------------------------------------------------
@pytest.mark.parametrize('d,heads,f', [(32, 4, 26), (16, 2, 5), (16, 8, 39)])
def test_batch_equals_its_slices_with_the_row_offset(nat, d, heads, f):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    rows_per_cta = max(1, 128 // (heads * f))
    b = sm * 8 * rows_per_cta * 2 + 77                   # every CTA makes more than two passes over the batch
    rate, seed = 0.3, 2024
    x, dy = torch.relu(rnd(b, f, 4 * d, seed=3)), rnd(b, f, d, seed=4)
    y = att_fwd(nat, x, heads, 1, rate, seed)
    g = att_bwd(nat, x, y, dy, heads, 1, 1, rate, seed)
    for lo, hi in ((0, 41), (41, b // 2), (b // 2, b)):
        ys = att_fwd(nat, x[lo:hi], heads, 1, rate, seed, row_offset=lo)
        gs = att_bwd(nat, x[lo:hi], ys, dy[lo:hi], heads, 1, 1, rate, seed, row_offset=lo)
        assert torch.equal(ys, y[lo:hi]) and torch.equal(gs, g[lo:hi]), f'rows {lo}:{hi}'
    assert not torch.equal(att_fwd(nat, x[41:82], heads, 1, rate, seed), y[41:82]), 'the row offset is not used'


# ---- 3. statistics of the mask -----------------------------------------------------------------------------------------------
def _weights(nat, b, f, rate, seed):
    """The dropped attention weights themselves: one head of width 32 >= F, V = the identity, no residual."""
    d = 32
    x = torch.zeros(b, f, 4 * d, device='cuda')
    x[:, :, :2 * d] = 0.3 * rnd(b, f, 2 * d, seed=5)
    x[:, :, 2 * d:2 * d + f] = torch.eye(f, device='cuda')
    return att_fwd(nat, x, 1, 0, rate, seed)[:, :, :f]


@pytest.mark.parametrize('rate', [0.1, 0.5])
def test_mask_statistics_and_scale(nat, rate):
    b, f = 1600, 26                                       # 1 081 600 weights
    w = _weights(nat, b, f, 0.0, 0)
    assert float(w.min()) > 0
    wd = _weights(nat, b, f, rate, 777)
    kept = wd > 0
    n = kept.numel()
    p = 1.0 - int(D.threshold(rate)) / 2 ** 32
    assert abs(int(kept.sum()) / n - p) < 4 * math.sqrt(p * (1 - p) / n)
    assert np.array_equal(kept.cpu().numpy(), D.attention_keep(777, rate, b, 1, f)[:, 0])
    # a kept weight is the float product of the weight and 1 / (1 - rate)
    assert torch.equal(wd[kept], w[kept] * float(D.scale(rate)))
    assert torch.equal(wd, _weights(nat, b, f, rate, 777))
    other = _weights(nat, b, f, rate, 778) > 0
    assert abs(float((other == kept).float().mean()) - (p * p + (1 - p) * (1 - p))) < 0.01


# ---- 4. seeds in device memory -----------------------------------------------------------------------------------------------
def test_device_seed_forms_give_the_bits_of_the_host_seed_forms(nat):
    seeds = [0, 1, 0xFFFFFFFFFFFF, 123456789012345]
    dev = torch.tensor(seeds, dtype=torch.int64, device='cuda')
    x = rnd(100003, seed=6)
    xa, dy = torch.relu(rnd(500, 26, 128, seed=7)), rnd(500, 26, 32, seed=8)
    for k, s in enumerate(seeds):
        y0, y1 = torch.empty_like(x), torch.empty_like(x)
        nat.check(nat.lib.dtb_dropout(nat.ptr(x), nat.ptr(y0), x.numel(), 0.3, s, None))
        nat.check(nat.lib.dtb_dropout_dev(nat.ptr(x), nat.ptr(y1), x.numel(), 0.3, nat.ptr(dev[k:]), None))
        assert torch.equal(y0, y1)
        assert np.array_equal((y0 != 0).cpu().numpy(), D.keep(s, np.arange(x.numel()), 0.3) & (x != 0).cpu().numpy())
        a0 = att_fwd(nat, xa, 4, 1, 0.1, s)
        a1 = att_fwd(nat, xa, 4, 1, 0.1, 999, seed_dev=dev[k:])         # the pointer wins over the value
        assert torch.equal(a0, a1)
        assert torch.equal(att_bwd(nat, xa, a0, dy, 4, 1, 1, 0.1, s), att_bwd(nat, xa, a0, dy, 4, 1, 1, 0.1, 999, dev[k:]))
    assert nat.lib.dtb_dropout_dev(nat.ptr(x), nat.ptr(x), x.numel(), 0.3, None, None) != 0


def test_seed_advance_adds_the_number_of_sites_modulo_2_to_the_48(nat):
    vals = [5, 0xFFFFFFFFFFFF, 0xFFFFFFFFFFFF - 2, 42]
    dev = torch.tensor(vals, dtype=torch.int64, device='cuda')
    nat.check(nat.lib.dtb_seed_advance(nat.ptr(dev), 4, None))
    assert dev.tolist() == [(v + 4) & D.SEED_MASK for v in vals] == [9, 3, 1, 46]


# ---- model-level helpers -----------------------------------------------------------------------------------------------------
def build(nets, vocab, dim, n_cont, seed=5, **cfg_kw):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    kw = dict(nets=nets, embeddings_output_dim=dim, embedding_dropout=0.3, dense_dropout=0.2, metrics=['AUC'],
              dnn_params={'hidden_units': ((16, 0.25, False), (8, 0.1, True)), 'activation': 'relu'},
              cin_params={'cross_layer_size': (8, 6), 'activation': 'relu', 'use_residual': False,
                          'use_bias': False, 'direct': False, 'reduce_D': False},
              autoint_params={'num_attention': 2, 'num_heads': 2, 'dropout_rate': 0.1, 'use_residual': True},
              afm_params={'attention_factor': 4, 'dropout_rate': 0.2})
    kw.update(cfg_kw)
    conf = deeptable.ModelConfig(**kw)
    cats = [CategoricalColumn(f'c{i}', v, dim) for i, v in enumerate(vocab)]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(n_cont)])] if n_cont else []
    model = DeepModel('binary', 2, conf, cats, conts, seed=seed)
    model._build_model()
    return model, conf


def distinct_batch(vocab, n_cont, b, seed):
    """rows without repeated ids: the table gradient has no atomics to reorder"""
    g = np.random.default_rng(seed)
    idx = np.stack([g.choice(v, size=b, replace=False) for v in vocab], axis=1).astype(np.int32)
    cont = g.normal(size=(b, n_cont)).astype(np.float32)
    y = (g.random(b) < 0.35).astype(np.float32)
    return idx, cont, y


def states_equal(a, b, what):
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f'{what}: {k} differs'


VOCAB, DIM, N_CONT, ROWS = [400, 300, 500, 350], 8, 2, 2
# dropout call sites of one training pass: the embedding block, the dense input, the DNN layers, AFM, attention layers
NETS = {
    'deepfm': (['linear', 'fm_nets', 'dnn_nets'], 4),
    'xdeepfm': (['cin_nets', 'dnn_nets'], 4),
    'autoint': (['autoint_nets'], 4),
    'afm': (['afm_nets'], 3),
}


def _run(nets, steps, grow_at=None):
    """`steps` train steps; returns the model, every step's predictions and losses.  grow_at: before that step the
    rate table is cut back to the steps done, so that it grows (and moves) again."""
    model, _ = build(nets, VOCAB, DIM, N_CONT)
    probs, losses, graphs = [], [], []
    for step in range(steps):
        if step == grow_at:
            model._rates.host = model._rates.host[:model._step + 1]
        idx, cont, y = distinct_batch(VOCAB, N_CONT, ROWS, seed=step)
        ti, tc = torch.tensor(idx).cuda(), torch.tensor(cont).cuda()
        ty = torch.tensor(y).cuda().view(-1, 1)
        model._loss_acc.zero_()
        probs.append(model.train_step(ti, tc, ty).clone())
        losses.append(float(model._loss_acc.item()))
        graphs.append([e[0] for e in model._graphs.values()])
    return model, probs, losses, graphs


@pytest.mark.parametrize('grow_at', [None, 5], ids=['plain', 'rate_table_grows'])
@pytest.mark.parametrize('name', list(NETS))
def test_graph_replay_of_dropout_steps_is_bit_identical_to_eager(monkeypatch, name, grow_at):
    nets, sites = NETS[name]
    steps = 9
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    eager, pe, le, _ = _run(nets, steps, grow_at)
    assert not eager._graphs and eager._scope.seed_sites == sites
    assert eager._scope._seed_counter == steps * sites
    monkeypatch.setenv('DTB_CUDA_GRAPH', '1')
    graphed, pg, lg, graphs = _run(nets, steps, grow_at)
    assert graphed._graphs and not graphed._graph_failed, 'the train step was not captured'
    assert graphs[2] and graphs[2] == graphs[4], 'steps after the capture were not replays of it'
    if grow_at is not None:
        assert graphs[grow_at][0] is not graphs[grow_at - 1][0], 'the step was not captured again'
    for step, (a, b) in enumerate(zip(pg, pe)):
        assert torch.equal(a, b), f'{name}: predictions of step {step}'
    assert lg == le
    states_equal(graphed, eager, f'{name}: graph replay vs eager')
    assert graphed._scope._seed_counter == eager._scope._seed_counter
    # the masks change from step to step: the same batch twice gives different training predictions
    idx, cont, y = distinct_batch(VOCAB, N_CONT, ROWS, seed=0)
    args = (torch.tensor(idx).cuda(), torch.tensor(cont).cuda(), torch.tensor(y).cuda().view(-1, 1))
    assert not torch.equal(graphed.train_step(*args).clone(), graphed.train_step(*args))


def test_fit_history_of_a_dropout_model_is_the_same_with_and_without_graph_replay(monkeypatch):
    parts = [distinct_batch(VOCAB, N_CONT, ROWS, seed) for seed in range(8)]
    idx, cont, y = (np.concatenate([p[k] for p in parts]) for k in range(3))
    X = pd.DataFrame({**{f'c{i}': idx[:, i] for i in range(len(VOCAB))}, **{f'n{i}': cont[:, i] for i in range(N_CONT)}})
    runs = {}
    for graphs in ('0', '1'):
        monkeypatch.setenv('DTB_CUDA_GRAPH', graphs)
        model, _ = build(['linear', 'fm_nets', 'dnn_nets', 'autoint_nets'], VOCAB, DIM, N_CONT)
        history = model.fit(X, y, batch_size=ROWS, epochs=3, verbose=0, shuffle=False, validation_data=(X.head(4), y[:4]))
        runs[graphs] = (model, history.history)
    (eager, he), (graphed, hg) = runs['0'], runs['1']
    assert graphed._graphs and not graphed._graph_failed and not eager._graphs
    assert he['loss'] == hg['loss'] and he['val_loss'] == hg['val_loss']
    states_equal(graphed, eager, 'fit: graph replay vs eager')


# ---- 6. inference ignores dropout --------------------------------------------------------------------------------------------
def test_inference_ignores_every_dropout_rate():
    nets = ['linear', 'fm_nets', 'dnn_nets', 'autoint_nets', 'afm_nets']
    with_dropout, _ = build(nets, VOCAB, DIM, N_CONT, autoint_params={'num_attention': 2, 'num_heads': 2,
                                                                      'dropout_rate': 0.3, 'use_residual': True})
    without, _ = build(nets, VOCAB, DIM, N_CONT, embedding_dropout=0, dense_dropout=0,
                       dnn_params={'hidden_units': ((16, 0, False), (8, 0, True)), 'activation': 'relu'},
                       autoint_params={'num_attention': 2, 'num_heads': 2, 'dropout_rate': 0, 'use_residual': True},
                       afm_params={'attention_factor': 4, 'dropout_rate': 0})
    states_equal(with_dropout, without, 'same seed, same initial weights')
    idx, cont, y = distinct_batch(VOCAB, N_CONT, 200, seed=1)
    X = pd.DataFrame({**{f'c{i}': idx[:, i] for i in range(len(VOCAB))}, **{f'n{i}': cont[:, i] for i in range(N_CONT)}})
    assert np.array_equal(with_dropout.predict(X), without.predict(X))
    assert dict(with_dropout.evaluate(X, y)) == dict(without.evaluate(X, y))
    ti, tc, ty = torch.tensor(idx).cuda(), torch.tensor(cont).cuda(), torch.tensor(y).cuda().view(-1, 1)
    assert not torch.equal(with_dropout.train_step(ti, tc, ty), without.train_step(ti, tc, ty))


# ---- 7. public surface -------------------------------------------------------------------------------------------------------
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


def test_deeptable_fit_autoint_with_attention_dropout_and_default_embedding_dropout(tmp_path):
    from deeptables_b200 import deeptable, deepnets
    df, y = _frame(3000)
    conf = deeptable.ModelConfig(nets=deepnets.AutoInt, metrics=['AUC'], auto_scale=True, earlystopping_patience=100,
                                 autoint_params={'num_attention': 3, 'num_heads': 2, 'dropout_rate': 0.1,
                                                 'use_residual': True})
    assert conf.embedding_dropout == 0.3
    dt = deeptable.DeepTable(config=conf)
    model, history = dt.fit(df, y, batch_size=128, epochs=8, verbose=0)
    loss = history.history['loss']
    assert np.isfinite(loss).all() and loss[-1] < loss[0]
    assert model._graphs and not model._graph_failed, 'the dropout train step was not replayed as a graph'
    assert np.isfinite(dt.evaluate(df, y, batch_size=512, verbose=0)['AUC'])
    proba = dt.predict_proba(df.head(100))
    dt.save(str(tmp_path / 'm'))
    dt2 = deeptable.DeepTable.load(str(tmp_path / 'm'))
    np.testing.assert_allclose(dt2.predict_proba(df.head(100)), proba, rtol=1e-5, atol=1e-6)


# ---- 8. data parallel --------------------------------------------------------------------------------------------------------
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
        vocab = [50, 40, 30, 20, 60]
        m, _ = build(['linear', 'fm_nets', 'dnn_nets', 'autoint_nets'], vocab, 8, 3, seed=11)
        g = np.random.default_rng(100 + rank)
        for step in range(6):
            idx = np.stack([g.integers(0, v, size=64) for v in vocab], axis=1).astype(np.int32)
            m.train_on_batch(idx, g.normal(size=(64, 3)).astype(np.float32), (g.random(64) < 0.35).astype(np.float32))
        m.sync_replica_buffers()
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), **{k: v.detach().cpu().numpy() for k, v in m.state_dict().items()})
    finally:
        dist.destroy_process_group()


def test_data_parallel_replicas_stay_bit_identical_with_dropout(tmp_path):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    r0, r1 = np.load(tmp_path / 'rank0.npz'), np.load(tmp_path / 'rank1.npz')
    for k in r0.files:
        assert np.array_equal(r0[k], r1[k]), f'replica 1 diverged from replica 0 on {k}'
