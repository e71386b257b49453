"""Denoising auto-encoder (fe.dae) on the GPU: dtb_dae_swap_batch bit for bit against dae_ref, one train step's gradient
against float64 autograd, CUDA-graph replay against eager launches, determinism, the reference's callbacks, the features
and a learning check."""
import numpy as np
import pytest
import torch

import dae_ref
from deeptables_b200 import _native as N, optimizers as O, schedules as S
from deeptables_b200._native import ptr, stream_ptr
from deeptables_b200.fe.dae import DAE

pytestmark = pytest.mark.gpu

LR = 2.0 ** 10            # SGD learning rate: g * LR is exact in float32 (tests/test_model_grads_gpu.py)
RTOL = 1e-4               # gradient bar, relative to max |g64| of the tensor
LOSS_RTOL = 1e-5
TAU = 3e-5                # a relu input within TAU * max |input| of its layer of zero may flip in float32


def _swap(X, p1, p2, step, first, batch_rows, rows, k, seed, graph=False):
    cols = X.shape[1]
    x_in = torch.full((rows, cols), -7.0, device='cuda')
    x_tgt = torch.full((rows, cols), -7.0, device='cuda')
    step_dev = torch.tensor([step], dtype=torch.int32, device='cuda')
    first_dev = torch.tensor([first], dtype=torch.int32, device='cuda')

    def launch():
        N.check(N.lib.dtb_dae_swap_batch(ptr(X), cols, ptr(p1), ptr(p2 if k else None), ptr(step_dev), ptr(first_dev),
                                         batch_rows, rows, k, seed, ptr(x_in), ptr(x_tgt), stream_ptr()),
                'dae_swap_batch')
    if graph:
        step_dev.fill_(0)                       # captured with another step: the replay must read the counter
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            launch()
        x_in.fill_(-7.0)
        x_tgt.fill_(-7.0)
        step_dev.fill_(step)
        g.replay()
    else:
        launch()
    torch.cuda.synchronize()
    return x_in.cpu().numpy(), x_tgt.cpu().numpy()


@pytest.mark.parametrize('rows,cols,k', [(1, 1, 0), (1, 1, 1), (128, 37, 5), (128, 200, 30), (4096, 221, 33),
                                         (7, 5000, 750), (64, 64, 64)])
def test_swap_batch_is_bit_exact(rows, cols, k):
    g = np.random.default_rng(rows * 7919 + cols * 31 + k)
    n = 3 * rows + 5
    X = g.random((n, cols), dtype=np.float32)
    p1, p2 = g.permutation(n), g.permutation(n)
    Xd = torch.from_numpy(X).cuda()
    p1d, p2d = torch.from_numpy(p1).cuda(), torch.from_numpy(p2).cuda()
    seed = 0xC0FFEE ^ (rows * cols)
    # (step, epoch's first step, batch rows): base 0, base = 2 batches in, and a partial batch at base 1 * batch_rows
    for step, first, batch_rows, r in ((0, 0, rows, rows), (9, 7, rows, rows), (1000, 999, rows + 2, rows)):
        want_in, want_tgt = dae_ref.swap_batch(X, p1, p2, step, first, batch_rows, r, k, seed)
        got_in, got_tgt = _swap(Xd, p1d, p2d, step, first, batch_rows, r, k, seed)
        np.testing.assert_array_equal(got_tgt, want_tgt)
        np.testing.assert_array_equal(got_in, want_in)
        if k:
            changed = (want_in != want_tgt).sum(axis=1)
            assert (changed <= k).all()
    rg_in, rg_tgt = _swap(Xd, p1d, p2d, 9, 7, rows, rows, k, seed, graph=True)
    e_in, e_tgt = _swap(Xd, p1d, p2d, 9, 7, rows, rows, k, seed)
    np.testing.assert_array_equal(rg_in, e_in)
    np.testing.assert_array_equal(rg_tgt, e_tgt)


def test_swap_batch_with_k_zero_and_x_in_copies_the_clean_rows():
    X = torch.rand(20, 9, device='cuda')
    p1 = torch.randperm(20, device='cuda')
    x_in, x_tgt = _swap(X, p1, None, 3, 2, 8, 8, 0, 5)
    np.testing.assert_array_equal(x_in, x_tgt)
    np.testing.assert_array_equal(x_tgt, X[p1[8:16]].cpu().numpy())


def test_swap_batch_refuses_bad_arguments():
    X = torch.rand(4, 3, device='cuda')
    p = torch.arange(4, device='cuda')
    s = torch.zeros(1, dtype=torch.int32, device='cuda')
    out = torch.empty(4, 3, device='cuda')
    for args in ((3, ptr(p), None, 4, 4, 1),      # k > 0 without donors
                 (3, ptr(p), ptr(p), 4, 4, 0),    # donors with k == 0
                 (3, ptr(p), ptr(p), 4, 4, 4),    # k > cols
                 (3, ptr(p), None, 2, 4, 0)):     # rows > batch_rows
        cols, p1, p2, batch_rows, rows, k = args
        rc = N.lib.dtb_dae_swap_batch(ptr(X), cols, p1, p2, ptr(s), ptr(s), batch_rows, rows, k, 1, ptr(out), ptr(out),
                                      stream_ptr())
        assert rc != 0


# ---- the gradient of one train step ---------------------------------------------------------------------------------
def _forward64(weights, plan, x, upto=None, record=None):
    for name, _, _, act in plan:
        z = x @ weights[f'{name}/kernel'] + weights[f'{name}/bias']
        if record is not None and act == 'relu':
            record.append(z.detach())
        x = torch.relu(z) if act == 'relu' else torch.tanh(z) if act == 'tanh' else z
        if name == upto:
            break
    return x


GRAD_CASES = {
    # feature_units=4 takes the narrow Dense kernels, the wider layers the wgmma ones; the relu cases have few enough
    # relu inputs per batch that one of the seeded batches has none within rounding of zero
    'relu_narrow_feature_odd_m': dict(encoder_units=(0, 64, 96), feature_units=4, activation='relu', cols=37, rows=24),
    'tanh_wide': dict(encoder_units=(500, 128), feature_units=64, activation='tanh', cols=65, rows=96),
    'linear_narrow_feature': dict(encoder_units=(1, 72, 80), feature_units=4, activation='linear', cols=33, rows=96),
    'relu_reference_shape': dict(encoder_units=(500, 500), feature_units=20, activation='relu', cols=29, rows=16),
}


@pytest.mark.parametrize('name', list(GRAD_CASES))
def test_train_step_gradient_matches_float64_autograd(name):
    c = dict(GRAD_CASES[name])
    cols, rows = c.pop('cols'), c.pop('rows')
    for data_seed in range(32):
        X = np.random.default_rng(data_seed).random((rows, cols), dtype=np.float32)
        dae = DAE(optimizer=O.SGD(learning_rate=LR), random_state=11, **c)
        ae0 = dae.build_dae(X)
        w0 = {k: v.double().clone() for k, v in ae0.weights.items()}
        rec = []
        x64 = torch.from_numpy(X).double().cuda()
        _forward64(w0, ae0.plan, x64, record=rec)
        if all((z.abs() > TAU * z.abs().max()).all() for z in rec):
            break
    else:
        pytest.fail('no batch without a relu input at rounding distance of zero')
    ae = dae.fit(X, batch_size=rows, epochs=1)       # one step over every row: the loss does not depend on the order
    w64 = {k: v.clone().requires_grad_(True) for k, v in w0.items()}
    out = _forward64(w64, ae.plan, x64)
    loss = ((out - x64) ** 2).mean(dim=1).mean()
    loss.backward()
    loss = float(loss.detach())
    assert abs(ae.history.history['loss'][0] - loss) <= LOSS_RTOL * loss
    assert ae.history.history['mse'] == ae.history.history['loss']
    for k, w1 in ae.weights.items():
        g = (w0[k] - w1.double()) / LR
        g64 = w64[k].grad
        bar = RTOL * float(g64.abs().max())
        err = float((g - g64).abs().max())
        assert err <= bar, f'{name}: {k}: max |g - g64| {err:.3e} > {bar:.3e}'


# ---- replay, determinism, callbacks, features --------------------------------------------------------------------------
# The Dense weight gradients and the loss sum add float partial sums with atomics across blocks, so bits repeat from run
# to run only where every reduction of a step stays in one block: the runs compared bit for bit use 8-row batches.
def _noisy_fit(monkeypatch, graphs, seed=3):
    monkeypatch.setenv('DTB_CUDA_GRAPH', graphs)
    X = np.random.default_rng(0).random((60, 23), dtype=np.float32)
    dae = DAE(encoder_units=(0, 48), feature_units=6, noise_rate=0.15, random_state=seed)
    return dae.fit(X, batch_size=8, epochs=3), X                  # 8 steps per epoch, the last one of 4 rows


def test_graph_replay_is_bit_identical_to_eager(monkeypatch):
    eager, _ = _noisy_fit(monkeypatch, '0')
    assert not eager._graphs
    replayed, _ = _noisy_fit(monkeypatch, '1')
    assert sorted(replayed._graphs) == [4, 8] and not replayed._graph_failed
    assert replayed._step == eager._step == 24
    assert replayed.history.history == eager.history.history
    for k, v in eager.weights.items():
        assert torch.equal(v, replayed.weights[k]), k


def _small(seed, call='fit_transform'):
    X = np.random.default_rng(1).random((60, 17), dtype=np.float32)
    dae = DAE(encoder_units=(0, 32), feature_units=5, noise_rate=0.2, random_state=seed)
    return getattr(dae, call)(X, batch_size=8, epochs=2), X


def test_same_random_state_gives_the_same_features():
    a, b, c = _small(5)[0], _small(5)[0], _small(6)[0]
    assert a.dtype == np.float32 and a.shape == (60, 5)
    np.testing.assert_array_equal(a, b)
    assert not np.array_equal(a, c)
    ae, X = _small(5, 'fit')
    np.testing.assert_array_equal(ae.apply(X, 'feature_layer', batch_size=8), a)


def test_callbacks_stop_cut_the_rate_and_restore():
    X = np.zeros((64, 6), dtype=np.float32)
    ae = DAE(encoder_units=(0, 16), feature_units=4, kernel_initializer='zeros', random_state=1).fit(
        X, batch_size=16, epochs=50)
    h = ae.history.history
    assert ae.history.epoch == list(range(6)) and ae.stop_training
    assert h['mse'] == [0.0] * 6 and h['loss'] == h['mse']
    np.testing.assert_allclose(h['learning_rate'], [1e-3] * 4 + [5e-4] * 2, rtol=1e-6)
    assert ae.optimizer.learning_rate == pytest.approx(5e-4, rel=1e-6)
    for k, v in ae.weights.items():
        assert not v.any(), k


def test_epochs_zero_trains_nothing():
    X = np.random.default_rng(2).random((40, 5), dtype=np.float32)
    dae = DAE(encoder_units=(0, 16), feature_units=3, random_state=4)
    ae = dae.fit(X, epochs=0)
    assert ae._step == 0 and ae.history.history == {}
    for k, v in dae.build_dae(X).weights.items():
        assert torch.equal(v, ae.weights[k])


def test_features_match_the_float64_encoder():
    X = np.random.default_rng(3).random((1000, 31), dtype=np.float32)
    ae = DAE(encoder_units=(500, 300, 200), feature_units=12, noise_rate=0.1, random_state=8).fit(
        X, batch_size=256, epochs=2)
    assert ae.name == 'AE' and list(ae.weights)[:2] == ['encoder_0/kernel', 'encoder_0/bias']
    assert list(ae.weights)[-1] == 'output_layer/bias'
    assert ae.count_params() == sum(i * o + o for _, i, o, _ in ae.plan)
    feats = ae.apply(X, 'feature_layer', batch_size=256)
    assert feats.dtype == np.float32 and feats.shape == (1000, 12)
    w = {k: v.double() for k, v in ae.weights.items()}
    want = _forward64(w, ae.plan, torch.from_numpy(X).double().cuda(), upto='feature_layer').cpu().numpy()
    np.testing.assert_allclose(feats, want, atol=1e-4 * np.abs(want).max(), rtol=0)
    rec = ae.predict(X)
    want = _forward64(w, ae.plan, torch.from_numpy(X).double().cuda()).cpu().numpy()
    assert rec.shape == X.shape and rec.dtype == np.float32
    np.testing.assert_allclose(rec, want, atol=1e-4 * np.abs(want).max(), rtol=0)
    with pytest.raises(ValueError, match='No such layer'):
        ae.apply(X, 'nope')


@pytest.mark.parametrize('opt', ['sgd', 'rmsprop', 'adagrad',
                                 O.Adam(learning_rate=S.ExponentialDecay(1e-3, decay_steps=10, decay_rate=0.9))],
                         ids=['sgd', 'rmsprop', 'adagrad', 'adam_schedule'])
def test_every_optimizer_trains(opt):
    X = np.random.default_rng(5).random((256, 12), dtype=np.float32)
    ae = DAE(encoder_units=(0, 32), feature_units=4, optimizer=opt, random_state=2).fit(X, batch_size=32, epochs=3)
    mse = ae.history.history['mse']
    assert len(mse) == 3 and np.isfinite(mse).all()
    assert ae._graphs and not ae._graph_failed


def test_learning_on_rank_5_data():
    g = np.random.default_rng(6)
    X = (g.random((4096, 5)) @ g.random((5, 40)) / 5).astype(np.float32)
    assert 0 <= X.min() and X.max() <= 1
    ae = DAE(feature_units=8, noise_rate=0.1, random_state=9).fit(X, batch_size=128, epochs=20)
    mse = ae.history.history['mse']
    assert min(mse) < 0.3 * mse[0], mse          # 0.14 on an H100
