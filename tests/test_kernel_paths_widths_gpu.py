"""The ragged flatten / concat kernels for columns of different embedding widths (fixed_embedding_dim=False): the
forward is a bit-exact gather on the fast and the generic path, out-of-range ids set the status bits, the backward
matches float64 and leaves the padding alone, and the profiler names the kernel each shape runs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def nat():
    from deeptables_b200 import _native
    return _native


# ---- kernels --------------------------------------------------------------------------------------------------------
def _table(vocab, dims, dmax, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    w = torch.rand(sum(vocab), dmax, device='cuda', generator=g) - 0.5
    offs = np.cumsum([0] + list(vocab))
    for i, d in enumerate(dims):
        w[offs[i]:offs[i + 1], d:] = 0.0
    return w, torch.tensor(offs, dtype=torch.int64, device='cuda'), offs


def _ids(vocab, b, seed, dup=False):
    g = np.random.default_rng(seed)
    hi = [min(v, 3) if dup else v for v in vocab]           # dup: few distinct ids, many repeats per table row
    return np.stack([g.integers(0, h, size=b) for h in hi], axis=1).astype(np.int32)


def _np_concat(w, offs, dims, ids, dense):
    w = w.cpu().numpy()
    parts = [w[offs[i] + ids[:, i], :d] for i, d in enumerate(dims)]
    if dense is not None:
        parts.append(dense.cpu().numpy())
    return np.concatenate(parts, axis=1)


def _fwd(nat, w, offs_d, dims, ids_d, dense, status=None):
    b, f = ids_d.shape
    c = 0 if dense is None else dense.shape[1]
    x = torch.full((b, sum(dims) + c), float('nan'), device='cuda')
    p = nat.ptr
    nat.check(nat.lib.dtb_ragged_concat_emb_dense_fwd(p(ids_d), p(w), p(offs_d), nat.int_array(dims), p(dense), p(x), b,
                                                      f, w.shape[1], c, p(status), nat.stream_ptr()), 'ragged fwd')
    return x


SHAPES = {                       # name: (vocab, dims, Dmax, C)
    'fast_c0': ([50, 40, 300, 7, 90], [4, 8, 12, 16, 20], 20, 0),
    'fast_c13': ([50, 40, 300, 7, 90], [4, 8, 12, 16, 20], 20, 13),
    'fast_c4': ([50, 40, 300], [8, 4, 16], 16, 4),                   # row stride % 4 == 0: 16-byte stores
    'generic_c0': ([50, 40, 300, 7], [3, 5, 4, 1], 5, 0),
    'generic_c13': ([50, 40, 300, 7], [3, 5, 4, 1], 5, 13),
    'generic_dmax_odd': ([11, 9], [4, 8], 9, 3),                      # widths % 4 == 0 but Dmax is not
    'criteo_like': ([1460, 583, 10131227 // 1000, 2202608 // 1000, 305, 24, 12517, 633, 3, 93145 // 100, 5683, 8351 // 10,
                     3194, 27, 14992, 5461 // 10, 10, 5652, 2173, 4, 7046 // 10, 18, 15, 286181 // 100, 105, 142572 // 100],
                    None, None, 13),
}


def _shape(name):
    vocab, dims, dmax, c = SHAPES[name]
    if dims is None:
        dims = [min(4 * int(v ** 0.25), 20) for v in vocab]
        dmax = max(dims)
    return vocab, dims, dmax, c


@pytest.mark.parametrize('name', list(SHAPES))
def test_forward_is_a_bit_exact_gather(nat, name):
    vocab, dims, dmax, c = _shape(name)
    w, offs_d, offs = _table(vocab, dims, dmax, seed=1)
    ids = _ids(vocab, 301, seed=2)
    dense = torch.randn(301, c, device='cuda') if c else None
    status = torch.zeros(1, dtype=torch.int32, device='cuda')
    x = _fwd(nat, w, offs_d, dims, torch.tensor(ids, device='cuda'), dense, status)
    torch.cuda.synchronize()
    assert np.array_equal(x.cpu().numpy(), _np_concat(w, offs, dims, ids, dense))
    assert int(status.item()) == 0


@pytest.mark.parametrize('name', ['fast_c13', 'generic_c13'])
def test_out_of_range_ids_set_status_bits_and_read_zero(nat, name):
    vocab, dims, dmax, c = _shape(name)
    w, offs_d, offs = _table(vocab, dims, dmax, seed=3)
    ids = _ids(vocab, 64, seed=4)
    ids[5, 1] = vocab[1]            # one past the end
    ids[9, 3] = -1
    dense = torch.randn(64, c, device='cuda')
    status = torch.zeros(1, dtype=torch.int32, device='cuda')
    x = _fwd(nat, w, offs_d, dims, torch.tensor(ids, device='cuda'), dense, status).cpu().numpy()
    assert int(status.item()) == (1 << 1) | (1 << 3)
    safe = ids.copy()
    safe[5, 1] = safe[9, 3] = 0
    want = _np_concat(w, offs, dims, safe, dense)
    cols = np.cumsum([0] + dims)
    want[5, cols[1]:cols[2]] = 0.0
    want[9, cols[3]:cols[4]] = 0.0
    assert np.array_equal(x, want)


@pytest.mark.parametrize('name', ['fast_c13', 'fast_c4', 'generic_c13', 'generic_dmax_odd', 'criteo_like'])
def test_backward_matches_float64_and_leaves_padding_alone(nat, name):
    vocab, dims, dmax, c = _shape(name)
    b = 513
    ids = _ids(vocab, b, seed=5, dup=True)
    ids_d = torch.tensor(ids, device='cuda')
    dx = torch.randn(b, sum(dims) + c, device='cuda')
    grad = torch.zeros(sum(vocab), dmax, device='cuda')
    p = nat.ptr
    nat.check(nat.lib.dtb_ragged_concat_emb_dense_bwd(p(ids_d), p(torch.tensor(np.cumsum([0] + vocab), device='cuda')),
                                                      nat.int_array(dims), p(dx), p(grad), b, len(vocab), dmax, c,
                                                      nat.stream_ptr()), 'ragged bwd')
    want = np.zeros((sum(vocab), dmax))
    offs, cols, g = np.cumsum([0] + vocab), np.cumsum([0] + dims), dx.double().cpu().numpy()
    for i, d in enumerate(dims):
        np.add.at(want, (offs[i] + ids[:, i], slice(0, d)), g[:, cols[i]:cols[i + 1]])
    got = grad.cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)
    for i, d in enumerate(dims):
        pad = got[offs[i]:offs[i + 1], d:]
        assert np.array_equal(pad, np.zeros_like(pad)) and not np.signbit(pad).any()


def _ragged_kernels(fn):
    from torch.profiler import profile, ProfilerActivity
    for _ in range(2):              # a profiler session occasionally records no device activity: profile once more
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if 'ragged_concat' in e.name}
        if names:
            return names
    return names


@pytest.mark.parametrize('name,vec', [('fast_c13', 4), ('fast_c4', 4), ('generic_c13', 1), ('generic_dmax_odd', 1),
                                      ('criteo_like', 4)])
def test_profiler_names_the_ragged_kernel_each_shape_runs(nat, name, vec):
    vocab, dims, dmax, c = _shape(name)
    w, offs_d, _ = _table(vocab, dims, dmax, seed=6)
    ids_d = torch.tensor(_ids(vocab, 128, seed=7), device='cuda')
    dense = torch.randn(128, c, device='cuda') if c else None
    grad = torch.zeros_like(w)
    dx = torch.randn(128, sum(dims) + c, device='cuda')

    def run():
        _fwd(nat, w, offs_d, dims, ids_d, dense)
        nat.check(nat.lib.dtb_ragged_concat_emb_dense_bwd(nat.ptr(ids_d), nat.ptr(offs_d), nat.int_array(dims), nat.ptr(dx),
                                                          nat.ptr(grad), 128, len(dims), dmax, c, nat.stream_ptr()), 'bwd')
    names = _ragged_kernels(run)
    other = 1 if vec == 4 else 4
    assert any(f'ragged_concat_fwd_kernel<{vec}>' in n for n in names), names
    assert any(f'ragged_concat_bwd_kernel<{vec}>' in n for n in names), names
    assert not any(f'_kernel<{other}>' in n for n in names), names
