"""Columns of different embedding widths (fixed_embedding_dim=False), the parts that need no GPU: the CPU oracle
against tests/golden/reference_widths.npz (written by tests/golden/make_reference_widths_golden.py through the reference's
own DeepModel.__build_model), the nets that
refuse mixed widths, the preprocessor's widths, the padded table layout and the C ABI of the ragged kernels."""
import json
import os

import numpy as np
import pandas as pd
import pytest
import torch

from oracle import model_ref as M

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = dict(rtol=1e-9, atol=1e-11)

Z = np.load(os.path.join(HERE, 'golden', 'reference_widths.npz'))
MANIFEST = json.loads(str(Z['__manifest__']))
MODEL_CASES = [m for m in MANIFEST if m['kind'] == 'model']
REFUSALS = next(m for m in MANIFEST if m['kind'] == 'refusals')


def model_config(p):
    from deeptables_b200 import deeptable
    kw = dict(p['config'])
    if 'dnn_params' in kw:
        kw['dnn_params'] = dict(kw['dnn_params'], hidden_units=tuple(tuple(h) for h in kw['dnn_params']['hidden_units']))
    return deeptable.ModelConfig(embedding_dropout=0, dense_dropout=0, fixed_embedding_dim=False, **kw)


def weights(case):
    pre = f'{case}/w/'
    return {k[len(pre):]: torch.tensor(Z[k], dtype=torch.float64) for k in Z.files if k.startswith(pre)}


def test_fixture_inventory():
    assert {m['case'] for m in MODEL_CASES} >= {'dnn', 'dnn_bn', 'dcn', 'cross_dnn', 'cross_concat_dnn', 'dnn_no_cont'}
    for m in MODEL_CASES:
        assert len(set(m['params']['dims'])) > 1


@pytest.mark.parametrize('meta', MODEL_CASES, ids=[m['case'] for m in MODEL_CASES])
def test_oracle_reproduces_reference_at_mixed_widths(meta):
    case, p = meta['case'], meta['params']
    conf = model_config(p)
    state = weights(case)
    spec, _ = M.param_spec(conf, p['vocab'], p['dims'], p['n_cont'], p['task'], p['num_classes'] or 2)
    for name, shape, _ in spec:
        assert tuple(state[name].shape) == tuple(shape), name
    for i, (v, d) in enumerate(zip(p['vocab'], p['dims'])):
        assert tuple(state[f'emb_categorical_vars_all/embeddings_{i}'].shape) == (v, d)
    ids = torch.tensor(Z[f'{case}/ids'])
    cont = torch.tensor(Z[f'{case}/cont'], dtype=torch.float64) if p['n_cont'] else None
    for training, key in ((False, 'out_infer'), (True, 'out_train')):
        got, _ = M.forward(state, conf, ids, cont, len(p['vocab']), training, task=p['task'])
        np.testing.assert_allclose(got.numpy(), Z[f'{case}/{key}'], **TOL, err_msg=f'{case} training={training}')


def test_refused_nets_are_the_ones_the_reference_cannot_build():
    from deeptables_b200 import deepnets
    raises = Z['nets_at_mixed_widths/raises']
    ref = {n for n, r in zip(REFUSALS['params']['nets'], raises) if r}
    assert ref == set(deepnets.EQUAL_WIDTH_NETS)
    assert {'dnn_nets', 'cross_nets', 'cross_dnn_nets', 'dcn_nets'}.isdisjoint(ref)


def test_preprocessor_widths():
    from deeptables_b200 import deeptable
    from deeptables_b200.deeptable import DefaultPreprocessor
    g = np.random.default_rng(0)
    n = 400
    df = pd.DataFrame({'small': g.choice(list('abc'), size=n), 'mid': g.integers(0, 60, size=n).astype(str),
                       'big': g.integers(0, 300, size=n).astype(str), 'x': g.normal(size=n)})
    y = g.integers(0, 2, size=n)

    def widths(**kw):
        pre = DefaultPreprocessor(deeptable.ModelConfig(**kw))
        pre.fit_transform(df, y)
        return {c.name: (c.vocabulary_size, c.embeddings_output_dim) for c in pre.categorical_columns}

    # reference preprocessor.py:477-493: min(4 * int(V ** 0.25), 20) per column
    for name, (v, d) in widths(fixed_embedding_dim=False).items():
        assert d == min(4 * int(v ** 0.25), 20), name
    assert len({d for _, d in widths(fixed_embedding_dim=False).values()}) > 1
    assert {d for _, d in widths(embeddings_output_dim=6).values()} == {6}
    # a fixed width of 0 is the default width 4 (EMBEDDING_OUT_DIM_DEFAULT), not the fourth root of the vocabulary
    assert {d for _, d in widths(embeddings_output_dim=0).values()} == {4}


def test_padded_table_layout_on_the_host():
    from deeptables_b200.engine import EmbeddingTable
    g = torch.Generator().manual_seed(5)
    t = EmbeddingTable([7, 20, 5], 12, 'cpu', generator=g, field_dims=[4, 12, 3])
    assert t.ragged and t.dim == 12 and tuple(t.weight.shape) == (32, 12)
    assert tuple(t.field_weight(0).shape) == (7, 4) and tuple(t.field_weight(2).shape) == (5, 3)
    assert torch.equal(t.weight[0:7, 4:], torch.zeros(7, 8)) and torch.equal(t.weight[27:32, 3:], torch.zeros(5, 9))
    assert not torch.signbit(t.weight[0:7, 4:]).any()
    assert float(t.field_weight(1).abs().max()) <= 0.05 and float(t.field_weight(1).abs().min()) > 0
    assert t.padding_share() == pytest.approx((7 * 8 + 5 * 9) / (32 * 12))
    t.slot_inits = (0.1, None, None)
    t.ensure_training_state()
    assert torch.equal(t.grad, torch.zeros(32, 12)) and torch.equal(t.slots[0], torch.full((32, 12), 0.1))
    with pytest.raises(ValueError):
        EmbeddingTable([7, 20], 4, 'cpu', field_dims=[4, 8])
    # equal widths: the uniform table, same draws as without field_dims
    a = EmbeddingTable([7, 20], 8, 'cpu', generator=torch.Generator().manual_seed(1))
    b = EmbeddingTable([7, 20], 8, 'cpu', generator=torch.Generator().manual_seed(1), field_dims=[8, 8])
    assert not b.ragged and torch.equal(a.weight, b.weight) and b.field_weight(1).is_contiguous()


def test_ragged_symbols_are_declared_and_bound():
    from deeptables_b200 import _native
    for sym in ('dtb_ragged_concat_emb_dense_fwd', 'dtb_ragged_concat_emb_dense_bwd'):
        assert sym in _native.declared_symbols() and sym in _native._SIGNATURES and hasattr(_native.lib, sym)


def test_ragged_entry_points_refuse_bad_widths_without_a_gpu():
    """Argument checks run on the host before any launch."""
    import ctypes
    from deeptables_b200 import _native as nat
    p = ctypes.c_void_p(16)
    for dims, dmax in (([4, 9], 8), ([0, 4], 8), ([4] * 961, 4)):
        arr = nat.int_array(dims)
        assert nat.lib.dtb_ragged_concat_emb_dense_fwd(p, p, p, arr, None, p, 4, len(dims), dmax, 0, None, None) != 0
        assert nat.lib.dtb_ragged_concat_emb_dense_bwd(p, p, arr, p, p, 4, len(dims), dmax, 0, None) != 0
        assert 'invalid argument' in nat.last_error()
