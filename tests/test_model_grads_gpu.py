"""The gradient of one real train step of the assembled model, for every trainable tensor, against float64 autograd of
the oracle model.

Most model-level checks elsewhere train with Adam, whose step m / sqrt(v) does not move when a gradient is scaled by a
constant, and run at toy shapes where the dispatch picks the small-shape kernels.  Here the model trains with SGD at a
power-of-two learning rate (momentum 0): sgd_update computes p - g * lr with an exact product, so (p_before - p_after) / lr
in float64 recovers the gradient g that `train_on_batch` applied -- the loss scaling, dp.scale_for_mean, the lazy or dense
table update and, from step 2 on, the captured CUDA graph included -- to within ulp(p_after) / (2 lr).  Every compared
step starts from the same restored snapshot of the weights and BatchNormalization statistics.

Bar, per tensor: max |g - g64| <= 1e-4 * max |g64|; the loss agrees to 1e-5 relative.  A float32 gradient that is small
through cancellation (a BatchNormalization beta feeding a Dense and another BatchNormalization is zero in exact arithmetic;
the AFM attention and SENET excitation kernels sum softmax- and mean-centred terms) carries the rounding error of its
terms, not of its result: a tensor's bar is RTOL of the larger of its own max |g64| and MODEL_SHARE of the model's
largest gradient, and neither bar goes below FP32_FLOOR times the error of the oracle's own float32 run of the same step
(which also reproduces float32's clip of probabilities at 1 - 1e-7 in the loss).  Each case also checks that the bar
rejects the float64 gradient of the same batch with one row's loss left out (the last row whose probability is not
clipped: a clipped row contributes no gradient).

An fp32 forward may take a relu or max decision the other way where the float64 input lies within rounding of the
threshold (oracle/layers_ref.py `recording`).  An entry is ambiguous when its margin is below TAU of its call's max
|input|.  A case picks, among BATCH_SEEDS seeded batches, the first without ambiguous entries and asserts there are none.
Where that is impractical -- at production shapes relu CIN, AutoInt, AFM and FGCNN, at toy shapes AFM over FGCNN's 21
fields -- the case may take the batch with the fewest instead, and the bar is widened element by element by
sum_i |delta_i|, delta_i being the first-order gradient contribution of ambiguous entry i (one float64 backward each); at
most MAX_WIDENED entries are allowed.  Relu inputs of exactly 0 and exact ties of a max come from exact
zeros or copies that the float32 forward reproduces, and are not ambiguous.

The cases at production shapes and the per-column-width cases also assert which of this library's kernels their train
step launched (recorded with torch.profiler in a child process, as tests/test_batch_passes_gpu.py explains), so that a
moved dispatch threshold cannot take a case off the path it is meant to check.
"""
import contextlib
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from deeptables_b200 import layers
from kernel_profile import launches, ran
from oracle import layers_ref as L
from oracle import model_ref as M
from test_model_gpu import NET_SETS

pytestmark = pytest.mark.gpu

LR = 2.0 ** 10            # SGD learning rate: g * LR is exact in float32
RTOL = 1e-4               # gradient bar, relative to max |g64| of the tensor
LOSS_RTOL = 1e-5
FP32_FLOOR = 10           # no bar below 10 x the rounding error of the oracle's own float32 run of the same step
MODEL_SHARE = 0.1         # no bar below RTOL x this share of the model's largest gradient
TAU = 3e-5                # ambiguous decision: margin below TAU * max |input| of its call
MAX_WIDENED = 64
BATCH_SEEDS = 32          # batches tried for a case that must have no ambiguous decision
DEV = 'cuda'              # where the float64 reference runs


# ---------------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------------
TOY_VOCAB, TOY_DIM, TOY_CONT, TOY_B = [11, 7, 13, 5, 9], 4, 3, 48        # tests/test_model_gpu.py's shapes
TOY_KW = dict(dnn_params={'hidden_units': ((16, 0, False), (8, 0, True)), 'activation': 'relu'},
              cross_params={'num_cross_layer': 3},
              autoint_params={'num_attention': 2, 'num_heads': 2, 'dropout_rate': 0, 'use_residual': True},
              cin_params={'cross_layer_size': (8, 6), 'activation': 'relu', 'use_residual': False, 'use_bias': False,
                          'direct': False, 'reduce_D': False})
# production paths: 26 fields with vocabularies of 50 .. 1000 (ids repeat within a batch) and 13 continuous columns
F26 = [50 + 950 * i // 25 for i in range(26)]


def cin3(act):
    return {'cross_layer_size': (128, 128, 128), 'activation': act, 'use_residual': False, 'use_bias': False,
            'direct': False, 'reduce_D': False}


def case(nets, vocab=TOY_VOCAB, dim=TOY_DIM, n_cont=TOY_CONT, b=TOY_B, task='binary', classes=2, kw=None, toy=True,
         kernels=(), widen=False, weighted=False, tweak=None, seed=5, table_mode=None):
    """A model and its batches.  dim: one width or one per column; kw: ModelConfig keywords over TOY_KW (toy) or the
    ModelConfig defaults; kernels: dtb kernels the train step must launch; widen: widen the bar by the ambiguous
    decisions instead of choosing a batch without any; tweak(snapshot): edits the weights before the step."""
    return dict(nets=nets, vocab=list(vocab), dims=list(dim) if isinstance(dim, (list, tuple)) else [dim] * len(vocab),
                n_cont=n_cont, b=b, task=task, classes=classes, kw={**(TOY_KW if toy else {}), **(kw or {})},
                kernels=tuple(kernels), widen=widen, weighted=weighted, tweak=tweak, seed=seed, prod=not toy,
                table_mode=table_mode)


def prod(nets, dim=16, b=32, kw=None, **more):
    return case(nets, F26, dim, 13, b, kw=kw, toy=False, **more)


DENSE_TC = ('dense_tc_rows_kernel<128>', 'dense_tc_rows_kernel<64>', 'dense_tc_wgrad_kernel', 'dense_narrow_fwd',
            'dense_narrow_bwd_dw')
CIN_WG = ('cin_wg_fwd_kernel', 'cin_wg_dgrad_kernel', 'cin_wg_wgrad_kernel')
FGCNN = ('conv_fields_fwd_kernel', 'maxpool_fields_fwd_kernel', 'conv_fields_bwd_dw_tiled_kernel')

# A: tests/test_model_gpu.py's matrix at its shapes
CASES_A = {'+'.join(n): case(n) for n in NET_SETS}
# AFM over the 21 fields after FGCNN: 210 pairs x 16 attention units per row make a batch without an ambiguous relu rare
# and give a few hundred at 48 rows; 8 rows keep them under MAX_WIDENED
CASES_A['fgcnn_afm_nets'] = case(['fgcnn_afm_nets'], b=8, widen=True)
CASES_A.update({
    'fibi_max_r2_field_all': case(['fibi_dnn_nets'], kw={'fibinet_params': {
        'senet_pooling_op': 'max', 'senet_reduction_ratio': 2, 'bilinear_type': 'field_all'}}),
    'fibi_mean_r3_field_each': case(['fibi_dnn_nets'], kw={'fibinet_params': {
        'senet_pooling_op': 'mean', 'senet_reduction_ratio': 3, 'bilinear_type': 'field_each'}}),
    'fgcnn_small_kernels': case(['fgcnn_dnn_nets'], kw={'fgcnn_params': {
        'fg_filters': (3, 4), 'fg_heights': (3, 2), 'fg_pool_heights': (2, 3), 'fg_new_feat_filters': (2, 1)}}),
    'afm_h5_linear': case(['afm_nets', 'dnn_nets'], kw={'afm_params': {'hidden_factor': 5, 'activation': 'linear',
                                                                        'dropout_rate': 0}}),
    'binary_focal_loss': case(['linear', 'dnn_nets'], kw={'loss': layers.BinaryFocalLoss(gamma=2.0, alpha=0.25)}),
})

# B: production kernel paths
CASES_B = {
    'deepfm_d16': prod(['linear', 'fm_nets', 'dnn_nets'], 16, kernels=('fm_linear_fwd_vec<1>',) + DENSE_TC),
    'deepfm_d32': prod(['linear', 'fm_nets', 'dnn_nets'], 32, kernels=('fm_linear_fwd_vec<2>',) + DENSE_TC),
    'xdeepfm_cin3x128_linear': prod(['linear', 'cin_nets', 'dnn_nets'], 16, kw={'cin_params': cin3('linear')},
                                    kernels=CIN_WG),
    'xdeepfm_cin3x128_relu': prod(['linear', 'cin_nets', 'dnn_nets'], 16, b=16, kw={'cin_params': cin3('relu')},
                                  kernels=CIN_WG, widen=True),
    'dcn6_autoint4x32': prod(['dcn_nets', 'autoint_nets'], 32, kw={
        'cross_params': {'num_cross_layer': 6},
        'autoint_params': {'num_attention': 3, 'num_heads': 4, 'dropout_rate': 0, 'use_residual': True}},
        kernels=('cross_fwd_reg_kernel', 'attention_core_fwd_t_kernel', 'attention_core_bwd_t_kernel'), widen=True),
    'cross_w1053': prod(['cross_nets'], 40, kernels=('cross_fwd_kernel', 'cross_bwd_smem_kernel')),
    'pnn_mat': prod(['pnn_nets'], 16, kw={'pnn_params': {'outer_product_kernel_type': 'mat'}},
                    kernels=('pnn_fwd_t_kernel<16>', 'pnn_bwd_de_t_kernel<16>', 'pnn_bwd_dk_t_kernel<16>')),
    'ipnn': prod(['ipnn_nets'], 16, kernels=('pnn_fwd_t_kernel<16>', 'pnn_bwd_de_t_kernel<16>')),
    'opnn_vec': prod(['opnn_nets'], 16, kw={'pnn_params': {'outer_product_kernel_type': 'vec'}},
                     kernels=('pnn_fwd_t_kernel<16>', 'pnn_bwd_de_t_kernel<16>')),
    'opnn_num': prod(['opnn_nets'], 16, kw={'pnn_params': {'outer_product_kernel_type': 'num'}},
                     kernels=('pnn_fwd_t_kernel<16>', 'pnn_bwd_de_t_kernel<16>')),
    'afm_d16': prod(['afm_nets'], 16, kernels=('afm_rows_kernel',), widen=True),
    'fgcnn_dnn_d16': prod(['fgcnn_dnn_nets'], 16, b=16, kernels=FGCNN, widen=True),
    'fgcnn_cin_d16': prod(['fgcnn_cin_nets'], 16, b=16, kernels=FGCNN, widen=True),
    'five_nets_d16': prod(['fm_nets', 'cin_nets', 'cross_nets', 'autoint_nets', 'pnn_nets'], 16, b=16,
                          kw={'cin_params': cin3('relu')},
                          kernels=CIN_WG + ('cross_fwd_reg_kernel', 'attention_core_fwd_t_kernel', 'pnn_fwd_t_kernel<16>'),
                          widen=True),
    'fm_d10': prod(['linear', 'fm_nets'], 10, kernels=('fm_linear_fwd_generic', 'fm_linear_bwd_generic')),
}
for _bt in ('field_all', 'field_each', 'field_interaction'):
    CASES_B[f'fibi_dnn_{_bt}'] = prod(['fibi_dnn_nets'], 16, kw={'fibinet_params': {
        'senet_pooling_op': 'mean', 'senet_reduction_ratio': 3, 'bilinear_type': _bt}},
        kernels=('bilinear_fwd_kernel', 'bilinear_bwd_dx_kernel', 'bilinear_bwd_dw_kernel'))


def senet_tie(snap):
    """Every row of field 0 takes its maximum in two coordinates: SENET's max pooling sees an exact tie."""
    w = snap['emb_categorical_vars_all/embeddings_0']
    top = w.abs().max(dim=1).values + 0.01
    w[:, 0] = top
    w[:, 1] = top


WIDTHS_KW = dict(fixed_embedding_dim=False, dnn_params={'hidden_units': ((16, 0, False), (8, 0, False)),
                                                        'activation': 'relu'}, cross_params={'num_cross_layer': 2})
# C: model-level variants
CASES_C = {
    'multiclass4': case(['linear', 'fm_nets', 'dnn_nets'], task='multiclass', classes=4),
    'regression': case(['linear', 'fm_nets', 'dnn_nets'], task='regression'),
    'sample_weights': case(['linear', 'fm_nets', 'dnn_nets'], weighted=True),
    'stacking_concat': case(['linear', 'dnn_nets', 'cin_nets'], kw={'stacking_op': 'concat'}),
    'dnn_bn_each_layer': case(['dnn_nets'], kw={'dnn_params': {'hidden_units': ((16, 0, True), (8, 0, True)),
                                                               'activation': 'relu'}}),
    'cin_bias_direct_residual': case(['cin_nets'], kw={'cin_params': {
        'cross_layer_size': (8, 6), 'activation': 'relu', 'use_residual': True, 'use_bias': True, 'direct': True,
        'reduce_D': False}}),
    'cin_bias_residual_d16': prod(['cin_nets'], 16, kw={'cin_params': {
        'cross_layer_size': (32, 32, 16), 'activation': 'linear', 'use_residual': True, 'use_bias': True,
        'direct': False, 'reduce_D': False}}, kernels=CIN_WG),
    'autoint_no_residual': case(['autoint_nets'], kw={'autoint_params': {'num_attention': 2, 'num_heads': 2,
                                                                          'dropout_rate': 0, 'use_residual': False}}),
    'senet_max_tie': case(['fibi_dnn_nets'], kw={'fibinet_params': {
        'senet_pooling_op': 'max', 'senet_reduction_ratio': 2, 'bilinear_type': 'field_interaction'}}, tweak=senet_tie),
    'categorical_only': case(['linear', 'fm_nets', 'dnn_nets', 'cin_nets'], n_cont=0),
    'continuous_only': case(['linear', 'dnn_nets', 'cross_nets'], vocab=[], n_cont=4),
}
# per-column widths on the nets tests/test_widths_gpu.py trains, on both ragged concatenation kernels: every width a
# multiple of 4 (the float4 kernels <4>; max width 16, so the table also updates row-wise -- forced: the toy batch
# touches too much of the table for the cost rule to pick it) and a width of 3 (the generic kernels <1>; max width 20,
# the dense sweep)
for _w, _dims, _vec in (('dmax16', [4, 16, 8, 12, 4], 4), ('dmax20', [20, 4, 8, 3, 12], 1)):
    for _n in ('dnn_nets', 'dcn_nets'):
        CASES_C[f'widths_{_w}_{_n}'] = case([_n], dim=_dims, kw=WIDTHS_KW, toy=False,
                                            table_mode='lazy' if _w == 'dmax16' else None,
                                            kernels=(f'ragged_concat_fwd_kernel<{_vec}>',
                                                     f'ragged_concat_bwd_kernel<{_vec}>'))

ALL = {**CASES_A, **CASES_B, **CASES_C}
PATH_CASES = {k: c for k, c in ALL.items() if c['kernels']}       # cases whose launches are recorded and asserted


# ---------------------------------------------------------------------------------------------------------------------
# the model, its batches and the gradient of its real train step
# ---------------------------------------------------------------------------------------------------------------------
def build(c, table_mode=None):
    from deeptables_b200 import deeptable, optimizers
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    conf = deeptable.ModelConfig(nets=c['nets'], embeddings_output_dim=c['dims'][0] if c['dims'] else 4,
                                 embedding_dropout=0, metrics=['AUC'],
                                 optimizer=optimizers.SGD(learning_rate=LR, momentum=0.0), **c['kw'])
    cats = [CategoricalColumn(f'c{i}', v, d) for i, (v, d) in enumerate(zip(c['vocab'], c['dims']))]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(c['n_cont'])])] if c['n_cont'] else []
    model = DeepModel(c['task'], c['classes'], conf, cats, conts, seed=c['seed'])
    model._build_model()
    model._table_mode_override = table_mode
    return model, conf


def make_batch(c, seed, b=None):
    """ids (with every field's first and last row, and one row repeated), continuous inputs, labels and weights."""
    b = c['b'] if b is None else b
    g = np.random.default_rng(1000 + seed)
    idx = None
    if c['vocab']:
        idx = np.stack([g.integers(0, v, size=b) for v in c['vocab']], axis=1).astype(np.int32)
        idx[0] = 0
        idx[1] = np.array(c['vocab']) - 1
        idx[b - 2] = idx[2]
    cont = g.normal(size=(b, c['n_cont'])).astype(np.float32) if c['n_cont'] else None
    if c['task'] == 'multiclass':
        y = np.eye(c['classes'], dtype=np.float32)[g.integers(0, c['classes'], size=b)]
    elif c['task'] == 'regression':
        y = g.normal(size=b).astype(np.float32)
    else:
        y = (g.random(b) < 0.35).astype(np.float32)
    w = g.uniform(0.0, 3.0, size=b).astype(np.float32) if c['weighted'] else None
    return idx, cont, y, w


def snapshot(model):
    return {k: v.detach().clone() for k, v in model.state_dict().items()}


def gpu_step(model, snap, batch):
    """Loss and recovered gradient of one train_on_batch from `snap`."""
    idx, cont, y, w = batch
    model.load_state_dict(snap)
    loss = model.train_on_batch(idx, cont, y, sample_weight=w)
    after = model.state_dict()
    return loss, {k: (snap[k].double() - after[k].double()) / LR for k in snap if M.is_trainable(k)}


# ---------------------------------------------------------------------------------------------------------------------
# the float64 reference (oracle.model_ref.RefTrainer.loss_and_grads, with Keras's per-row weights and the recorder)
# ---------------------------------------------------------------------------------------------------------------------
def state64(snap, dtype=torch.float64):
    return {k: v.detach().to(DEV, dtype) for k, v in snap.items()}


def reference(st, conf, c, batch, row_weight=None, record=False):
    """Loss, {name: float64 gradient} and, with `record`, the relu / max decisions of the forward with the graph kept.
    row_weight: Keras's sample weights, sum_r w_r l_r / rows (the sample weights of the batch when None)."""
    idx, cont, y, w = batch
    idx = torch.tensor(idx).to(DEV) if idx is not None else None
    dtype = next(iter(st.values())).dtype
    cont = torch.tensor(cont, dtype=dtype).to(DEV) if cont is not None else None
    if row_weight is None and w is not None:
        row_weight = torch.tensor(w, dtype=dtype).to(DEV)
    params = {k: v.clone().requires_grad_(M.is_trainable(k)) for k, v in st.items()}
    entries = []
    with L.recording(entries) if record else contextlib.nullcontext():
        out, _ = M.forward(params, conf, idx, cont, len(c['vocab']), True, c['task'])
    yt = torch.tensor(y, dtype=dtype).to(DEV).reshape(out.shape[0], -1)
    if row_weight is None:
        loss = M.loss_fn(c['task'], yt, out, conf.loss)
    else:
        rows = out.shape[0]
        loss = sum(row_weight[r] * M.loss_fn(c['task'], yt[r:r + 1], out[r:r + 1], conf.loss)
                   for r in range(rows) if row_weight[r] != 0) / rows
    names = [k for k in params if M.is_trainable(k)]
    grads = torch.autograd.grad(loss, [params[k] for k in names], allow_unused=True, retain_graph=record)
    gd = {k: (g if g is not None else torch.zeros_like(params[k])) for k, g in zip(names, grads)}
    return float(loss.detach()), {k: v.double() for k, v in gd.items()}, (entries, loss, params, names) if record else None


def decisions(entries):
    """(ambiguous entries [(site, x, y, index, (first, second) of a max, reduced axis of a max)], exact entries).
    A relu entry is ambiguous when 0 < |x| < TAU * max|x| of the call; a max when the runner-up is within TAU * max|x|.
    Exact entries -- a relu input of exactly 0, an exact tie of a max -- come from exact zeros or copies (a row whose
    relu inputs upstream all died, a duplicated embedding value) that the fp32 forward reproduces exactly."""
    amb, ties = [], 0
    for site, x, y, dim in entries:
        xd = x.detach()
        scale = float(xd.abs().max())
        if dim is None:
            ties += int((xd == 0).sum())
            hit = ((xd != 0) & (xd.abs() < TAU * scale)).nonzero()
            amb += [(site, x, y, tuple(i.tolist()), None, None) for i in hit]
            continue
        xs = xd.movedim(dim, -1)
        if xs.shape[-1] < 2:
            continue
        top = xs.topk(2, dim=-1)
        margin = top.values[..., 0] - top.values[..., 1]
        ties += int((margin == 0).sum())
        hit = ((margin > 0) & (margin < TAU * scale)).nonzero()
        amb += [(site, x, y, tuple(i.tolist()), top.indices[tuple(i.tolist())].tolist(), dim) for i in hit]
    return amb, ties


def widening(rec, amb):
    """Element-wise sum over the ambiguous entries of |first-order change of the gradient had the decision gone the
    other way|: relu, dL/dy_i * dx_i/dtheta; max, dL/dy * d(x_first - x_second)/dtheta."""
    _, loss, params, names = rec
    ys = list({id(y): y for _, _, y, *_ in amb}.values())
    gys = dict(zip(map(id, ys), torch.autograd.grad(loss, ys, retain_graph=True, allow_unused=True)))
    wide = {k: torch.zeros_like(params[k]) for k in names}
    for site, x, y, i, top, dim in amb:
        gy = gys[id(y)]
        if gy is None:
            continue
        if top is None:
            s = gy[i] * x[i]
        else:
            xm = x.movedim(dim, -1)
            s = gy[i] * (xm[i + (top[0],)] - xm[i + (top[1],)])
        d = torch.autograd.grad(s, [params[k] for k in names], retain_graph=True, allow_unused=True)
        for k, g in zip(names, d):
            if g is not None:
                wide[k] += g.abs()
    return wide



def choose_batch(c, st, conf, seeds):
    """First batch among `seeds` without an ambiguous decision (failing that, a case that may widen its bar takes the
    one with the fewest), its reference and its decisions."""
    report, fewest = [], None
    for s in seeds:
        batch = make_batch(c, s)
        loss, g64, rec = reference(st, conf, c, batch, record=True)
        amb, ties = decisions(rec[0])
        if not amb:
            return batch, loss, g64, rec, amb, ties
        if fewest is None or len(amb) < len(fewest[4]):
            fewest = (batch, loss, g64, rec, amb, ties)
        sites = {}
        for site, x, *_ in amb:
            sites[f'{site} {tuple(x.shape)}'] = sites.get(f'{site} {tuple(x.shape)}', 0) + 1
        report.append(f'seed {s}: {len(amb)} ambiguous, at {sites}')
    if c['widen']:
        return fewest
    pytest.fail('every batch tried has ambiguous relu / max decisions:\n' + '\n'.join(report))


# ---------------------------------------------------------------------------------------------------------------------
# the comparison
# ---------------------------------------------------------------------------------------------------------------------
def compare(name, c, st, conf, batch, loss_g, g, loss64, g64, rec, amb, ties, loss32, g32):
    wide = None
    if c['widen']:
        assert len(amb) <= MAX_WIDENED, f'{name}: {len(amb)} ambiguous decisions (at most {MAX_WIDENED} may widen the bar)'
        wide = widening(rec, amb) if amb else None
    else:
        assert not amb, f'{name}: ambiguous decisions at {sorted({s for s, *_ in amb})}'
    loss_bar = max(LOSS_RTOL * abs(loss64), FP32_FLOOR * abs(loss32 - loss64))
    assert abs(loss_g - loss64) <= loss_bar, f'{name}: loss {loss_g!r} against float64 {loss64!r} (float32 oracle {loss32!r})'
    # the same batch with its last row's loss left out (batch statistics unchanged)
    # (a row whose probability is clipped contributes no gradient: then the last row that does)
    top = max(float(v.abs().max()) for v in g64.values())
    for r in reversed(range(c['b'])):
        keep = torch.ones(c['b'], dtype=torch.float64, device=DEV)
        if batch[3] is not None:
            keep *= torch.tensor(batch[3], dtype=torch.float64, device=DEV)
        keep[r] = 0
        _, g_short, _ = reference(st, conf, c, batch, row_weight=keep)
        if any(bool((g_short[k] != g64[k]).any()) for k in g64):
            break
    worst, worst_key, seen, floored = 0.0, None, 0.0, 0
    for k, want in g64.items():
        got = g[k]
        assert got.shape == want.shape, f'{name}: {k} has shape {tuple(got.shape)}, float64 {tuple(want.shape)}'
        bar = want.new_tensor(RTOL * max(float(want.abs().max()), MODEL_SHARE * top) + 1e-30)
        floor = FP32_FLOOR * (g32[k] - want).abs().max()
        floored += int(floor > bar)
        bar = torch.maximum(bar, floor)
        if wide is not None:
            bar = bar + wide[k]
        err = float(((got - want).abs() / bar).max())
        if err > worst:
            worst, worst_key = err, k
        seen = max(seen, float(((g_short[k] - want).abs() / bar).max()))
        assert err <= 1, (f'{name}: gradient of {k} off by {err:.3g} of its bar (max |g64| {float(want.abs().max()):.3e}, '
                          f'max |g - g64| {float((got - want).abs().max()):.3e})')
    print(f'{name}: worst error / bar {worst:.3g} ({worst_key}), ambiguous {len(amb)}, exact {ties}, '
          f'row {r} left out {seen:.3g} x bar, float32 floor on {floored} of {len(g64)} tensors')
    assert seen > 1, f'{name}: the bar does not see row {r} left out ({seen:.3g} of the bar)'
    return ties


def check(name, c, seeds=range(BATCH_SEEDS), model=None, snap=None, conf=None):
    if model is None:
        model, conf = build(c, c['table_mode'])
        snap = snapshot(model)
        if c['tweak'] is not None:
            c['tweak'](snap)
    st = state64(snap)
    batch, loss64, g64, rec, amb, ties = choose_batch(c, st, conf, seeds)
    loss32, g32, _ = reference(state64(snap, torch.float32), conf, c, batch)
    loss_g, g = gpu_step(model, snap, batch)
    return compare(name, c, st, conf, batch, loss_g, g, loss64, g64, rec, amb, ties, loss32, g32), model


@pytest.fixture(autouse=True)
def _release():
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.mark.parametrize('name', list(CASES_A))
def test_toy_matrix_gradient(name):
    check(name, CASES_A[name])


def assert_path(recorded, name):
    ks = recorded[name]
    missing = [k for k in PATH_CASES[name]['kernels'] if not ran([(n, None, None) for n in ks], k)]
    assert not missing, f'{name}: {missing} did not run; the train step launched {sorted(set(ks))}'


@pytest.mark.parametrize('name', list(CASES_B))
def test_production_path_gradient(recorded, name):
    assert_path(recorded, name)
    _, model = check(name, CASES_B[name])
    model.release()


@pytest.mark.parametrize('name', list(CASES_C))
def test_model_variant_gradient(recorded, name):
    c = CASES_C[name]
    if name in PATH_CASES:
        assert_path(recorded, name)
    ties, model = check(name, c)
    if name == 'senet_max_tie':
        assert ties >= c['b'], f'{name}: SENET max pooling saw {ties} exact ties'
    if name.startswith('widths_'):
        assert model.table.ragged and model.table.lazy_active == ('dmax16' in name)


@pytest.mark.parametrize('name', ['linear+fm_nets+dnn_nets', 'deepfm_d16'])
def test_eager_capture_and_replay_steps(name):
    """Step 1 runs eagerly, step 2 captures the CUDA graph of the train step and step 3 replays it; each from the
    restored snapshot, on its own batch."""
    c = ALL[name]
    model, conf = build(c)
    snap = snapshot(model)
    for step in range(3):
        check(f'{name} step {step + 1}', c, seeds=range(100 * step, 100 * step + BATCH_SEEDS), model=model, snap=snap,
              conf=conf)
        assert model._step == step + 1 and len(model._graphs) == (0 if step == 0 else 1)
    model.release()


# ---------------------------------------------------------------------------------------------------------------------
# the launches of each case that names its kernels, recorded in a child process
# ---------------------------------------------------------------------------------------------------------------------
def _record(path):
    rec = {}
    for name, c in PATH_CASES.items():
        model, _ = build(c, c['table_mode'])
        idx, cont, y, _ = make_batch(c, 0)
        kernels, _ = launches(lambda: model.train_on_batch(idx, cont, y))
        rec[name] = [k for k, _, _ in kernels]
        model.release()
        del model
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    with open(path, 'w') as f:
        json.dump(rec, f)


@pytest.fixture(scope='module')
def recorded(tmp_path_factory):
    path = str(tmp_path_factory.mktemp('launches') / 'launches.json')
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f'import sys; sys.path[:0] = [{here!r}, {os.path.dirname(here)!r}]; import test_model_grads_gpu as t; '
            f't._record({path!r})')
    flags = ['-s'] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ['-c', code], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, f'recording the launches failed:\n{r.stdout[-4000:]}\n{r.stderr[-4000:]}'
    with open(path) as f:
        return json.load(f)


# ---------------------------------------------------------------------------------------------------------------------
# E: data parallel over NCCL, two ranks on different shards that share table rows
# ---------------------------------------------------------------------------------------------------------------------
DP_CASE = case(['linear', 'fm_nets', 'dnn_nets', 'cin_nets'], vocab=[20, 15, 30, 10, 25], dim=8, n_cont=3, b=32,
               kw={'cin_params': {'cross_layer_size': (16, 16), 'activation': 'relu', 'use_residual': False,
                                  'use_bias': False, 'direct': False, 'reduce_D': False}})


def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_worker(rank, world, port, out_dir, table_mode, seeds):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        model, _ = build(DP_CASE, table_mode)
        assert model.world_size == world
        snap = snapshot(model)
        loss, g = gpu_step(model, snap, make_batch(DP_CASE, seeds[rank]))
        assert model.table.lazy_active == (table_mode == 'lazy')
        torch.save({'loss': loss, 'g': {k: v.cpu() for k, v in g.items()},
                    'snap': {k: v.cpu() for k, v in snap.items()}}, os.path.join(out_dir, f'rank{rank}.pt'))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('table_mode', ['dense', 'lazy'])
def test_data_parallel_gradient_is_the_mean_of_the_shards(tmp_path, table_mode):
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f'needs {world} GPUs')
    c = DP_CASE
    model, conf = build(c)
    st = state64(snapshot(model))
    model.release()
    # two shards without ambiguous decisions; small vocabularies make them share rows
    seeds = []
    for s in range(4 * BATCH_SEEDS):
        if not decisions(reference(st, conf, c, make_batch(c, s), record=True)[2][0])[0]:
            seeds.append(s)
        if len(seeds) == world:
            break
    assert len(seeds) == world, 'no two shards without ambiguous decisions'
    shards = [make_batch(c, s) for s in seeds]
    shared = sum(len(set(shards[0][0][:, f]) & set(shards[1][0][:, f])) for f in range(len(c['vocab'])))
    assert shared > 0
    import torch.multiprocessing as mp
    mp.spawn(_dp_worker, args=(world, _free_port(), str(tmp_path), table_mode, seeds), nprocs=world, join=True)
    refs = [reference(st, conf, c, b) for b in shards]           # each replica's own batch statistics
    want = {k: sum(r[1][k] for r in refs) / world for k in refs[0][1]}
    refs32 = [reference(state64(st, torch.float32), conf, c, b) for b in shards]
    want32 = {k: sum(r[1][k] for r in refs32) / world for k in want}
    top = max(float(w.abs().max()) for w in want.values())
    bars = {k: torch.maximum(w.new_tensor(RTOL * max(float(w.abs().max()), MODEL_SHARE * top) + 1e-30),
                             FP32_FLOOR * (want32[k] - w).abs().max()) for k, w in want.items()}
    # the bar sees rank 0's last row left out of the loss (batch statistics unchanged)
    keep = torch.ones(c['b'], dtype=torch.float64, device=DEV)
    keep[-1] = 0
    short0 = reference(st, conf, c, shards[0], row_weight=keep)[1]
    seen = max(float(((short0[k] + refs[1][1][k]) / world - w).abs().div(bars[k]).max()) for k, w in want.items())
    assert seen > 1, f'the bar does not see rank 0\'s last row left out ({seen:.3g} of the bar)'
    for rank in range(world):
        got = torch.load(tmp_path / f'rank{rank}.pt')
        for k, v in got['snap'].items():
            assert torch.equal(v.to(DEV).double(), st[k]), f'rank {rank} started from other weights ({k})'
        assert abs(got['loss'] - refs[rank][0]) <= max(LOSS_RTOL * abs(refs[rank][0]),
                                                       FP32_FLOOR * abs(refs32[rank][0] - refs[rank][0]))
        worst = 0.0
        for k, w in want.items():
            err = float(((got['g'][k].to(DEV) - w).abs() / bars[k]).max())
            worst = max(worst, err)
            assert err <= 1, f'rank {rank}: gradient of {k} off by {err:.3g} of its bar from the mean of the shards'
        print(f'data parallel ({table_mode}), rank {rank}: worst error / bar {worst:.3g}, {shared} shared ids, '
              f'rank 0\'s last row left out {seen:.3g} x bar')
