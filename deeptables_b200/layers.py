"""Interaction layers with the reference's names and constructor arguments
(reference deeptables/models/layers.py), executed by hand-written sm_90a kernels through the
C ABI.  Layers are define-by-run: calling one inside a model scope creates (first call) or looks
up (later calls) its weights under the Keras-style layer name, so net builders -- the built-in
ones in deepnets.py and user callables with the same 6-argument signature -- read exactly like
the reference's.

Tensors are torch CUDA tensors; ``FieldBlock`` (engine.py) is the lazy (B,F,D) embedding block
that lets FM / CIN / linear / PNN fuse the categorical gather into their kernels.
"""
import math
import os
import re
import threading

import torch

from . import engine as E, regularizers as R
from .engine import FieldBlock, EmbeddingList

_tls = threading.local()


def current_scope():
    scope = getattr(_tls, 'scope', None)
    if scope is None:
        raise RuntimeError('layers can only be called inside a DeepModel forward pass '
                           '(net builders are invoked by DeepModel with an active scope)')
    return scope


class scope_guard:
    def __init__(self, scope):
        self.scope = scope

    def __enter__(self):
        self.prev = getattr(_tls, 'scope', None)
        _tls.scope = self.scope
        self.scope._begin_pass()
        return self.scope

    def __exit__(self, *exc):
        _tls.scope = self.prev
        return False


def _snake(name):
    s = re.sub(r'(.)([A-Z][a-z0-9]+)', r'\1_\2', name)
    s = re.sub(r'([a-z0-9])([A-Z])', r'\1_\2', s).lower()
    return s


# ---------------------------------------------------------------------------------------------
# keras initialisers (fan computation as keras.initializers.VarianceScaling)
# ---------------------------------------------------------------------------------------------
def _fans(shape):
    if len(shape) == 1:
        return shape[0], shape[0]
    if len(shape) == 2:
        return shape[0], shape[1]
    rf = 1
    for s in shape[:-2]:
        rf *= s
    return shape[-2] * rf, shape[-1] * rf


def init_tensor(shape, kind, device, generator=None):
    shape = tuple(int(s) for s in shape)
    t = torch.empty(shape, dtype=torch.float32, device=device)
    if kind == 'zeros':
        return t.zero_()
    if kind == 'ones':
        return t.fill_(1.0)
    fan_in, fan_out = _fans(shape)
    if kind == 'glorot_normal':
        # keras GlorotNormal: truncated normal (2 sigma) with stddev sqrt(2 / (fan_in + fan_out)) / 0.87962566
        std = math.sqrt(2.0 / (fan_in + fan_out)) / 0.87962566103423978
        return torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=generator)
    if kind == 'uniform':
        lim = 0.05
    elif kind == 'glorot_uniform':
        lim = math.sqrt(6.0 / (fan_in + fan_out))
    elif kind == 'he_uniform':
        lim = math.sqrt(6.0 / fan_in)
    else:
        raise NotImplementedError(f'initializer {kind!r}')
    return t.uniform_(-lim, lim, generator=generator)


class Layer:
    """Base: resolves the Keras-style unique layer name inside the active model scope."""

    def __init__(self, name=None, **kwargs):
        regs = sorted(k for k, v in kwargs.items() if k.endswith('regularizer') and v is not None)
        if regs:      # only Dense kernels and the embedding tables take regularizers, as in the reference
            raise NotImplementedError(f'{type(self).__name__}({", ".join(regs)}): regularizers on this layer are not '
                                      f'built natively')
        self._given_name = name
        self.name = name

    def __call__(self, *args, **kwargs):
        scope = current_scope()
        self.name = scope.full_name(self._given_name, _snake(type(self).__name__))
        out = self.call(scope, *args, **kwargs)
        scope.record_output(self.name, out)
        return out

    def get_config(self):
        return {'name': self._given_name}


def _materialize(x):
    return x.materialize() if isinstance(x, FieldBlock) else x


# ---------------------------------------------------------------------------------------------
# generic keras layers used by the builders
# ---------------------------------------------------------------------------------------------
class Dense(Layer):
    def __init__(self, units, activation=None, use_bias=True, kernel_initializer='glorot_uniform',
                 kernel_regularizer=None, activity_regularizer=None, name=None):
        super().__init__(name)
        if activation not in E.ACT_CODES:
            raise NotImplementedError(f'activation {activation!r} (supported: relu, linear/None)')
        R.reject_activity(activity_regularizer, 'Dense(activity_regularizer)')
        self.kernel_regularizer = R.resolve(kernel_regularizer, 'Dense(kernel_regularizer)')
        self.units, self.activation, self.use_bias = int(units), activation, use_bias
        self.kernel_initializer = kernel_initializer

    def call(self, scope, x):
        x = _materialize(x)
        in_dim = x.shape[-1]
        kernel = scope.param(f'{self.name}/kernel', (in_dim, self.units), self.kernel_initializer,
                             regularizer=self.kernel_regularizer)
        bias = scope.param(f'{self.name}/bias', (self.units,), 'zeros') if self.use_bias else None
        return E.DenseFn.apply(x, kernel, bias, E.ACT_CODES[self.activation])


class BatchNormalization(Layer):
    def call(self, scope, x):
        x = _materialize(x)
        width = x.shape[-1]
        gamma = scope.param(f'{self.name}/gamma', (width,), 'ones')
        beta = scope.param(f'{self.name}/beta', (width,), 'zeros')
        mm = scope.buffer(f'{self.name}/moving_mean', (width,), 0.0)
        mv = scope.buffer(f'{self.name}/moving_variance', (width,), 1.0)
        if scope.training:
            return E.BatchNormFn.apply(x, gamma, beta, mm, mv)
        return E.batchnorm_infer(x, gamma, beta, mm, mv)


class Activation(Layer):
    def __init__(self, activation, name=None):
        super().__init__(name)
        if activation not in E.ACT_CODES:
            raise NotImplementedError(f'activation {activation!r}')
        self.activation = activation

    def call(self, scope, x):
        return torch.relu(x) if self.activation == 'relu' else x


class Dropout(Layer):
    def __init__(self, rate, name=None):
        super().__init__(name)
        self.rate = float(rate)

    def call(self, scope, x):
        if self.rate > 0 and scope.training:
            return E.DropoutFn.apply(_materialize(x), self.rate, scope.next_seed())
        return x


class Concatenate(Layer):
    def __init__(self, axis=-1, name=None):
        super().__init__(name)
        self.axis = axis

    def call(self, scope, inputs):
        if isinstance(inputs, EmbeddingList):
            if self.axis == 1:
                return inputs.block                              # lazy (B,F,D)
            return scope.flatten_embeddings(inputs).unsqueeze(1)  # (B,1,F*D)
        return torch.cat([_materialize(t) for t in inputs], dim=self.axis)


class Flatten(Layer):
    def call(self, scope, x):
        x = _materialize(x)
        return x.reshape(x.shape[0], -1)


class Add(Layer):
    def call(self, scope, inputs):
        out = inputs[0]
        for t in inputs[1:]:
            out = out + t
        return out


# ---------------------------------------------------------------------------------------------
# interaction layers (reference names)
# ---------------------------------------------------------------------------------------------
def _as_block(x):
    if isinstance(x, FieldBlock):
        return x
    if isinstance(x, EmbeddingList):
        return x.block
    if isinstance(x, (list, tuple)):
        x = torch.cat(list(x), dim=1)
    if x.dim() != 3:
        raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
    return FieldBlock.from_tensor(x)


class LinearLogit(Layer):
    """The whole of deepnets.linear (reference deepnets.py:43-66) as one fused launch:
    sum_d of every field embedding, concat with the continuous inputs, Dense(1, no bias)."""

    def call(self, scope, embeddings, dense_layer):
        f = len(embeddings) if embeddings is not None else 0
        c = dense_layer.shape[1] if dense_layer is not None else 0
        kernel = scope.param(f'{self.name}/kernel', (f + c, 1), 'glorot_uniform')
        block = _as_block(embeddings) if f else None
        anchor = block.table.anchor if block is not None else scope.anchor
        return E.FMLinearFn.apply(anchor, dense_layer, kernel.reshape(-1), block, True, False)


class FM(Layer):
    """Factorization Machine second-order term (reference layers.py:27-62)."""

    def call(self, scope, x):
        block = _as_block(x)
        return E.FMLinearFn.apply(block.table.anchor, None, None, block, False, True)


class CIN(Layer):
    """Compressed Interaction Network (reference layers.py:589-739)."""

    def __init__(self, params, name=None):
        super().__init__(name)
        self.params = params
        self.cross_layer_size = tuple(params.get('cross_layer_size', (128, 128,)))
        self.activation = params.get('activation', 'relu')
        self.use_residual = params.get('use_residual', False)
        self.use_bias = params.get('use_bias', False)
        self.direct = params.get('direct', False)
        self.reduce_D = params.get('reduce_D', False)
        # test hook: DTB_CIN_PRECISION overrides the auto choice (0) so the whole GPU suite can be run on another CIN mode
        self.precision = params.get('precision', 0) or int(os.environ.get('DTB_CIN_PRECISION', 0))   # engine knob: 0 auto (fused bf16x3 where supported, else any-shape), 1 any-shape, 2 bf16x3, 3 bf16x1, 4 fp16x1
        if len(self.cross_layer_size) == 0:
            raise ValueError('cross_layer_size must be a list(tuple) of length greater than 1')
        if self.activation not in E.ACT_CODES:
            raise NotImplementedError(f'CIN activation {self.activation!r} (supported: relu, linear)')

    def field_nums(self, f0):
        nums = [int(f0)]
        for i, size in enumerate(self.cross_layer_size):
            if self.direct:
                nums.append(size)
            else:
                if i != len(self.cross_layer_size) - 1 and size % 2 > 0:
                    raise ValueError(
                        'cross_layer_size must be even number except for the last layer when direct=True')
                nums.append(size // 2)
        return nums

    def call(self, scope, x):
        block = _as_block(x)
        _, f0, dim = block.shape
        nums = self.field_nums(f0)
        filters = []
        for i, size in enumerate(self.cross_layer_size):
            if self.reduce_D:
                f0_ = scope.param(f'{self.name}/f0_{i}', (1, size, nums[0], dim), 'he_uniform')
                f__ = scope.param(f'{self.name}/f__{i}', (1, size, dim, nums[i]), 'he_uniform')
                f_m = torch.matmul(f0_, f__)                                   # tiny weight-only reparam
                filt = f_m.reshape(1, size, nums[0] * nums[i]).permute(0, 2, 1)
            else:
                filt = scope.param(f'{self.name}/f_{i}', (1, nums[i] * nums[0], size), 'he_uniform')
            filters.append(filt.reshape(-1))
        weights = torch.cat(filters) if len(filters) > 1 else filters[0]
        bias = None
        if self.use_bias:
            bs = [scope.param(f'{self.name}/bias{i}', (size,), 'zeros')
                  for i, size in enumerate(self.cross_layer_size)]
            bias = torch.cat(bs) if len(bs) > 1 else bs[0]
        pooled = E.CINFn.apply(block.table.anchor, weights.contiguous(), bias, block,
                               tuple(self.cross_layer_size), bool(self.direct),
                               E.ACT_CODES[self.activation], int(self.precision),
                               bool(scope.training and torch.is_grad_enabled()))
        with scope.name_prefix(self.name):
            if self.use_residual:
                out0 = Dense(self.cross_layer_size[-1], activation=self.activation,
                             kernel_initializer='he_uniform', name='exFM_out0')(pooled)
                ex_in = torch.cat([out0, pooled], dim=1)
                return Dense(1, activation=None, name='exFM_out')(ex_in)
            return Dense(1, activation=None, name='exFM_out')(pooled)

    def get_config(self):
        return {'params': self.params, 'name': self._given_name}


class Cross(Layer):
    """Cross network (reference layers.py:385-441)."""

    def __init__(self, params, name=None):
        super().__init__(name)
        self.params = params
        self.num_cross_layer = params.get('num_cross_layer', 2)

    def call(self, scope, x):
        if x.dim() != 2:
            raise ValueError(f'Wrong dimensions of x, expected 2 but input {x.dim()}.')
        w = x.shape[-1]
        ks = [scope.param(f'{self.name}/kernels_{i}', (w, 1), 'glorot_uniform')
              for i in range(self.num_cross_layer)]
        bs = [scope.param(f'{self.name}/bias_{i}', (w, 1), 'zeros') for i in range(self.num_cross_layer)]
        if self.num_cross_layer == 0:
            return x
        kernels = torch.cat([k.reshape(1, w) for k in ks], dim=0)
        biases = torch.cat([b.reshape(1, w) for b in bs], dim=0)
        return E.CrossFn.apply(x, kernels, biases)


class MultiheadAttention(Layer):
    """AutoInt interacting layer (reference layers.py:65-158)."""

    def __init__(self, params, name=None):
        super().__init__(name)
        self.params = params
        self.num_heads = params.get('num_heads', 1)
        self.dropout_rate = params.get('dropout_rate', 0)
        self.use_residual = params.get('use_residual', True)
        if self.dropout_rate:
            raise NotImplementedError('attention dropout_rate > 0 is not supported')

    def call(self, scope, x):
        x = _materialize(x)
        if x.dim() != 3:
            raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
        d = x.shape[-1]
        if d % self.num_heads:
            raise ValueError(f'num_heads={self.num_heads} must divide the embedding size {d}')
        ws, bs = [], []
        for proj in ('dense_Q', 'dense_K', 'dense_V', 'dense_residual'):
            ws.append(scope.param(f'{self.name}/{proj}/kernel', (d, d), 'he_uniform'))
            bs.append(scope.param(f'{self.name}/{proj}/bias', (d,), 'zeros'))
        # the four relu(Dense) projections as ONE GEMM: kernels side by side -> [B, F, 4D] = [Q|K|V|R]
        # the attention backward has the relu outputs in shared memory and applies their mask itself, so the [B*F, 4D]
        # activation-gradient pass (and the gradient clone it needs) of the projection layer is skipped
        qkvr = E.DenseFn.apply(x, torch.cat(ws, dim=1), torch.cat(bs), E.ACT_CODES['relu'], True)
        out = E.AttentionCoreFn.apply(qkvr, int(self.num_heads), bool(self.use_residual), True)
        with scope.name_prefix(self.name):
            return BatchNormalization(name='batch_normalize')(out)


class InnerProduct(Layer):
    """PNN inner products (reference layers.py:444-490)."""

    def call(self, scope, x):
        block = _as_block(x)
        return E.PNNFn.apply(block.table.anchor, None, block, True, False, 'mat')


class OuterProduct(Layer):
    """PNN kernelised outer products (reference layers.py:493-586)."""

    def __init__(self, params, name=None):
        super().__init__(name)
        self.params = params
        self.kernel_type = params.get('outer_product_kernel_type', 'mat')
        if self.kernel_type not in ['mat', 'vec', 'num']:
            raise ValueError('kernel_type must be mat,vec or num')

    def call(self, scope, x):
        block = _as_block(x)
        _, f, d = block.shape
        pairs = f * (f - 1) // 2
        shape = {'mat': (d, pairs, d), 'vec': (pairs, d), 'num': (pairs, 1)}[self.kernel_type]
        kernel = scope.param(f'{self.name}/kernel', shape, 'glorot_uniform')
        return E.PNNFn.apply(block.table.anchor, kernel, block, False, True, self.kernel_type)


class InnerOuterProduct(Layer):
    """pnn_nets needs both products of the same block: one fused launch (deepnets.py:151-156)."""

    def __init__(self, params, ip_name, op_name):
        super().__init__(op_name)
        self.kernel_type = params.get('outer_product_kernel_type', 'mat')
        self.ip_name = ip_name

    def call(self, scope, x):
        block = _as_block(x)
        _, f, d = block.shape
        pairs = f * (f - 1) // 2
        shape = {'mat': (d, pairs, d), 'vec': (pairs, d), 'num': (pairs, 1)}[self.kernel_type]
        kernel = scope.param(f'{self.name}/kernel', shape, 'glorot_uniform')
        ip, op = E.PNNFn.apply(block.table.anchor, kernel, block, True, True, self.kernel_type)
        scope.record_output(self.ip_name, ip)
        return ip, op


# layers the reference exports that are outside the hot path (SURVEY.md section 8f, rank 3)
def _out_of_scope(name):
    class _Stub(Layer):
        def __init__(self, *a, **k):
            raise NotImplementedError(f'{name} is outside the hot path of this build '
                                      f'(SURVEY.md 8f): not implemented')
    _Stub.__name__ = name
    return _Stub


class AFM(Layer):
    """Attentional FM (reference layers.py:742-812).  Weight names: <name>/dense_attention/{kernel,bias},
    <name>/projection_h, <name>/dense_out/kernel."""

    def __init__(self, params, name=None):
        super().__init__(name)
        self.params = params
        self.hidden_factor = params.get('hidden_factor', 16)
        self.dropout_rate = params.get('dropout_rate', 0)
        self.activation_function = params.get('activation', 'relu')
        if self.activation_function not in ('relu', 'linear', None):
            raise NotImplementedError(f'AFM attention activation {self.activation_function!r}: relu or linear')

    def call(self, scope, x):
        if torch.is_tensor(x):
            if x.dim() != 3 or x.shape[1] < 2:           # the (B, F, D) block a list of F (B, 1, D) tensors concatenates to
                raise ValueError('A `AttentionalFM` layer should be called on a list of at least 2 inputs')
        elif not isinstance(x, (list, tuple, EmbeddingList)) or len(x) < 2:
            raise ValueError('A `AttentionalFM` layer should be called on a list of at least 2 inputs')
        block = _as_block(x)
        _, f, d = block.shape
        h = int(self.hidden_factor)
        wa = scope.param(f'{self.name}/dense_attention/kernel', (d, h), 'glorot_normal')
        ba = scope.param(f'{self.name}/dense_attention/bias', (h,), 'zeros')
        wo = scope.param(f'{self.name}/dense_out/kernel', (d, 1), 'glorot_uniform')
        ph = scope.param(f'{self.name}/projection_h', (h, 1), 'glorot_uniform')
        act = E.ACT_CODES['relu'] if self.activation_function == 'relu' else E.ACT_CODES['linear']
        pooled = E.AFMFn.apply(block.table.anchor, wa, ba, ph, block, act)
        if self.dropout_rate and scope.training:
            pooled = E.DropoutFn.apply(pooled, float(self.dropout_rate), scope.next_seed())
        return E.DenseFn.apply(pooled, wo, None, E.ACT_CODES['linear'])


class FGCNN(Layer):
    """Feature generation by a convolution along the fields, max pooling and a recombination Dense layer (reference
    layers.py:161-242).  x: (B, F, D, C).  Returns (pooling_output (B, ceil(F/pool), D, filters), new_features
    (B, F*new_filters, D)).  Weight names: <name>/conv2d/{kernel,bias}, <name>/dense_output/{kernel,bias}."""

    def __init__(self, filters, kernel_height, new_filters, pool_height, activation='tanh', name=None):
        super().__init__(name)
        self.filters, self.kernel_height = int(filters), int(kernel_height)
        self.new_filters, self.pool_height = int(new_filters), int(pool_height)
        self.activation = activation
        if activation not in E.ACT_CODES:
            raise NotImplementedError(f'FGCNN activation {activation!r}: tanh, relu or linear')

    def call(self, scope, x):
        x = _materialize(x)
        if x.dim() != 4:
            raise ValueError(f'Wrong dimensions of inputs, expected 4 but input {x.dim()}.')
        b, h, w, cin = x.shape
        act = E.ACT_CODES[self.activation]
        ck = scope.param(f'{self.name}/conv2d/kernel', (self.kernel_height, 1, cin, self.filters), 'glorot_uniform')
        cb = scope.param(f'{self.name}/conv2d/bias', (self.filters,), 'zeros')
        h_out = -(-h // self.pool_height)
        dk = scope.param(f'{self.name}/dense_output/kernel', (h_out * w * self.filters, h * w * self.new_filters), 'glorot_uniform')
        db = scope.param(f'{self.name}/dense_output/bias', (h * w * self.new_filters,), 'zeros')
        out = E.ConvFieldsFn.apply(x, ck, cb, act)
        pooled = E.MaxPoolFieldsFn.apply(out, self.pool_height)
        new_features = E.DenseFn.apply(pooled.reshape(b, -1), dk, db, act)
        return pooled, new_features.reshape(b, h * self.new_filters, w)

    def __call__(self, *args, **kwargs):
        scope = current_scope()
        self.name = scope.full_name(self._given_name, 'fgcnn')
        out = self.call(scope, *args, **kwargs)
        scope.record_output(self.name, out[1])
        return out




class SENET(Layer):
    """Squeeze-and-excitation re-weighting of the field embeddings (reference layers.py:245-311).
    Weight names: <name>/dense_att1/{kernel,bias}, <name>/dense_att2/{kernel,bias}."""

    def __init__(self, pooling_op='mean', reduction_ratio=3, name=None):
        super().__init__(name)
        self.pooling_op = pooling_op
        self.reduction_ratio = reduction_ratio

    def call(self, scope, x):
        x = _materialize(x)
        if x.dim() != 3:
            raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
        f = x.shape[1]
        red = max(f // self.reduction_ratio, 1)
        w1 = scope.param(f'{self.name}/dense_att1/kernel', (f, red), 'he_uniform')
        b1 = scope.param(f'{self.name}/dense_att1/bias', (red,), 'zeros')
        w2 = scope.param(f'{self.name}/dense_att2/kernel', (red, f), 'he_uniform')
        b2 = scope.param(f'{self.name}/dense_att2/bias', (f,), 'zeros')
        z = E.SenetPoolFn.apply(x, 1 if self.pooling_op == 'max' else 0)
        a1 = E.DenseFn.apply(z, w1, b1, E.ACT_CODES['relu'])
        a2 = E.DenseFn.apply(a1, w2, b2, E.ACT_CODES['relu'])
        return E.SenetScaleFn.apply(x, a2)


class BilinearInteraction(Layer):
    """(x_i W) * x_j over the field pairs (reference layers.py:314-382); the per-pair / per-field matrices are one stacked
    tensor here, exposed under the reference's names (bilinear_weight, bilinear_weight<i>, bilinear_weight<i>_<j>)."""

    def __init__(self, bilinear_type='field_interaction', name=None):
        super().__init__(name)
        if bilinear_type not in E.BILINEAR_TYPES:
            bilinear_type = 'field_interaction'          # the reference's else branch (layers.py:350)
        self.bilinear_type = bilinear_type

    def call(self, scope, x):
        x = _materialize(x)
        if x.dim() != 3:
            raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
        _, f, d = x.shape
        if self.bilinear_type == 'field_all':
            names = [f'{self.name}/bilinear_weight']
        elif self.bilinear_type == 'field_each':
            names = [f'{self.name}/bilinear_weight{i}' for i in range(f - 1)]
        else:
            names = [f'{self.name}/bilinear_weight{i}_{j}' for i in range(f) for j in range(i + 1, f)]
        w = scope.param_stack(names, (d, d), 'glorot_uniform')
        return E.BilinearFn.apply(x, w, self.bilinear_type)


VarLenColumnEmbedding = _out_of_scope('VarLenColumnEmbedding')


class BinaryFocalLoss:
    """``ModelConfig(loss=BinaryFocalLoss(gamma, alpha))`` for binary / multilabel tasks (reference layers.py:983-1022):
    FL = -alpha (1 - p_t)^gamma log p_t on the sigmoid probabilities, averaged over every element."""

    def __init__(self, gamma=2., alpha=.25, reduction=None, name='focal_loss'):
        self.gamma, self.alpha, self.name = float(gamma), float(alpha), name

    def get_config(self):
        return {'gamma': self.gamma, 'alpha': self.alpha, 'name': self.name}


class CategoricalFocalLoss(BinaryFocalLoss):
    """Softmax form for multiclass tasks (reference layers.py:1025-1083): sum_c alpha (1 - p_c)^gamma (-y_c log p_c)."""


def GHMCLoss(*a, **k):
    raise NotImplementedError('GHMCLoss (a TF1-style stateful helper, layers.py:1086-1163) is not implemented')

dt_custom_objects = {
    'FM': FM, 'CIN': CIN, 'Cross': Cross, 'MultiheadAttention': MultiheadAttention,
    'InnerProduct': InnerProduct, 'OuterProduct': OuterProduct, 'AFM': AFM, 'SENET': SENET,
    'BilinearInteraction': BilinearInteraction, 'FGCNN': FGCNN, 'BinaryFocalLoss': BinaryFocalLoss,
    'CategoricalFocalLoss': CategoricalFocalLoss,
}


def register_custom_objects(objs: dict):
    for k, v in objs.items():
        if dt_custom_objects.get(k) is None:
            dt_custom_objects[k] = v
