"""CPU oracle: restatement of the reference's interaction layers as plain torch-CPU ops.

TEST INFRASTRUCTURE ONLY.  Nothing under ``deeptables_b200/`` may import this module; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs use it, and only as the checker (or as the timed CPU baseline), never as the product path.

PARITY: PINNED FOR THE FORWARD LOGIC, UNPINNED FOR TENSORFLOW'S OWN ARITHMETIC.  The reference's arithmetic
lives in TensorFlow + Keras 3, which is neither vendored under /root/reference nor installable here (no
network, not in /opt/wheelhouse), and the reference's own tests pin no numerics for this path
(``AUC >= 0.0``, deeptables/tests/models/nets_test.py:44).  So:
  * every function below follows the reference's TF op sequence line by line (file:line cited) and is
    cross-checked in tests/test_oracle.py against an independent brute-force definition
    (oracle/bruteforce.py, numpy float64 loops);
  * tests/test_reference_golden.py pins them against golden vectors produced by the reference's OWN layer
    classes, net builders and ``DeepModel.__build_model``, imported unmodified from /root/reference and run
    eagerly in float64 over a stand-in for the ~25 TensorFlow/Keras primitives they call
    (tests/golden/tf_shim.py, tests/golden/make_reference_golden.py; agreement to 1e-9 on 19 layer cases and
    14 assembled models, inference and training-mode BatchNormalization);
  * NOT pinned by anything but the public Keras documentation: the losses, the Adam update and the
    BatchNormalization moving-statistics update (they run inside ``keras.Model.fit``), and TensorFlow's
    floating-point summation order.

Every function takes/returns torch tensors on CPU; dtype follows the inputs (float32 mirrors the
reference, float64 gives a high-precision check), and autograd through these functions is the
backward oracle.
"""
import contextlib
import math
import sys
import torch

# ---------------------------------------------------------------------------------------------
# Optional record of the relu and max decisions a forward pass takes (off unless `recording` installs a list).
# A float32 forward can decide an entry the other way where the float64 input lies within rounding of the
# threshold or of the runner-up; a gradient check needs to know which entries those are.
# ---------------------------------------------------------------------------------------------
_recorder = None


@contextlib.contextmanager
def recording(entries):
    """While active, every relu (`activation(..., 'relu')`, the bare relus of multihead_attention and senet) and every
    max (SENET's amax, each maxpool_fields window) appends (site, x, y, dim) to `entries`: the input x, the output y
    and the reduced axis of a max (None for a relu).  site names the oracle function that took the decision."""
    global _recorder
    prev, _recorder = _recorder, entries
    try:
        yield entries
    finally:
        _recorder = prev


def _decision(x, y, dim=None):
    if _recorder is None:
        return y
    frame = sys._getframe(1)
    while frame.f_code.co_name in ('_decision', 'activation', 'dense', 'relu'):
        frame = frame.f_back
    _recorder.append((frame.f_code.co_name, x, y, dim))
    return y


def relu(x):
    return _decision(x, torch.relu(x))


# ---------------------------------------------------------------------------------------------
# Keras-default facts the reference relies on implicitly (SURVEY.md section 8c)
# ---------------------------------------------------------------------------------------------
BN_EPS = 1e-3          # keras BatchNormalization epsilon default
BN_MOMENTUM = 0.99     # keras BatchNormalization momentum default
ADAM_LR, ADAM_B1, ADAM_B2, ADAM_EPS = 1e-3, 0.9, 0.999, 1e-7   # keras.optimizers.Adam defaults
BCE_EPS = 1e-7         # keras backend epsilon used to clip probabilities in binary_crossentropy


def activation(x, name):
    """keras Activation(name) for the names the hot path uses (layers.py:672, deepnets.py:424)."""
    if name is None or name == 'linear':
        return x
    if name == 'relu':
        return relu(x)
    if name == 'sigmoid':
        return torch.sigmoid(x)
    if name == 'tanh':
        return torch.tanh(x)
    raise ValueError(f'oracle: unsupported activation {name!r}')


def embedding_lookup(tables, indices):
    """MultiColumnEmbedding.call (layers.py:889-904), dropout off.

    tables: list of F tensors (V_i, D_i); indices: (B, F) any numeric dtype.  The reference casts
    non-integer inputs to int32 (layers.py:893-895) -- exact for ids < 2**24 when they arrive as
    float32 (dataset_generator.py:41-42).  Returns a list of F tensors (B, 1, D_i).
    """
    if indices.dtype not in (torch.int32, torch.int64):
        indices = indices.to(torch.int32)
    idx = indices.long()
    out = []
    for i, tab in enumerate(tables):
        col = idx[:, i:i + 1]                                   # tf.split(inputs, F, axis=1)
        if bool((col < 0).any()) or bool((col >= tab.shape[0]).any()):
            raise IndexError(f'embedding index out of range for column {i}')  # TF-CPU raises too
        out.append(tab[col])                                    # embedding_lookup -> (B,1,D)
    return out


def concat_embeddings(embeddings):
    """deepnets._concat_embeddings (deepnets.py:30-40): Concatenate(axis=1) -> (B, F, D)."""
    if embeddings is None or len(embeddings) == 0:
        return None
    if len(embeddings) == 1:
        return embeddings[0]
    return torch.cat(embeddings, dim=1)


def flatten_embeddings(embeddings):
    """deepmodel.py:269-274: Concatenate(axis=-1) -> (B,1,sum D) -> Flatten -> (B, sum D), field-major."""
    if len(embeddings) == 0:
        return None
    if len(embeddings) == 1:
        return embeddings[0].reshape(embeddings[0].shape[0], -1)
    return torch.cat(embeddings, dim=-1).reshape(embeddings[0].shape[0], -1)


def batch_norm(x, gamma, beta, moving_mean, moving_var, training, eps=BN_EPS, momentum=BN_MOMENTUM):
    """keras BatchNormalization(axis=-1) (deepmodel.py:359, layers.py:112,152, deepnets.py:422).

    Training: biased batch moments over every axis but the last; returns (y, new_mean, new_var)
    with moving = moving*momentum + batch*(1-momentum).  Inference: moving statistics.
    """
    if training:
        red = tuple(range(x.dim() - 1))
        mean = x.mean(dim=red)
        # keras ops.moments -> tf.nn.moments: mean(squared_difference(x, stop_gradient(mean)))
        var = torch.square(x - mean.detach()).mean(dim=red)
        y = (x - mean) * torch.rsqrt(var + eps) * gamma + beta
        new_mean = moving_mean * momentum + mean.detach() * (1.0 - momentum)
        new_var = moving_var * momentum + var.detach() * (1.0 - momentum)
        return y, new_mean, new_var
    y = (x - moving_mean) * torch.rsqrt(moving_var + eps) * gamma + beta
    return y, moving_mean, moving_var


def dense(x, kernel, bias=None, act=None):
    """keras Dense: x @ kernel (+ bias) -> activation."""
    y = x @ kernel
    if bias is not None:
        y = y + bias
    return activation(y, act)


def linear(embeddings, dense_layer, kernel):
    """deepnets.linear (deepnets.py:43-66): sum each field embedding over D, concat the
    continuous inputs, Dense(1, no bias)."""
    x_emb = None
    cat = concat_embeddings(embeddings)
    if cat is not None:
        x_emb = cat.sum(dim=-1)                                 # keras.ops.sum(axis=-1) -> (B,F)
    if x_emb is not None and dense_layer is not None:
        x = torch.cat([x_emb, dense_layer], dim=-1)
    elif x_emb is not None:
        x = x_emb
    elif dense_layer is not None:
        x = dense_layer
    else:
        raise ValueError('No input layer exists.')
    return x @ kernel                                           # (B,1)


def fm(x):
    """FM.call (layers.py:53-62): 0.5 * sum_d[(sum_f x)^2 - sum_f x^2] -> (B,1)."""
    if x.dim() != 3:
        raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
    square_of_sum = torch.square(x.sum(dim=1, keepdim=True))
    sum_of_square = (x * x).sum(dim=1, keepdim=True)
    cross = square_of_sum - sum_of_square
    return 0.5 * cross.sum(dim=2, keepdim=False)


def cin_field_nums(f0, cross_layer_size, direct):
    """CIN.build field bookkeeping (layers.py:643,665-671)."""
    field_nums = [int(f0)]
    for i, size in enumerate(cross_layer_size):
        if direct:
            field_nums.append(size)
        else:
            if i != len(cross_layer_size) - 1 and size % 2 > 0:
                raise ValueError(
                    'cross_layer_size must be even number except for the last layer when direct=True')
            field_nums.append(size // 2)
    return field_nums


def cin(x, params, weights):
    """CIN.call (layers.py:682-734).

    x: (B, F0, D).  weights: dict with 'f_{k}' (1, F0*H_k, L_k) [or 'f0_{k}' (1,L,F0,D) and
    'f__{k}' (1,L,D,H_k) when reduce_D], optional 'bias{k}' (L_k,), 'exFM_out/kernel'
    (P,1) + 'exFM_out/bias' (1,), and for use_residual 'exFM_out0/kernel' (P, L_last) + bias.
    The TF op sequence (split / batched matmul / reshape / transpose / conv1d) is kept verbatim.
    """
    if x.dim() != 3:
        raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
    sizes = tuple(params.get('cross_layer_size', (128, 128)))
    act = params.get('activation', 'relu')
    use_residual = params.get('use_residual', False)
    use_bias = params.get('use_bias', False)
    direct = params.get('direct', False)
    reduce_d = params.get('reduce_D', False)
    b, f0, dim = x.shape
    field_nums = cin_field_nums(f0, sizes, direct)
    hidden = [x]
    final_result = []
    split0 = x.permute(2, 0, 1).unsqueeze(-1)                   # tf.split(x, D*[1], 2) -> (D,B,F0,1)
    for idx, layer_size in enumerate(sizes):
        split = hidden[-1].permute(2, 0, 1).unsqueeze(-1)       # (D,B,H,1)
        # tf.matmul(split0, split, transpose_b=True): (D,B,F0,1) x (D,B,1,H) -> (D,B,F0,H).  An inner
        # dimension of 1 makes every output a single product, so the broadcast multiply below is
        # bit-identical to the batched matmul and far cheaper on CPU.
        dot_m = split0 * split.transpose(-1, -2)
        dot_o = dot_m.reshape(dim, -1, field_nums[0] * field_nums[idx])
        dot = dot_o.permute(1, 0, 2)                            # (B,D,F0*H)
        if reduce_d:
            f_m = weights[f'f0_{idx}'] @ weights[f'f__{idx}']   # (1,L,F0,H)
            f_o = f_m.reshape(1, layer_size, field_nums[0] * field_nums[idx])
            filters = f_o.permute(0, 2, 1)
        else:
            filters = weights[f'f_{idx}']
        curr = dot @ filters[0]                                 # conv1d, width 1, VALID == GEMM (B,D,L)
        if use_bias:
            curr = curr + weights[f'bias{idx}']
        curr = activation(curr, act)
        curr = curr.permute(0, 2, 1)                            # (B,L,D)
        if direct:
            direct_connect, next_hidden = curr, curr
        else:
            if idx != len(sizes) - 1:
                next_hidden, direct_connect = torch.split(curr, 2 * [layer_size // 2], dim=1)
            else:
                direct_connect, next_hidden = curr, None
        final_result.append(direct_connect)
        hidden.append(next_hidden)
    result = torch.cat(final_result, dim=1).sum(dim=-1)        # (B, sum L')
    if use_residual:
        out0 = dense(result, weights['exFM_out0/kernel'], weights['exFM_out0/bias'], act)
        ex_in = torch.cat([out0, result], dim=1)
        return dense(ex_in, weights['exFM_out/kernel'], weights['exFM_out/bias'])
    return dense(result, weights['exFM_out/kernel'], weights['exFM_out/bias'])


def cin_pooled_width(f0, params):
    sizes = tuple(params.get('cross_layer_size', (128, 128)))
    direct = params.get('direct', False)
    if direct:
        return sum(sizes)
    return sum(s // 2 for s in sizes[:-1]) + sizes[-1]


def cross(x, kernels, biases):
    """Cross.call (layers.py:428-436): x_{l+1} = x0 (x_l^T w_l) + x_l + b_l.
    kernels[i], biases[i]: (W, 1)."""
    if x.dim() != 2:
        raise ValueError(f'Wrong dimensions of x, expected 2 but input {x.dim()}.')
    x_f = x.unsqueeze(-1)                                       # (B,W,1)
    x_n = x_f
    for w, bias in zip(kernels, biases):
        xw = torch.tensordot(x_n, w, dims=([1], [0]))           # (B,1,1)
        x_n = x_f @ xw + x_n + bias
    return x_n.reshape(-1, x_f.shape[1])


def multihead_attention(x, params, weights, bn_state, training):
    """MultiheadAttention.call (layers.py:115-153), dropout_rate 0.

    weights: 'dense_Q|K|V|residual/kernel' (D,D) and '/bias' (D,), 'batch_normalize/gamma|beta'.
    bn_state: dict moving_mean / moving_variance (D,).  Returns (y, new_bn_state)."""
    if x.dim() != 3:
        raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
    num_heads = params.get('num_heads', 1)
    use_residual = params.get('use_residual', True)
    q = dense(x, weights['dense_Q/kernel'], weights['dense_Q/bias'], 'relu')
    k = dense(x, weights['dense_K/kernel'], weights['dense_K/bias'], 'relu')
    v = dense(x, weights['dense_V/kernel'], weights['dense_V/bias'], 'relu')
    if use_residual:
        v_res = dense(x, weights['dense_residual/kernel'], weights['dense_residual/bias'], 'relu')
    q_ = torch.cat(torch.chunk(q, num_heads, dim=2), dim=0)     # split on last axis, stack on batch
    k_ = torch.cat(torch.chunk(k, num_heads, dim=2), dim=0)
    v_ = torch.cat(torch.chunk(v, num_heads, dim=2), dim=0)
    w = q_ @ k_.transpose(1, 2)
    w = w / (k_.shape[-1] ** 0.5)
    w = torch.softmax(w, dim=-1)
    out = w @ v_
    out = torch.cat(torch.chunk(out, num_heads, dim=0), dim=2)
    if use_residual:
        out = out + v_res
    out = relu(out)
    y, nm, nv = batch_norm(out, weights['batch_normalize/gamma'], weights['batch_normalize/beta'],
                           bn_state['moving_mean'], bn_state['moving_variance'], training)
    return y, {'moving_mean': nm, 'moving_variance': nv}


def pair_lists(num_inputs):
    """InnerProduct/OuterProduct pair ordering (layers.py:478-483, 546-551): i<j, row-major."""
    row, col = [], []
    for i in range(num_inputs - 1):
        for j in range(i + 1, num_inputs):
            row.append(i)
            col.append(j)
    return row, col


def inner_product(embeddings):
    """InnerProduct.call (layers.py:473-487)."""
    n = len(embeddings)
    num_pairs = int(n * (n - 1) / 2)
    row, col = pair_lists(n)
    p = torch.cat([embeddings[i] for i in row], dim=1)
    q = torch.cat([embeddings[j] for j in col], dim=1)
    return (p * q).sum(dim=-1).reshape(-1, num_pairs)


def outer_product(embeddings, kernel, kernel_type='mat'):
    """OuterProduct.call (layers.py:541-581).  mat kernel (D,P,D); vec (P,D); num (P,1)."""
    if kernel_type not in ('mat', 'vec', 'num'):
        raise ValueError('kernel_type must be mat,vec or num')
    n = len(embeddings)
    row, col = pair_lists(n)
    p = torch.cat([embeddings[i] for i in row], dim=1)          # (B,P,D)
    q = torch.cat([embeddings[i] for i in col], dim=1)
    if kernel_type == 'mat':
        p4 = p.unsqueeze(1)                                     # (B,1,P,D)
        inner = (p4 * kernel).sum(dim=-1)                       # (B,D,P)   sum_d p[b,p,d] K[k,p,d]
        kp = (inner.permute(0, 2, 1) * q).sum(dim=-1)           # (B,P)
    else:
        kp = (p * q * kernel.unsqueeze(0)).sum(dim=-1)
    return kp


def afm(embeddings, att_kernel, att_bias, projection_h, out_kernel, act='relu'):
    """AFM.call (layers.py:790-807): list of F tensors (B,1,D) -> (B,1).
    bi = e_i * e_j over itertools.combinations (same order as pair_lists); attention MLP Dense(hidden_factor, act)
    (kernel (D,H), bias (H)); score = softmax over the PAIRS of (attention . projection_h (H,1)); the score-weighted sum of
    the pair products (B,D) goes through Dense(1, use_bias=False) (kernel (D,1)).  Dropout is identity (rate 0 / inference)."""
    if embeddings[0].dim() != 3:
        raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {embeddings[0].dim()}.')
    row, col = pair_lists(len(embeddings))
    p = torch.cat([embeddings[i] for i in row], dim=1)          # (B,P,D)
    q = torch.cat([embeddings[i] for i in col], dim=1)
    bi = p * q
    att = activation(bi @ att_kernel + att_bias, act)           # (B,P,H)
    score = torch.softmax(torch.tensordot(att, projection_h, dims=([-1], [0])), dim=1)      # (B,P,1)
    pooled = (score * bi).sum(dim=1)                            # (B,D)
    return pooled @ out_kernel                                  # (B,1)


def afm_pooled(embeddings, att_kernel, att_bias, projection_h, act='relu'):
    """The (B,D) attention-pooled pair product of afm() (what the fused kernel emits, before Dropout and Dense(1))."""
    row, col = pair_lists(len(embeddings))
    bi = torch.cat([embeddings[i] for i in row], dim=1) * torch.cat([embeddings[i] for i in col], dim=1)
    att = activation(bi @ att_kernel + att_bias, act)
    score = torch.softmax(torch.tensordot(att, projection_h, dims=([-1], [0])), dim=1)
    return (score * bi).sum(dim=1)


def senet(x, att1_kernel, att1_bias, att2_kernel, att2_bias, pooling_op='mean'):
    """SENET.call (layers.py:291-303): x (B,F,D).  Z = mean (or max) over the embedding axis (B,F);
    A = relu(Dense(F)(relu(Dense(max(F // reduction_ratio, 1))(Z)))); V = x * A[:, :, None]."""
    if x.dim() != 3:
        raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
    # amax: ties share the gradient, as tf.reduce_max does
    z = _decision(x, x.amax(dim=-1), -1) if pooling_op == 'max' else x.mean(dim=-1)
    a1 = relu(z @ att1_kernel + att1_bias)
    a2 = relu(a1 @ att2_kernel + att2_bias)
    return x * a2.unsqueeze(2)


def bilinear_interaction(x, weights, bilinear_type='field_interaction'):
    """BilinearInteraction.call (layers.py:358-372): x (B,F,D) -> (B,P,D), pair order of itertools.combinations.
    field_all: one W (D,D), (v_i W) * v_j;  field_each: W_i per first field (F-1 of them);
    field_interaction: one W per pair, in pair order."""
    if x.dim() != 3:
        raise ValueError(f'Wrong dimensions of inputs, expected 3 but input {x.dim()}.')
    f = x.shape[1]
    row, col = pair_lists(f)
    outs = []
    for n, (i, j) in enumerate(zip(row, col)):
        if bilinear_type == 'field_all':
            w = weights[0]
        elif bilinear_type == 'field_each':
            w = weights[i]
        else:
            w = weights[n]
        outs.append((x[:, i:i + 1, :] @ w) * x[:, j:j + 1, :])
    return torch.cat(outs, dim=1)


def same_padding(size, k, stride):
    """TensorFlow 'SAME' padding along one axis: (before, after, output size)."""
    out = -(-size // stride)
    total = max((out - 1) * stride + k - size, 0)
    return total // 2, total - total // 2, out


def conv_fields(x, kernel, bias, act='tanh'):
    """Conv2D(filters, kernel_size=(kh, 1), strides 1, padding='same', channels_last) of FGCNN.build (layers.py:204-212):
    x (B, H, W, Cin), kernel (kh, 1, Cin, Cout); the convolution runs along the FIELD axis H only."""
    kh = kernel.shape[0]
    before, after, _ = same_padding(x.shape[1], kh, 1)
    xp = torch.nn.functional.pad(x, (0, 0, 0, 0, before, after))          # pad H
    h = x.shape[1]
    y = sum(torch.einsum('bhwc,co->bhwo', xp[:, t:t + h], kernel[t, 0]) for t in range(kh))
    return activation(y + bias, act)


def maxpool_fields(x, pool):
    """MaxPooling2D(pool_size=(pool, 1), padding='same') (layers.py:214): windows of `pool` fields, stride `pool`,
    TensorFlow 'SAME' padding (padded cells never win)."""
    before, _, out = same_padding(x.shape[1], pool, pool)
    rows = []
    for o in range(out):
        lo, hi = max(o * pool - before, 0), min(o * pool - before + pool, x.shape[1])
        win = x[:, lo:hi]
        rows.append(_decision(win, win.max(dim=1).values, 1))   # the gradient goes to the first maximum (TensorFlow's MaxPoolGrad argmax)
    return torch.stack(rows, dim=1)


def fgcnn(x, conv_kernel, conv_bias, dense_kernel, dense_bias, pool_height, new_filters, act='tanh'):
    """FGCNN.call (layers.py:223-232): x (B, F, D, C) -> (pooling_output (B, F', D, filters), new_features (B, F*new_filters, D))."""
    out = conv_fields(x, conv_kernel, conv_bias, act)
    pooled = maxpool_fields(out, pool_height)
    new = activation(pooled.reshape(pooled.shape[0], -1) @ dense_kernel + dense_bias, act)
    return pooled, new.reshape(-1, out.shape[1] * new_filters, out.shape[2])


def dnn(x, params, weights, bn_state, training, cellname='dnn'):
    """deepnets.dnn (deepnets.py:401-427): [Dense(use_bias=not bn) -> BN? -> act -> Dropout?]*.
    Dropout layers are identity in this oracle (parity runs use rate 0 / inference)."""
    hidden_units = params.get('hidden_units', ((128, 0, True), (64, 0, False)))
    act = params.get('activation', 'relu')
    if len(hidden_units) <= 0:
        raise ValueError('[hidden_units] must be a list of tuple([units],[dropout_rate],[use_bn]) '
                         'and at least one tuple.')
    new_state = {}
    for index, (units, dropout, use_bn) in enumerate(hidden_units, start=1):
        name = f'{cellname}_dense_{index}'
        x = dense(x, weights[f'{name}/kernel'], None if use_bn else weights[f'{name}/bias'])
        if use_bn:
            bn = f'{cellname}_bn_{index}'
            x, nm, nv = batch_norm(x, weights[f'{bn}/gamma'], weights[f'{bn}/beta'],
                                   bn_state[f'{bn}/moving_mean'], bn_state[f'{bn}/moving_variance'],
                                   training)
            new_state[f'{bn}/moving_mean'] = nm
            new_state[f'{bn}/moving_variance'] = nv
        x = activation(x, act)
    return x, new_state


def binary_crossentropy(y_true, y_pred, eps=BCE_EPS):
    """keras binary_crossentropy on probabilities + 'sum_over_batch_size' reduction
    (deepmodel.py:327-329): clip to [eps, 1-eps], mean over the last axis, mean over the batch."""
    p = torch.clamp(y_pred, eps, 1.0 - eps)
    bce = y_true * torch.log(p) + (1.0 - y_true) * torch.log(1.0 - p)
    return (-bce).mean(dim=-1).mean()


def mean_squared_error(y_true, y_pred):
    return torch.square(y_pred - y_true).mean(dim=-1).mean()


def categorical_crossentropy(y_true, y_pred, eps=BCE_EPS):
    """keras categorical_crossentropy on probabilities: renormalise, clip, -sum y log p."""
    p = y_pred / y_pred.sum(dim=-1, keepdim=True)
    p = torch.clamp(p, eps, 1.0 - eps)
    return (-(y_true * torch.log(p)).sum(dim=-1)).mean()


def binary_focal_loss(y_true, y_pred, gamma=2.0, alpha=0.25, eps=BCE_EPS):
    """BinaryFocalLoss.call (layers.py:1006-1017) on probabilities: a SCALAR, both terms averaged over every element.
    pt_1 = p where y == 1 else 1; pt_0 = p where y == 0 else 0; both clipped to [eps, 1 - eps]."""
    pt_1 = torch.where(y_true == 1, y_pred, torch.ones_like(y_pred)).clamp(eps, 1.0 - eps)
    pt_0 = torch.where(y_true == 0, y_pred, torch.zeros_like(y_pred)).clamp(eps, 1.0 - eps)
    return -(alpha * torch.pow(1.0 - pt_1, gamma) * torch.log(pt_1)).mean() \
        - ((1.0 - alpha) * torch.pow(pt_0, gamma) * torch.log(1.0 - pt_0)).mean()


def categorical_focal_loss(y_true, y_pred, gamma=2.0, alpha=0.25, eps=BCE_EPS):
    """CategoricalFocalLoss.call (layers.py:1061-1077) on probabilities: per-sample losses (B,) -- renormalise, clip,
    alpha (1 - p)^gamma (-y log p) summed over the classes.  Keras then averages over the batch."""
    p = y_pred / y_pred.sum(dim=-1, keepdim=True)
    p = torch.clamp(p, eps, 1.0 - eps)
    return (alpha * torch.pow(1.0 - p, gamma) * (-y_true * torch.log(p))).sum(dim=1)


def adam_step(p, g, m, v, step, lr=ADAM_LR, b1=ADAM_B1, b2=ADAM_B2, eps=ADAM_EPS):
    """keras.optimizers.Adam.update_step (dense semantics; deepmodel.py:321-322).
    step is 1-based.  Updates p, m, v in place (all same shape)."""
    b1p = b1 ** step
    b2p = b2 ** step
    alpha = lr * math.sqrt(1.0 - b2p) / (1.0 - b1p)
    m.add_((g - m) * (1.0 - b1))
    v.add_((g * g - v) * (1.0 - b2))
    p.sub_(m * alpha / (torch.sqrt(v) + eps))
