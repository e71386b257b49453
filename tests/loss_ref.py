"""Float64 restatement of the Keras 3 losses ``ModelConfig.loss`` takes (deeptables_b200/losses.py) and a reference
trainer that trains with one of them.

Keras is not installed here; the formulas are Keras 3's ``keras/src/losses/losses.py`` as the header of
``dtb_keras_loss_fwd_bwd`` states them.  Gradients come from ``torch.autograd`` and follow TensorFlow's conventions
because of how the formulas are written: ``torch.clamp`` passes the gradient on [lo, hi] as ``tf.clip_by_value`` does,
``maximum`` below sends it to its first argument on ties as ``tf.maximum`` does (``torch.maximum`` would split it),
``torch.abs`` has ``abs'(0) = 0``, ``torch.amax`` splits it among tied maxima as ``tf.reduce_max`` does, and
``torch.where`` sends it to the branch it takes."""
import math

import numpy as np
import torch

import optim_ref as OR
from oracle import model_ref as M

# the float32 constants Keras computes with: epsilon and the upper clip bound 1 - epsilon, 0.99999988 in float32 (1.19e-7
# below 1, not 1e-7: the loss of a clipped probability differs by 19% or, through log(1 - p), by 1%)
EPS = float(np.float32(1e-7))
ONE_MINUS_EPS = float(np.float32(1.0 - 1e-7))


def maximum(a, b):
    """tf.maximum: the gradient goes to ``a`` where a >= b."""
    b = torch.as_tensor(b, dtype=a.dtype)
    return torch.where(a >= b, a, b)


def output(z, task):
    """The task output of the pre-activation z."""
    if task in ('binary', 'multilabel'):
        return torch.sigmoid(z)
    if task == 'multiclass':
        return torch.softmax(z, dim=-1)
    return z


def labels_are_binary(y):
    """keras convert_binary_labels_to_hinge: every label of the batch is 0 or 1."""
    return bool(((y == 0) | (y == 1)).all())


def per_row(kind, y, p, delta=1.0, label_smoothing=0.0, binary=None):
    """The per-row loss of Keras class ``kind`` on labels y and outputs p, both (rows, C).  ``binary`` is the hinge
    losses' batch-wide flag (computed from y when None)."""
    c = y.shape[-1]
    if kind == 'MeanSquaredError':
        return ((p - y) ** 2).mean(-1)
    if kind == 'MeanAbsoluteError':
        return (y - p).abs().mean(-1)
    if kind == 'MeanAbsolutePercentageError':
        return 100.0 * ((y - p) / maximum(y.abs(), EPS)).abs().mean(-1)
    if kind == 'MeanSquaredLogarithmicError':
        return ((torch.log(maximum(p, EPS) + 1.0) - torch.log(maximum(y, EPS) + 1.0)) ** 2).mean(-1)
    if kind == 'Huber':
        e = p - y
        return torch.where(e.abs() <= delta, 0.5 * e * e, delta * e.abs() - 0.5 * delta * delta).mean(-1)
    if kind == 'LogCosh':
        e = p - y
        return (e + torch.nn.functional.softplus(-2.0 * e) - math.log(2.0)).mean(-1)
    if kind == 'Poisson':
        return (p - y * torch.log(p + EPS)).mean(-1)
    if kind in ('Hinge', 'SquaredHinge'):
        if binary is None:
            binary = labels_are_binary(y)
        yy = 2.0 * y - 1.0 if binary else y
        h = maximum(1.0 - yy * p, 0.0)
        return (h * h if kind == 'SquaredHinge' else h).mean(-1)
    if kind == 'CategoricalHinge':
        pos = (y * p).sum(-1)
        neg = ((1.0 - y) * p).amax(-1)
        return maximum(neg - pos + 1.0, 0.0)
    if kind == 'KLDivergence':
        yh, ph = torch.clamp(y, EPS, 1.0), torch.clamp(p, EPS, 1.0)
        return (yh * torch.log(yh / ph)).sum(-1)
    if kind == 'BinaryCrossentropy':
        ys = y * (1.0 - label_smoothing) + 0.5 * label_smoothing
        pc = torch.clamp(p, EPS, ONE_MINUS_EPS)
        return -(ys * torch.log(pc) + (1.0 - ys) * torch.log(1.0 - pc)).mean(-1)
    if kind == 'CategoricalCrossentropy':
        ys = y * (1.0 - label_smoothing) + label_smoothing / c
        q = torch.clamp(p / p.sum(-1, keepdim=True), EPS, ONE_MINUS_EPS)
        return -(ys * torch.log(q)).sum(-1)
    raise ValueError(kind)


def spec_args(spec):
    """(kind, delta, label_smoothing) of a losses.LossSpec, with the float32 values the kernel reads."""
    return spec.kind, float(np.float32(spec.delta)), float(np.float32(spec.label_smoothing))


def batch_loss(spec, y, p, weights=None):
    """Keras's sum_over_batch_size: sum_r w_r l_r / rows."""
    kind, delta, s = spec_args(spec)
    per = per_row(kind, y, p, delta, s)
    if weights is not None:
        per = per * weights
    return per.sum() / y.shape[0]


class LossRefTrainer(OR.OptimRefTrainer):
    """OptimRefTrainer (float64 by default) whose loss is ``spec`` (a losses.LossSpec) on the task output."""

    def __init__(self, state, config, n_fields, spec, task='binary', optimizer=None, dtype=torch.float64):
        super().__init__(state, config, n_fields, task, dtype, optimizer)
        self.spec = spec

    def loss_and_grads(self, cat_idx, cont, y):
        params = {k: v.detach().clone().requires_grad_(M.is_trainable(k)) for k, v in self.state.items()}
        out, new_bn = M.forward(params, self.config, cat_idx, cont, self.n_fields, True, self.task)
        loss = batch_loss(self.spec, y.to(out.dtype).reshape(out.shape[0], -1), out)
        names = [k for k in params if M.is_trainable(k)]
        grads = torch.autograd.grad(loss, [params[k] for k in names], allow_unused=True)
        gd = {k: (g if g is not None else torch.zeros_like(params[k])) for k, g in zip(names, grads)}
        return loss.detach(), gd, {k: v.detach() for k, v in new_bn.items()}, out.detach()

    def loss(self, cat_idx, cont, y):
        """The evaluation loss (training=False forward) of one batch."""
        out = self.predict(cat_idx, cont)
        return float(batch_loss(self.spec, y.to(out.dtype).reshape(out.shape[0], -1), out))
