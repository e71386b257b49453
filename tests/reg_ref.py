"""Float64 restatement of Keras 3's L1 / L2 / L1L2 weight regularizers and a reference trainer that trains with them.

Keras 3 (what the reference runs on) adds ``l1 * sum|w| + l2 * sum w^2`` of every regularized weight to the training
loss, taken on the weights before the step; its gradient ``l1 * sign(w) + 2 * l2 * w`` (``sign(0) = 0``, TensorFlow's
gradient of ``abs``) joins the data gradient that the optimiser sees.  The formulas are checked against
``torch.autograd`` in tests/test_regularizers_cpu.py."""
import re

import torch

import optim_ref as OR


def reg_loss(w, l1, l2):
    return l1 * w.abs().sum() + l2 * (w * w).sum()


def reg_grad(w, l1, l2):
    return l1 * torch.sign(w) + 2.0 * l2 * w


def regularized_weights(state, emb_reg=None, kernel_reg=None, kernel_pattern=r'^dnn_dense_\d+/kernel$'):
    """state key -> (l1, l2): the embedding tables under ``emb_reg`` and the DNN tower's Dense kernels (the reference's
    ``dnn()`` passes ``kernel_regularizer`` to them, not to their biases) under ``kernel_reg``.  Both are
    ``regularizers.RegSpec`` or None."""
    out = {}
    for k in state:
        if emb_reg is not None and re.search(r'/embeddings_\d+$', k):
            out[k] = (emb_reg.l1, emb_reg.l2)
        elif kernel_reg is not None and re.match(kernel_pattern, k):
            out[k] = (kernel_reg.l1, kernel_reg.l2)
    return out


class RegRefTrainer(OR.OptimRefTrainer):
    """OptimRefTrainer (any optimiser, float64 by default) whose loss includes the regularization terms of
    ``regs`` (state key -> (l1, l2))."""

    def __init__(self, state, config, n_fields, regs, optimizer, dtype=torch.float64):
        super().__init__(state, config, n_fields, dtype=dtype, optimizer=optimizer)
        self.regs = dict(regs)

    def reg_term(self):
        return sum(float(reg_loss(self.state[k], *r)) for k, r in self.regs.items())

    def train_step(self, cat_idx, cont, y):
        loss, grads, new_bn, _ = self.loss_and_grads(cat_idx, cont, y)
        total = float(loss) + self.reg_term()
        for k, r in self.regs.items():
            grads[k] = grads[k] + reg_grad(self.state[k], *r)
        self.step += 1
        for k, g in grads.items():
            OR.step(self.opt, self.state[k], g, self.slots[k], self.step)
        self.state.update(new_bn)
        return total
