"""CPU restatement of Keras 3's SGD, RMSprop and Adagrad ``update_step`` (dense semantics: every trainable weight steps
every iteration, with g = 0 where it has no gradient), and a ``RefTrainer`` that trains with any of them.

Keras is not installable here; these formulas are checked against ``torch.optim`` in float64 where the two forms
coincide (tests/test_optimizers_cpu.py).  ``opt`` is any object with the fields of
``deeptables_b200.optimizers.OptimizerSpec`` (kind, learning_rate, beta_1, beta_2, epsilon, momentum, nesterov, rho,
centered, initial_accumulator_value)."""
import torch

from oracle import layers_ref as L
from oracle import model_ref as M


def sgd_step(p, g, m, lr=0.01, momentum=0.0, nesterov=False):
    """keras.optimizers.SGD.update_step; m is unused (may be None) when momentum == 0."""
    if momentum == 0:
        p.sub_(g * lr)
        return
    m.copy_(m * momentum - g * lr)
    if nesterov:
        p.add_(m * momentum - g * lr)
    else:
        p.add_(m)


def rmsprop_step(p, g, v, a, mom, lr=0.001, rho=0.9, momentum=0.0, epsilon=1e-7, centered=False):
    """keras.optimizers.RMSprop.update_step; a (average gradient) only when centered, mom only when momentum > 0."""
    v.copy_(rho * v + (1 - rho) * g * g)
    if centered:
        a.copy_(rho * a + (1 - rho) * g)
        den = v - a * a + epsilon
    else:
        den = v + epsilon
    inc = lr * g / torch.sqrt(den)
    if momentum > 0:
        mom.copy_(momentum * mom + inc)
        p.sub_(mom)
    else:
        p.sub_(inc)


def adagrad_step(p, g, acc, lr=0.001, epsilon=1e-7):
    """keras.optimizers.Adagrad.update_step; acc starts at initial_accumulator_value."""
    acc.add_(g * g)
    p.sub_(lr * g / torch.sqrt(acc + epsilon))


def new_slots(opt, like):
    """The optimiser's state for one weight, as (s0, s1, s2) like the engine's slots (None where unused)."""
    z = lambda: torch.zeros_like(like)
    if opt.kind == 'adam':
        return (z(), z(), None)
    if opt.kind == 'sgd':
        return (z() if opt.momentum > 0 else None, None, None)
    if opt.kind == 'rmsprop':
        return (z(), z() if opt.centered else None, z() if opt.momentum > 0 else None)
    return (torch.full_like(like, opt.initial_accumulator_value), None, None)


def step(opt, p, g, slots, t):
    """One update of weight p with gradient g; t is the 1-based step (Adam's bias correction)."""
    s0, s1, s2 = slots
    if opt.kind == 'adam':
        L.adam_step(p, g, s0, s1, t, lr=opt.learning_rate, b1=opt.beta_1, b2=opt.beta_2, eps=opt.epsilon)
    elif opt.kind == 'sgd':
        sgd_step(p, g, s0, opt.learning_rate, opt.momentum, opt.nesterov)
    elif opt.kind == 'rmsprop':
        rmsprop_step(p, g, s0, s1, s2, opt.learning_rate, opt.rho, opt.momentum, opt.epsilon, opt.centered)
    elif opt.kind == 'adagrad':
        adagrad_step(p, g, s0, opt.learning_rate, opt.epsilon)
    else:
        raise ValueError(opt.kind)


class OptimRefTrainer(M.RefTrainer):
    """oracle.model_ref.RefTrainer with the optimiser as a parameter (default: Adam(1e-3), RefTrainer's own)."""

    def __init__(self, state, config, n_fields, task='binary', dtype=torch.float32, optimizer=None):
        super().__init__(state, config, n_fields, task, dtype)
        self.opt = optimizer
        if optimizer is not None:
            self.slots = {k: new_slots(optimizer, self.state[k]) for k in self.m}

    def train_step(self, cat_idx, cont, y):
        if self.opt is None:
            return super().train_step(cat_idx, cont, y)
        loss, grads, new_bn, _ = self.loss_and_grads(cat_idx, cont, y)
        self.step += 1
        for k, g in grads.items():
            step(self.opt, self.state[k], g, self.slots[k], self.step)
        self.state.update(new_bn)
        return float(loss)
