"""The optimiser surface without a GPU: the CPU restatements of Keras's SGD / RMSprop / Adagrad against torch.optim in
float64 (where the two forms coincide), and ModelConfig.optimizer resolution."""
import pickle

import numpy as np
import pytest
import torch

import optim_ref as R
from deeptables_b200 import optimizers as O

STEPS = 20
ZERO_STEPS = {4, 9, 10, 15}          # whole-gradient zero steps (after the first, so that RMSprop's v > 0 with eps = 0)


def _grads(n=37, seed=0):
    g = torch.Generator().manual_seed(seed)
    out = []
    for s in range(STEPS):
        x = torch.randn(n, generator=g, dtype=torch.float64)
        if s in ZERO_STEPS:
            x.zero_()
        out.append(x)
    return out


def _run_torch(make_opt, p0, grads):
    p = torch.nn.Parameter(p0.clone())
    opt = make_opt([p])
    for g in grads:
        p.grad = g.clone()
        opt.step()
    return p.detach()


def _run_ref(spec, p0, grads):
    p = p0.clone()
    slots = R.new_slots(spec, p)
    for t, g in enumerate(grads, 1):
        R.step(spec, p, g, slots, t)
    return p


@pytest.mark.parametrize('momentum,nesterov', [(0.0, False), (0.9, False), (0.9, True), (0.5, True)])
def test_sgd_matches_torch(momentum, nesterov):
    p0 = torch.randn(37, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    grads = _grads()
    spec = O.resolve(O.SGD(learning_rate=0.05, momentum=momentum, nesterov=nesterov))
    want = _run_torch(lambda ps: torch.optim.SGD(ps, lr=0.05, momentum=momentum, nesterov=nesterov), p0, grads)
    torch.testing.assert_close(_run_ref(spec, p0, grads), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('momentum', [0.0, 0.9])
@pytest.mark.parametrize('centered', [False, True])
def test_rmsprop_matches_torch(momentum, centered):
    """torch's RMSprop adds eps after the square root, Keras inside it: they coincide at eps = 0 (alpha = rho)."""
    p0 = torch.randn(37, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    grads = _grads(seed=3)
    spec = O.resolve(O.RMSprop(learning_rate=0.01, rho=0.8, momentum=momentum, epsilon=0.0, centered=centered))
    want = _run_torch(lambda ps: torch.optim.RMSprop(ps, lr=0.01, alpha=0.8, eps=0.0, momentum=momentum,
                                                     centered=centered), p0, grads)
    torch.testing.assert_close(_run_ref(spec, p0, grads), want, rtol=1e-12, atol=1e-12)


def test_adagrad_matches_torch():
    """torch's Adagrad adds eps after the square root, Keras inside it: they coincide at eps = 0."""
    p0 = torch.randn(37, dtype=torch.float64, generator=torch.Generator().manual_seed(4))
    grads = _grads(seed=5)
    spec = O.resolve(O.Adagrad(learning_rate=0.1, initial_accumulator_value=0.1, epsilon=0.0))
    want = _run_torch(lambda ps: torch.optim.Adagrad(ps, lr=0.1, initial_accumulator_value=0.1, eps=0.0), p0, grads)
    torch.testing.assert_close(_run_ref(spec, p0, grads), want, rtol=1e-12, atol=1e-12)


def test_names_resolve_to_keras_defaults_in_any_case():
    assert O.resolve('SGD') == O.resolve('sgd') == O.OptimizerSpec('sgd', 0.01, momentum=0.0, nesterov=False)
    assert O.resolve('RMSprop') == O.resolve('rmsprop') == O.resolve('RMSPROP') == \
        O.OptimizerSpec('rmsprop', 0.001, epsilon=1e-7, momentum=0.0, rho=0.9, centered=False)
    assert O.resolve('Adagrad') == O.resolve('adagrad') == \
        O.OptimizerSpec('adagrad', 0.001, epsilon=1e-7, initial_accumulator_value=0.1)
    auto = O.resolve('auto')
    assert auto == O.OptimizerSpec('adam', 0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7)
    assert O.resolve('adam') == O.resolve('Adam') == O.resolve(O.Adam()) == auto
    assert hash(auto) == hash(O.resolve(O.Adam()))
    assert [O.resolve(n).keras_name for n in ('auto', 'sgd', 'rmsprop', 'adagrad')] == ['Adam', 'SGD', 'RMSprop', 'Adagrad']


def test_instances_and_keras_like_objects_resolve():
    spec = O.resolve(O.RMSprop(learning_rate=3e-3, rho=0.95, momentum=0.5, epsilon=1e-6, centered=True))
    assert spec == O.OptimizerSpec('rmsprop', 3e-3, epsilon=1e-6, momentum=0.5, rho=0.95, centered=True)
    assert O.resolve(O.SGD(0.1, 0.9, True)) == O.OptimizerSpec('sgd', 0.1, momentum=0.9, nesterov=True)
    assert O.resolve(O.Adam(learning_rate=3e-3, beta_1=0.8, beta_2=0.99, epsilon=1e-6)) == \
        O.OptimizerSpec('adam', 3e-3, beta_1=0.8, beta_2=0.99, epsilon=1e-6)

    class RMSprop:               # what keras.optimizers.RMSprop() is: read through get_config()
        def get_config(self):
            return {'name': 'rmsprop', 'learning_rate': 0.0010000000474974513, 'weight_decay': None, 'clipnorm': None,
                    'global_clipnorm': None, 'clipvalue': None, 'use_ema': False, 'ema_momentum': 0.99,
                    'ema_overwrite_frequency': None, 'loss_scale_factor': None, 'gradient_accumulation_steps': None,
                    'rho': 0.9, 'momentum': 0.0, 'epsilon': 1e-07, 'centered': False}

    spec = O.resolve(RMSprop())
    assert spec.kind == 'rmsprop' and spec.rho == 0.9 and not spec.centered
    assert np.float32(spec.learning_rate) == np.float32(0.001)
    # the optimiser objects pickle with the ModelConfig that holds them (DeepTable.save / load)
    opt = pickle.loads(pickle.dumps(O.Adagrad(learning_rate=0.05, initial_accumulator_value=0.2)))
    assert O.resolve(opt) == O.OptimizerSpec('adagrad', 0.05, epsilon=1e-7, initial_accumulator_value=0.2)
    assert opt.learning_rate == 0.05 and opt.get_config()['name'] == 'adagrad'


@pytest.mark.parametrize('optimizer,named', [
    ('nadam', 'nadam'), ('Adamax', 'Adamax'), ('adamw', 'adamw'), ('ftrl', 'ftrl'), ('adadelta', 'adadelta'),
    ('lion', 'lion'), (object(), 'object'),
    (O.Adam(amsgrad=True), 'amsgrad'),
    (O.SGD(weight_decay=0.01), 'weight_decay'), (O.RMSprop(clipnorm=1.0), 'clipnorm'), (O.Adam(clipvalue=0.5), 'clipvalue'),
    (O.Adagrad(global_clipnorm=1.0), 'global_clipnorm'), (O.SGD(use_ema=True), 'use_ema'),
    (O.Adam(loss_scale_factor=128.0), 'loss_scale_factor'), (O.RMSprop(gradient_accumulation_steps=4),
                                                              'gradient_accumulation_steps'),
    (O.Adam(learning_rate={'class_name': 'ExponentialDecay'}), 'learning_rate')])
def test_unsupported_options_are_rejected_by_name(optimizer, named):
    with pytest.raises(NotImplementedError, match=named):
        O.resolve(optimizer)


def test_weight_decay_zero_and_unknown_keywords():
    assert O.resolve(O.SGD(weight_decay=0.0)) == O.resolve('sgd')
    with pytest.raises(TypeError):
        O.SGD(decay=0.1)
    with pytest.raises(ValueError):
        O.resolve(O.SGD(momentum=1.5))


def test_state_slots():
    assert O.slot_inits(O.resolve('sgd')) == (None, None, None)
    assert O.slot_inits(O.resolve(O.SGD(momentum=0.9))) == (0.0, None, None)
    assert O.slot_inits(O.resolve('rmsprop')) == (0.0, None, None)
    assert O.slot_inits(O.resolve(O.RMSprop(momentum=0.9, centered=True))) == (0.0, 0.0, 0.0)
    assert O.slot_inits(O.resolve(O.Adagrad(initial_accumulator_value=0.3))) == (0.3, None, None)
