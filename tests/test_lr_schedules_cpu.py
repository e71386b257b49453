"""Learning-rate schedules and callbacks on the host: the six Keras 3 schedules against a float64 restatement,
``resolve`` of every accepted form and the rejections, the checkpoint text of unscheduled optimisers, the callbacks
against a fake model, and the rate table the engine builds."""
import json
import math
import types

import numpy as np
import pytest

import lr_ref
from deeptables_b200 import callbacks as C
from deeptables_b200 import optimizers as O
from deeptables_b200 import schedules as S

CASES = {
    'exp': S.ExponentialDecay(0.1, decay_steps=300, decay_rate=0.5),
    'exp_staircase': S.ExponentialDecay(0.1, decay_steps=300, decay_rate=0.5, staircase=True),
    'piecewise': S.PiecewiseConstantDecay(boundaries=[100, 1000, 2500], values=[0.1, 0.05, 0.2, 0.01]),
    'poly': S.PolynomialDecay(0.1, decay_steps=2000, end_learning_rate=0.001, power=2.0),
    'poly_cycle': S.PolynomialDecay(0.1, decay_steps=700, end_learning_rate=0.001, power=0.5, cycle=True),
    'inverse': S.InverseTimeDecay(0.1, decay_steps=200, decay_rate=0.7),
    'inverse_staircase': S.InverseTimeDecay(0.1, decay_steps=200, decay_rate=0.7, staircase=True),
    'cosine': S.CosineDecay(0.1, decay_steps=3000, alpha=0.1),
    'cosine_warmup': S.CosineDecay(0.01, decay_steps=3000, alpha=0.05, warmup_target=0.2, warmup_steps=500),
    'restarts_t1': S.CosineDecayRestarts(0.1, first_decay_steps=400, t_mul=1.0, m_mul=0.8, alpha=0.01),
    'restarts_t2': S.CosineDecayRestarts(0.1, first_decay_steps=300, t_mul=2.0, m_mul=0.9),
}


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


# ---- 1. per-step rates against float64 ---------------------------------------------------------------------------------
@pytest.mark.parametrize('case', list(CASES))
def test_schedule_rates_match_float64(case):
    sched = CASES[case]
    desc = S.resolve(sched)
    name, config = S.to_config(desc)
    t = np.arange(0, 5001)
    got = S.rates(desc, t)
    want = np.array([lr_ref.rate(name, config, x) for x in t])
    # one float32 rounding of float64 values; numpy's vector cos / pow may differ from libm's in the last float64 bit
    assert _ulps(got, want).max() <= 1, case
    assert np.array_equal(got, got.astype(np.float32).astype(np.float64)), 'rates are float32 values'
    assert float(sched(17)) == float(got[17])


def test_schedule_boundaries():
    pw = S.resolve(CASES['piecewise'])
    r = S.rates(pw, [0, 100, 101, 1000, 1001, 2500, 2501, 10 ** 6])
    assert list(r) == [float(np.float32(v)) for v in (0.1, 0.1, 0.05, 0.05, 0.2, 0.2, 0.01, 0.01)]
    stair = S.rates(S.resolve(CASES['exp_staircase']), [0, 299, 300, 599, 600])
    assert list(stair) == [float(np.float32(v)) for v in (0.1, 0.1, 0.05, 0.05, 0.025)]
    poly = S.resolve(CASES['poly'])
    assert S.rates(poly, [2000])[0] == S.rates(poly, [9000])[0] == float(np.float32(0.001))
    cyc = S.resolve(CASES['poly_cycle'])
    # with cycle the decay restarts at every multiple of decay_steps; t = 0 uses a multiplier of 1
    assert S.rates(cyc, [0])[0] == float(np.float32(0.1))
    assert S.rates(cyc, [700])[0] == float(np.float32(0.001))
    assert S.rates(cyc, [701])[0] > S.rates(cyc, [700])[0]
    warm = S.resolve(CASES['cosine_warmup'])
    r = S.rates(warm, [0, 250, 500, 3500, 9000])
    assert r[0] == float(np.float32(0.01)) and r[2] == float(np.float32(0.2))
    assert r[1] == float(np.float32(0.01 + (0.2 - 0.01) * 0.5))
    assert r[3] == r[4] == float(np.float32(0.2 * 0.05))
    t1 = S.resolve(CASES['restarts_t1'])
    assert S.rates(t1, [400])[0] == float(np.float32(0.1 * (0.99 * 0.8 + 0.01)))     # first restart: m_mul once
    t2 = S.resolve(CASES['restarts_t2'])
    assert S.rates(t2, [300, 900])[0] == float(np.float32(0.1 * 0.9))
    assert S.rates(t2, [900])[0] == float(np.float32(0.1 * 0.81))         # periods 300, 600: second restart at 900


# ---- 2. resolve -------------------------------------------------------------------------------------------------------------
def test_resolve_instance_keras_object_and_serialized_dict():
    want = S.resolve(S.ExponentialDecay(0.01, 1000, 0.96))

    class ExponentialDecay:                      # what a real keras.optimizers.schedules.ExponentialDecay reports
        def get_config(self):
            return {'initial_learning_rate': 0.01, 'decay_steps': 1000, 'decay_rate': 0.96, 'staircase': False,
                    'name': 'ExponentialDecay'}

    assert S.resolve(ExponentialDecay()) == want
    ser = {'module': 'keras.optimizers.schedules', 'class_name': 'ExponentialDecay',
           'config': ExponentialDecay().get_config(), 'registered_name': None}
    assert S.resolve(ser) == want
    spec = O.resolve(O.Adam(learning_rate=ser))
    assert spec.schedule == want and spec.learning_rate == float(np.float32(0.01))
    for opt in (O.SGD, O.RMSprop, O.Adagrad):
        assert O.resolve(opt(learning_rate=S.CosineDecay(0.1, 100))).schedule == S.resolve(S.CosineDecay(0.1, 100))
    hash(spec)


def test_keras_optimizer_config_with_a_schedule():
    """A real keras.optimizers.Adam(learning_rate=ExponentialDecay(...)).get_config() holds the serialized schedule."""
    class Adam:
        def get_config(self):
            return {'name': 'adam', 'learning_rate': {
                'module': 'keras.optimizers.schedules', 'class_name': 'CosineDecay', 'registered_name': None,
                'config': {'initial_learning_rate': 0.001, 'decay_steps': 500, 'alpha': 0.0, 'name': 'CosineDecay',
                           'warmup_target': 0.01, 'warmup_steps': 100}},
                'weight_decay': None, 'clipnorm': None, 'global_clipnorm': None, 'clipvalue': None, 'use_ema': False,
                'ema_momentum': 0.99, 'ema_overwrite_frequency': None, 'loss_scale_factor': None,
                'gradient_accumulation_steps': None, 'beta_1': 0.9, 'beta_2': 0.999, 'epsilon': 1e-07,
                'amsgrad': False}

    spec = O.resolve(Adam())
    assert spec.kind == 'adam' and spec.schedule[0] == 'CosineDecay'


class _Custom:
    def get_config(self):
        return {}


@pytest.mark.parametrize('lr,exc', [
    ({'class_name': 'ExponentialDecay'}, NotImplementedError),                 # serialized without a config
    ({'class_name': 'MySchedule', 'config': {}}, NotImplementedError),
    (_Custom(), NotImplementedError),
    (lambda: 0.1, NotImplementedError),
    ('0.1', NotImplementedError),
    ({'class_name': 'ExponentialDecay', 'config': {'initial_learning_rate': 0.1}}, NotImplementedError),
    (-0.01, ValueError), (float('nan'), ValueError), (float('inf'), ValueError),
    ({'class_name': 'ExponentialDecay', 'config': {'initial_learning_rate': -0.1, 'decay_steps': 100,
                                                   'decay_rate': 0.9}}, ValueError),
    ({'class_name': 'PolynomialDecay', 'config': {'initial_learning_rate': 0.1, 'decay_steps': 100,
                                                  'power': -1.0}}, ValueError),             # infinite at the end
])
def test_rejections_name_learning_rate(lr, exc):
    with pytest.raises(exc, match='learning_rate'):
        O.resolve(O.SGD(learning_rate=lr))


@pytest.mark.parametrize('make', [
    lambda: S.ExponentialDecay(-0.1, 100, 0.9), lambda: S.PiecewiseConstantDecay([10], [0.1, float('inf')]),
    lambda: S.PolynomialDecay(0.1, 0), lambda: S.PiecewiseConstantDecay([10, 20], [0.1, 0.2]),
    lambda: S.CosineDecay(0.1, 100, warmup_target=float('nan'), warmup_steps=10)])
def test_schedule_constructors_reject_bad_rates(make):
    with pytest.raises(ValueError, match='learning_rate'):
        make()


def test_other_options_stay_rejected_with_a_schedule():
    sched = S.ExponentialDecay(0.1, 100, 0.9)
    for opt, named in ((O.SGD(learning_rate=sched, weight_decay=0.01), 'weight_decay'),
                       (O.Adam(learning_rate=sched, amsgrad=True), 'amsgrad'),
                       (O.RMSprop(learning_rate=sched, clipnorm=1.0), 'clipnorm')):
        with pytest.raises(NotImplementedError, match=named):
            O.resolve(opt)


# ---- 3. checkpoint text ----------------------------------------------------------------------------------------------------
def test_describe_without_schedule_is_unchanged():
    base = dict(beta_1=None, beta_2=None, centered=None, epsilon=None, initial_accumulator_value=None, momentum=None,
                nesterov=None, rho=None)
    want = {
        'auto': dict(base, kind='adam', learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-07),
        'sgd': dict(base, kind='sgd', learning_rate=0.01, momentum=0.0, nesterov=False),
        'rmsprop': dict(base, kind='rmsprop', learning_rate=0.001, rho=0.9, momentum=0.0, epsilon=1e-07,
                        centered=False),
        'adagrad': dict(base, kind='adagrad', learning_rate=0.001, epsilon=1e-07, initial_accumulator_value=0.1),
    }
    for name, d in want.items():
        assert O.resolve(name).describe() == json.dumps(d, sort_keys=True), name
    assert O.resolve('auto').describe() == (
        '{"beta_1": 0.9, "beta_2": 0.999, "centered": null, "epsilon": 1e-07, "initial_accumulator_value": null, '
        '"kind": "adam", "learning_rate": 0.001, "momentum": null, "nesterov": null, "rho": null}')


def test_describe_with_schedule_differs_by_schedule():
    a = O.resolve(O.Adam(learning_rate=S.ExponentialDecay(0.001, 100, 0.9))).describe()
    b = O.resolve(O.Adam(learning_rate=S.ExponentialDecay(0.001, 100, 0.8))).describe()
    assert a != b and 'schedule' in a and a != O.resolve('auto').describe()


# ---- 4. callbacks ----------------------------------------------------------------------------------------------------------
class _FakeModel:
    def __init__(self, lr):
        self.optimizer = types.SimpleNamespace(learning_rate=lr)


def _plateau_run(cb, values, lr=1.0, key='val_loss'):
    model = _FakeModel(lr)
    cb.set_model(model)
    cb.on_train_begin()
    rates, logged = [], []
    for epoch, v in enumerate(values):
        logs = {key: v}
        cb.on_epoch_end(epoch, logs)
        logged.append(logs['learning_rate'])
        rates.append(model.optimizer.learning_rate)
    return rates, logged


def test_reduce_lr_on_plateau_patience_and_logs():
    rates, logged = _plateau_run(C.ReduceLROnPlateau(patience=2, factor=0.5), [5, 4, 4, 4, 4, 4, 3])
    assert rates == [1.0, 1.0, 1.0, 0.5, 0.5, 0.25, 0.25]
    assert logged == [1.0, 1.0, 1.0, 1.0, 0.5, 0.5, 0.25], 'logs hold the rate before the decision'


def test_reduce_lr_on_plateau_min_delta_cooldown_min_lr():
    # an improvement smaller than min_delta counts as none
    rates, _ = _plateau_run(C.ReduceLROnPlateau(patience=1, factor=0.5, min_delta=0.1), [1.0, 0.95, 0.9, 0.5])
    assert rates == [1.0, 0.5, 0.25, 0.25]
    # cooldown: the epochs counted down after a reduction do not count towards patience (the epoch that ends it does)
    rates, _ = _plateau_run(C.ReduceLROnPlateau(patience=1, factor=0.5, cooldown=2), [1, 1, 1, 1, 1, 1])
    assert rates == [1.0, 0.5, 0.5, 0.25, 0.25, 0.125]
    # min_lr floors the rate, and once there nothing more happens
    rates, _ = _plateau_run(C.ReduceLROnPlateau(patience=1, factor=0.1, min_lr=0.05), [1, 1, 1, 1])
    assert rates == [1.0, 0.1, 0.05, 0.05]


def test_reduce_lr_on_plateau_modes():
    # auto maximises a monitor containing 'acc' and minimises every other one (AUC too)
    rates, _ = _plateau_run(C.ReduceLROnPlateau(monitor='val_accuracy', patience=1, factor=0.5), [0.5, 0.6, 0.55],
                            key='val_accuracy')
    assert rates == [1.0, 1.0, 0.5]
    rates, _ = _plateau_run(C.ReduceLROnPlateau(monitor='val_auc', patience=1, factor=0.5), [0.5, 0.6, 0.55],
                            key='val_auc')
    assert rates == [1.0, 0.5, 0.25]
    rates, _ = _plateau_run(C.ReduceLROnPlateau(monitor='val_auc', mode='max', patience=1, factor=0.5),
                            [0.5, 0.6, 0.55], key='val_auc')
    assert rates == [1.0, 1.0, 0.5]
    with pytest.raises(ValueError):
        C.ReduceLROnPlateau(factor=1.0)
    with pytest.warns(UserWarning):
        C.ReduceLROnPlateau(mode='sideways')


def test_learning_rate_scheduler_both_call_forms():
    model = _FakeModel(0.1)
    seen = []

    def two(epoch, lr):
        seen.append((epoch, lr))
        return lr * 0.5

    cb = C.LearningRateScheduler(two)
    cb.set_model(model)
    for epoch in range(3):
        cb.on_epoch_begin(epoch)
        logs = {}
        cb.on_epoch_end(epoch, logs)
        assert logs['learning_rate'] == model.optimizer.learning_rate
    assert seen == [(0, 0.1), (1, 0.05), (2, 0.025)] and model.optimizer.learning_rate == 0.0125
    cb = C.LearningRateScheduler(lambda epoch: 0.01 * (epoch + 1))
    cb.set_model(model)
    cb.on_epoch_begin(4)
    assert model.optimizer.learning_rate == 0.05
    cb = C.LearningRateScheduler(lambda epoch, lr: 1)
    cb.set_model(model)
    with pytest.raises(ValueError, match='float'):
        cb.on_epoch_begin(0)


# ---- 5. the engine's rate table and optimiser object ------------------------------------------------------------------------
def _rates(optimizer):
    from deeptables_b200.deepmodel import _StepRates
    return _StepRates(O.resolve(optimizer), 'cpu')


def test_rate_table_follows_the_schedule_and_a_set_rate():
    sched = CASES['cosine_warmup']
    r = _rates(O.SGD(learning_rate=sched))
    r.ensure(5000)
    name, c = S.to_config(S.resolve(sched))
    want = lr_ref.step_rates(name, c, len(r.host) - 1)
    assert _ulps(r.host, want).max() <= 1
    plain = _rates(O.RMSprop(learning_rate=0.003))
    plain.ensure(10)
    assert (plain.host[1:] == np.float32(0.003)).all()
    plain.set(0.0007, after=6)
    assert (plain.host[1:7] == np.float32(0.003)).all() and (plain.host[7:] == np.float32(0.0007)).all()
    assert plain.rate(7) == float(np.float32(0.0007))
    assert bool((plain.dev.numpy() == plain.host).all())
    grown = len(plain.host)
    assert plain.ensure(grown + 5) and (plain.host[grown:] == np.float32(0.0007)).all()


def test_adam_table_keeps_the_constant_rate_bits():
    from deeptables_b200.engine import adam_alpha
    r = _rates(O.Adam(learning_rate=3e-3, beta_1=0.8, beta_2=0.99))
    r.ensure(3000)
    want = np.array([0.0] + [adam_alpha(s, 3e-3, 0.8, 0.99) for s in range(1, len(r.host))], dtype=np.float32)
    assert np.array_equal(r.host, want)
    assert r.lazy_ok


def test_adam_replay_bound():
    """The lazy replay's early exit needs fl(fl(7 * 2^-149 * max alpha) / eps) < 2^-108."""
    assert _rates('auto').ensure(10) and _rates('auto').lazy_ok
    big = _rates(O.Adam(learning_rate=S.PiecewiseConstantDecay([100], [1e-3, 1.0]), epsilon=1e-13))
    big.ensure(10)
    assert not big.lazy_ok
    ok = _rates(O.Adam(learning_rate=1.0, epsilon=1e-7))
    ok.ensure(10)
    assert ok.lazy_ok
    low = _rates(O.Adam(learning_rate=0.001, epsilon=1e-13))
    low.ensure(10)
    assert low.lazy_ok
    low.set(1.0, after=3)
    assert not low.lazy_ok


def test_setting_a_scheduled_rate_is_a_type_error():
    from deeptables_b200.deepmodel import _ModelOptimizer, _StepRates

    def fake(optimizer):
        spec = O.resolve(optimizer)
        return types.SimpleNamespace(_rates=_StepRates(spec, 'cpu'), _opt=spec, _step=0)

    m = fake(O.Adam(learning_rate=S.ExponentialDecay(0.01, 10, 0.5)))
    opt = _ModelOptimizer(m)
    assert opt.learning_rate == float(np.float32(0.01)) and opt.iterations == 0
    m._step = 10
    assert opt.learning_rate == float(np.float32(0.005)) and opt.iterations == 10
    with pytest.raises(TypeError, match='not settable'):
        opt.learning_rate = 0.1
    m = fake(O.SGD(learning_rate=0.1))
    opt = _ModelOptimizer(m)
    opt.learning_rate = 0.3
    assert opt.learning_rate == float(np.float32(0.3))
    with pytest.raises(ValueError, match='learning_rate'):
        opt.learning_rate = -1.0
    assert math.isclose(opt.learning_rate, 0.3, rel_tol=1e-7)
