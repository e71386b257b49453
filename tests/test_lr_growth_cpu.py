"""Schedules whose rate grows: the engine's rate table runs far ahead of training, and a rate that overflows float32 at
a step that never runs must not stop training.  Such a step is refused only when it is about to run.  Also Adam's
replay bound as a prefix of the table, and PolynomialDecay(power=0)."""
import numpy as np
import pytest

from deeptables_b200 import optimizers as O
from deeptables_b200 import schedules as S


def _rates(optimizer):
    from deeptables_b200.deepmodel import _StepRates
    return _StepRates(O.resolve(optimizer), 'cpu')


@pytest.mark.parametrize('optimizer', [
    O.Adam(learning_rate=S.ExponentialDecay(1e-6, decay_steps=100, decay_rate=10.0)),     # learning-rate range test
    O.SGD(learning_rate=S.CosineDecayRestarts(0.1, first_decay_steps=10, t_mul=1.0, m_mul=2.0)),
    O.RMSprop(learning_rate=S.ExponentialDecay(0.01, decay_steps=1, decay_rate=1e50, staircase=True))],
    ids=['range_test', 'restarts_growing', 'jump_to_inf'])
def test_growing_schedule_fills_the_table_and_refuses_only_the_overflowing_step(optimizer):
    r = _rates(optimizer)
    assert r.ensure(3, reserve=200000)                      # what the first captured step asks for
    first = int(np.flatnonzero(~np.isfinite(r.host[1:]))[0]) + 1
    for s in range(1, first):
        r.check_step(s)
    with pytest.raises(ValueError, match='learning_rate'):
        r.check_step(first)
    with pytest.raises(ValueError, match='learning_rate'):
        r.check_step(first + 1000)


def test_range_test_schedule_runs_its_600_steps():
    r = _rates(O.Adam(learning_rate=S.ExponentialDecay(1e-6, decay_steps=100, decay_rate=10.0)))
    r.ensure(2, reserve=200000)
    for s in range(1, 601):
        r.check_step(s)
    assert r.rate(600) == float(np.float32(1e-6 * 10.0 ** (599 / 100)))


def test_adam_replay_bound_is_a_prefix():
    """Lazy replay through step s needs the bound only on the alphas of steps 1..s."""
    r = _rates(O.Adam(learning_rate=S.ExponentialDecay(1e-3, decay_steps=2, decay_rate=10.0), epsilon=1e-12))
    r.ensure(10)
    u = (np.float32(7 * 2.0 ** -149) * r.host) / np.float32(1e-12)
    first_break = int(np.flatnonzero(~(u[1:] < np.float32(2.0 ** -108)))[0]) + 1
    assert 1 < first_break < 20
    assert r.lazy_ok_through(first_break - 1) and not r.lazy_ok_through(first_break)
    assert not r.lazy_ok
    plain = _rates(O.Adam(learning_rate=1e-3, epsilon=1e-12))
    plain.ensure(10)
    assert plain.lazy_ok_through(10 ** 6) and plain.lazy_ok
    plain.set(10.0, after=4)
    assert plain.lazy_ok_through(4) and not plain.lazy_ok_through(5)


def test_polynomial_power_zero_is_the_constant_rate():
    """Keras accepts power=0: (1 - t/decay_steps)**0 = 1, including 0**0 at the end of the decay."""
    desc = O.resolve(O.SGD(learning_rate=S.PolynomialDecay(0.05, decay_steps=100, power=0.0))).schedule
    assert set(S.rates(desc, np.arange(0, 300)).tolist()) == {float(np.float32(0.05))}
    cyc = S.resolve(S.PolynomialDecay(0.05, decay_steps=100, power=0.0, cycle=True))
    assert set(S.rates(cyc, np.arange(0, 300)).tolist()) == {float(np.float32(0.05))}
