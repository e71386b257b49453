"""Keras 3's built-in learning-rate schedules, for the ``learning_rate`` of the optimisers in ``optimizers.py``.

``ExponentialDecay``, ``PiecewiseConstantDecay``, ``PolynomialDecay``, ``InverseTimeDecay``, ``CosineDecay`` and
``CosineDecayRestarts`` take Keras 3's keywords.  ``resolve`` also accepts any object of one of those class names with
``get_config()`` (a real ``keras.optimizers.schedules`` object) and the serialized form a Keras 3 optimiser's
``get_config()`` holds under ``learning_rate``.  It turns each into a hashable description that ``rates`` evaluates.

Step ``s`` of the optimiser (1-based) uses the rate of ``t = s - 1``, the iterations completed before it, as in Keras.
Keras evaluates the formulas in float32 tensor ops; ``rates`` evaluates them in float64 and rounds once to float32, a
difference of a few float32 ulp at most.  Custom ``LearningRateSchedule`` subclasses and callables are not built.
"""
import math
import numbers

import numpy as np


class _Schedule:
    _keys = ()

    def __init__(self, name=None, **config):
        self.name = type(self).__name__ if name is None else name
        self._config = config
        _check_config(type(self).__name__, config)

    def get_config(self):
        return {**self._config, 'name': self.name}

    def __call__(self, step):
        """The rate at ``step`` completed iterations (float32, as a Python float)."""
        return float(rates(resolve(self), np.asarray([step]), check=False)[0])

    def __getattr__(self, item):
        d = self.__dict__
        if '_config' in d and item in d['_config']:
            return d['_config'][item]
        raise AttributeError(item)

    def __repr__(self):
        return f'{type(self).__name__}({", ".join(f"{k}={v!r}" for k, v in self._config.items())})'


class ExponentialDecay(_Schedule):
    """keras.optimizers.schedules.ExponentialDecay: ``lr0 * rate ** (t / decay_steps)`` (exponent floored if staircase)."""

    def __init__(self, initial_learning_rate, decay_steps, decay_rate, staircase=False, name=None):
        super().__init__(name, initial_learning_rate=initial_learning_rate, decay_steps=decay_steps,
                         decay_rate=decay_rate, staircase=staircase)


class PiecewiseConstantDecay(_Schedule):
    """keras.optimizers.schedules.PiecewiseConstantDecay: ``values[i]`` for ``boundaries[i-1] < t <= boundaries[i]``."""

    def __init__(self, boundaries, values, name=None):
        super().__init__(name, boundaries=list(boundaries), values=list(values))


class PolynomialDecay(_Schedule):
    """keras.optimizers.schedules.PolynomialDecay."""

    def __init__(self, initial_learning_rate, decay_steps, end_learning_rate=0.0001, power=1.0, cycle=False,
                 name=None):
        super().__init__(name, initial_learning_rate=initial_learning_rate, decay_steps=decay_steps,
                         end_learning_rate=end_learning_rate, power=power, cycle=cycle)


class InverseTimeDecay(_Schedule):
    """keras.optimizers.schedules.InverseTimeDecay: ``lr0 / (1 + rate * t / decay_steps)`` (floored if staircase)."""

    def __init__(self, initial_learning_rate, decay_steps, decay_rate, staircase=False, name=None):
        super().__init__(name, initial_learning_rate=initial_learning_rate, decay_steps=decay_steps,
                         decay_rate=decay_rate, staircase=staircase)


class CosineDecay(_Schedule):
    """keras.optimizers.schedules.CosineDecay, with the optional linear warmup to ``warmup_target``."""

    def __init__(self, initial_learning_rate, decay_steps, alpha=0.0, name=None, warmup_target=None, warmup_steps=0):
        super().__init__(name, initial_learning_rate=initial_learning_rate, decay_steps=decay_steps, alpha=alpha,
                         warmup_target=warmup_target, warmup_steps=warmup_steps)


class CosineDecayRestarts(_Schedule):
    """keras.optimizers.schedules.CosineDecayRestarts (SGDR)."""

    def __init__(self, initial_learning_rate, first_decay_steps, t_mul=2.0, m_mul=1.0, alpha=0.0, name=None):
        super().__init__(name, initial_learning_rate=initial_learning_rate, first_decay_steps=first_decay_steps,
                         t_mul=t_mul, m_mul=m_mul, alpha=alpha)


CLASSES = {c.__name__: c for c in (ExponentialDecay, PiecewiseConstantDecay, PolynomialDecay, InverseTimeDecay,
                                   CosineDecay, CosineDecayRestarts)}
_STEP_KEYS = ('decay_steps', 'first_decay_steps')
_FLAGS = ('staircase', 'cycle')


def _real(cls_name, key, value, positive=False):
    if isinstance(value, bool) or not isinstance(value, numbers.Real) or not math.isfinite(value) or value < 0 or \
            (positive and value == 0):
        need = 'a finite number > 0' if positive else 'a finite number >= 0'
        raise ValueError(f'{cls_name}({key}={value!r}) for learning_rate: must be {need}')
    return float(value)


def _check_config(cls_name, config):
    """Raise ValueError naming learning_rate for a config whose rates are not finite and non-negative."""
    for key, value in config.items():
        if key in _FLAGS:
            continue
        if key in ('boundaries', 'values'):
            for v in value:
                _real(cls_name, key, v)
        elif key == 'warmup_target':
            if value is not None:
                _real(cls_name, key, value)
        else:
            _real(cls_name, key, value, positive=key in _STEP_KEYS or key == 't_mul')
    if cls_name == 'PiecewiseConstantDecay':
        b, v = config['boundaries'], config['values']
        if len(v) != len(b) + 1:
            raise ValueError(f'PiecewiseConstantDecay for learning_rate: values must have one more entry than '
                             f'boundaries, got {len(b)} boundaries and {len(v)} values')
        if any(x >= y for x, y in zip(b, b[1:])):
            raise ValueError('PiecewiseConstantDecay for learning_rate: boundaries must increase')


def _describe(cls_name, config):
    items = []
    for key in sorted(config):
        if key == 'name':
            continue
        value = config[key]
        if key in _FLAGS:
            value = bool(value)
        elif isinstance(value, (list, tuple)):
            value = tuple(float(v) for v in value)
        elif value is not None:
            value = float(value)
        items.append((key, value))
    return (cls_name, tuple(items))


def resolve(schedule):
    """A schedule -> its hashable description ``(class name, ((key, value), ...))``.

    Accepts an instance of the classes above, any object of one of their class names with ``get_config()``, and the
    serialized dict ``{'class_name': ..., 'config': {...}, ...}``.  Raises NotImplementedError naming learning_rate
    for anything else, ValueError for a rate that is not finite and non-negative."""
    if isinstance(schedule, dict):
        cls_name = schedule.get('class_name')
        config = schedule.get('config')
        if cls_name not in CLASSES:
            raise NotImplementedError(f'learning_rate schedule {cls_name!r} is not built natively; use one of '
                                      f'{sorted(CLASSES)}')
        if not isinstance(config, dict):
            raise NotImplementedError(f'learning_rate: the serialized {cls_name} has no config')
    else:
        cls_name = type(schedule).__name__
        if cls_name not in CLASSES or not callable(getattr(schedule, 'get_config', None)):
            raise NotImplementedError(f'learning_rate={schedule!r}: custom schedules and callables are not built '
                                      f'natively; pass a number or one of {sorted(CLASSES)}')
        config = schedule.get_config()
    try:
        built = CLASSES[cls_name](**dict(config))
    except TypeError as exc:
        raise NotImplementedError(f'learning_rate: {cls_name} config {config!r} not understood ({exc})') from None
    return _describe(cls_name, built.get_config())


def to_config(desc):
    """The description back to (class name, keyword arguments)."""
    cls_name, items = desc
    return cls_name, {k: (list(v) if isinstance(v, tuple) else v) for k, v in items}


def rates(desc, t, check=True):
    """float32 rates (as float64) of schedule ``desc`` at the completed-iteration counts ``t`` (int array).

    ``check``: raise ValueError naming learning_rate if one of them is not finite or negative.  A schedule whose rate
    grows (ExponentialDecay with decay_rate > 1, CosineDecayRestarts with m_mul > 1) overflows float32 at some step;
    callers that fill tables ahead of training pass False and refuse such a step only when it is about to run."""
    cls_name, c = to_config(desc)
    t = np.asarray(t, dtype=np.float64)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        r = _EVAL[cls_name](t, **c)
        r = np.broadcast_to(np.asarray(r, dtype=np.float64), t.shape).astype(np.float32)
    if check and (not np.isfinite(r).all() or (r < 0).any()):
        bad = int(np.flatnonzero(~np.isfinite(r) | (r < 0))[0])
        raise ValueError(f'learning_rate: {cls_name} gives {r[bad]} at step {int(t[bad])}; rates must be finite and '
                         f'non-negative')
    return r.astype(np.float64)


def _exponential(t, initial_learning_rate, decay_steps, decay_rate, staircase):
    p = t / decay_steps
    if staircase:
        p = np.floor(p)
    return initial_learning_rate * np.power(decay_rate, p)


def _inverse_time(t, initial_learning_rate, decay_steps, decay_rate, staircase):
    p = t / decay_steps
    if staircase:
        p = np.floor(p)
    return initial_learning_rate / (1.0 + decay_rate * p)


def _piecewise(t, boundaries, values):
    # values[i] where boundaries[i-1] < t <= boundaries[i]
    return np.asarray(values, dtype=np.float64)[np.searchsorted(np.asarray(boundaries, dtype=np.float64), t,
                                                                side='left')]


def _polynomial(t, initial_learning_rate, decay_steps, end_learning_rate, power, cycle):
    if cycle:
        decay_steps = decay_steps * np.where(t == 0, 1.0, np.ceil(t / decay_steps))
    else:
        t = np.minimum(t, decay_steps)
    return (initial_learning_rate - end_learning_rate) * np.power(1.0 - t / decay_steps, power) + end_learning_rate


def _cosine_decayed(t, decay_steps, alpha):
    return (1.0 - alpha) * (0.5 * (1.0 + np.cos(math.pi * (t / decay_steps)))) + alpha


def _cosine(t, initial_learning_rate, decay_steps, alpha, warmup_target, warmup_steps):
    if warmup_target is None:
        return initial_learning_rate * _cosine_decayed(np.minimum(t, decay_steps), decay_steps, alpha)
    t = np.minimum(t, decay_steps + warmup_steps)
    warm = (warmup_target - initial_learning_rate) * (t / warmup_steps) + initial_learning_rate
    decay = warmup_target * _cosine_decayed(t - warmup_steps, decay_steps, alpha)
    return np.where(t < warmup_steps, warm, decay)


def _cosine_restarts(t, initial_learning_rate, first_decay_steps, t_mul, m_mul, alpha):
    f = t / first_decay_steps
    if t_mul == 1.0:
        i = np.floor(f)
        f = f - i
    else:
        i = np.floor(np.log(1.0 - f * (1.0 - t_mul)) / math.log(t_mul))
        f = (f - (1.0 - np.power(t_mul, i)) / (1.0 - t_mul)) / np.power(t_mul, i)
    return initial_learning_rate * ((1.0 - alpha) * (0.5 * np.power(m_mul, i) * (1.0 + np.cos(math.pi * f))) + alpha)


_EVAL = {'ExponentialDecay': _exponential, 'InverseTimeDecay': _inverse_time, 'PiecewiseConstantDecay': _piecewise,
         'PolynomialDecay': _polynomial, 'CosineDecay': _cosine, 'CosineDecayRestarts': _cosine_restarts}
