"""Optimisers for ``ModelConfig.optimizer``: Keras 3's ``Adam``, ``SGD``, ``RMSprop`` and ``Adagrad``.

``ModelConfig.optimizer`` takes ``'auto'`` (Adam 1e-3, the reference's default, deepmodel.py:319-322), one of the
names ``'adam'``, ``'sgd'``, ``'rmsprop'`` and ``'adagrad'`` (any case, Keras defaults), an instance of the classes
below, or any object of one of those four class names with ``get_config()`` -- a real ``keras.optimizers.RMSprop()``
included, as in the reference's own example.  ``resolve`` turns each of them into an ``OptimizerSpec``: a plain,
hashable description that the engine runs and that checkpoints record.

``learning_rate`` is a non-negative number or one of Keras 3's built-in schedules (``schedules.py``), in any form
``schedules.resolve`` accepts.

Every trainable weight, every embedding row included, takes a step every iteration (Keras's dense semantics; a row
with no gradient steps with g = 0).  Custom learning-rate schedules, weight decay, clipping, EMA, loss scaling,
gradient accumulation, AMSGrad and the other Keras optimisers are not built: ``resolve`` rejects them with
``NotImplementedError`` naming the option.
"""
import json
import math
import numbers
from typing import NamedTuple, Optional

from . import schedules as S

# keyword -> default of keras.optimizers.Optimizer (Keras 3) that every optimiser class accepts
_BASE_DEFAULTS = dict(weight_decay=None, clipnorm=None, clipvalue=None, global_clipnorm=None, use_ema=False,
                      ema_momentum=0.99, ema_overwrite_frequency=None, loss_scale_factor=None,
                      gradient_accumulation_steps=None)
# only meaningful with use_ema=True, which is rejected on its own
_EMA_DETAILS = ('ema_momentum', 'ema_overwrite_frequency')


class OptimizerSpec(NamedTuple):
    """What the engine runs.  Fields an optimiser does not use are None."""
    kind: str                                   # 'adam' | 'sgd' | 'rmsprop' | 'adagrad'
    learning_rate: float
    beta_1: Optional[float] = None              # adam
    beta_2: Optional[float] = None              # adam
    epsilon: Optional[float] = None             # adam, rmsprop, adagrad
    momentum: Optional[float] = None            # sgd, rmsprop
    nesterov: Optional[bool] = None             # sgd
    rho: Optional[float] = None                 # rmsprop
    centered: Optional[bool] = None             # rmsprop
    initial_accumulator_value: Optional[float] = None   # adagrad
    schedule: Optional[tuple] = None            # schedules.resolve description; learning_rate is then its step-1 rate

    @property
    def keras_name(self):
        """The Keras class name (what the reference's ModelDesc.optimizer_info shows)."""
        return _KERAS_NAMES[self.kind]

    def describe(self):
        """Stable text form, stored in checkpoints: a saved optimiser state resumes only under the same description."""
        d = self._asdict()
        if d['schedule'] is None:       # the text of an optimiser without a schedule is what it always was
            del d['schedule']
        return json.dumps(d, sort_keys=True)


class _KerasOptimizer:
    _name = None

    def __init__(self, hparams, name, base):
        unknown = sorted(set(base) - set(_BASE_DEFAULTS))
        if unknown:
            raise TypeError(f'{type(self).__name__}() got unexpected keyword argument(s) {unknown}')
        self.name = self._name if name is None else name
        self._hparams = dict(hparams)
        self._base = {**_BASE_DEFAULTS, **base}

    def get_config(self):
        return {'name': self.name, **self._hparams, **self._base}

    def __getattr__(self, item):
        # hyperparameters read as attributes, as on a Keras optimiser (optimizer.learning_rate, .momentum, ...)
        d = self.__dict__
        for src in ('_hparams', '_base'):
            if src in d and item in d[src]:
                return d[src][item]
        raise AttributeError(item)

    def __repr__(self):
        return f'{type(self).__name__}({", ".join(f"{k}={v!r}" for k, v in self._hparams.items())})'


class Adam(_KerasOptimizer):
    """keras.optimizers.Adam."""
    _name = 'adam'

    def __init__(self, learning_rate=0.001, beta_1=0.9, beta_2=0.999, epsilon=1e-7, amsgrad=False, name=None, **base):
        super().__init__(dict(learning_rate=learning_rate, beta_1=beta_1, beta_2=beta_2, epsilon=epsilon,
                              amsgrad=amsgrad), name, base)


class SGD(_KerasOptimizer):
    """keras.optimizers.SGD."""
    _name = 'SGD'

    def __init__(self, learning_rate=0.01, momentum=0.0, nesterov=False, name=None, **base):
        super().__init__(dict(learning_rate=learning_rate, momentum=momentum, nesterov=nesterov), name, base)


class RMSprop(_KerasOptimizer):
    """keras.optimizers.RMSprop."""
    _name = 'rmsprop'

    def __init__(self, learning_rate=0.001, rho=0.9, momentum=0.0, epsilon=1e-7, centered=False, name=None, **base):
        super().__init__(dict(learning_rate=learning_rate, rho=rho, momentum=momentum, epsilon=epsilon,
                              centered=centered), name, base)


class Adagrad(_KerasOptimizer):
    """keras.optimizers.Adagrad."""
    _name = 'adagrad'

    def __init__(self, learning_rate=0.001, initial_accumulator_value=0.1, epsilon=1e-7, name=None, **base):
        super().__init__(dict(learning_rate=learning_rate, initial_accumulator_value=initial_accumulator_value,
                              epsilon=epsilon), name, base)


_CLASSES = {'Adam': Adam, 'SGD': SGD, 'RMSprop': RMSprop, 'Adagrad': Adagrad}
_KERAS_NAMES = {'adam': 'Adam', 'sgd': 'SGD', 'rmsprop': 'RMSprop', 'adagrad': 'Adagrad'}
_SUPPORTED = "'auto', 'adam', 'sgd', 'rmsprop', 'adagrad' or an Adam / SGD / RMSprop / Adagrad instance"


def resolve(optimizer):
    """``ModelConfig.optimizer`` -> ``OptimizerSpec``.  Raises NotImplementedError naming what is not built."""
    if isinstance(optimizer, str):
        key = 'adam' if optimizer.lower() == 'auto' else optimizer.lower()
        if key not in _KERAS_NAMES:
            raise NotImplementedError(f'optimizer {optimizer!r} is not built natively; use {_SUPPORTED}')
        cls_name, config = _KERAS_NAMES[key], {}
    else:
        cls_name = type(optimizer).__name__
        if cls_name not in _CLASSES or not callable(getattr(optimizer, 'get_config', None)):
            raise NotImplementedError(f'optimizer {cls_name} is not built natively; use {_SUPPORTED}')
        config = dict(optimizer.get_config())
    cfg = {**_CLASSES[cls_name]().get_config(), **config}
    for key, default in _BASE_DEFAULTS.items():
        if key in _EMA_DETAILS:
            continue
        value = cfg.get(key, default)
        if not (value == default or (key == 'weight_decay' and value == 0)):
            raise NotImplementedError(f'{cls_name}({key}={value!r}) is not built natively: weight decay, clipping, '
                                      f'EMA, loss scaling and gradient accumulation are not supported')
    lr, sched = _learning_rate(cls_name, cfg['learning_rate'])
    if cls_name == 'Adam':
        if cfg['amsgrad']:
            raise NotImplementedError('Adam(amsgrad=True) is not built natively')
        return OptimizerSpec('adam', lr, beta_1=float(cfg['beta_1']), beta_2=float(cfg['beta_2']),
                             epsilon=float(cfg['epsilon']), schedule=sched)
    if cls_name == 'SGD':
        momentum = float(cfg['momentum'])
        if not 0.0 <= momentum <= 1.0:
            raise ValueError(f'SGD momentum must be in [0, 1], got {momentum}')
        return OptimizerSpec('sgd', lr, momentum=momentum, nesterov=bool(cfg['nesterov']), schedule=sched)
    if cls_name == 'RMSprop':
        return OptimizerSpec('rmsprop', lr, epsilon=float(cfg['epsilon']), momentum=float(cfg['momentum']),
                             rho=float(cfg['rho']), centered=bool(cfg['centered']), schedule=sched)
    return OptimizerSpec('adagrad', lr, epsilon=float(cfg['epsilon']),
                         initial_accumulator_value=float(cfg['initial_accumulator_value']), schedule=sched)


def _learning_rate(cls_name, lr):
    """learning_rate -> (rate of the first step, schedule description or None)."""
    if isinstance(lr, bool) or not isinstance(lr, numbers.Real):
        try:
            sched = S.resolve(lr)
        except NotImplementedError as exc:
            raise NotImplementedError(f'{cls_name}(learning_rate=...): {exc}') from None
        return float(S.rates(sched, [0])[0]), sched
    lr = float(lr)
    if not math.isfinite(lr) or lr < 0:
        raise ValueError(f'{cls_name}(learning_rate={lr!r}): the learning rate must be finite and non-negative')
    return lr, None


def slot_inits(spec):
    """Initial values of the state slots s0, s1, s2 of SGD / RMSprop / Adagrad (None: slot not used)."""
    if spec.kind == 'sgd':
        return (0.0 if spec.momentum > 0 else None, None, None)
    if spec.kind == 'rmsprop':
        return (0.0, 0.0 if spec.centered else None, 0.0 if spec.momentum > 0 else None)
    if spec.kind == 'adagrad':
        return (spec.initial_accumulator_value, None, None)
    raise ValueError(f'{spec.kind} keeps its own state (m, v)')
