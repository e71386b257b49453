"""Losses for ``ModelConfig.loss``: Keras 3's regression, hinge, divergence and crossentropy losses.

``ModelConfig.loss`` takes ``'auto'`` (the task's BCE / MSE / CCE), one of the reference's focal-loss objects
(``layers.BinaryFocalLoss`` / ``CategoricalFocalLoss``, handled by the model as before), or a Keras loss: an instance of
the classes below, any object of one of those class names with ``get_config()`` -- a real
``keras.losses.Huber(delta=2.0)`` included --, a serialized ``{'class_name': ..., 'config': {...}}``, a Keras loss
function such as ``keras.losses.mean_absolute_error``, or a name, in any case: a class name, a Keras function name or
one of the aliases ``'mse'``, ``'mae'``, ``'mape'``, ``'msle'``, ``'kld'``, ``'bce'``.  ``resolve`` turns it into a
hashable ``LossSpec``.

Semantics (Keras 3, float32; ``p`` the task output -- sigmoid, softmax or identity --, ``eps = 1e-7``): the per-row
formulas of ``include/deeptables_b200.h`` (``dtb_keras_loss_fwd_bwd``), reduced as Keras's ``sum_over_batch_size``: the
batch loss is ``sum_r w_r l_r / rows`` with ``w`` the sample (or class) weights, 1 without.  The labels are those the
model trains on: 0 / 1 for binary and multilabel tasks, one-hot rows for multiclass, the targets for regression.

Refused with ``NotImplementedError`` naming the option: ``from_logits=True`` (the output layer already applies its
activation), a ``reduction`` other than ``'sum_over_batch_size'``, ``axis`` other than -1, a ``dtype`` other than
float32, every other loss class (``CosineSimilarity``, Keras's focal crossentropies, ...) and custom callables.
Refused with ``ValueError``: ``SparseCategoricalCrossentropy`` (the labels are one-hot), ``label_smoothing`` outside
[0, 1] and a Huber ``delta`` that is not positive and finite.
"""
import math
import numbers
from collections import OrderedDict
from typing import NamedTuple

from . import consts

EPSILON = 1e-7          # keras.backend.epsilon()
REDUCTION = 'sum_over_batch_size'


class _KerasLoss:
    _fn = None              # the Keras loss function's name
    _default_name = None    # the object's default ``name``
    _params = ()            # ((keyword, default), ...) in Keras's positional order, before reduction, name and dtype

    def __init__(self, *args, **kwargs):
        names = [k for k, _ in self._params] + ['reduction', 'name', 'dtype']
        if len(args) > len(names):
            raise TypeError(f'{type(self).__name__}() takes at most {len(names)} positional arguments')
        unknown = sorted(set(kwargs) - set(names))
        if unknown:
            raise TypeError(f'{type(self).__name__}() got unexpected keyword argument(s) {unknown}')
        given = {**dict(zip(names, args)), **kwargs}
        self._config = {k: given.get(k, d) for k, d in self._params}
        self.reduction = given.get('reduction', REDUCTION)
        self.name = given.get('name') or self._default_name
        self.dtype = given.get('dtype')
        for k, v in self._config.items():
            setattr(self, k, v)

    def get_config(self):
        return {'name': self.name, 'reduction': self.reduction, 'dtype': self.dtype, **self._config}

    def __repr__(self):
        return f'{type(self).__name__}({", ".join(f"{k}={v!r}" for k, v in self._config.items())})'


def _loss(class_name, fn, default_name=None, params=()):
    return type(class_name, (_KerasLoss,), {'_fn': fn, '_default_name': default_name or fn, '_params': tuple(params),
                                            '__doc__': f'keras.losses.{class_name}.'})


_CROSSENTROPY = (('from_logits', False), ('label_smoothing', 0.0), ('axis', -1))
MeanSquaredError = _loss('MeanSquaredError', 'mean_squared_error')
MeanAbsoluteError = _loss('MeanAbsoluteError', 'mean_absolute_error')
MeanAbsolutePercentageError = _loss('MeanAbsolutePercentageError', 'mean_absolute_percentage_error')
MeanSquaredLogarithmicError = _loss('MeanSquaredLogarithmicError', 'mean_squared_logarithmic_error')
Huber = _loss('Huber', 'huber', 'huber_loss', (('delta', 1.0),))
LogCosh = _loss('LogCosh', 'log_cosh')
Poisson = _loss('Poisson', 'poisson')
Hinge = _loss('Hinge', 'hinge')
SquaredHinge = _loss('SquaredHinge', 'squared_hinge')
CategoricalHinge = _loss('CategoricalHinge', 'categorical_hinge')
KLDivergence = _loss('KLDivergence', 'kl_divergence')
BinaryCrossentropy = _loss('BinaryCrossentropy', 'binary_crossentropy', params=_CROSSENTROPY)
CategoricalCrossentropy = _loss('CategoricalCrossentropy', 'categorical_crossentropy', params=_CROSSENTROPY)

_CLASSES = OrderedDict((c.__name__, c) for c in (
    MeanSquaredError, MeanAbsoluteError, MeanAbsolutePercentageError, MeanSquaredLogarithmicError, Huber, LogCosh,
    Poisson, Hinge, SquaredHinge, CategoricalHinge, KLDivergence, BinaryCrossentropy, CategoricalCrossentropy))
# DTB_LOSS_* (include/deeptables_b200.h)
CODES = {name: i + 1 for i, name in enumerate(_CLASSES)}
_FUNCTIONS = {c._fn: name for name, c in _CLASSES.items()}
_NAMES = {**{name.lower(): name for name in _CLASSES}, **_FUNCTIONS,
          'mse': 'MeanSquaredError', 'mae': 'MeanAbsoluteError', 'mape': 'MeanAbsolutePercentageError',
          'msle': 'MeanSquaredLogarithmicError', 'kld': 'KLDivergence', 'bce': 'BinaryCrossentropy'}
_SPARSE = ('sparsecategoricalcrossentropy', 'sparse_categorical_crossentropy')
# the three (loss, task) pairs 'auto' already runs: they keep dtb_loss_fwd_bwd
_BUILTIN = {'BinaryCrossentropy': (consts.TASK_BINARY, consts.TASK_MULTILABEL),
            'MeanSquaredError': (consts.TASK_REGRESSION,), 'CategoricalCrossentropy': (consts.TASK_MULTICLASS,)}


class LossSpec(NamedTuple):
    """What the kernels run: the Keras class name, Huber's ``delta`` and the crossentropies' ``label_smoothing``."""
    kind: str
    delta: float = 1.0
    label_smoothing: float = 0.0

    @property
    def code(self):
        return CODES[self.kind]

    @property
    def hinge(self):
        """Hinge and SquaredHinge decide on the device whether the batch's labels are 0 / 1."""
        return self.kind in ('Hinge', 'SquaredHinge')

    def builtin(self, task):
        """True where 'auto' computes the same loss: the existing kernel runs it, with the same bits."""
        return task in _BUILTIN.get(self.kind, ()) and self.label_smoothing == 0.0

    def __str__(self):
        """The Keras function name, with the parameters that differ from Keras's defaults."""
        shown = []
        if self.kind == 'Huber' and self.delta != 1.0:
            shown.append(f'delta={self.delta!r}')
        if self.label_smoothing:
            shown.append(f'label_smoothing={self.label_smoothing!r}')
        fn = _CLASSES[self.kind]._fn
        return f'{fn}({", ".join(shown)})' if shown else fn


def _sparse(name):
    return ValueError(f'loss={name!r}: the labels are one-hot rows (as the reference builds them), so '
                      f"SparseCategoricalCrossentropy does not fit; use 'categorical_crossentropy'")


def _supported():
    return "'auto', " + ', '.join(_CLASSES) + ' (instances, names or Keras functions)'


def _dtype_name(dtype):
    if isinstance(dtype, dict):                      # a serialized keras DTypePolicy
        return dtype.get('config', {}).get('name')
    if dtype is None or isinstance(dtype, str):
        return dtype
    return getattr(dtype, 'name', dtype)             # a DTypePolicy object


def resolve(loss, task, num_classes=None):
    """``ModelConfig.loss`` (anything but 'auto' and the focal objects) -> ``LossSpec``.  ``task`` and ``num_classes``
    are the model's; every loss applies to every task's output."""
    if isinstance(loss, LossSpec):
        return loss
    if isinstance(loss, dict) and loss.get('class_name') == 'function' and isinstance(loss.get('config'), str):
        loss = loss['config']                        # a serialized Keras loss function
    if isinstance(loss, str):
        if loss.lower() in _SPARSE:
            raise _sparse(loss)
        if loss.lower() not in _NAMES:
            raise NotImplementedError(f'loss={loss!r} is not built natively; use {_supported()}')
        cls_name, config = _NAMES[loss.lower()], {}
    elif isinstance(loss, dict):
        cls_name, config = loss.get('class_name'), loss.get('config') or {}
        if not isinstance(config, dict):
            raise NotImplementedError(f'loss={loss!r}: a serialized loss needs a config dict')
        config = dict(config)
        if isinstance(cls_name, str) and cls_name.lower() in _SPARSE:
            raise _sparse(cls_name)
        if cls_name not in _CLASSES:
            raise NotImplementedError(f'loss {cls_name!r} is not built natively; use {_supported()}')
    elif isinstance(loss, type):
        raise NotImplementedError(f'loss={loss!r}: pass an instance, such as {loss.__name__}(), not the class')
    elif callable(getattr(loss, 'get_config', None)):
        cls_name = type(loss).__name__
        if cls_name.lower() in _SPARSE:
            raise _sparse(cls_name)
        if cls_name not in _CLASSES:
            raise NotImplementedError(f'loss {cls_name} is not built natively; use {_supported()}')
        config = dict(loss.get_config())
    elif callable(loss):
        name = getattr(loss, '__name__', '')
        keras_fn = str(getattr(loss, '__module__', '') or '').startswith('keras')
        if keras_fn and name in _SPARSE:
            raise _sparse(name)
        if not keras_fn or name not in _NAMES:
            raise NotImplementedError(f'loss={loss!r}: custom loss functions are not built natively; use {_supported()}')
        cls_name, config = _NAMES[name], {}
    else:
        raise NotImplementedError(f'loss={loss!r} is not built natively; use {_supported()}')
    return _spec(cls_name, config)


def _spec(cls_name, config):
    defaults = dict(_CLASSES[cls_name]._params)
    cfg = {**defaults, 'reduction': REDUCTION, 'dtype': None, **config}
    for key in cfg:
        if key not in defaults and key not in ('reduction', 'name', 'dtype'):
            raise NotImplementedError(f'{cls_name}({key}={cfg[key]!r}) is not built')
    if cfg['reduction'] != REDUCTION:
        raise NotImplementedError(f'{cls_name}(reduction={cfg["reduction"]!r}) is not built: the batch loss is '
                                  f"Keras's {REDUCTION!r}")
    if _dtype_name(cfg['dtype']) not in (None, 'float32'):
        raise NotImplementedError(f'{cls_name}(dtype={cfg["dtype"]!r}) is not built: losses are float32')
    if 'from_logits' in cfg and cfg['from_logits']:
        raise NotImplementedError(f'{cls_name}(from_logits=True) is not built: the output layer already applies '
                                  f'its sigmoid or softmax')
    if 'axis' in cfg and cfg['axis'] != -1:
        raise NotImplementedError(f'{cls_name}(axis={cfg["axis"]!r}) is not built: the loss runs over the last axis')
    delta, smoothing = 1.0, 0.0
    if 'delta' in cfg:
        delta = cfg['delta']
        if isinstance(delta, bool) or not isinstance(delta, numbers.Real) or not math.isfinite(delta) or delta <= 0:
            raise ValueError(f'Huber(delta={delta!r}): delta must be positive and finite')
        delta = float(delta)
    if 'label_smoothing' in cfg:
        smoothing = cfg['label_smoothing']
        if isinstance(smoothing, bool) or not isinstance(smoothing, numbers.Real) or not 0.0 <= smoothing <= 1.0:
            raise ValueError(f'{cls_name}(label_smoothing={smoothing!r}): must be in [0, 1]')
        smoothing = float(smoothing)
    return LossSpec(cls_name, delta, smoothing)
