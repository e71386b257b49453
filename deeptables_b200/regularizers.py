"""Weight regularizers for ``ModelConfig.embeddings_regularizer`` and ``dnn_params['kernel_regularizer']``: Keras 3's
``L1``, ``L2`` and ``L1L2``.

Each argument takes ``None``, one of the names ``'l1'``, ``'l2'``, ``'l1_l2'`` (or the class names; Keras defaults),
a Keras serialization dict ``{'class_name': 'L2', 'config': {'l2': 1e-5}}``, an instance of the classes below, or any
object of one of those three class names with ``get_config()`` -- a real ``keras.regularizers.L2(1e-5)`` included.
``resolve`` turns each of them into a ``RegSpec(l1, l2)``, or ``None`` when both factors are 0.

Semantics (Keras 3): the training loss is the data loss plus ``l1 * sum|w| + l2 * sum w^2`` of every regularized
weight, taken on the weights before the step, and its gradient ``l1 * sign(w) + 2 * l2 * w`` (``sign(0) = 0``) is added
to the data gradient the optimiser sees.  Under that rule every row of a regularized embedding table steps every
iteration, so the table's optimiser runs as one dense sweep with the regularization fused into it.

Activity regularizers, ``OrthogonalRegularizer`` and custom callables are not built: ``resolve`` rejects them with
``NotImplementedError`` naming them.
"""
import math
import numbers
from typing import NamedTuple


class RegSpec(NamedTuple):
    """What the kernels run: the L1 and L2 factors, not both 0."""
    l1: float
    l2: float

    def __str__(self):
        if self.l1 and self.l2:
            return f'L1L2(l1={self.l1!r}, l2={self.l2!r})'
        return f'L1(l1={self.l1!r})' if self.l1 else f'L2(l2={self.l2!r})'


def _factor(value, name):
    # keras.src.regularizers.regularizers.validate_float_arg
    if isinstance(value, bool) or not isinstance(value, numbers.Real) or not math.isfinite(value) or value < 0:
        raise ValueError(f'Invalid value for argument {name}: expected a non-negative float. Received: {name}={value!r}')
    return float(value)


class L1:
    """keras.regularizers.L1."""

    def __init__(self, l1=0.01):
        self.l1 = _factor(0.01 if l1 is None else l1, 'l1')

    def get_config(self):
        return {'l1': self.l1}


class L2:
    """keras.regularizers.L2."""

    def __init__(self, l2=0.01):
        self.l2 = _factor(0.01 if l2 is None else l2, 'l2')

    def get_config(self):
        return {'l2': self.l2}


class L1L2:
    """keras.regularizers.L1L2."""

    def __init__(self, l1=0.0, l2=0.0):
        self.l1 = _factor(0.0 if l1 is None else l1, 'l1')
        self.l2 = _factor(0.0 if l2 is None else l2, 'l2')

    def get_config(self):
        return {'l1': self.l1, 'l2': self.l2}


_CLASSES = {'L1': L1, 'L2': L2, 'L1L2': L1L2}
_NAMES = {'l1': 'L1', 'l2': 'L2', 'l1_l2': 'L1L2', 'L1': 'L1', 'L2': 'L2', 'L1L2': 'L1L2'}
_ORTHOGONAL = ('OrthogonalRegularizer', 'orthogonal_regularizer')
_SUPPORTED = "None, 'l1', 'l2', 'l1_l2' or an L1 / L2 / L1L2 instance"


def resolve(regularizer, what='regularizer'):
    """A regularizer argument -> ``RegSpec`` or None (no regularization).  ``what`` names the argument in errors."""
    if regularizer is None or isinstance(regularizer, RegSpec):
        return regularizer
    if isinstance(regularizer, str):
        cls_name, config = _NAMES.get(regularizer), {}
        name = regularizer
    elif isinstance(regularizer, dict):
        name = regularizer.get('class_name')
        cls_name, config = (name if name in _CLASSES else None), dict(regularizer.get('config') or {})
    else:
        name = type(regularizer).__name__
        cls_name = name if name in _CLASSES and callable(getattr(regularizer, 'get_config', None)) else None
        config = dict(regularizer.get_config()) if cls_name else {}
    if cls_name is None:
        if name in _ORTHOGONAL:
            raise NotImplementedError(f'{what}={name} is not built natively: OrthogonalRegularizer is not supported; '
                                      f'use {_SUPPORTED}')
        if callable(regularizer):
            raise NotImplementedError(f'{what}={regularizer!r}: custom callables are not built natively as '
                                      f'regularizers; use {_SUPPORTED}')
        raise NotImplementedError(f'{what}={regularizer!r} is not built natively; use {_SUPPORTED}')
    reg = _CLASSES[cls_name](**{k: v for k, v in config.items() if k in ('l1', 'l2')})
    spec = RegSpec(getattr(reg, 'l1', 0.0), getattr(reg, 'l2', 0.0))
    return spec if (spec.l1 or spec.l2) else None


def reject_activity(regularizer, what):
    """Activity regularizers are not built: Keras 2 and Keras 3 disagree on whether their term is divided by the
    batch size."""
    if regularizer is not None:
        raise NotImplementedError(f'{what}={regularizer!r}: activity regularizers are not built natively (Keras 2 '
                                  f'and Keras 3 scale their term differently)')
