"""Keras 3's learning-rate callbacks, ``ReduceLROnPlateau`` and ``LearningRateScheduler``, for ``DeepTable.fit``.

Both work through ``model.optimizer.learning_rate`` (``DeepModel.optimizer``), which is all a real Keras callback of
these two kinds touches, so ``keras.callbacks.ReduceLROnPlateau`` objects work as well.  A rate set during ``fit``
applies from the next optimiser step on.  ``DeepModel.fit`` records ``history`` after the callbacks' ``on_epoch_end``,
as Keras's ``History`` does, so the ``learning_rate`` they write into ``logs`` appears in ``history``.
"""
import warnings

import numpy as np


class Callback:
    """keras.callbacks.Callback: every hook a no-op."""

    def __init__(self):
        self.model = None

    def set_model(self, model):
        self.model = model

    def on_train_begin(self, logs=None):
        pass

    def on_train_end(self, logs=None):
        pass

    def on_epoch_begin(self, epoch, logs=None):
        pass

    def on_epoch_end(self, epoch, logs=None):
        pass


def _current_lr(model):
    return float(np.asarray(model.optimizer.learning_rate))


class ReduceLROnPlateau(Callback):
    """keras.callbacks.ReduceLROnPlateau: multiply the rate by ``factor`` once ``monitor`` has not improved by
    ``min_delta`` for ``patience`` epochs, then wait ``cooldown`` epochs.  In ``'auto'`` mode a monitor whose name
    contains ``'acc'`` is maximised, every other one minimised."""

    def __init__(self, monitor='val_loss', factor=0.1, patience=10, verbose=0, mode='auto', min_delta=1e-4, cooldown=0,
                 min_lr=0.0, **kwargs):
        super().__init__()
        self.monitor = monitor
        if factor >= 1.0:
            raise ValueError(f'ReduceLROnPlateau does not support a factor >= 1.0. Received factor={factor}')
        self.factor = factor
        self.min_lr = min_lr
        self.min_delta = min_delta
        self.patience = patience
        self.verbose = verbose
        self.cooldown = cooldown
        self.cooldown_counter = 0
        self.wait = 0
        self.best = 0
        self.mode = mode
        self.monitor_op = None
        self._reset()

    def _reset(self):
        if self.mode not in {'auto', 'min', 'max'}:
            warnings.warn(f'Learning rate reduction mode {self.mode} is unknown, fallback to auto mode.', stacklevel=2)
            self.mode = 'auto'
        if self.mode == 'min' or (self.mode == 'auto' and 'acc' not in self.monitor):
            self.monitor_op = lambda a, b: np.less(a, b - self.min_delta)
            self.best = np.inf
        else:
            self.monitor_op = lambda a, b: np.greater(a, b + self.min_delta)
            self.best = -np.inf
        self.cooldown_counter = 0
        self.wait = 0

    def on_train_begin(self, logs=None):
        self._reset()

    def on_epoch_end(self, epoch, logs=None):
        logs = logs if logs is not None else {}
        logs['learning_rate'] = _current_lr(self.model)
        current = logs.get(self.monitor)
        if current is None:
            warnings.warn(f'Learning rate reduction is conditioned on metric `{self.monitor}` which is not available. '
                          f'Available metrics are: {",".join(logs)}.', stacklevel=2)
            return
        if self.in_cooldown():
            self.cooldown_counter -= 1
            self.wait = 0
        if self.monitor_op(current, self.best):
            self.best = current
            self.wait = 0
        elif not self.in_cooldown():
            self.wait += 1
            if self.wait >= self.patience:
                old_lr = _current_lr(self.model)
                if old_lr > np.float32(self.min_lr):
                    new_lr = max(old_lr * self.factor, self.min_lr)
                    self.model.optimizer.learning_rate = new_lr
                    if self.verbose > 0:
                        print(f'\nEpoch {epoch + 1}: ReduceLROnPlateau reducing learning rate to {new_lr}.')
                    self.cooldown_counter = self.cooldown
                    self.wait = 0

    def in_cooldown(self):
        return self.cooldown_counter > 0


class LearningRateScheduler(Callback):
    """keras.callbacks.LearningRateScheduler: at the start of each epoch the rate becomes ``schedule(epoch, lr)``, or
    ``schedule(epoch)`` for a function of one argument."""

    def __init__(self, schedule, verbose=0):
        super().__init__()
        self.schedule = schedule
        self.verbose = verbose

    def on_epoch_begin(self, epoch, logs=None):
        try:
            learning_rate = self.schedule(epoch, _current_lr(self.model))
        except TypeError:           # the one-argument form
            learning_rate = self.schedule(epoch)
        if not isinstance(learning_rate, (float, np.float32, np.float64)):
            raise ValueError(f'The output of the `schedule` function should be a float. Got: {learning_rate}')
        self.model.optimizer.learning_rate = learning_rate
        if self.verbose > 0:
            print(f'\nEpoch {epoch + 1}: LearningRateScheduler setting learning rate to {learning_rate}.')

    def on_epoch_end(self, epoch, logs=None):
        logs = logs if logs is not None else {}
        logs['learning_rate'] = _current_lr(self.model)
