"""Denoising auto-encoder features on the device (the work behind ``fe.dae``; reference deeptables/fe/dae.py).

``DAE(...).fit_transform(X)`` trains the reference's ``build_dae`` MLP to reconstruct X and returns the activations of
its ``feature_layer``.  With ``noise_rate > 0`` the net reads swap noise: in each row, ``k = int(M * noise_rate)`` of
the M values come from another random row (the donor), and the target is the clean row.

The data set is cast to float32 and uploaded once.  Each epoch draws a permutation ``p1`` of the rows and, with noise,
an independent permutation ``p2`` of the donors, both from the auto-encoder's device generator.  A step runs wholly on
the device: ``dtb_dae_swap_batch`` builds the batch (clean rows ``p1[j*bs:(j+1)*bs]``, donors ``p2`` at the same
positions, the swapped columns chosen by a counter hash of (seed, step, batch row, column)), the Dense layers run
forward and backward, ``dtb_loss_fwd_bwd`` computes Keras's MSE (the mean over the columns, then over the rows), and
the optimiser sweeps the flat parameters.  The step is captured in a CUDA graph once per batch shape and replayed
(``DTB_CUDA_GRAPH=0`` disables it): the batch kernel and the optimiser read the step from device memory, so one graph
serves every full batch of every epoch and another the partial last batch.  The epoch's summed loss stays in a device
float64 and is read once per epoch.
"""
import numbers
import os
from collections import OrderedDict

import numpy as np
import torch

from . import callbacks as CB, consts, deepmodel as DM, engine as E, layers as L, optimizers as O
from . import _native as N
from ._native import check, ptr, stream_ptr
from .analysis import draw_seed

_DEFAULT_OPTIMIZER = O.Adam(learning_rate=0.001)


def layer_plan(encoder_units, feature_units, activation, cols):
    """The reference's build_dae as (name, in, out, activation) rows: encoder_units[0] is never used."""
    n_stacks = len(encoder_units) - 1
    plan, width = [], cols
    for name, units, act in ([(f'encoder_{i}', encoder_units[i + 1], activation) for i in range(n_stacks)] +
                             [('feature_layer', feature_units, None)] +
                             [(f'decoder_{i}', encoder_units[i], activation) for i in range(n_stacks, 0, -1)] +
                             [('output_layer', cols, activation)]):
        plan.append((name, width, int(units), act))
        width = int(units)
    return plan


def swap_count(cols, noise_rate):
    """Columns swapped per row: the reference's int(M * noise_rate), in Python float arithmetic."""
    return int(cols * noise_rate)


def _count(name, value, low):
    if isinstance(value, bool) or not isinstance(value, numbers.Integral) or value < low:
        raise ValueError(f'{name} must be an int >= {low}, got {value!r}')
    return int(value)


def as_matrix(X):
    """X (2-D numeric numpy array or DataFrame of numeric columns) -> float32 C-contiguous [N, M] ndarray.  ValueError,
    naming the column, for a non-numeric column or a NaN or infinite value."""
    if hasattr(X, 'columns') and hasattr(X, 'dtypes'):
        import pandas as pd
        names = list(X.columns)
        for name in names:
            if not pd.api.types.is_numeric_dtype(X[name].dtype):
                raise ValueError(f'column {name!r} is not numeric ({X[name].dtype}); DAE takes numeric columns only')
        arr = X.to_numpy(dtype=np.float32)
    else:
        arr = np.asarray(X)
        if arr.ndim != 2:
            raise ValueError(f'X must be 2-D, got shape {arr.shape}')
        if arr.dtype.kind not in 'biuf':
            raise ValueError(f'X has dtype {arr.dtype}; DAE takes numeric values only')
        names = list(range(arr.shape[1]))
        arr = arr.astype(np.float32)
    if arr.ndim != 2 or arr.shape[0] == 0 or arr.shape[1] == 0:
        raise ValueError(f'X must have at least one row and one column, got shape {arr.shape}')
    bad = ~np.isfinite(arr).all(axis=0)
    if bad.any():
        raise ValueError(f'column {names[int(np.argmax(bad))]!r} has NaN or infinite values')
    return np.ascontiguousarray(arr)


class AutoEncoder:
    """The trained (or, from ``DAE.build_dae``, initialised) auto-encoder: the reference's Keras ``Model`` named 'AE'.
    ``optimizer.learning_rate``, ``stop_training`` and ``state_dict`` / ``load_state_dict`` are what the Keras callbacks
    of ``DAE.fit`` use."""

    name = 'AE'

    def __init__(self, plan, kernel_initializer, spec, seed, device):
        """plan: layer_plan rows; spec: optimizers.OptimizerSpec; seed: the 32-bit seed of weights, permutations and
        noise."""
        self.device = torch.device(device)
        self.plan = plan
        self.seed = seed
        self._scope = DM._Scope(self.device, seed)
        self._layers = [L.Dense(out, activation=act, kernel_initializer=kernel_initializer, name=name)
                        for name, _, out, act in plan]
        self._opt = spec
        self._opt_native = None if self._opt.kind == 'adam' else DM._native_optim_params(self._opt)
        self._rates = DM._StepRates(self._opt, self.device)
        with torch.no_grad():
            self._forward(torch.zeros(2, plan[0][1], dtype=torch.float32, device=self.device))
        self._scope.freeze(None if self._opt.kind == 'adam' else O.slot_inits(self._opt))
        self._step = 0
        self._step_dev = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._epoch_first_dev = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._loss_acc = torch.zeros(1, dtype=torch.float64, device=self.device)
        self._graphs = {}
        self._graph_failed = False
        self.stop_training = False
        self.history = DM.History()

    # ---- the Keras model surface ---------------------------------------------------------------------------------------
    @property
    def optimizer(self):
        """``learning_rate`` (get / set) and ``iterations``, as callbacks see them."""
        return DM._ModelOptimizer(self)

    @property
    def weights(self):
        """Keras weight name (``encoder_0/kernel``, ..., ``output_layer/bias``) -> tensor, in layer order."""
        return self.state_dict()

    def count_params(self):
        return sum(p.numel() for p in self._scope.params.values())

    def state_dict(self):
        return OrderedDict((k, v.detach()) for k, v in self._scope.params.items())

    def load_state_dict(self, sd):
        own = self.state_dict()
        if set(sd) != set(own):
            raise KeyError(f'state dict mismatch: expected {list(own)}, got {list(sd)}')
        with torch.no_grad():
            for k, v in sd.items():
                own[k].copy_(torch.as_tensor(v).to(self.device, torch.float32).reshape(own[k].shape))

    def predict(self, X, batch_size=128):
        """The reconstruction of X (float32 ndarray [N, M])."""
        return self.apply(X, 'output_layer', batch_size)

    def apply(self, X, output_layer='feature_layer', batch_size=128):
        """The activations of layer ``output_layer`` for X (float32 ndarray); the forward stops at that layer."""
        x = as_matrix(X)
        if x.shape[1] != self.plan[0][1]:
            raise ValueError(f'X has {x.shape[1]} columns, the auto-encoder was built for {self.plan[0][1]}')
        return self._apply(torch.from_numpy(x).to(self.device), output_layer, _count('batch_size', batch_size, 1))

    def _apply(self, x, output_layer, batch_size):
        names = [p[0] for p in self.plan]
        if output_layer not in names:
            raise ValueError(f'No such layer: {output_layer!r}; the layers are {names}')
        with torch.no_grad():
            parts = [self._forward(x[lo:lo + batch_size], output_layer) for lo in range(0, x.shape[0], batch_size)]
        return torch.cat(parts).cpu().numpy()

    def _forward(self, x, upto=None):
        with L.scope_guard(self._scope):
            for layer in self._layers:
                x = layer(x)
                if layer.name == upto:
                    break
        return x

    # ---- training ------------------------------------------------------------------------------------------------------
    def _fit(self, x, batch_size, epochs, k, noise, callbacks):
        """Train on the device-resident float32 [N, M] ``x``: ``epochs`` epochs of ceil(N / batch_size) steps, k columns
        swapped per row when ``noise``.  Returns the History."""
        n = x.shape[0]
        gen = self._scope.generator
        p1 = torch.empty(n, dtype=torch.int64, device=self.device)
        p2 = torch.empty(n, dtype=torch.int64, device=self.device) if noise else None
        batch = (x, p1, p2 if k else None, batch_size, k)
        self._graphs.clear()           # graphs captured the data pointers of an earlier fit
        history = self.history = DM.History()
        for cb in callbacks:
            cb.set_model(self)
        self.stop_training = False
        for cb in callbacks:
            DM._call(cb, 'on_train_begin', None)
        for epoch in range(epochs):
            for cb in callbacks:
                DM._call(cb, 'on_epoch_begin', epoch, None)
            torch.randperm(n, generator=gen, out=p1)
            if p2 is not None:
                torch.randperm(n, generator=gen, out=p2)
            self._epoch_first_dev.fill_(self._step)
            self._loss_acc.zero_()
            for lo in range(0, n, batch_size):
                self._train_step(batch, min(batch_size, n - lo))
            loss = float(self._loss_acc.item()) / n
            logs = {'loss': loss, 'mse': loss}
            for cb in callbacks:
                DM._call(cb, 'on_epoch_end', epoch, logs)
            history.epoch.append(epoch)
            for key, v in logs.items():
                history.history.setdefault(key, []).append(v)
            if self.stop_training:
                break
        for cb in callbacks:
            DM._call(cb, 'on_train_end', None)
        return history

    def _train_step(self, batch, rows):
        if self._rates.ensure(self._step + 1):
            self._graphs.clear()                       # the table moved: captured pointers are stale
        self._rates.check_step(self._step + 1)
        if self._step >= 1 and not self._graph_failed and os.environ.get('DTB_CUDA_GRAPH', '1') != '0':
            if self._rates.ensure(self._step + 2, reserve=200000):
                self._graphs.clear()
            entry = self._graphs.get(rows)
            if entry is None:
                entry = DM.capture_step(lambda _: self._step_body(batch, rows, dev_step=True))
                if entry is None:
                    self._graph_failed = True
                else:
                    self._graphs[rows] = entry
            if entry is not None:
                graph, _, n_launch = entry
                graph.replay()
                N.lib.dtb_launch_count_add(n_launch)
                self._step += 1
                return
        self._step_body(batch, rows, dev_step=False)
        self._step += 1
        self._step_dev.fill_(self._step)

    def _step_body(self, batch, rows, dev_step):
        """One optimiser step on the batch of ``rows`` rows that starts at row (*step_dev - *epoch_first_dev) * bs of the
        epoch's permutation.  dev_step: the CUDA-graph form (the step is read from device memory and incremented)."""
        x, p1, p2, batch_size, k = batch
        cols = x.shape[1]
        x_tgt = torch.empty(rows, cols, dtype=torch.float32, device=self.device)
        x_in = torch.empty_like(x_tgt) if k else None
        check(N.lib.dtb_dae_swap_batch(ptr(x), cols, ptr(p1), ptr(p2), ptr(self._step_dev), ptr(self._epoch_first_dev),
                                       batch_size, rows, k, self.seed, ptr(x_in), ptr(x_tgt), stream_ptr()),
              'dae_swap_batch')
        out = self._forward(x_in if k else x_tgt)
        _, dz = E.loss_forward_backward(out, x_tgt, consts.TASK_REGRESSION, None, True, self._loss_acc)
        out.backward(dz)
        DM.dense_step(self._scope, self._opt, self._opt_native, self._rates, self._step + 1,
                      self._step_dev if dev_step else None)
        if dev_step:
            check(N.lib.dtb_step_increment(ptr(self._step_dev), stream_ptr()), 'step_increment')


class DAE:
    """Denoising auto-encoder feature extractor (reference fe/dae.py).  ``random_state`` (an int in [0, 2^32), or None
    for a seed drawn from numpy's global generator at each fit) fixes the weight initialisation, the epoch permutations
    and the noise."""

    def __init__(self, encoder_units=(500, 500), feature_units=20, activation='relu',
                 kernel_initializer='glorot_uniform', optimizer=_DEFAULT_OPTIMIZER, noise_rate=0, *, random_state=None):
        self.encoder_units = encoder_units
        self.feature_units = feature_units
        self.activate = activation
        self.kernel_initializer = kernel_initializer
        self.optimizer = optimizer
        self.noise_rate = noise_rate
        self.random_state = random_state

    def _check(self):
        units = tuple(self.encoder_units)
        if not units:
            raise ValueError('encoder_units must not be empty')
        for name, u in [(f'encoder_units[{i}]', u) for i, u in enumerate(units) if i] + \
                       [('feature_units', self.feature_units)]:      # encoder_units[0] is never used
            _count(name, u, 1)
        rate = self.noise_rate
        if isinstance(rate, bool) or not isinstance(rate, numbers.Real) or not 0 <= rate <= 1:
            raise ValueError(f'noise_rate must be a number in [0, 1], got {rate!r}')
        return units

    def _build(self, cols):
        units = self._check()
        plan = layer_plan(units, self.feature_units, self.activate, cols)
        L.Dense(1, activation=self.activate)         # NotImplementedError, before any device work, for what Dense lacks
        spec = O.resolve(self.optimizer)
        seed = draw_seed(self.random_state)
        return AutoEncoder(plan, self.kernel_initializer, spec, seed, torch.device('cuda', torch.cuda.current_device()))

    def build_dae(self, X):
        """The auto-encoder for X's column count, weights initialised, untrained."""
        return self._build(as_matrix(X).shape[1])

    def _fit(self, X, batch_size, epochs):
        x = as_matrix(X)
        batch_size, epochs = _count('batch_size', batch_size, 1), _count('epochs', epochs, 0)
        ae = self._build(x.shape[1])
        x_dev = torch.from_numpy(x).to(ae.device)
        from .deeptable import EarlyStopping
        # the reference's callbacks, silent: nothing is printed
        es = EarlyStopping(monitor='mse', min_delta=0.001, patience=5, mode='min', restore_best_weights=True)
        rlr = CB.ReduceLROnPlateau(monitor='mse', factor=0.5, patience=3, min_lr=1e-6, mode='min')
        ae._fit(x_dev, batch_size, epochs, swap_count(x.shape[1], self.noise_rate), self.noise_rate > 0, [es, rlr])
        return ae, x_dev

    def fit(self, X, batch_size=128, epochs=1000):
        """Train the auto-encoder on X (float32 MSE reconstruction, with swap noise when noise_rate > 0)."""
        return self._fit(X, batch_size, epochs)[0]

    def fit_transform(self, X, batch_size=128, epochs=1000):
        """fit, then the feature_layer activations of X: float32 ndarray [N, feature_units]."""
        ae, x_dev = self._fit(X, batch_size, epochs)
        return ae._apply(x_dev, 'feature_layer', batch_size)
