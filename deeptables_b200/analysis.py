"""What the model-analysis tools share: permutation importance (``importance``), Kernel SHAP and expected gradients
(``explain``), partial dependence (``utils.partial_dependence``) and the boosted-leaf booster (``gbm``).

Data parallel: every rank calls a tool with the same arguments, computes the items ``rank_share(n)`` gives it and
returns the full result assembled by ``gather_strided``, so every rank returns what one process would.
"""
import collections
import contextlib
import numbers
import time

import numpy as np
import torch

from . import dp, engine as E


def fitted_model(dt_model):
    """The current model of ``dt_model``; ValueError when there is none, or when it is a list (a model set)."""
    model = dt_model.get_model() if dt_model is not None else None
    if model is None or isinstance(model, list) or getattr(model, 'model', None) is None:
        raise ValueError('dt_model: the DeepTable has no fitted model')
    return model


def model_columns(model):
    """The names of the model's encoded columns: (categorical, continuous), in the order of its input tensors."""
    return ([c.name for c in model.categorical_columns],
            [name for c in model.continuous_columns for name in c.column_names])


def forward_rows(model, cat, cont, pred, batch_size):
    """The inference forward of ``model`` over the first ``len(pred)`` rows of the device inputs ``cat`` / ``cont``
    (either may be None), ``batch_size`` rows per call, its outputs written into ``pred`` [rows, cols] float32.  The
    caller brings the embedding rows up to date first (``model.flush_optimizer_state()``)."""
    with torch.no_grad():
        for lo in range(0, pred.shape[0], batch_size):
            hi = min(lo + batch_size, pred.shape[0])
            bc = cat[lo:hi] if cat is not None else None
            bx = cont[lo:hi] if cont is not None else None
            z = model._forward(bc, bx, training=False)
            p, _ = E.loss_forward_backward(z, torch.zeros_like(z), model.task, None, False, None)
            pred[lo:hi].copy_(p)


def is_int(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, (bool, np.bool_))


def check_positive_int(value, name):
    if not is_int(value) or value < 1:
        raise ValueError(f'{name} must be a positive integer, got {value!r}')


def draw_seed(random_state):
    """A 32-bit seed: ``random_state`` itself, or (None) one drawn from numpy's global generator, rank 0's under data
    parallel."""
    if random_state is None:
        seed = int(np.random.randint(0, 2 ** 32, dtype=np.uint64))
        if dp.is_distributed():
            box = [seed]
            torch.distributed.broadcast_object_list(box, src=0)
            seed = int(box[0])
        return seed
    if not is_int(random_state) or not 0 <= random_state < 2 ** 32:
        raise ValueError(f'random_state must be None or an integer in [0, 2**32), got {random_state!r}')
    return int(random_state)


def rank_share(n):
    """The items of ``range(n)`` this rank computes: ``range(rank, n, world)``, all of them without data parallel."""
    if not dp.is_distributed():
        return range(n)
    return range(torch.distributed.get_rank(), n, dp.world_size())


def gather_strided(local, n, axis=0):
    """The full array of ``n`` items along ``axis`` on every rank, from each rank's part ``local`` (its items of
    ``rank_share(n)``, in order): rank r's part goes to positions ``r::world``.  ``local`` itself without data
    parallel."""
    if not dp.is_distributed() or dp.world_size() == 1:
        return local
    world = dp.world_size()
    parts = [None] * world
    torch.distributed.all_gather_object(parts, local)
    shape = list(local.shape)
    shape[axis] = n
    out = np.empty(shape, local.dtype)
    for r, part in enumerate(parts):
        np.moveaxis(out, axis, 0)[r::world] = np.moveaxis(part, axis, 0)
    return out


class Stages:
    """Seconds spent per stage, added into the dict ``stages`` by ``finish``; nothing is timed when it is None.

    ``with timer.device(name):`` times the device work the block enqueues (CUDA events, read at ``finish``);
    ``timer.host(name, t0)`` adds the host clock since ``t0`` (``time.perf_counter()``)."""

    def __init__(self, stages):
        self.stages = stages
        self.events = []
        self.seconds = collections.defaultdict(float)

    def device(self, name):
        return contextlib.nullcontext() if self.stages is None else self._events(name)

    @contextlib.contextmanager
    def _events(self, name):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        yield
        end.record()
        self.events.append((name, start, end))

    def host(self, name, t0):
        if self.stages is not None:
            self.seconds[name] += time.perf_counter() - t0

    def finish(self):
        if self.stages is None:
            return
        torch.cuda.synchronize()
        for name, start, end in self.events:
            self.seconds[name] += start.elapsed_time(end) / 1e3
        for name, s in self.seconds.items():
            self.stages[name] = self.stages.get(name, 0.0) + s
