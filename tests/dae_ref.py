"""numpy restatement of the denoising auto-encoder's layer plan, swap count, noise choice, batch builder and epoch
schedule (reference fe/dae.py; csrc/dae.cu's dtb_dae_swap_batch)."""
import math

import numpy as np

from importance_ref import mix32

_S32 = np.uint64(32)


def layer_plan(encoder_units, feature_units, activation, cols):
    """(name, in, out, activation) of each Dense layer the reference's build_dae creates, in order."""
    plan = []
    width = cols

    def dense(units, act, name):
        nonlocal width
        plan.append((name, width, units, act))
        width = units

    n_stacks = len(encoder_units) - 1
    for i in range(n_stacks):
        dense(encoder_units[i + 1], activation, 'encoder_%d' % i)
    dense(feature_units, None, 'feature_layer')
    for i in range(n_stacks, 0, -1):
        dense(encoder_units[i], activation, 'decoder_%d' % i)
    dense(cols, activation, 'output_layer')
    return plan


def swap_count(cols, noise_rate):
    """mix_generator's num_swap."""
    return int(cols * noise_rate)


def steps_per_epoch(n, batch_size):
    """Keras fit: ceil(N / batch_size) steps, the last one partial."""
    return math.ceil(n / batch_size)


def batch_rows(n, batch_size):
    """Rows of each step of an epoch."""
    return [min(batch_size, n - lo) for lo in range(0, n, batch_size)]


def row_hashes(seed, step, row, cols):
    """h(seed, step, row, c) for c < cols, uint64 holding 32-bit values."""
    a = mix32((np.uint64(seed) << _S32) | np.uint64(step & 0xFFFFFFFF))
    b = mix32((a << _S32) | np.uint64(row & 0xFFFFFFFF))
    return mix32((b << _S32) | np.arange(cols, dtype=np.uint64))


def swapped_columns(seed, step, row, cols, k):
    """The k columns with the smallest keys (h << 32) | c, ascending by column."""
    keys = (row_hashes(seed, step, row, cols) << _S32) | np.arange(cols, dtype=np.uint64)
    return np.sort(np.argsort(keys, kind='stable')[:k])


def swap_batch(X, p1, p2, step_dev, epoch_first, batch_size, rows, k, seed):
    """(x_in, x_tgt) of dtb_dae_swap_batch."""
    base = (step_dev - epoch_first) * batch_size
    tgt = X[p1[base:base + rows]].copy()
    x_in = tgt.copy()
    if k:
        donors = X[p2[base:base + rows]]
        for i in range(rows):
            c = swapped_columns(seed, step_dev + 1, i, X.shape[1], k)
            x_in[i, c] = donors[i, c]
    return x_in, tgt
