"""Float64 restatement of Keras 3's built-in learning-rate schedules, one step at a time with ``math``.

``rate(name, config, t)`` is the rate after ``t`` completed optimiser iterations.  It is written from the formulas of
keras/src/optimizers/schedules/learning_rate_schedule.py independently of ``deeptables_b200.schedules`` (which
evaluates whole tables with numpy), so the two check each other.  ``step_rates`` gives the float32 rates the optimiser
kernels read, step s (1-based) taking ``rate(t = s - 1)``, and ``adam_alphas`` Adam's alpha table with the rate folded
in."""
import math

import numpy as np


def rate(name, c, t):
    t = float(t)
    if name == 'ExponentialDecay':
        p = t / c['decay_steps']
        if c.get('staircase'):
            p = math.floor(p)
        return c['initial_learning_rate'] * c['decay_rate'] ** p
    if name == 'InverseTimeDecay':
        p = t / c['decay_steps']
        if c.get('staircase'):
            p = math.floor(p)
        return c['initial_learning_rate'] / (1 + c['decay_rate'] * p)
    if name == 'PiecewiseConstantDecay':
        b, v = c['boundaries'], c['values']
        for i, x in enumerate(b):
            if t <= x:
                return v[i]
        return v[-1]
    if name == 'PolynomialDecay':
        steps = c['decay_steps']
        if c.get('cycle'):
            steps = steps * (1.0 if t == 0 else math.ceil(t / steps))
        else:
            t = min(t, steps)
        end = c.get('end_learning_rate', 0.0001)
        return (c['initial_learning_rate'] - end) * (1 - t / steps) ** c.get('power', 1.0) + end
    if name == 'CosineDecay':
        lr0, steps, alpha = c['initial_learning_rate'], c['decay_steps'], c.get('alpha', 0.0)
        target, warm = c.get('warmup_target'), c.get('warmup_steps', 0)

        def decayed(x, frm):
            return frm * ((1 - alpha) * 0.5 * (1 + math.cos(math.pi * min(x, steps) / steps)) + alpha)

        if target is None:
            return decayed(t, lr0)
        t = min(t, steps + warm)
        if t < warm:
            return lr0 + (target - lr0) * (t / warm)
        return decayed(t - warm, target)
    if name == 'CosineDecayRestarts':
        lr0, first = c['initial_learning_rate'], c['first_decay_steps']
        t_mul, m_mul, alpha = c.get('t_mul', 2.0), c.get('m_mul', 1.0), c.get('alpha', 0.0)
        f = t / first
        if t_mul == 1.0:
            i = math.floor(f)
            f -= i
        else:
            i = math.floor(math.log(1 - f * (1 - t_mul)) / math.log(t_mul))
            f = (f - (1 - t_mul ** i) / (1 - t_mul)) / t_mul ** i
        return lr0 * ((1 - alpha) * 0.5 * m_mul ** i * (1 + math.cos(math.pi * f)) + alpha)
    raise ValueError(name)


def step_rates(name, c, steps):
    """float32 rates of steps 0..steps (entry 0 unused, 0): what the SGD / RMSprop / Adagrad table holds."""
    return np.array([0.0] + [rate(name, c, s - 1) for s in range(1, steps + 1)], dtype=np.float32)


def adam_alphas(rates32, beta_1, beta_2):
    """Adam's alpha table from per-step float32 rates: alpha[s] = rate[s] * sqrt(1 - b2^s) / (1 - b1^s)."""
    out = [0.0] + [float(rates32[s]) * math.sqrt(1.0 - beta_2 ** s) / (1.0 - beta_1 ** s)
                   for s in range(1, len(rates32))]
    return np.array(out, dtype=np.float32)
