"""Float64 numpy restatement of the Keras 3 metrics that deeptables_b200/metrics.py runs on the GPU.

Written from the Keras 3 sources (keras/src/metrics/*.py, keras/src/losses/losses.py, keras/src/backend) as the author
knows them; TensorFlow / Keras are not installed where this suite runs, so these restatements are the contract and
each docstring names the Keras code it restates.  Nothing here imports deeptables_b200.

Every metric is ``Ref(...)``: ``update(y_true, y_pred)`` per batch (float32 [rows, cols]), ``result()`` at the end.
All of them are functions of sums over rows, so ``result()`` works on the concatenation.  Inputs stay float32 where
Keras compares float32 values (``y_pred > threshold``); everything after the comparison is float64, rounded once to
float32 as Keras's float32 result is.

Two places where Keras's float32 arithmetic is not restated bit for bit, on purpose: Keras accumulates float32 sums
batch by batch, this file (and the GPU path) sums in float64; and R2Score of constant labels is 0 here where Keras
returns 0 for -inf but nan for 0/0.
"""
import numpy as np

EPS = 1e-7      # keras.backend.epsilon()


def divide_no_nan(a, b):
    """keras.src.ops.divide_no_nan: 0 where the denominator is 0."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    out = np.zeros(np.broadcast(a, b).shape)
    np.divide(a, b, out=out, where=b != 0)
    return out


def auc_thresholds(num_thresholds=200, thresholds=None):
    """keras.metrics.AUC.__init__: ``[(i + 1) / (num_thresholds - 1) for i in range(num_thresholds - 2)]`` (or the sorted
    user list) between ``0 - epsilon`` and ``1 + epsilon``; compared as float32 tensors."""
    inner = sorted(thresholds) if thresholds is not None else \
        [(i + 1) * 1.0 / (num_thresholds - 1) for i in range(num_thresholds - 2)]
    return np.asarray([0.0 - EPS] + list(inner) + [1.0 + EPS], dtype=np.float32)


def confusion(y_true, y_pred, thresholds):
    """metrics_utils.update_confusion_matrix_variables: labels cast to bool, prediction positive when
    ``y_pred > threshold`` (float32 comparison; a NaN prediction is never positive).  Returns tp, fp, tn, fn [T, cols]."""
    t = np.asarray(thresholds, np.float32).reshape(-1, 1, 1)
    pred = y_pred.astype(np.float32)[None] > t
    label = (y_true != 0)[None]
    f = lambda m: m.sum(1).astype(np.float64)
    return f(pred & label), f(pred & ~label), f(~pred & ~label), f(~pred & label)


def auc_from_counts(tp, fp, tn, fn, curve='ROC', summation_method='interpolation'):
    """keras.metrics.AUC.result() for one label column (counts at ascending thresholds), including
    interpolate_pr_auc for curve='PR' with 'interpolation'."""
    if curve == 'PR' and summation_method == 'interpolation':
        dtp = tp[:-1] - tp[1:]
        p = tp + fp
        dp = p[:-1] - p[1:]
        prec_slope = divide_no_nan(dtp, np.maximum(dp, 0))
        intercept = tp[1:] - prec_slope * p[1:]
        safe_p_ratio = np.where((p[:-1] > 0) & (p[1:] > 0), divide_no_nan(p[:-1], np.maximum(p[1:], 0)), 1.0)
        inc = divide_no_nan(prec_slope * (dtp + intercept * np.log(safe_p_ratio)), np.maximum(tp[1:] + fn[1:], 0))
        return inc.sum()
    recall = divide_no_nan(tp, tp + fn)
    if curve == 'ROC':
        x, y = divide_no_nan(fp, fp + tn), recall
    else:
        x, y = recall, divide_no_nan(tp, tp + fp)
    if summation_method == 'interpolation':
        heights = (y[:-1] + y[1:]) / 2.0
    elif summation_method == 'minoring':
        heights = np.minimum(y[:-1], y[1:])
    else:
        heights = np.maximum(y[:-1], y[1:])
    return ((x[:-1] - x[1:]) * heights).sum()


def fbeta(tp, fp, fn, beta=1.0, average=None):
    """keras.metrics.FBetaScore.result(): precision = tp / (tp + fp + eps), recall = tp / (tp + fn + eps),
    score = (1 + beta^2) * precision * recall / (beta^2 * precision + recall + eps); 'micro' sums the counts over the
    classes first, 'weighted' weighs the classes by their number of positives."""
    support = tp + fn
    if average == 'micro':
        tp, fp, fn = tp.sum(), fp.sum(), fn.sum()
    precision = tp / (tp + fp + EPS)
    recall = tp / (tp + fn + EPS)
    score = precision * recall / (beta ** 2 * precision + recall + EPS) * (1 + beta ** 2)
    if average == 'weighted':          # weights = support / (sum(support) + epsilon)
        return (score * support / (support.sum() + EPS)).sum()
    if average == 'macro':
        return score.mean()
    return score


def _clip(p):
    """backend.binary_crossentropy / categorical_crossentropy clip to [epsilon, 1 - epsilon] in float32."""
    return np.clip(p, np.float64(np.float32(EPS)), np.float64(np.float32(1.0) - np.float32(EPS)))


def row_values(kind, y, p):
    """The per-row value whose mean over rows is the metric (keras.losses functions, mean over the last axis)."""
    y, p = y.astype(np.float64), p.astype(np.float64)
    e = np.float64(np.float32(EPS))
    if kind == 'mse':       # mean_squared_error
        return ((y - p) ** 2).mean(-1)
    if kind == 'mae':       # mean_absolute_error
        return np.abs(y - p).mean(-1)
    if kind == 'mape':      # mean_absolute_percentage_error: 100 * mean |(y - p) / max(|y|, eps)|
        return 100.0 * np.abs((y - p) / np.maximum(np.abs(y), e)).mean(-1)
    if kind == 'msle':      # mean_squared_logarithmic_error: log(max(., eps) + 1)
        return ((np.log(np.maximum(p, e) + 1.0) - np.log(np.maximum(y, e) + 1.0)) ** 2).mean(-1)
    if kind == 'logcosh':   # log_cosh: x + softplus(-2x) - log 2, x = p - y
        x = p - y
        return (x + np.logaddexp(-2.0 * x, 0.0) - np.log(2.0)).mean(-1)
    if kind == 'bce':       # binary_crossentropy on probabilities
        q = _clip(p)
        return -(y * np.log(q) + (1.0 - y) * np.log(1.0 - q)).mean(-1)
    if kind == 'cce':       # categorical_crossentropy on probabilities: renormalise, clip, -sum y log p
        q = _clip(p / p.sum(-1, keepdims=True))
        return -(y * np.log(q)).sum(-1)
    raise KeyError(kind)


class Ref:
    """One metric: ``kind`` is a Keras class name; keywords as Keras's."""

    def __init__(self, kind, **kw):
        self.kind, self.kw, self.y, self.p = kind, kw, [], []

    def update(self, y_true, y_pred):
        y_pred = np.asarray(y_pred, np.float32)
        self.p.append(y_pred.reshape(len(y_pred), 1) if y_pred.ndim == 1 else y_pred)
        self.y.append(np.asarray(y_true, np.float32).reshape(self.p[-1].shape))

    def result(self):
        out = np.asarray(self._result(np.concatenate(self.y), np.concatenate(self.p)), np.float64).astype(np.float32)
        return float(out) if out.ndim == 0 else [float(v) for v in out]

    def _result(self, y, p):
        kind, kw = self.kind, self.kw
        if kind in ('Precision', 'Recall', 'TruePositives', 'FalsePositives', 'TrueNegatives', 'FalseNegatives'):
            th = kw.get('thresholds')
            scalar = th is None or np.isscalar(th)
            th = [0.5 if th is None else th] if scalar else list(th)
            if kw.get('class_id') is not None:
                y, p = y[:, [kw['class_id']]], p[:, [kw['class_id']]]
            tp, fp, tn, fn = (a.sum(-1) for a in confusion(y, p, th))
            v = {'Precision': divide_no_nan(tp, tp + fp), 'Recall': divide_no_nan(tp, tp + fn), 'TruePositives': tp,
                 'FalsePositives': fp, 'TrueNegatives': tn, 'FalseNegatives': fn}[kind]
            return v[0] if scalar else v
        if kind == 'AUC':
            th = auc_thresholds(kw.get('num_thresholds', 200), kw.get('thresholds'))
            counts = confusion(y, p, th)
            if not kw.get('multi_label', False):        # the columns are flattened into one label
                counts = [a.sum(-1, keepdims=True) for a in counts]
            per_label = [auc_from_counts(*(a[:, c] for a in counts), kw.get('curve', 'ROC'),
                                         kw.get('summation_method', 'interpolation'))
                         for c in range(counts[0].shape[1])]
            return np.mean(per_label)
        if kind in ('F1Score', 'FBetaScore'):
            if kw.get('threshold') is None:
                # FBetaScore._update_state: y_pred = (y_pred >= row max) & (|y_pred| > 1e-9)
                pred = (p >= p.max(-1, keepdims=True)) & (np.abs(p) > 1e-9)
            else:
                pred = p > np.float32(kw['threshold'])
            label = y != 0
            tp, fp, fn = ((pred & label).sum(0), (pred & ~label).sum(0), (~pred & label).sum(0))
            return fbeta(*(a.astype(np.float64) for a in (tp, fp, fn)), kw.get('beta', 1.0), kw.get('average'))
        if kind == 'BinaryAccuracy':        # binary_accuracy: mean((y_pred > threshold) == y_true) over all elements
            return ((p > np.float32(kw.get('threshold', 0.5))).astype(np.float32) == y).mean() if y.size else 0.0
        if kind == 'CategoricalAccuracy':   # argmax(y_true) == argmax(y_pred), first maximum
            return (y.argmax(-1) == p.argmax(-1)).mean() if len(y) else 0.0
        if kind == 'TopKCategoricalAccuracy':
            # in_top_k(argmax(y_true), y_pred, k) with TensorFlow's rule: the target's prediction is finite and fewer
            # than k classes have a strictly larger one (ties count as inside)
            target = np.take_along_axis(p, y.argmax(-1)[:, None], -1)
            return (np.isfinite(target[:, 0]) & ((p > target).sum(-1) < kw.get('k', 5))).mean() if len(y) else 0.0
        if kind == 'R2Score':               # 1 - sum (y - p)^2 / sum (y - mean y)^2 per output, uniform average
            y64, p64 = y.astype(np.float64), p.astype(np.float64)
            res, tot = ((y64 - p64) ** 2).sum(0), ((y64 - y64.mean(0)) ** 2).sum(0) if len(y) else np.zeros(y.shape[1])
            return np.where(tot != 0, 1.0 - divide_no_nan(res, tot), 0.0).mean()
        names = {'MeanSquaredError': 'mse', 'RootMeanSquaredError': 'mse', 'MeanAbsoluteError': 'mae',
                 'MeanAbsolutePercentageError': 'mape', 'MeanSquaredLogarithmicError': 'msle', 'LogCoshError': 'logcosh',
                 'BinaryCrossentropy': 'bce', 'CategoricalCrossentropy': 'cce'}
        v = row_values(names[kind], y, p).mean() if len(y) else 0.0
        return np.sqrt(v) if kind == 'RootMeanSquaredError' else v     # sqrt(sum of squares / count)
