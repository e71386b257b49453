"""The oracle of partial dependence: a scikit-learn adapter over a fitted DeepTable, for
``sklearn.inspection.partial_dependence(..., method='brute')``, and a host loop for what scikit-learn has no estimator
for (multilabel).  Both compose on pandas frames and call ``predict_proba`` / ``predict`` once per grid point, so every
grid value goes through the preprocessor exactly as a user's frame would."""
import numpy as np
import pandas as pd
from sklearn.base import BaseEstimator, ClassifierMixin, RegressorMixin

BATCH = 4096          # rows per forward call of the host predictions


def _frame(X, columns):
    return X if isinstance(X, pd.DataFrame) else pd.DataFrame(np.asarray(X), columns=columns).infer_objects()


class DeepTableClassifier(ClassifierMixin, BaseEstimator):
    """``predict_proba`` of a fitted binary or multiclass DeepTable, with its labels as ``classes_``."""

    def __init__(self, dt=None, columns=None):
        self.dt = dt
        self.columns = columns

    def fit(self, X, y=None):
        return self

    def __sklearn_is_fitted__(self):
        return True

    @property
    def classes_(self):
        return np.asarray(self.dt.classes_)

    def predict_proba(self, X):
        return self.dt.predict_proba(_frame(X, self.columns), batch_size=BATCH)

    def predict(self, X):
        return self.dt.predict(_frame(X, self.columns), batch_size=BATCH)


class DeepTableRegressor(RegressorMixin, BaseEstimator):
    """``predict`` of a fitted regression DeepTable, one value per row."""

    def __init__(self, dt=None, columns=None):
        self.dt = dt
        self.columns = columns

    def fit(self, X, y=None):
        return self

    def __sklearn_is_fitted__(self):
        return True

    def predict(self, X):
        return np.asarray(self.dt.predict(_frame(X, self.columns), batch_size=BATCH)).reshape(-1)


def adapter(dt):
    return DeepTableRegressor(dt) if dt.task == 'regression' else DeepTableClassifier(dt)


def host_loop(dt, X, features, grid, sample_weight=None):
    """(average float64 [outputs, points], individual float32 [outputs, rows, points]) by setting the feature columns of
    every row of X to each grid point in turn and calling ``predict_proba``: every output column is one output (the
    multilabel task's label probabilities; on binary, keep output 1)."""
    preds = []
    for point in grid:
        f = X.copy()
        for name, v in zip(features, point):
            f[name] = [v] * len(f)
        p = np.asarray(dt.predict_proba(f, batch_size=BATCH))
        preds.append(p.reshape(len(f), -1))
    ind = np.stack(preds, axis=-1).transpose(1, 0, 2)                      # [outputs, rows, points]
    w = np.ones(len(X)) if sample_weight is None else np.asarray(sample_weight, np.float64)
    avg = np.einsum('orp,r->op', ind.astype(np.float64), w) / w.sum()
    return avg, ind


def block_order_mean(pred, weight, block_rows):
    """The device path's order of a weighted mean over the rows of ``pred`` [rows, cols] float32 (one grid point):
    float64 block sums restated lane by lane (``block_sums_restated``), added block by block in index order, divided by
    the weights' sum taken in the same order."""
    rows = len(pred)
    w = np.ones(rows) if weight is None else np.asarray(weight, np.float64)
    sums = block_sums_restated(pred[None], None if weight is None else w, block_rows)[0]
    acc = np.zeros(pred.shape[1])
    for b in range(sums.shape[0]):
        acc += sums[b]
    if weight is None:
        total = float(rows)
    else:
        wb = block_sums_restated(np.ones((1, rows, 1), np.float32), w, block_rows)[0, :, 0]
        total = 0.0
        for b in range(len(wb)):
            total += wb[b]
    return acc / total


def block_sums_restated(prob, weight, block_rows):
    """``dtb_pdp_block_sums`` in numpy: prob [groups, rows, cols] float32, weight [rows] float64 or None ->
    float64 [groups, blocks, cols].  Lane l of a block adds rows l, l+32, ... in order; then the butterfly
    ``v += shfl_xor(v, o)`` for o = 16, 8, 4, 2, 1, whose lane-0 result is returned."""
    groups, rows, cols = prob.shape
    blocks = (rows + block_rows - 1) // block_rows
    p = prob.astype(np.float64)
    if weight is not None:
        p = np.asarray(weight, np.float64)[None, :, None] * p
    out = np.empty((groups, blocks, cols))
    for b in range(blocks):
        lo, hi = b * block_rows, min((b + 1) * block_rows, rows)
        seg = p[:, lo:hi]
        # lane l's rows as column l of [passes, 32], after a leading 0.0 (the accumulator's start); the zero padding
        # of the last pass adds nothing.  cumsum adds along the passes in order.
        seg = np.concatenate([np.zeros((groups, 32, cols)), seg, np.zeros((groups, (lo - hi) % 32, cols))],
                             axis=1)
        lanes = np.cumsum(seg.reshape(groups, -1, 32, cols), axis=1)[:, -1]
        for o in (16, 8, 4, 2, 1):
            lanes = lanes + lanes[:, np.arange(32) ^ o]
        out[:, b] = lanes[:, 0]
    return out
