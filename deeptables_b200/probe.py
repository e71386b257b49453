"""Linear probes of intermediate layers on the GPU: ``deeptable.probe_evaluate`` (reference deeptable.py
``probe_evaluate``) and the estimator it fits, scikit-learn 1.9's lbfgs ``LogisticRegression`` over device features.

The estimator minimises scikit-learn's objective

    (1/n) sum_i l_i + (1/(2 C n)) ||W||^2        (the intercept is not penalised)

with binary l = log(1 + e^z) - y z over the positive class's column, or the symmetric multinomial
l = logsumexp(z) - z_y over one column per class.  Each evaluation is one ``dtb_probe_loss_grad`` pass over the
float32 features, in float64, and one ``dtb_probe_join``; the optimiser is the call scikit-learn makes,
``scipy.optimize.minimize(method='L-BFGS-B')`` from zeros.
"""
import time
import warnings
from collections.abc import Mapping

import numpy as np
import scipy.optimize
import torch
from sklearn.exceptions import ConvergenceWarning
from sklearn.metrics import roc_auc_score

from . import _native as N, consts, dp
from ._native import check, ptr, stream_ptr
from .analysis import Stages, check_positive_int, fitted_model, rank_share

BLOCK_ROWS = 1024          # DTB_PROBE_BLOCK_ROWS
MAX_CLASSES = 64           # DTB_PROBE_MAX_CLASSES


def fits_on_device(width, classes):
    """Whether the kernels take a probe of ``classes`` classes over ``width`` features (a row must fit in shared
    memory, and at most MAX_CLASSES classes)."""
    K = 1 if classes == 2 else classes
    return K <= MAX_CLASSES and N.lib.dtb_probe_tile_rows(int(width), K) > 0


def _features(X):
    if not isinstance(X, torch.Tensor) or X.dtype != torch.float32 or X.dim() != 2 or X.stride(1) != 1:
        raise ValueError('X must be a 2-D float32 tensor with unit column stride')
    return X


class DeviceObjective:
    """``W`` (float64 [K, d + 1]) -> (sum of the row losses, their gradient [K, d + 1]) over the device features ``X``
    [n, d] and class codes ``codes`` [n] (int32; binary: 0 / 1)."""

    def __init__(self, X, codes, K, fit_intercept, tile_rows=0):
        self.X, self.codes, self.K, self.fit_intercept, self.tile_rows = X, codes, K, fit_intercept, tile_rows
        n, d = X.shape
        self.blocks = (n + BLOCK_ROWS - 1) // BLOCK_ROWS
        self.width = 1 + K * (d + 1)
        self.partials = torch.empty(self.blocks * self.width, dtype=torch.float64, device=X.device)
        self.sums = torch.empty(self.width, dtype=torch.float64, device=X.device)
        self.W = torch.empty(K * (d + 1), dtype=torch.float64, device=X.device)
        self.evaluations = 0

    def __call__(self, W):
        n, d = self.X.shape
        self.W.copy_(torch.from_numpy(np.ascontiguousarray(W, np.float64).reshape(-1)))
        check(N.lib.dtb_probe_loss_grad(ptr(self.X), self.X.stride(0), ptr(self.codes), ptr(self.W), n, d, self.K,
                                        int(self.fit_intercept), self.tile_rows, ptr(self.partials), stream_ptr()),
              'probe_loss_grad')
        check(N.lib.dtb_probe_join(ptr(self.partials), self.blocks, self.width, ptr(self.sums), stream_ptr()),
              'probe_join')
        self.evaluations += 1
        s = self.sums.cpu().numpy()
        return float(s[0]), s[1:].reshape(self.K, d + 1)


class LogisticProbe:
    """scikit-learn's ``LogisticRegression(penalty='l2', solver='lbfgs')`` over float32 device features: ``fit``,
    ``predict_proba``, ``predict``, ``coef_``, ``intercept_``, ``n_iter_``, ``classes_``."""

    objective = DeviceObjective

    def __init__(self, C=1.0, tol=1e-4, max_iter=100, fit_intercept=True):
        self.C, self.tol, self.max_iter, self.fit_intercept = C, tol, max_iter, fit_intercept

    def fit(self, X, y):
        """X: float32 [n, d] tensor; y: the n labels (host array-like)."""
        X = _features(X)
        y = np.asarray(y).reshape(-1)
        n, d = X.shape
        if len(y) != n:
            raise ValueError(f'y has {len(y)} rows, X has {n}')
        self.classes_ = np.unique(y)
        if len(self.classes_) < 2:
            raise ValueError(f'y: needs samples of at least 2 classes, got one class: {self.classes_[0]!r}')
        K = 1 if len(self.classes_) == 2 else len(self.classes_)
        if K > MAX_CLASSES:
            raise ValueError(f'y: a probe takes at most {MAX_CLASSES} classes, got {K}')
        codes = torch.as_tensor(np.searchsorted(self.classes_, y).astype(np.int32)).to(X.device)
        obj = self.objective(X, codes, K, self.fit_intercept)
        cols = d + 1 if self.fit_intercept else d
        l2 = 1.0 / (self.C * n)
        full = np.zeros((K, d + 1))

        def fun(w):
            full[:, :cols] = w.reshape(K, cols)
            loss, grad = obj(full)
            coef = full[:, :d]
            g = grad[:, :cols] / n
            g[:, :d] += l2 * coef
            return loss / n + 0.5 * l2 * float(np.dot(coef.ravel(), coef.ravel())), g.ravel()

        res = scipy.optimize.minimize(fun, np.zeros(K * cols), method='L-BFGS-B', jac=True,
                                      options={'maxiter': self.max_iter, 'maxls': 50, 'gtol': self.tol,
                                               'ftol': 64 * np.finfo(float).eps})
        self.n_iter_ = np.array([min(res.nit, self.max_iter)])
        self.n_evaluations_ = res.nfev
        self.stop_message_ = res.message       # which stopping rule of L-BFGS-B fired
        if res.status != 0:
            warnings.warn(f'lbfgs failed to converge after {self.n_iter_[0]} iteration(s) (status={res.status}):\n'
                          f'{res.message}', ConvergenceWarning, stacklevel=2)
        W = res.x.reshape(K, cols)
        self._W = np.zeros((K, d + 1))
        self._W[:, :cols] = W
        self.coef_ = W[:, :d].copy()
        self.intercept_ = W[:, d].copy() if self.fit_intercept else np.zeros(K)
        return self

    def _predict(self, X):
        """(probabilities float64 [n, classes], class codes int32 [n]: indices into ``classes_``) on the device."""
        X = _features(X)
        n, d = X.shape
        K = self._W.shape[0]
        W = torch.as_tensor(self._W).to(X.device)
        proba = torch.empty(n, max(K, 2), dtype=torch.float64, device=X.device)
        codes = torch.empty(n, dtype=torch.int32, device=X.device)
        check(N.lib.dtb_probe_predict(ptr(X), X.stride(0), ptr(W), n, d, K, int(self.fit_intercept), ptr(proba),
                                      ptr(codes), stream_ptr()), 'probe_predict')
        return proba, codes

    def predict_proba(self, X):
        return self._predict(X)[0]

    def predict(self, X):
        """The predicted labels (values of ``classes_``), int64 on the device."""
        codes = self._predict(X)[1]
        return torch.as_tensor(self.classes_.astype(np.int64)).to(X.device)[codes.long()]


def count_correct(pred, truth):
    """The number of rows where the int32 device codes ``pred`` and ``truth`` agree."""
    count = torch.zeros(1, dtype=torch.int64, device=pred.device)
    check(N.lib.dtb_probe_correct(ptr(pred), ptr(truth), pred.shape[0], ptr(count), stream_ptr()), 'probe_correct')
    return int(count.item())


def deal(n, fn):
    """[fn(0), ..., fn(n - 1)]: under data parallel this rank calls fn on ``rank_share(n)`` and the other items come
    from the ranks that computed them, so every rank returns the same list."""
    local = {i: fn(i) for i in rank_share(n)}
    if dp.is_distributed() and dp.world_size() > 1:
        parts = [None] * dp.world_size()
        torch.distributed.all_gather_object(parts, local)
        local = {i: v for part in parts for i, v in part.items()}
    return [local[i] for i in range(n)]


def _add_count(stages, name, value):
    if stages is not None:
        stages[name] = stages.get(name, 0) + value


def _probe_layer(model, train, test, layer, y, y_test, score_fn, batch_size, timer, stages):
    """The scores of one layer: a probe fitted on ``train`` (device inputs, rows) and scored on ``test``."""
    with timer.device('forward'):
        x = model.captured_outputs(*train, batch_size, [layer])[0]
        x = x.reshape(x.shape[0], -1)
    t0 = time.perf_counter()
    clf = LogisticProbe().fit(x, y)
    timer.host('fit', t0)
    _add_count(stages, 'fit_iterations', int(clf.n_iter_[0]))
    _add_count(stages, 'fit_evaluations', int(clf.n_evaluations_))
    del x
    with timer.device('forward'):
        x = model.captured_outputs(*test, batch_size, [layer])[0]
        x = x.reshape(x.shape[0], -1)
    t0 = time.perf_counter()
    proba, codes = clf._predict(x)
    if not score_fn:
        pos = np.minimum(np.searchsorted(clf.classes_, y_test), len(clf.classes_) - 1)
        truth = np.where(clf.classes_[pos] == y_test, pos, -1).astype(np.int32)
        scores = {'accuracy': count_correct(codes, torch.as_tensor(truth).to(codes.device)) / len(y_test)}
    else:
        p1 = proba[:, 1].cpu().numpy()
        pred = clf.classes_[codes.cpu().numpy()]
        scores = {name: fn(y_test, p1 if fn is roc_auc_score else pred) for name, fn in score_fn.items()}
    timer.host('score', t0)
    return scores


def probe_evaluate(dt, X, y, X_test, y_test, layers, score_fn={}, *, batch_size=65536, stages=None):
    """``deeptable.probe_evaluate`` (its documentation); ``stages``: a dict that receives the seconds spent encoding,
    in the forwards, fitting and scoring, and the probes' L-BFGS iteration and objective evaluation counts."""
    model = fitted_model(dt)
    check_positive_int(batch_size, 'batch_size')
    if isinstance(layers, str) or not isinstance(layers, (list, tuple)) or not layers:
        raise ValueError(f'layers must be a non-empty list of layer names, got {layers!r}')
    widths = model.layer_widths()
    unknown = [name for name in layers if name not in widths]
    if unknown:
        raise ValueError(f'layers: no layer named {unknown} in the model')
    if len(X) != len(y):
        raise ValueError(f'y has {len(y)} rows, X has {len(X)}')
    if len(X_test) != len(y_test):
        raise ValueError(f'y_test has {len(y_test)} rows, X_test has {len(X_test)}')
    if not isinstance(score_fn, Mapping) or not all(callable(fn) for fn in score_fn.values()):
        raise ValueError(f'score_fn must be a mapping of names to callables, got {score_fn!r}')
    if dt.task not in (consts.TASK_BINARY, consts.TASK_MULTICLASS):
        raise ValueError(f'y: a logistic probe needs binary or multiclass labels; the task is {dt.task}')
    y = dt.preprocessor.transform_y(y)
    y_test = dt.preprocessor.transform_y(y_test)
    classes = len(np.unique(y))
    if classes < 2:
        raise ValueError(f'y: needs samples of at least 2 classes, got one class: {y[0]!r}')
    if classes > MAX_CLASSES:
        raise ValueError(f'y: a probe takes at most {MAX_CLASSES} classes, got {classes}')
    wide = [name for name in layers if widths[name] is not None and not fits_on_device(widths[name], classes)]
    if wide:
        raise ValueError(f'layers: {wide} are too wide for a {classes}-class probe (widths '
                         f'{[widths[name] for name in wide]}; a row must fit in shared memory)')

    timer = Stages(stages)
    t0 = time.perf_counter()
    model.flush_optimizer_state()
    pre = dt.preprocessor
    train = (*model._to_device_inputs(pre.transform_X(X)), len(X))
    test = (*model._to_device_inputs(pre.transform_X(X_test)), len(X_test))
    timer.host('encode', t0)
    results = deal(len(layers), lambda i: _probe_layer(model, train, test, layers[i], y, y_test, score_fn,
                                                       batch_size, timer, stages))
    timer.finish()
    return {name: r for name, r in zip(layers, results)}
