"""Permutation feature importance on the device (the work behind ``utils.feature_importance``).

The frame is encoded by the preprocessor and uploaded once; a pass permutes the rows of one encoded column in a working
copy of the model's inputs (``dtb_perm_keys`` + ``torch.sort`` + ``dtb_shuffle_column``), runs the inference forward
over the copy in batches, scores the predictions into one float64 slot of a device array and puts the column back.
The host reads the slots once, after the last pass.  DefaultPreprocessor encodes each column on its own and row by
row, so permuting an encoded column is permuting the raw one.  Quantile-bin columns (``auto_discrete``) and
gradient-boosted leaf columns (``apply_gbm_features``) are recomputed from the permuted columns on the device, the bin
columns first; they are not columns of X, so they get no importance.

Data parallel: every rank calls this with the same frame; pass ``s`` (0 is the unpermuted base) runs on rank
``s % world`` and the slots are all-gathered, so every rank returns what one process would.
"""
import collections
import ctypes

import numpy as np
import torch

from . import _native as N, consts, discrete, engine as E, metrics as M
from ._native import check, ptr, stream_ptr
from .analysis import check_positive_int, draw_seed, fitted_model, forward_rows, gather_strided, model_columns, \
    rank_share

AUC, LOG_LOSS, ACCURACY, F1, F1_MACRO, MSE, RMSE, MAE, R2 = range(1, 10)     # DTB_IMPORTANCE_* (deeptables_b200.h)
STREAMING, AUC_OVO = 0, -1     # streaming metrics of metrics.py; multiclass one-vs-one AUC (scikit-learn, host)

# the names fit_cross_validation(oof_metrics=) scores with scikit-learn (deeptable._OOF_SKLEARN_NAMES)
SKLEARN_METRICS = {'auc': AUC, 'roc_auc': AUC, 'log_loss': LOG_LOSS, 'logloss': LOG_LOSS, 'accuracy': ACCURACY,
                   'acc': ACCURACY, 'f1': F1, 'f1_score': F1, 'mse': MSE, 'mean_squared_error': MSE, 'rmse': RMSE,
                   'mae': MAE, 'mean_absolute_error': MAE, 'r2': R2, 'r2_score': R2}
_PROBA_METRICS = ('auc', 'roc_auc', 'log_loss', 'logloss')
_REGRESSION_KINDS = (MSE, RMSE, MAE, R2)

Scorer = collections.namedtuple('Scorer', 'name kind spec')
Result = collections.namedtuple('Result', 'columns decreases passes seed')


def uses_probabilities(metric):
    """Whether a metric scores predicted probabilities rather than predicted labels: the reference's 'auc' and
    'log_loss', their aliases 'roc_auc' and 'logloss', and the streaming metrics (which take the model output, as in
    fit_cross_validation)."""
    if isinstance(metric, str) and metric.lower() in SKLEARN_METRICS:
        return metric.lower() in _PROBA_METRICS
    return True


def resolve_metric(metric, task, num_classes):
    """``metric`` -> Scorer; ValueError for a name or object that is not a metric or does not fit the task."""
    if isinstance(metric, str) and metric.lower() in SKLEARN_METRICS:
        name = metric.lower()
        kind = SKLEARN_METRICS[name]
        if task == consts.TASK_MULTILABEL:
            raise ValueError(f'metric {metric!r}: the multilabel task takes only the streaming metrics of metrics.py')
        if (kind in _REGRESSION_KINDS) != (task == consts.TASK_REGRESSION):
            raise ValueError(f'metric {metric!r} does not fit the {task} task')
        if kind == F1 and task == consts.TASK_MULTICLASS:
            kind = F1_MACRO
        return Scorer(name, kind, None)
    if M.is_metric_object(metric) or M.is_metric_name(metric):
        try:
            spec = M.resolve(metric, task, num_classes)
        except NotImplementedError as e:
            raise ValueError(str(e)) from e
        cols = 1 if task in (consts.TASK_BINARY, consts.TASK_REGRESSION) else num_classes
        plan = M.Plan([spec], cols)
        value = plan.finish(np.zeros(plan.words, np.uint64))[spec.key]
        if isinstance(value, list):
            raise ValueError(f'metric {metric!r} has a vector result; an importance needs one number per pass')
        return Scorer(spec.key, STREAMING, spec)
    raise ValueError(f'Unsupported metric: {metric!r}')


def _sorted_keys(rows, seed, iteration, column, device):
    """The keys of pass (iteration, column) in ascending order: their low halves are its permutation."""
    keys = torch.empty(rows, dtype=torch.int64, device=device)
    check(N.lib.dtb_perm_keys(ptr(keys), rows, seed, iteration, column, stream_ptr()), 'perm_keys')
    return torch.sort(keys).values


def permutation(rows, seed, iteration, column, device):
    """The permutation of pass (iteration, column): int64 [rows] on ``device``; row b of the pass reads row perm[b]."""
    return _sorted_keys(rows, seed, iteration, column, device) & 0xFFFFFFFF


def _class_ranks(labels):
    """Class code -> its position among the sorted labels (scikit-learn's column order for log loss and AUC)."""
    try:
        order = sorted(range(len(labels)), key=lambda i: labels[i])
    except TypeError:
        order = list(range(len(labels)))
    ranks = np.empty(len(labels), np.int64)
    ranks[order] = np.arange(len(labels))
    return ranks


class _Targets:
    """What the scoring kernels read about y, in device memory, built once."""

    def __init__(self, dt_model, model, y, scorer, device):
        task = model.task
        self.y = y = np.asarray(y)
        self.classes = dt_model.classes_
        self.label = self.sk_col = self.positive = self.target = self.onehot = None
        self.aux, self.pos = 0.0, 0
        if scorer.kind == STREAMING:
            labels = dt_model.preprocessor.transform_y(y) if task in (consts.TASK_BINARY, consts.TASK_MULTICLASS) else y
            self.onehot = model._to_device_labels(labels, device)
            return
        if task == consts.TASK_REGRESSION:
            t = y.astype(np.float64).reshape(-1)
            self.target = torch.as_tensor(t).to(device)
            if scorer.kind == R2:          # sklearn r2_score's denominator
                self.aux = float(np.sum((t - np.average(t)) ** 2))
            return
        enc = np.asarray(dt_model.preprocessor.transform_y(y), np.int64).reshape(-1)
        self.label = torch.as_tensor(enc.astype(np.int32)).to(device)
        sk_col = _class_ranks(self.classes)[enc]
        self.sk_col = torch.as_tensor(sk_col.astype(np.int32)).to(device)
        if scorer.kind == AUC and task == consts.TASK_BINARY:
            if len(np.unique(sk_col)) < 2:
                raise ValueError('Only one class present in y_true. ROC AUC score is not defined in that case.')
            self.positive = torch.as_tensor((sk_col == 1).astype(np.int32)).to(device)
        if scorer.kind == F1:
            self.pos = int(dt_model.preprocessor.transform_y([dt_model.pos_label])[0])


def score_decreases(dt_model, X, y, metric, n_iter=5, mode='min', random_state=None, batch_size=65536):
    """The score decreases of every pass: Result(columns, decreases [n_iter, columns] float64, passes run on this
    rank, seed).  Columns the model does not read decrease by exactly 0.0 and cost no pass."""
    if mode not in ('min', 'max'):
        raise ValueError(f'Unsupported mode:{mode}')
    check_positive_int(n_iter, 'n_iter')
    check_positive_int(batch_size, 'batch_size')
    model = fitted_model(dt_model)
    scorer = resolve_metric(metric, model.task, model.num_classes)
    if scorer.kind == AUC and model.task == consts.TASK_MULTICLASS:
        scorer = scorer._replace(kind=AUC_OVO)
    columns = X.columns.to_list()
    rows = len(X)
    if rows < 1 or rows >= 2 ** 32:
        raise ValueError(f'X must have between 1 and 2**32 - 1 rows, got {rows}')
    if len(np.asarray(y)) != rows:
        raise ValueError(f'y has {len(np.asarray(y))} rows for {rows} rows of X')
    seed = draw_seed(random_state)
    device = model.device
    targets = _Targets(dt_model, model, y, scorer, device)

    cat, cont = model._to_device_inputs(dt_model.preprocessor.transform_X(X))
    cat_names, cont_names = model_columns(model)
    read = []                                   # (position in X, working array key, column in that array)
    for j, c in enumerate(columns):
        if str(c) in cat_names:
            read.append((j, 'cat', cat_names.index(str(c))))
        elif str(c) in cont_names:
            read.append((j, 'cont', cont_names.index(str(c))))
    src = {'cat': cat, 'cont': cont}
    work = {k: (v.clone() if v is not None else None) for k, v in src.items()}

    cols = model._output_dim()
    pred = torch.empty(rows, cols, dtype=torch.float32, device=device)
    n_slots = 1 + n_iter * len(read)
    scores = torch.full((n_slots,), float('nan'), dtype=torch.float64, device=device)
    scratch = torch.empty(N.lib.dtb_importance_scratch_bytes(cols) // 8, dtype=torch.float64, device=device)
    host_scores = {}
    state = states = None
    if scorer.kind == STREAMING:
        state = E.MetricsState(M.Plan([scorer.spec], cols), device)
        states = torch.zeros(n_slots, state.state.numel(), dtype=torch.int64, device=device)

    def forward():
        forward_rows(model, work['cat'], work['cont'], pred, batch_size)

    def score(slot):
        out = _ptr_at(scores, slot)
        k = scorer.kind
        if k == STREAMING:
            state.reset()
            state.update(pred, targets.onehot)
            states[slot].copy_(state.state)
        elif k == AUC_OVO:                      # copies the pass's probabilities to the host: slow
            from sklearn.metrics import roc_auc_score
            host_scores[slot] = roc_auc_score(targets.y, pred.cpu().numpy(), multi_class='ovo', labels=targets.classes)
        elif k == AUC:
            sp, order = torch.sort(pred[:, 0])
            check(N.lib.dtb_importance_auc(ptr(sp), ptr(order), ptr(targets.positive), rows, ptr(scratch), out,
                                           stream_ptr()), 'importance_auc')
        elif k in (ACCURACY, F1, F1_MACRO):
            check(N.lib.dtb_importance_labels(k, ptr(pred), ptr(targets.label), rows, cols, targets.pos, ptr(scratch),
                                              out, stream_ptr()), 'importance_labels')
        else:
            check(N.lib.dtb_importance_sums(k, ptr(pred), ptr(targets.sk_col), ptr(targets.target), rows, cols,
                                            targets.aux, ptr(scratch), out, stream_ptr()), 'importance_sums')

    model.flush_optimizer_state()               # every embedding row current: the forward needs no per-batch catch-up
    mine = rank_share(n_slots)
    passes = 0
    for slot in mine:
        if slot == 0:
            forward()
        else:
            it, (j, key, col) = divmod(slot - 1, len(read))[0], read[(slot - 1) % len(read)]
            arr = work[key]
            perm = _sorted_keys(rows, seed, it, j, device)
            check(N.lib.dtb_shuffle_column(ptr(src[key]), ptr(arr), ptr(perm), rows, arr.shape[1], col, stream_ptr()),
                  'shuffle_column')
            discrete.rewrite_derived(dt_model.preprocessor, work['cat'], work['cont'])
            forward()
            check(N.lib.dtb_shuffle_column(ptr(src[key]), ptr(arr), None, rows, arr.shape[1], col, stream_ptr()),
                  'shuffle_column')
            discrete.rewrite_derived(dt_model.preprocessor, work['cat'], work['cont'])
            passes += 1
        score(slot)

    if states is not None:
        raw_states = gather_strided(states.cpu().numpy().view(np.uint64)[mine], n_slots)
        values = np.array([float(state.plan.finish(raw_states[s])[scorer.spec.key]) for s in range(n_slots)])
    else:
        values = scores.cpu().numpy()
        for slot, v in host_scores.items():
            values[slot] = v
        values = gather_strided(values[mine], n_slots)
    signed = -values if mode == 'min' else values
    decreases = np.zeros((n_iter, len(columns)), np.float64)
    for i in range(n_slots - 1):
        it, (j, _, _) = divmod(i, len(read))[0], read[i % len(read)]
        decreases[it, j] = signed[0] - signed[1 + i]
    return Result(columns, decreases, passes, seed)


def _ptr_at(t, index):
    """Device pointer of element ``index`` of a contiguous tensor."""
    return ctypes.c_void_p(t.data_ptr() + index * t.element_size())
