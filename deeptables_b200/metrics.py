"""Metrics for ``ModelConfig.metrics``: Keras 3's streaming metrics, kept as counters in device memory.

An entry of ``ModelConfig.metrics`` may be an instance of the classes below, any object of one of those class names
with ``get_config()`` -- a real ``keras.metrics.Precision(thresholds=0.3)`` included -- or a Keras name: the class
names in any case, Keras's snake-case names (``'precision'``, ``'binary_accuracy'``, ``'f1_score'``, ...) and the
aliases ``'mape'``, ``'msle'``, ``'logcosh'``, ``'logloss'`` / ``'bce'``.  ``resolve`` turns one entry into a
``MetricSpec``; ``Plan`` lays the specs of a model out as ONE device buffer that ``dtb_metrics_update`` adds every batch
to (include/deeptables_b200.h), and ``Plan.finish`` turns a copy of that buffer into the values Keras's ``result()``
gives: suffix sums, ratios, AUC's Riemann sums, F-score averaging, in float64 rounded once to float32.

The strings ``'auc'``, ``'accuracy'`` / ``'acc'``, ``'mse'``, ``'rmse'``, ``'mae'`` (and their long forms) and plain
functions ``fn(y_true, y_pred)`` are older than this module and do not come here (deepmodel._resolve_metrics): the
string ``'AUC'`` is the exact rank-sum AUC, the object ``AUC()`` Keras's 200-threshold approximation.

Metrics are unweighted, as Keras's ``metrics=`` are even when sample or class weights are given.  Labels are 0 / 1
(one-hot for multiclass); a label counts as positive when it is not 0.  Not built, and refused by name with
``NotImplementedError``: ``top_k`` of Precision / Recall, ``label_weights``, ``from_logits=True``, ``label_smoothing``,
a ``dtype`` other than float32, R2Score's other aggregations and every metric class not listed here.
"""
import math
import numbers
from collections import OrderedDict
from typing import NamedTuple

import numpy as np

from . import consts

EPSILON = 1e-7          # keras.backend.epsilon()
MAX_LISTS, MAX_THRESHOLDS = 8, 2048         # DTB_METRIC_MAX_LISTS, DTB_METRIC_MAX_THRESHOLDS
# DTB_METRIC_SUM_* bits; the first seven are also the word of the sum in the state
SUM_SE, SUM_AE, SUM_APE, SUM_SLE, SUM_LOGCOSH, SUM_BCE, SUM_CCE, SUM_R2 = (1 << i for i in range(8))


class MetricSpec(NamedTuple):
    """What the engine runs: the Keras class name, the history key and the honoured options (sorted pairs)."""
    kind: str
    key: str
    params: tuple

    def get(self, name):
        return dict(self.params)[name]

    def __str__(self):
        shown = ', '.join(f'{k}={v!r}' for k, v in self.params)
        return f'{self.kind}({shown})' if self.key == _CLASSES[self.kind]._name else \
            f"{self.kind}({shown}{', ' if shown else ''}name={self.key!r})"


class _KerasMetric:
    _name = None
    _params = ()            # ((keyword, default), ...) in Keras's positional order, without name and dtype

    def __init__(self, *args, name=None, dtype=None, **kwargs):
        names = [k for k, _ in self._params]
        if len(args) > len(names):
            raise TypeError(f'{type(self).__name__}() takes at most {len(names)} positional arguments')
        unknown = sorted(set(kwargs) - set(names))
        if unknown:
            raise TypeError(f'{type(self).__name__}() got unexpected keyword argument(s) {unknown}')
        self._config = {**dict(self._params), **dict(zip(names, args)), **kwargs}
        self.name = self._name if name is None else name
        self.dtype = dtype

    def get_config(self):
        return {'name': self.name, 'dtype': self.dtype, **self._config}

    def __getattr__(self, item):
        config = self.__dict__.get('_config', {})
        if item in config:
            return config[item]
        raise AttributeError(item)

    def __repr__(self):
        return f'{type(self).__name__}({", ".join(f"{k}={v!r}" for k, v in self._config.items())})'


def _metric(class_name, default_name, params=(), doc=None):
    return type(class_name, (_KerasMetric,), {'_name': default_name, '_params': tuple(params),
                                               '__doc__': doc or f'keras.metrics.{class_name}.'})


_THRESHOLDED = (('thresholds', None),)
Precision = _metric('Precision', 'precision', (('thresholds', None), ('top_k', None), ('class_id', None)))
Recall = _metric('Recall', 'recall', (('thresholds', None), ('top_k', None), ('class_id', None)))
TruePositives = _metric('TruePositives', 'true_positives', _THRESHOLDED)
FalsePositives = _metric('FalsePositives', 'false_positives', _THRESHOLDED)
TrueNegatives = _metric('TrueNegatives', 'true_negatives', _THRESHOLDED)
FalseNegatives = _metric('FalseNegatives', 'false_negatives', _THRESHOLDED)
AUC = _metric('AUC', 'auc', (('num_thresholds', 200), ('curve', 'ROC'), ('summation_method', 'interpolation'),
                             ('thresholds', None), ('multi_label', False), ('num_labels', None),
                             ('label_weights', None), ('from_logits', False)),
              'keras.metrics.AUC: the Riemann sum over num_thresholds thresholds, not the exact rank-sum AUC.')
F1Score = _metric('F1Score', 'f1_score', (('average', None), ('threshold', None)))
FBetaScore = _metric('FBetaScore', 'fbeta_score', (('average', None), ('beta', 1.0), ('threshold', None)))
BinaryAccuracy = _metric('BinaryAccuracy', 'binary_accuracy', (('threshold', 0.5),))
CategoricalAccuracy = _metric('CategoricalAccuracy', 'categorical_accuracy')
TopKCategoricalAccuracy = _metric('TopKCategoricalAccuracy', 'top_k_categorical_accuracy', (('k', 5),))
MeanSquaredError = _metric('MeanSquaredError', 'mean_squared_error')
RootMeanSquaredError = _metric('RootMeanSquaredError', 'root_mean_squared_error')
MeanAbsoluteError = _metric('MeanAbsoluteError', 'mean_absolute_error')
MeanAbsolutePercentageError = _metric('MeanAbsolutePercentageError', 'mean_absolute_percentage_error')
MeanSquaredLogarithmicError = _metric('MeanSquaredLogarithmicError', 'mean_squared_logarithmic_error')
LogCoshError = _metric('LogCoshError', 'logcosh')
_CROSSENTROPY = (('from_logits', False), ('label_smoothing', 0))
BinaryCrossentropy = _metric('BinaryCrossentropy', 'binary_crossentropy', _CROSSENTROPY)
CategoricalCrossentropy = _metric('CategoricalCrossentropy', 'categorical_crossentropy', _CROSSENTROPY + (('axis', -1),))
R2Score = _metric('R2Score', 'r2_score', (('class_aggregation', 'uniform_average'), ('num_regressors', 0)))

_CLASSES = OrderedDict((c.__name__, c) for c in (
    Precision, Recall, TruePositives, FalsePositives, TrueNegatives, FalseNegatives, AUC, F1Score, FBetaScore,
    BinaryAccuracy, CategoricalAccuracy, TopKCategoricalAccuracy, MeanSquaredError, RootMeanSquaredError,
    MeanAbsoluteError, MeanAbsolutePercentageError, MeanSquaredLogarithmicError, LogCoshError, BinaryCrossentropy,
    CategoricalCrossentropy, R2Score))
_NAMES = {}
for _cls in _CLASSES.values():
    _NAMES[_cls.__name__.lower()] = _NAMES[_cls._name] = _cls.__name__
_NAMES.update(mape='MeanAbsolutePercentageError', msle='MeanSquaredLogarithmicError', logcosh='LogCoshError',
              log_cosh_error='LogCoshError', logloss='BinaryCrossentropy', bce='BinaryCrossentropy')

_COUNTS = ('TruePositives', 'FalsePositives', 'TrueNegatives', 'FalseNegatives')
_ROW_SUMS = {'MeanSquaredError': SUM_SE, 'RootMeanSquaredError': SUM_SE, 'MeanAbsoluteError': SUM_AE,
             'MeanAbsolutePercentageError': SUM_APE, 'MeanSquaredLogarithmicError': SUM_SLE, 'LogCoshError': SUM_LOGCOSH,
             'BinaryCrossentropy': SUM_BCE, 'CategoricalCrossentropy': SUM_CCE, 'R2Score': SUM_R2}
_MULTICLASS_ONLY = ('CategoricalAccuracy', 'TopKCategoricalAccuracy', 'CategoricalCrossentropy')


def is_metric_object(metric):
    """An instance of this module's classes or a look-alike (same class name, has ``get_config()``)."""
    return not isinstance(metric, str) and type(metric).__name__ in _CLASSES and \
        callable(getattr(metric, 'get_config', None))


def is_metric_name(name):
    return isinstance(name, str) and name.lower() in _NAMES


def _threshold_list(cls_name, keyword, value):
    values = [value] if isinstance(value, numbers.Real) else list(value)
    if not values:
        raise ValueError(f'{cls_name}({keyword}=[]): at least one threshold is needed')
    for t in values:
        if isinstance(t, bool) or not isinstance(t, numbers.Real) or not 0.0 <= t <= 1.0:
            raise ValueError(f'{cls_name}({keyword}={value!r}): thresholds must be numbers in [0, 1]')
    return tuple(float(t) for t in values)


def auc_thresholds(num_thresholds=200, thresholds=None):
    """keras.metrics.AUC's threshold list: the given ones, sorted, or (i + 1) / (T - 1) for i < T - 2, between the end
    points -1e-7 and 1 + 1e-7."""
    inner = sorted(thresholds) if thresholds is not None else \
        [(i + 1) * 1.0 / (num_thresholds - 1) for i in range(num_thresholds - 2)]
    return tuple([0.0 - EPSILON] + list(inner) + [1.0 + EPSILON])


def resolve(metric, task, num_classes=None):
    """One entry of ``ModelConfig.metrics`` -> ``MetricSpec``.  NotImplementedError names what is not built, ValueError a
    metric that does not fit the task."""
    if isinstance(metric, str):
        if metric.lower() not in _NAMES:
            raise NotImplementedError(f'metric {metric!r}')
        cls_name, config, key = _NAMES[metric.lower()], {}, metric
    elif is_metric_object(metric):
        cls_name, config = type(metric).__name__, dict(metric.get_config())
        key = config.get('name') or getattr(metric, 'name', None) or _CLASSES[cls_name]._name
    else:
        raise NotImplementedError(f'metric {metric!r}')
    cfg = {**_CLASSES[cls_name]().get_config(), **config}
    dtype = cfg.get('dtype')
    if isinstance(dtype, dict):             # a serialized keras DTypePolicy
        dtype = dtype.get('config', {}).get('name')
    if dtype not in (None, 'float32'):
        raise NotImplementedError(f'{cls_name}(dtype={cfg["dtype"]!r}) is not built: metrics are float32')
    for option, default in (('top_k', None), ('label_weights', None), ('from_logits', False), ('label_smoothing', 0),
                            ('class_aggregation', 'uniform_average'), ('num_regressors', 0), ('axis', -1)):
        if option in cfg and not (cfg[option] == default or cfg[option] is default):
            raise NotImplementedError(f'{cls_name}({option}={cfg[option]!r}) is not built')
    is_error = cls_name in _ROW_SUMS and 'Crossentropy' not in cls_name          # the regression errors and R2Score
    if (task == consts.TASK_REGRESSION and not is_error) or (task != consts.TASK_REGRESSION and cls_name == 'R2Score'):
        raise ValueError(f'metric {cls_name} does not fit a {task} task')
    if cls_name in _MULTICLASS_ONLY and task != consts.TASK_MULTICLASS:
        raise ValueError(f'metric {cls_name} needs one-hot labels: it does not fit a {task} task')
    p = {}
    if cls_name in ('Precision', 'Recall') + _COUNTS:
        p['thresholds'] = _threshold_list(cls_name, 'thresholds', 0.5 if cfg['thresholds'] is None else cfg['thresholds'])
        p['scalar'] = cfg['thresholds'] is None or isinstance(cfg['thresholds'], numbers.Real)
        if 'class_id' in cfg:
            p['class_id'] = _class_id(cls_name, cfg['class_id'], task, num_classes)
    elif cls_name == 'AUC':
        curve, method = str(cfg['curve']).upper(), str(cfg['summation_method']).lower()
        if curve not in ('ROC', 'PR'):
            raise ValueError(f"AUC(curve={cfg['curve']!r}): expected 'ROC' or 'PR'")
        if method not in ('interpolation', 'minoring', 'majoring'):
            raise ValueError(f"AUC(summation_method={cfg['summation_method']!r}): expected 'interpolation', "
                             f"'minoring' or 'majoring'")
        n, given = cfg['num_thresholds'], None
        if cfg['thresholds'] is not None:           # Keras then ignores num_thresholds
            given = tuple(sorted(_threshold_list('AUC', 'thresholds', cfg['thresholds'])))
            n = len(given) + 2
        elif isinstance(n, bool) or not isinstance(n, numbers.Integral) or n <= 1:
            raise ValueError(f'AUC(num_thresholds={n!r}): must be an integer > 1')
        p = dict(num_thresholds=int(n), given_thresholds=given, curve=curve, summation_method=method,
                 multi_label=bool(cfg['multi_label']))
    elif cls_name in ('F1Score', 'FBetaScore'):
        if cfg['average'] not in (None, 'micro', 'macro', 'weighted'):
            raise ValueError(f"{cls_name}(average={cfg['average']!r}): expected None, 'micro', 'macro' or 'weighted'")
        beta = float(cfg.get('beta', 1.0))
        if not beta > 0.0:
            raise ValueError(f'{cls_name}(beta={beta!r}): must be > 0')
        t = cfg['threshold']
        if t is not None and (isinstance(t, bool) or not isinstance(t, numbers.Real) or not 0.0 < t <= 1.0):
            raise ValueError(f'{cls_name}(threshold={t!r}): must be None or in (0, 1]')
        p = dict(average=cfg['average'], beta=beta, threshold=None if t is None else float(t))
    elif cls_name == 'BinaryAccuracy':
        t = cfg['threshold']
        if isinstance(t, bool) or not isinstance(t, numbers.Real) or not 0.0 < t < 1.0:
            raise ValueError(f'BinaryAccuracy(threshold={t!r}): must be in (0, 1)')
        p = dict(threshold=float(t))
    elif cls_name == 'TopKCategoricalAccuracy':
        k = cfg['k']
        if isinstance(k, bool) or not isinstance(k, numbers.Integral) or k < 1:
            raise ValueError(f'TopKCategoricalAccuracy(k={k!r}): must be an integer >= 1')
        p = dict(k=int(k))
    if not isinstance(key, str) or not key:
        raise ValueError(f'{cls_name}(name={key!r}): the name must be a non-empty string')
    return MetricSpec(cls_name, key, tuple(sorted(p.items())))


def _class_id(cls_name, class_id, task, num_classes):
    if class_id is None:
        return None
    cols = num_classes if task == consts.TASK_MULTICLASS else None
    if isinstance(class_id, bool) or not isinstance(class_id, numbers.Integral) or class_id < 0 or \
            (cols is not None and class_id >= cols):
        raise ValueError(f'{cls_name}(class_id={class_id!r}): not a class of this {task} task')
    return int(class_id)


def _divide_no_nan(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.where(b != 0, a / np.where(b != 0, b, 1.0), 0.0)


def _f32(value):
    """A float64 result rounded once to the float32 Keras returns: a float, or a list of floats for a vector."""
    a = np.asarray(value, dtype=np.float64).astype(np.float32)
    return float(a) if a.ndim == 0 else [float(v) for v in a]


class Plan:
    """The device state of a model's streaming metrics: what ``dtb_metric_plan`` says, where each spec's counters are,
    and how to finish them.  ``cols`` is the width of the prediction / label rows."""

    def __init__(self, specs, cols):
        self.specs, self.cols = tuple(specs), int(cols)
        self.lists, self.sums, self.argmax, self.top_k = [], 0, False, 1
        self._where = {}                    # spec -> (list index, position of each of its thresholds in that list)
        top_k = None
        for s in self.specs:
            thresholds = self._thresholds_of(s)
            if thresholds is not None:
                wanted = [np.float32(t) for t in thresholds]
                ordered = tuple(sorted(set(wanted)))
                if ordered not in self.lists:
                    self.lists.append(ordered)
                self._where[s] = (self.lists.index(ordered), [ordered.index(t) for t in wanted])
            self.sums |= _ROW_SUMS.get(s.kind, 0)
            if s.kind in ('CategoricalAccuracy', 'TopKCategoricalAccuracy') or \
                    (s.kind in ('F1Score', 'FBetaScore') and s.get('threshold') is None):
                self.argmax = True
            if s.kind == 'TopKCategoricalAccuracy':
                if top_k not in (None, s.get('k')):
                    raise NotImplementedError('TopKCategoricalAccuracy with two different k in one model is not built')
                top_k = s.get('k')
            if dict(s.params).get('class_id') is not None and s.get('class_id') >= self.cols:
                raise ValueError(f'{s.kind}(class_id={s.get("class_id")}): the model has {self.cols} output column(s)')
        self.top_k = top_k or 1
        if len(self.lists) > MAX_LISTS or sum(len(t) for t in self.lists) > MAX_THRESHOLDS:
            raise NotImplementedError(f'metrics with more than {MAX_LISTS} different threshold lists or '
                                      f'{MAX_THRESHOLDS} thresholds in all are not built')
        self.list_off = [int(v) for v in np.cumsum([0] + [len(t) for t in self.lists])[:-1]]
        self.counters = 8 + 3 * self.cols           # first counter word
        self.hist_off, n = [], 3 + 3 * self.cols
        for t in self.lists:
            self.hist_off.append(n)
            n += self.cols * 2 * (len(t) + 1)
        self.words = self.counters + n

    @staticmethod
    def _thresholds_of(spec):
        p = dict(spec.params)
        if 'thresholds' in p:
            return p['thresholds']
        if spec.kind == 'AUC':
            return auc_thresholds(p['num_thresholds'], p['given_thresholds'])
        if spec.kind == 'BinaryAccuracy' or (spec.kind in ('F1Score', 'FBetaScore') and p['threshold'] is not None):
            return (p['threshold'],)
        return None

    def thresholds(self):
        """All lists back to back, float32: ``thresholds_dev``."""
        return np.asarray([t for lst in self.lists for t in lst], dtype=np.float32)

    def merge(self, counters, sums_by_rank):
        """The state of all data-parallel ranks' batches together: ``counters`` is the elementwise total of the ranks'
        counter words (integers: exact in any order), ``sums_by_rank`` [world, 8 + 3 cols] their float64 words, added here
        in rank order so that every rank gets the same bits."""
        total = np.zeros(self.counters, np.float64)
        for rank_sums in np.asarray(sums_by_rank, np.float64):
            total = total + rank_sums
        return np.concatenate([total.view(np.uint64), np.asarray(counters).view(np.uint64)])

    # ---- finishing ----------------------------------------------------------------------------------------------
    def confusion(self, state, li):
        """float64 (tp, fp, tn, fn), each [cols, T], at the thresholds of list ``li`` (prediction positive: p > t)."""
        T = len(self.lists[li])
        lo = self.counters + self.hist_off[li]
        h = np.asarray(state[lo:lo + self.cols * 2 * (T + 1)], dtype=np.uint64).reshape(self.cols, 2, T + 1)
        above = np.flip(np.cumsum(np.flip(h, -1), -1), -1)[..., 1:].astype(np.float64)   # buckets i+1.. : p > t_i
        total = h.sum(-1, keepdims=True).astype(np.float64)
        tp, fp = above[:, 1], above[:, 0]
        return tp, fp, total[:, 0] - fp, total[:, 1] - tp

    def finish(self, state):
        """history key -> value of every spec (a float, or a list of floats where Keras returns a vector)."""
        state = np.asarray(state, dtype=np.uint64)
        sums = state[:self.counters].view(np.float64)
        cnt = state[self.counters:]
        rows = float(cnt[0])
        out = OrderedDict()
        for s in self.specs:
            p = dict(s.params)
            if s in self._where:
                li, pos = self._where[s]
                tp, fp, tn, fn = self.confusion(state, li)
            if s.kind in ('Precision', 'Recall') + _COUNTS:
                sel = slice(None) if p.get('class_id') is None else [p['class_id']]
                tp, fp, tn, fn = (a[sel].sum(0)[pos] for a in (tp, fp, tn, fn))
                v = {'Precision': _divide_no_nan(tp, tp + fp), 'Recall': _divide_no_nan(tp, tp + fn),
                     'TruePositives': tp, 'FalsePositives': fp, 'TrueNegatives': tn, 'FalseNegatives': fn}[s.kind]
                out[s.key] = _f32(v[0] if p['scalar'] else v)
            elif s.kind == 'AUC':
                if not p['multi_label']:
                    tp, fp, tn, fn = (a.sum(0, keepdims=True) for a in (tp, fp, tn, fn))
                out[s.key] = _f32(np.mean([_auc(p['curve'], p['summation_method'], *col)
                                           for col in zip(tp, fp, tn, fn)]))
            elif s.kind == 'BinaryAccuracy':
                out[s.key] = _f32(_divide_no_nan((tp + tn).sum(), rows * self.cols))
            elif s.kind in ('F1Score', 'FBetaScore'):
                if p['threshold'] is None:
                    tp, fp, fn = (cnt[3 + k * self.cols:3 + (k + 1) * self.cols].astype(np.float64) for k in range(3))
                else:
                    tp, fp, fn = tp[:, 0], fp[:, 0], fn[:, 0]
                out[s.key] = _f32(_fbeta(tp, fp, fn, p['beta'], p['average']))
            elif s.kind == 'CategoricalAccuracy':
                out[s.key] = _f32(_divide_no_nan(float(cnt[1]), rows))
            elif s.kind == 'TopKCategoricalAccuracy':
                out[s.key] = _f32(_divide_no_nan(float(cnt[2]), rows))
            elif s.kind == 'R2Score':
                sy, syy, sdd = (sums[8 + k:8 + 3 * self.cols:3] for k in range(3))
                # keras R2Score: 1 - sum (y - p)^2 / sum (y - mean y)^2 per output, then the mean over the outputs;
                # sum (y - mean y)^2 = sum y^2 - (sum y)^2 / n
                total = syy - _divide_no_nan(sy * sy, rows)
                out[s.key] = _f32(np.mean(np.where(total != 0, 1.0 - _divide_no_nan(sdd, total), 0.0)))   # constant y: 0
            else:
                word = int(math.log2(_ROW_SUMS[s.kind]))
                v = _divide_no_nan(sums[word], rows)
                out[s.key] = _f32(np.sqrt(v) if s.kind == 'RootMeanSquaredError' else v)
        return out


def _auc(curve, method, tp, fp, tn, fn):
    """keras.metrics.AUC.result() from the confusion counts at its thresholds (ascending)."""
    if curve == 'PR' and method == 'interpolation':
        # AUC.interpolate_pr_auc (Davis & Goadrich 2006): precision is not linear in recall between two thresholds
        dtp = tp[:-1] - tp[1:]
        pos = tp + fp
        slope = _divide_no_nan(dtp, np.maximum(pos[:-1] - pos[1:], 0))
        intercept = tp[1:] - slope * pos[1:]
        both = (pos[:-1] > 0) & (pos[1:] > 0)
        ratio = np.where(both, _divide_no_nan(pos[:-1], np.maximum(pos[1:], 0)), 1.0)
        return float(np.sum(_divide_no_nan(slope * (dtp + intercept * np.log(ratio)), np.maximum(tp[1:] + fn[1:], 0))))
    recall = _divide_no_nan(tp, tp + fn)
    if curve == 'ROC':
        x, y = _divide_no_nan(fp, fp + tn), recall
    else:
        x, y = recall, _divide_no_nan(tp, tp + fp)
    heights = {'interpolation': (y[:-1] + y[1:]) / 2.0, 'minoring': np.minimum(y[:-1], y[1:]),
               'majoring': np.maximum(y[:-1], y[1:])}[method]
    return float(np.sum((x[:-1] - x[1:]) * heights))


def _fbeta(tp, fp, fn, beta, average):
    """keras.metrics.FBetaScore.result() from per-class counts."""
    weights = tp + fn
    if average == 'micro':
        tp, fp, fn = tp.sum(), fp.sum(), fn.sum()
    precision = tp / (tp + fp + EPSILON)
    recall = tp / (tp + fn + EPSILON)
    b2 = beta * beta
    score = precision * recall / (b2 * precision + recall + EPSILON) * (1.0 + b2)
    if average == 'weighted':
        return float(np.sum(score * weights / (weights.sum() + EPSILON)))
    return float(np.mean(score)) if average == 'macro' else score
