"""metrics.py without a GPU: what ``resolve`` accepts and refuses, that the spellings older than metrics.py keep their
functions, and ``Plan.finish`` / ``Plan.merge`` on counter states made by hand against the Keras restatement in
metrics_ref.py."""
import numpy as np
import pytest
import torch

import metrics_ref as MR
import metrics_state_ref as SR
from deeptables_b200 import deepmodel, metrics as M


class _LookAlike:
    """Stands for a real keras.metrics object: matched by class name and get_config()."""

    def __init__(self, **config):
        self._config = config

    def get_config(self):
        return dict(self._config)


def _look_alike(class_name, **config):
    return type(class_name, (_LookAlike,), {})(**config)


KERAS_DEFAULTS = {      # keras.metrics.<class>().get_config() without dtype, Keras 3
    'Precision': dict(name='precision', thresholds=None, top_k=None, class_id=None),
    'Recall': dict(name='recall', thresholds=None, top_k=None, class_id=None),
    'TruePositives': dict(name='true_positives', thresholds=None),
    'FalsePositives': dict(name='false_positives', thresholds=None),
    'TrueNegatives': dict(name='true_negatives', thresholds=None),
    'FalseNegatives': dict(name='false_negatives', thresholds=None),
    'AUC': dict(name='auc', num_thresholds=200, curve='ROC', summation_method='interpolation', thresholds=None,
                multi_label=False, num_labels=None, label_weights=None, from_logits=False),
    'F1Score': dict(name='f1_score', average=None, threshold=None),
    'FBetaScore': dict(name='fbeta_score', average=None, beta=1.0, threshold=None),
    'BinaryAccuracy': dict(name='binary_accuracy', threshold=0.5),
    'CategoricalAccuracy': dict(name='categorical_accuracy'),
    'TopKCategoricalAccuracy': dict(name='top_k_categorical_accuracy', k=5),
    'MeanSquaredError': dict(name='mean_squared_error'),
    'RootMeanSquaredError': dict(name='root_mean_squared_error'),
    'MeanAbsoluteError': dict(name='mean_absolute_error'),
    'MeanAbsolutePercentageError': dict(name='mean_absolute_percentage_error'),
    'MeanSquaredLogarithmicError': dict(name='mean_squared_logarithmic_error'),
    'LogCoshError': dict(name='logcosh'),
    'BinaryCrossentropy': dict(name='binary_crossentropy', from_logits=False, label_smoothing=0),
    'CategoricalCrossentropy': dict(name='categorical_crossentropy', from_logits=False, label_smoothing=0, axis=-1),
    'R2Score': dict(name='r2_score', class_aggregation='uniform_average', num_regressors=0),
}


def _task_of(class_name):
    if class_name in ('CategoricalAccuracy', 'TopKCategoricalAccuracy', 'CategoricalCrossentropy'):
        return 'multiclass'
    return 'regression' if class_name in ('R2Score', 'MeanSquaredError') else 'binary'


@pytest.mark.parametrize('class_name', sorted(KERAS_DEFAULTS))
def test_defaults_are_keras3s_and_every_form_resolves_alike(class_name):
    cls = getattr(M, class_name)
    config = cls().get_config()
    assert config.pop('dtype') is None
    assert config == KERAS_DEFAULTS[class_name]
    task = _task_of(class_name)
    spec = M.resolve(cls(), task, 3)
    assert spec.kind == class_name and spec.key == KERAS_DEFAULTS[class_name]['name']
    hash(spec)
    assert M.resolve(_look_alike(class_name, **KERAS_DEFAULTS[class_name], dtype='float32'), task, 3) == spec
    for name in (class_name, class_name.lower(), class_name.upper(), spec.key):
        by_name = M.resolve(name, task, 3)
        assert by_name.key == name and by_name._replace(key=spec.key) == spec


def test_aliases_and_positional_arguments():
    for alias, kind in [('mape', 'MeanAbsolutePercentageError'), ('msle', 'MeanSquaredLogarithmicError'),
                        ('LogCosh', 'LogCoshError')]:
        assert M.resolve(alias, 'regression').kind == kind
    for alias in ('logloss', 'bce', 'Binary_Crossentropy'):
        assert M.resolve(alias, 'binary').kind == 'BinaryCrossentropy'
    assert M.resolve('categorical_crossentropy', 'multiclass', 4).kind == 'CategoricalCrossentropy'
    assert M.Precision(0.3).thresholds == 0.3 and M.AUC(50, 'PR').curve == 'PR' and M.TopKCategoricalAccuracy(2).k == 2
    assert M.resolve(M.Precision(0.3, name='p30'), 'binary').key == 'p30'
    assert M.resolve(M.Recall(thresholds=[0.7, 0.3]), 'binary').get('thresholds') == (0.7, 0.3)
    with pytest.raises(TypeError, match='bogus'):
        M.Precision(bogus=1)


@pytest.mark.parametrize('metric, named', [
    (M.Precision(top_k=2), 'top_k'), (M.Recall(top_k=1), 'top_k'), (M.AUC(label_weights=[1.0]), 'label_weights'),
    (M.AUC(from_logits=True), 'from_logits'), (M.BinaryCrossentropy(from_logits=True), 'from_logits'),
    (M.BinaryCrossentropy(label_smoothing=0.1), 'label_smoothing'), (M.Precision(dtype='float64'), 'dtype'),
    (M.Precision(dtype='bfloat16'), 'dtype'), (_look_alike('Precision', thresholds=None, top_k=3), 'top_k')])
def test_options_that_are_not_built_are_refused_by_name(metric, named):
    with pytest.raises(NotImplementedError, match=named):
        M.resolve(metric, 'binary', 2)


def test_unknown_metrics_and_bad_values_are_refused():
    for metric in ('mean_io_u', 'hinge', _look_alike('MeanIoU', num_classes=2), 3.5):
        with pytest.raises(NotImplementedError, match='metric'):
            M.resolve(metric, 'binary', 2)
    with pytest.raises(NotImplementedError, match='class_aggregation'):
        M.resolve(M.R2Score(class_aggregation='variance_weighted_average'), 'regression')
    for bad in (M.Precision(thresholds=1.5), M.AUC(num_thresholds=1), M.AUC(curve='XY'), M.AUC(summation_method='x'),
                M.F1Score(average='samples'), M.F1Score(threshold=0.0), M.FBetaScore(beta=0.0),
                M.TopKCategoricalAccuracy(k=0), M.Precision(class_id=5), M.BinaryAccuracy(threshold=1.0)):
        with pytest.raises(ValueError, match=type(bad).__name__):
            M.resolve(bad, 'multiclass', 3)


@pytest.mark.parametrize('metric, task', [
    ('categorical_accuracy', 'regression'), ('CategoricalAccuracy', 'binary'), (M.TopKCategoricalAccuracy(), 'multilabel'),
    ('r2_score', 'binary'), (M.R2Score(), 'multiclass'), ('precision', 'regression'), (M.AUC(), 'regression'),
    ('binary_crossentropy', 'regression'), ('categorical_crossentropy', 'binary')])
def test_a_metric_that_does_not_fit_the_task_is_a_value_error(metric, task):
    name = metric if isinstance(metric, str) else type(metric).__name__
    with pytest.raises(ValueError, match=f'(?i){name.replace("_", "")}.*{task}'):
        M.resolve(metric, task, 3)


# ---- ModelConfig.metrics as a whole ------------------------------------------------------------------------------------
OLD_SPELLINGS = ['auc', 'AUC', 'acc', 'accuracy', 'Accuracy', 'mse', 'MSE', 'mean_squared_error', 'rmse',
                 'RootMeanSquaredError', 'root_mean_squared_error', 'mae', 'mean_absolute_error']


def _named(y_true, y_pred):
    return float(np.mean(y_pred))


@pytest.mark.parametrize('task', ['binary', 'multiclass', 'regression'])
def test_the_older_spellings_keep_their_functions(task):
    """Every string _resolve_metrics knows, and plain functions, go where they went: same key, same value."""
    g = torch.Generator().manual_seed(3)
    cols = 3 if task == 'multiclass' else 1
    p = torch.rand(64, cols, generator=g)
    t = torch.nn.functional.one_hot(torch.randint(0, 3, (64,), generator=g), 3).float() if task == 'multiclass' \
        else (torch.rand(64, 1, generator=g) < 0.4).float()
    for entry in OLD_SPELLINGS + [_named]:
        fns, specs, keys = deepmodel._plan_metrics([entry], task, 3)
        want = deepmodel._resolve_metrics([entry], task)
        assert not specs and list(fns) == list(want) == list(keys)
        (key, fn), = fns.items()
        assert fn(t, p) == want[key](t, p)
    assert deepmodel._plan_metrics(['AUC'], task, 3)[0]['AUC'] is deepmodel._auc


def test_plan_metrics_orders_keys_and_refuses_duplicates():
    fns, specs, keys = deepmodel._plan_metrics(['AUC', M.AUC(name='auc_200'), 'Precision', _named, M.Recall(), 'logloss'],
                                               'binary', 2)
    assert keys == ('AUC', 'auc_200', 'Precision', '_named', 'recall', 'logloss')
    assert list(fns) == ['AUC', '_named'] and [s.key for s in specs] == ['auc_200', 'Precision', 'recall', 'logloss']
    # an object of a known class name is a streaming metric whatever its name
    assert deepmodel._plan_metrics([M.AUC(name='mse')], 'binary', 2)[1][0].kind == 'AUC'
    for pair in (['AUC', M.AUC()], ['precision', M.Precision()], [M.Recall(), M.Recall(thresholds=0.3)], ['mse', 'MSE']):
        with pytest.raises(ValueError, match='two entries'):
            deepmodel._plan_metrics(pair, 'binary', 2)
    with pytest.raises(NotImplementedError, match='metric'):
        deepmodel._plan_metrics(['cosine_similarity'], 'binary', 2)
    assert deepmodel._plan_metrics(None, 'binary', 2) == ({}, [], ())


def test_early_stopping_mode_auto():
    from deeptables_b200.deeptable import EarlyStopping
    for name in ('val_precision', 'val_recall', 'val_auc_200', 'val_f1_score', 'val_fbeta_score', 'val_r2_score',
                 'val_true_positives', 'val_true_negatives', 'val_binary_accuracy', 'val_AUC', 'val_accuracy'):
        assert EarlyStopping(monitor=name).mode == 'max', name
    for name in ('val_loss', 'val_logloss', 'val_mape', 'val_mse', 'val_false_positives', 'val_false_negatives',
                 'val_mean_squared_error', 'val_rmse'):
        assert EarlyStopping(monitor=name).mode == 'min', name


# ---- finishing: Plan.finish on states made by hand ------------------------------------------------------------------------
BINARY = [M.AUC(), M.AUC(curve='PR', name='pr'), M.AUC(num_thresholds=3, summation_method='minoring', name='lo'),
          M.AUC(num_thresholds=50, curve='PR', summation_method='majoring', name='hi'),
          M.AUC(thresholds=[0.9, 0.25, 0.5], name='given'), M.Precision(), M.Recall(thresholds=[0.7, 0.3]),
          M.TruePositives(), M.FalsePositives(0.3), M.TrueNegatives([0.3, 0.7]), M.FalseNegatives(),
          M.BinaryAccuracy(), M.BinaryAccuracy(threshold=0.3, name='acc30'), 'f1_score',
          M.F1Score(threshold=0.5, name='f1_t'), M.FBetaScore(beta=2.0, threshold=0.3, average='micro'), 'logloss',
          'mape', 'msle', 'logcosh', M.MeanSquaredError(), M.RootMeanSquaredError(), M.MeanAbsoluteError()]


def _ref_of(spec):
    p = {k: v for k, v in spec.params if k not in ('scalar',)}
    if 'scalar' in dict(spec.params) and spec.get('scalar'):
        p['thresholds'] = p['thresholds'][0]
    if spec.kind == 'AUC':
        p['thresholds'] = p.pop('given_thresholds')
    return MR.Ref(spec.kind, **p)


def _check(entries, task, num_classes, y, p, batches=1):
    specs = [M.resolve(e, task, num_classes) for e in entries]
    plan = M.Plan(specs, y.shape[1])
    got = plan.finish(SR.state_of(plan, y, p))
    assert list(got) == [s.key for s in specs]
    for s in specs:
        ref = _ref_of(s)
        for yb, pb in zip(np.array_split(y, batches), np.array_split(p, batches)):
            ref.update(yb, pb)
        want = ref.result()
        assert type(got[s.key]) is type(want), s
        np.testing.assert_allclose(got[s.key], want, rtol=2e-6, atol=1e-7, err_msg=str(s))
    return got


def _binary_case(case, n=500):
    g = np.random.default_rng(5)
    y = (g.random((n, 1)) < 0.3).astype(np.float32)
    p = g.random((n, 1)).astype(np.float32)
    if case == 'on_thresholds':         # float32 values of AUC's and the other lists' thresholds, and their neighbours
        t = np.concatenate([MR.auc_thresholds(200), np.float32([0.3, 0.5, 0.7])])
        t = np.concatenate([t, np.nextafter(t, np.float32(2)), np.nextafter(t, np.float32(-2))])
        p = np.clip(g.choice(t, size=(n, 1)), 0, 1).astype(np.float32)
    elif case == 'zeros_and_ones':
        p = g.integers(0, 2, size=(n, 1)).astype(np.float32)
    elif case == 'all_equal':
        p[:] = 0.5
    elif case == 'only_positives':
        y[:] = 1
    elif case == 'only_negatives':
        y[:] = 0
    elif case == 'nan':
        p[::7] = np.nan
    elif case == 'empty':
        y, p = y[:0], p[:0]
    return y, p


@pytest.mark.parametrize('case', ['random', 'on_thresholds', 'zeros_and_ones', 'all_equal', 'only_positives',
                                  'only_negatives', 'empty'])
def test_finish_binary(case):
    y, p = _binary_case(case)
    got = _check(BINARY, 'binary', 2, y, p, batches=3)
    if case == 'random':
        from sklearn import metrics as SK
        np.testing.assert_allclose(got['precision'], SK.precision_score(y, p > 0.5), rtol=1e-6)
        np.testing.assert_allclose(got['recall'], [SK.recall_score(y, p > 0.7), SK.recall_score(y, p > 0.3)], rtol=1e-6)
        np.testing.assert_allclose(got['f1_t'], [SK.f1_score(y, p > 0.5)], rtol=1e-6)
        many = M.Plan([M.resolve(M.AUC(num_thresholds=2000), 'binary')], 1)
        np.testing.assert_allclose(many.finish(SR.state_of(many, y, p))['auc'], SK.roc_auc_score(y, p), atol=2e-3)
    if case == 'empty':
        assert all(v in (0.0, [0.0], [0.0, 0.0]) for v in got.values())


def test_finish_with_nan_predictions_counts_them_below_every_threshold():
    y, p = _binary_case('nan')
    confusion = [e for e in BINARY if not isinstance(e, str) and type(e).__name__ not in
                 ('MeanSquaredError', 'RootMeanSquaredError', 'MeanAbsoluteError')]
    _check(confusion, 'binary', 2, y, p)


def test_finish_multilabel_and_class_id():
    g = np.random.default_rng(8)
    y = (g.random((300, 4)) < 0.3).astype(np.float32)
    p = g.random((300, 4)).astype(np.float32)
    _check([M.AUC(multi_label=True), M.AUC(name='flat'), M.AUC(curve='PR', multi_label=True, name='pr'), M.Precision(),
            M.Precision(class_id=2, name='p2'), M.Recall(thresholds=[0.2, 0.6], class_id=0), M.BinaryAccuracy(),
            M.F1Score(threshold=0.5), M.F1Score(threshold=0.5, average='macro', name='macro'),
            M.FBetaScore(beta=0.5, threshold=0.4, average='weighted'), M.F1Score(name='argmax'), 'bce'],
           'multilabel', 4, y, p, batches=2)


def test_finish_multiclass():
    g = np.random.default_rng(9)
    labels = g.integers(0, 5, size=400)
    y = np.eye(5, dtype=np.float32)[labels]
    z = g.normal(size=(400, 5)) + 1.5 * y
    p = (np.exp(z) / np.exp(z).sum(-1, keepdims=True)).astype(np.float32)
    p[:40] = p[:40].round(1)            # ties between classes
    got = _check(['categorical_accuracy', M.TopKCategoricalAccuracy(k=2), 'f1_score', M.F1Score(average='macro', name='macro'),
                  M.F1Score(average='micro', name='micro'), M.F1Score(average='weighted', name='weighted'),
                  M.FBetaScore(beta=2.0), 'categorical_crossentropy', 'precision', M.Recall(class_id=3), M.AUC(),
                  'binary_accuracy'], 'multiclass', 5, y, p, batches=4)
    from sklearn import metrics as SK
    clean = slice(40, None)
    plan = M.Plan([M.resolve(M.F1Score(average='macro'), 'multiclass', 5)], 5)
    np.testing.assert_allclose(plan.finish(SR.state_of(plan, y[clean], p[clean]))['f1_score'],
                               SK.f1_score(labels[clean], p[clean].argmax(-1), average='macro'), rtol=1e-5)
    assert 0 < got['categorical_accuracy'] <= got['top_k_categorical_accuracy'] <= 1


def test_finish_regression():
    g = np.random.default_rng(10)
    y = g.normal(2.0, 1.0, size=(300, 1)).astype(np.float32)
    p = (y + g.normal(0, 0.5, size=y.shape)).astype(np.float32)
    got = _check(['r2_score', 'mape', 'msle', 'logcosh', M.MeanSquaredError(), M.RootMeanSquaredError(),
                  M.MeanAbsoluteError()], 'regression', None, y, p, batches=3)
    from sklearn import metrics as SK
    np.testing.assert_allclose(got['r2_score'], SK.r2_score(y, p), rtol=1e-5)
    constant = M.Plan([M.resolve('r2_score', 'regression')], 1)
    assert constant.finish(SR.state_of(constant, np.ones((9, 1)), p[:9]))['r2_score'] == 0.0


def test_metrics_sharing_a_threshold_list_share_one_histogram():
    specs = [M.resolve(e, 'binary') for e in (M.Precision(), M.Recall(), M.F1Score(threshold=0.5), M.BinaryAccuracy(),
                                               M.AUC(), M.AUC(curve='PR', name='pr'))]
    plan = M.Plan(specs, 1)
    assert [len(t) for t in plan.lists] == [1, 200] and plan.sums == 0 and not plan.argmax
    assert plan.words == 8 + 3 + (3 + 3) + 2 * 2 + 2 * 201
    np.testing.assert_array_equal(plan.thresholds()[1:], MR.auc_thresholds(200))
    with pytest.raises(NotImplementedError, match='threshold'):
        M.Plan([M.resolve(M.Precision(thresholds=0.05 * i, name=f'p{i}'), 'binary') for i in range(1, 10)], 1)
    with pytest.raises(NotImplementedError, match='two different k'):
        M.Plan([M.resolve(M.TopKCategoricalAccuracy(k=k, name=f'k{k}'), 'multiclass', 9) for k in (2, 3)], 9)


def test_merge_is_the_state_of_all_rows_together():
    y, p = _binary_case('random', n=600)
    specs = [M.resolve(e, 'binary') for e in (M.AUC(), M.Precision(), 'logloss')]
    plan = M.Plan(specs, 1)
    c = plan.counters
    parts = [SR.state_of(plan, y[i::3], p[i::3]) for i in range(3)]
    whole = SR.state_of(plan, y, p)
    merged = plan.merge(sum(s[c:] for s in parts).view(np.int64), np.stack([s[:c].view(np.float64) for s in parts]))
    np.testing.assert_array_equal(merged[c:], whole[c:])
    np.testing.assert_allclose(merged[:c].view(np.float64), whole[:c].view(np.float64), rtol=1e-12)
    assert plan.finish(merged) == plan.finish(whole)
    shard_mean = np.mean([plan.finish(s)['precision'] for s in parts])
    assert plan.finish(merged)['precision'] != shard_mean         # the metric of all rows is not the mean of shards
