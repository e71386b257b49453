"""Streaming metrics on the GPU: ``dtb_metrics_update`` through the C ABI against the numpy restatement of its state
(counters equal, float64 sums to 1e-12), and through DeepModel.fit / evaluate against the Keras restatement in
metrics_ref.py fed with the same predictions."""
import os
import socket

import numpy as np
import pandas as pd
import pytest
import torch

import metrics_ref as MR
import metrics_state_ref as SR
from test_metrics_cpu import _ref_of

pytestmark = pytest.mark.gpu


def _state(plan):
    from deeptables_b200 import engine as E
    return E.MetricsState(plan, torch.device('cuda', 0))


def _plan(entries, task, num_classes, cols):
    from deeptables_b200 import metrics as M
    return M.Plan([M.resolve(e, task, num_classes) for e in entries], cols)


def _assert_state(plan, got, y, p, what):
    want = SR.state_of(plan, y, p)
    c = plan.counters
    np.testing.assert_array_equal(got[c:], want[c:], err_msg=f'{what}: counters')
    np.testing.assert_allclose(got[:c].view(np.float64), want[:c].view(np.float64), rtol=1e-12, atol=1e-300,
                               err_msg=f'{what}: float64 sums')


def _update(st, y, p, splits=1):
    st.reset()
    for yb, pb in zip(np.array_split(y, splits), np.array_split(p, splits)):
        st.update(torch.as_tensor(pb).cuda(), torch.as_tensor(yb).cuda())
    return st.read()


def _binary_data(rows, kind, seed=0):
    g = np.random.default_rng(seed)
    y = (g.random((rows, 1)) < 0.25).astype(np.float32)
    if kind == 'random':
        p = g.random((rows, 1)).astype(np.float32)
    elif kind == 'equal':
        p = np.full((rows, 1), 0.5, np.float32)
    else:                               # on the thresholds of every list under test, and one float32 either side
        t = np.concatenate([MR.auc_thresholds(200), MR.auc_thresholds(1000), np.float32([0.5, 0.013, 0.2, 0.77, 0.9])])
        t = np.concatenate([t, np.nextafter(t, np.float32(2)), np.nextafter(t, np.float32(-2))])
        p = np.clip(g.choice(t, size=(rows, 1)), 0, 1).astype(np.float32)
    return y, p


def _binary_entries():
    from deeptables_b200 import metrics as M
    return {
        't1': [M.Precision(), M.Recall(), 'logloss'],
        't2': [M.Recall(thresholds=[0.3, 0.7])],
        't200': [M.AUC(), M.Precision(), M.MeanSquaredError()],
        't1000': [M.AUC(num_thresholds=1000), M.AUC(curve='PR', name='pr')],
        'irregular': [M.AUC(thresholds=[0.013, 0.2, 0.77, 0.9]), M.TruePositives([0.9, 0.2, 0.013]), 'mape', 'msle',
                      'logcosh', M.MeanAbsoluteError()],
    }


@pytest.mark.parametrize('rows', [1, 31, 1000, 8192, 65536])
@pytest.mark.parametrize('plan_name', ['t1', 't2', 't200', 't1000', 'irregular'])
def test_update_binary(plan_name, rows):
    plan = _plan(_binary_entries()[plan_name], 'binary', 2, 1)
    st = _state(plan)
    for kind in ('random', 'equal', 'on_thresholds'):
        y, p = _binary_data(rows, kind, seed=rows)
        _assert_state(plan, _update(st, y, p), y, p, f'{plan_name} rows {rows} {kind}')


def test_updates_accumulate_and_reset_zeroes():
    plan = _plan(_binary_entries()['t200'], 'binary', 2, 1)
    st = _state(plan)
    y, p = _binary_data(5000, 'random')
    once, many = _update(st, y, p), _update(st, y, p, splits=7)
    np.testing.assert_array_equal(once[plan.counters:], many[plan.counters:])
    np.testing.assert_allclose(once[:plan.counters].view(np.float64), many[:plan.counters].view(np.float64), rtol=1e-12)
    again = _update(st, y, p)
    np.testing.assert_array_equal(once[plan.counters:], again[plan.counters:])      # counters do not depend on scheduling
    st.reset()
    assert not st.read().any()
    nan = p.copy()
    nan[::5] = np.nan
    counts_only = _plan(_binary_entries()['t200'][:2], 'binary', 2, 1)         # a NaN lands below every threshold
    _assert_state(counts_only, _update(_state(counts_only), y, nan), y, nan, 'NaN predictions')


@pytest.mark.parametrize('rows', [1, 31, 777, 8192])
def test_update_multilabel_multiclass_regression(rows):
    from deeptables_b200 import metrics as M
    g = np.random.default_rng(rows)
    y = (g.random((rows, 4)) < 0.3).astype(np.float32)
    p = g.random((rows, 4)).astype(np.float32)
    plan = _plan([M.AUC(multi_label=True), M.Precision(class_id=1), M.F1Score(threshold=0.4), M.F1Score(name='am'), 'bce'],
                 'multilabel', 4, 4)
    _assert_state(plan, _update(_state(plan), y, p, splits=2), y, p, 'multilabel')
    labels = g.integers(0, 6, size=rows)
    y = np.eye(6, dtype=np.float32)[labels]
    z = g.normal(size=(rows, 6)) + y
    p = (np.exp(z) / np.exp(z).sum(-1, keepdims=True)).astype(np.float32)
    p[: rows // 4] = p[: rows // 4].round(1)            # ties, and rows of zeros and ones
    for entries in (['categorical_accuracy', M.TopKCategoricalAccuracy(k=2), 'f1_score', 'categorical_crossentropy',
                     'precision', M.AUC()],
                    [M.AUC(num_thresholds=1000), 'categorical_accuracy']):     # 12 012 counters: past shared memory
        plan = _plan(entries, 'multiclass', 6, 6)
        _assert_state(plan, _update(_state(plan), y, p, splits=3), y, p, 'multiclass')
    y = g.normal(1.0, 2.0, size=(rows, 1)).astype(np.float32)
    p = (y + g.normal(0, 0.7, size=y.shape)).astype(np.float32)
    plan = _plan(['r2_score', 'mape', 'msle', 'logcosh', M.MeanSquaredError(), M.MeanAbsoluteError()], 'regression', None, 1)
    _assert_state(plan, _update(_state(plan), y, p, splits=2), y, p, 'regression')


def test_bad_plans_are_refused_not_run():
    from deeptables_b200 import _native as N
    bad = N.MetricPlan(cols=1, n_lists=9)
    assert N.lib.dtb_metrics_state_bytes(bad) == 0
    st = _state(_plan(['precision'], 'binary', 2, 1))
    with pytest.raises(ValueError, match='expected'):
        st.update(torch.zeros(4, 2).cuda(), torch.zeros(4, 2).cuda())
    t = torch.zeros(4, 1).cuda()
    assert N.lib.dtb_metrics_update(N.ptr(t), N.ptr(t), N.ptr(st.state), None, 4, bad, None) == -1
    assert 'bad plan' in N.last_error()


# ---- through the model ---------------------------------------------------------------------------------------------------
VOCAB, DIM, N_CONT = [50, 40, 30, 20, 60], 8, 3


class _Recorder:
    """A plain-function metric: records what the epoch functions are given, which is what the streaming metrics saw."""
    __name__ = 'recorded'

    def __init__(self):
        self.calls = []

    def __call__(self, y_true, y_pred):
        self.calls.append((np.array(y_true), np.array(y_pred)))
        return 0.0


def _build(metrics, task='binary', num_classes=2, nets=None, seed=11):
    from deeptables_b200 import deeptable, deepnets
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    conf = deeptable.ModelConfig(nets=nets or deepnets.DeepFM, embeddings_output_dim=DIM, embedding_dropout=0,
                                 metrics=metrics)
    cats = [CategoricalColumn(f'c{i}', v, DIM) for i, v in enumerate(VOCAB)]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(N_CONT)])]
    return DeepModel(task, num_classes, conf, cats, conts, seed=seed)


def _data(n, task='binary', seed=0):
    g = np.random.default_rng(seed)
    idx = np.stack([g.integers(0, v, size=n) for v in VOCAB], axis=1)
    cont = g.normal(size=(n, N_CONT)).astype(np.float32)
    X = pd.DataFrame({**{f'c{i}': idx[:, i] for i in range(len(VOCAB))}, **{f'n{i}': cont[:, i] for i in range(N_CONT)}})
    signal = cont[:, 0] + (idx[:, 0] % 3 == 0) - 0.5
    if task == 'binary':
        y = (g.random(n) < 1 / (1 + np.exp(-2 * signal))).astype(np.float32)
    elif task == 'multiclass':
        y = np.clip(np.round(signal + g.normal(0, 0.5, size=n) + 1.5), 0, 3).astype(np.int64)
    else:
        y = (2.0 + signal + g.normal(0, 0.3, size=n)).astype(np.float32)
    return X, y


def _binary_metrics():
    from deeptables_b200 import metrics as M
    return ['AUC', M.AUC(name='auc_200'), M.AUC(curve='PR', name='auc_pr'), M.Precision(),
            M.Recall(thresholds=[0.3, 0.7]), 'f1_score', 'logloss']


def _assert_logs(model, logs, prefix, y, p, what):
    for spec in model._metrics_train.plan.specs:
        ref = _ref_of(spec)
        ref.update(y, p)
        np.testing.assert_allclose(logs[prefix + spec.key], ref.result(), rtol=2e-6, atol=1e-7,
                                   err_msg=f'{what}: {prefix}{spec.key}')


def test_fit_history_equals_the_reference_on_the_same_predictions(monkeypatch):
    from deeptables_b200 import deepmodel
    # The recorder is an epoch function, and epoch functions on training batches are only right with eager steps: a
    # replayed step returns the same output tensor every time, so fit collects the last batch's predictions once per
    # batch (a defect older than the streaming metrics, which read the predictions inside the step; README).  Replay is
    # covered by test_replayed_steps_give_the_eager_history_and_leave_training_untouched.
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    rec = _Recorder()
    model = _build(_binary_metrics() + [rec])
    X, y = _data(4096)
    Xv, yv = _data(1024, seed=1)
    h = model.fit(X, y, batch_size=256, epochs=2, verbose=0, validation_data=(Xv, yv)).history
    keys = ['AUC', 'auc_200', 'auc_pr', 'precision', 'recall', 'f1_score', 'logloss', 'recorded']
    assert list(h.keys()) == ['loss'] + [k.lower() for k in keys] + ['val_loss'] + ['val_' + k.lower() for k in keys]
    assert len(rec.calls) == 4          # train and validation of two epochs
    for epoch in range(2):
        for prefix, (t, p) in (('', rec.calls[2 * epoch]), ('val_', rec.calls[2 * epoch + 1])):
            logs = {k: v[epoch] for k, v in h.items()}
            _assert_logs(model, logs, prefix, t, p, f'epoch {epoch}')
            exact = deepmodel._auc(torch.as_tensor(t), torch.as_tensor(p))
            assert logs[prefix + 'auc'] == pytest.approx(exact, rel=1e-12)
            assert abs(logs[prefix + 'auc_200'] - exact) < 5e-3
    assert h['precision'][1] > 0 and len(h['recall'][0]) == 2
    ev = model.evaluate(Xv, yv, batch_size=256)
    t, p = rec.calls[-1]
    assert set(ev.keys()) == {'loss'} | {k.lower() for k in keys}
    _assert_logs(model, ev, '', t, p, 'evaluate')
    assert 'Precision(' in str(model.model_desc) and 'auc_200' in str(model.model_desc)


# Two-row batches without a repeated id in any column, and a small DNN: the setting in which this suite's other replay
# tests get the same bits from every run (no two rows add into one embedding-gradient row).
EXACT_VOCAB, EXACT_ROWS = [400, 300, 500, 350], 2


def _exact_model(metrics):
    from deeptables_b200 import deeptable
    from deeptables_b200.deepmodel import DeepModel
    from deeptables_b200.metainfo import CategoricalColumn, ContinuousColumn
    conf = deeptable.ModelConfig(nets=['linear', 'fm_nets', 'dnn_nets'], embeddings_output_dim=DIM, embedding_dropout=0,
                                 metrics=metrics,
                                 dnn_params={'hidden_units': ((16, 0, False), (8, 0, True)), 'activation': 'relu'})
    cats = [CategoricalColumn(f'c{i}', v, DIM) for i, v in enumerate(EXACT_VOCAB)]
    conts = [ContinuousColumn('input_continuous_all', [f'n{i}' for i in range(N_CONT)])]
    return DeepModel('binary', 2, conf, cats, conts, seed=5)


def _exact_data(batches):
    parts = []
    for seed in range(batches):
        g = np.random.default_rng(seed)
        idx = np.stack([g.choice(v, size=EXACT_ROWS, replace=False) for v in EXACT_VOCAB], axis=1)
        cont = g.normal(size=(EXACT_ROWS, N_CONT)).astype(np.float32)
        parts.append((idx, cont, (g.random(EXACT_ROWS) < 0.4).astype(np.float32)))
    idx, cont, y = (np.concatenate([p[k] for p in parts]) for k in range(3))
    X = pd.DataFrame({**{f'c{i}': idx[:, i] for i in range(len(EXACT_VOCAB))},
                      **{f'n{i}': cont[:, i] for i in range(N_CONT)}})
    return X, y


def _states_equal(a, b, what):
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), f'{what}: {k} differs'


def test_replayed_steps_give_the_eager_history_and_leave_training_untouched(monkeypatch):
    """The update kernel as a node of the captured train step: one more launch, the history of the eager run bit for
    bit (which in turn is the reference on the eager run's recorded predictions), and the weights of a model without
    streaming metrics bit for bit."""
    from deeptables_b200 import metrics as M
    X, y = _exact_data(48)
    streaming = [M.AUC(name='auc_200'), M.AUC(curve='PR', name='auc_pr'), M.Precision(thresholds=0.4),
                 M.Recall(thresholds=[0.3, 0.45]), M.F1Score(threshold=0.4, name='f1'), M.TruePositives(0.4),
                 M.FalsePositives(0.4), M.BinaryAccuracy(), 'logloss']
    runs = {}
    for name, graphs, metrics in (('eager', '0', streaming), ('replayed', '1', streaming), ('plain', '1', [])):
        monkeypatch.setenv('DTB_CUDA_GRAPH', graphs)
        rec = _Recorder()
        model = _exact_model(metrics + [rec])
        h = model.fit(X, y, batch_size=EXACT_ROWS, epochs=3, verbose=0, shuffle=False,
                      validation_data=(X.head(24), y[:24])).history
        runs[name] = (model, dict(h), rec)
    (eager, he, rec), (replayed, hg, _), (plain, hp, _) = runs['eager'], runs['replayed'], runs['plain']
    assert not eager._graphs and replayed._graphs and not replayed._graph_failed, 'the train step was not captured'
    (with_metrics,), (without,) = [e[-1] for e in replayed._graphs.values()], [e[-1] for e in plain._graphs.values()]
    assert with_metrics == without + 1          # one more launch per step, whatever the number of metrics
    keys = [k for k in he if 'recorded' not in k]
    assert len(keys) == 2 * (1 + len(streaming))
    for k in keys:
        assert hg[k] == he[k], k                # counters and, in one stream with one warp per launch, the sums too
    assert he['true_positives'][-1] + he['false_positives'][-1] > 0 and 0 < he['auc_200'][-1] < 1
    for epoch in range(3):                      # and the eager history is the reference on what the eager steps predicted
        logs = {k: v[epoch] for k, v in he.items()}
        _assert_logs(eager, logs, '', *rec.calls[2 * epoch], f'epoch {epoch}')
        _assert_logs(eager, logs, 'val_', *rec.calls[2 * epoch + 1], f'epoch {epoch}')
    _states_equal(replayed, eager, 'replayed vs eager')
    _states_equal(replayed, plain, 'with vs without streaming metrics')
    assert hg['loss'] == hp['loss'] and hg['val_loss'] == hp['val_loss']


def test_a_monitored_vector_metric_is_refused_by_name():
    from deeptables_b200 import deeptable, metrics as M
    model = _build([M.Recall(thresholds=[0.3, 0.7])])
    X, y = _data(512)
    with pytest.raises(ValueError, match="EarlyStopping monitors 'val_recall'.*one value per threshold"):
        model.fit(X, y, batch_size=256, epochs=1, verbose=0, validation_data=_data(512, seed=1),
                  callbacks=[deeptable.EarlyStopping(monitor='val_recall', mode='max')])


def test_oof_metrics_take_the_streaming_names(tmp_path):
    """fit_cross_validation(oof_metrics=): the names it took stay sklearn's; metrics.py's names and objects are scored
    per fold on the GPU.  Counts add up over the folds to the counts of the whole out-of-fold matrix."""
    from deeptables_b200 import deeptable, deepnets, metrics as M
    g = np.random.default_rng(3)
    n = 600
    df = pd.DataFrame({'a': g.choice(list('abcdef'), size=n), 'b': g.choice(['x', 'y', 'z'], size=n),
                       'u': g.normal(size=n), 'v': g.exponential(size=n)})
    y = np.where(g.random(n) < 1 / (1 + np.exp(-((df['a'] == 'a') * 2.0 + df['u'] * 1.5 - 0.5))), 1, 0)
    conf = deeptable.ModelConfig(nets=deepnets.DeepFM, embedding_dropout=0, metrics=['AUC'], auto_scale=True,
                                 earlystopping_patience=3, home_dir=str(tmp_path / 'out'))
    dt = deeptable.DeepTable(config=conf)
    oof, _, _, scores = dt.fit_cross_validation(
        df, y, num_folds=3, stratified=True, batch_size=64, epochs=3, verbose=0,
        oof_metrics=['auc', 'precision', M.Recall(thresholds=0.3, name='recall30'), 'true_positives', 'false_positives',
                     M.AUC(name='auc_200')])
    assert [list(sc) for sc in scores] == [['auc', 'precision', 'recall30', 'true_positives', 'false_positives', 'auc_200']] * 3
    p = oof[:, 1].astype(np.float32)
    assert sum(sc['true_positives'] for sc in scores) == ((p > 0.5) & (y == 1)).sum()
    assert sum(sc['false_positives'] for sc in scores) == ((p > 0.5) & (y == 0)).sum()
    for sc in scores:
        np.testing.assert_allclose(sc['precision'], sc['true_positives'] / max(sc['true_positives'] + sc['false_positives'], 1),
                                   rtol=1e-6)
        assert abs(sc['auc_200'] - sc['auc']) < 2e-2 and 0 < sc['recall30'] <= 1
    with pytest.raises(NotImplementedError, match='oof metric'):
        deeptable._calc_scores(y, y, oof, 'binary', ['cosine_similarity'], 1, [0, 1])


def test_early_stopping_and_monitor_metric_take_the_new_names():
    from deeptables_b200 import deeptable, deepnets, metrics as M
    es = deeptable.EarlyStopping(monitor='val_precision', patience=0)
    assert es.mode == 'max'
    model = _build([M.Precision()])
    X, y = _data(2048)
    h = model.fit(X, y, batch_size=256, epochs=3, verbose=0, validation_data=_data(512, seed=1), callbacks=[es]).history
    assert es.best == max(h['val_precision']) and len(h['val_precision']) <= 3
    df = X.copy()
    conf = deeptable.ModelConfig(nets=deepnets.DeepFM, embedding_dropout=0, metrics=['Precision', 'Recall'],
                                 monitor_metric='val_recall', earlystopping_patience=1)
    dt = deeptable.DeepTable(config=conf)
    _, history = dt.fit(df, y, batch_size=256, epochs=2, verbose=0)
    assert 'val_recall' in history.history and 'precision' in history.history
    assert set(dt.evaluate(df, y, batch_size=256).keys()) >= {'precision', 'recall', 'loss'}


def test_multiclass_and_regression_epochs(monkeypatch):
    from deeptables_b200 import metrics as M
    monkeypatch.setenv('DTB_CUDA_GRAPH', '0')
    for task, num_classes, metrics in (
            ('multiclass', 4, ['categorical_accuracy', M.TopKCategoricalAccuracy(k=2), M.F1Score(average='macro')]),
            ('regression', None, ['r2_score', 'mape', 'msle'])):
        rec = _Recorder()
        model = _build(metrics + [rec], task=task, num_classes=num_classes)
        X, y = _data(2048, task)
        h = model.fit(X, y, batch_size=256, epochs=1, verbose=0, validation_data=_data(512, task, seed=1)).history
        logs = {k: v[0] for k, v in h.items()}
        _assert_logs(model, logs, '', *rec.calls[0], task)
        _assert_logs(model, logs, 'val_', *rec.calls[1], task)


def test_wrong_metrics_raise_when_the_model_is_built():
    from deeptables_b200 import metrics as M
    with pytest.raises(ValueError, match='R2Score'):
        _build(['r2_score'])._build_model()
    with pytest.raises(NotImplementedError, match='top_k'):
        _build([M.Precision(top_k=1)])._build_model()
    with pytest.raises(ValueError, match='two entries'):
        _build(['AUC', M.AUC()])._build_model()


# ---- data parallel ---------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _dp_metrics():
    from deeptables_b200 import metrics as M
    return [M.Precision(), M.AUC(), 'logloss']


def _dp_worker(rank, world, port, out_dir):
    import json
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        rec = _Recorder()
        model = _build(_dp_metrics() + [rec])
        X, y = _data(2048)
        Xv, yv = _data(1024, seed=1)
        shard, vshard = slice(rank, None, world), slice(rank * 512, (rank + 1) * 512)
        h = model.fit(X[shard], y[shard], batch_size=128, epochs=1, verbose=0, shuffle=False,
                      validation_data=(Xv[vshard], yv[vshard]), validation_steps=4).history
        with open(os.path.join(out_dir, f'rank{rank}.json'), 'w') as f:
            json.dump(dict(h), f)
        np.savez(os.path.join(out_dir, f'rank{rank}.npz'), ty=rec.calls[0][0], tp=rec.calls[0][1], vy=rec.calls[1][0],
                 vp=rec.calls[1][1])
    finally:
        dist.destroy_process_group()


def test_data_parallel_logs_the_metric_of_all_shards(tmp_path):
    """Both ranks log the same values, and they are the metrics of the two shards' rows together (from what each rank
    predicted), not the mean of the shards' metrics."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    import json
    import torch.multiprocessing as mp
    from deeptables_b200 import metrics as M
    out = str(tmp_path)
    mp.spawn(_dp_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    h0, h1 = (json.load(open(os.path.join(out, f'rank{r}.json'))) for r in range(2))
    seen = [np.load(os.path.join(out, f'rank{r}.npz')) for r in range(2)]
    for prefix, yk, pk in (('', 'ty', 'tp'), ('val_', 'vy', 'vp')):
        for entry in _dp_metrics():
            spec = M.resolve(entry, 'binary', 2)
            ref = _ref_of(spec)
            for r in range(2):
                ref.update(seen[r][yk], seen[r][pk])
            key = prefix + spec.key
            assert h0[key] == h1[key], key
            np.testing.assert_allclose(h0[key][0], ref.result(), rtol=2e-6, atol=1e-7, err_msg=key)
