"""DeepTable -- the user-facing estimator of the reference (deeptables/models/deeptable.py) over the
H100 engine: ``DeepTable(config).fit(X, y) / predict / predict_proba / evaluate / save / load``.

The train/score hot path (DeepModel) is the product; what surrounds it here is the thinnest host
layer that makes the README flow work on a pandas DataFrame: a pandas/sklearn ``DefaultPreprocessor``
with the reference's column conventions (label-encoded categoricals with ``nunique + 2`` vocabulary
slots, reference preprocessor.py:333; one continuous group named ``input_continuous_all``,
preprocessor.py:495-500), early stopping injected as the reference does (deeptable.py:709-754) and
the binary ``[1-p, p]`` probability fix (deeptable.py:689-691), the quantile-bin columns of ``auto_discrete``
(discrete.py) and the gradient-boosted leaf columns of ``apply_gbm_features`` (gbm.py).  Var-len columns and the
model-set leaderboard are out of scope (SURVEY.md 8f).
"""
import copy
import os
import pickle
import time

import numpy as np
import pandas as pd

from . import consts, deepmodel
from .config import ModelConfig
from .metainfo import CategoricalColumn, ContinuousColumn


class EarlyStopping:
    """keras.callbacks.EarlyStopping subset the reference injects (deeptable.py:742-749)."""

    def __init__(self, monitor='val_loss', min_delta=0, patience=0, verbose=0, mode='auto',
                 restore_best_weights=False):
        self.monitor, self.min_delta, self.patience = monitor, abs(min_delta), patience
        self.verbose, self.restore_best_weights = verbose, restore_best_weights
        if mode == 'auto':
            lower = monitor.lower()
            mode = 'max' if any(k in lower for k in ('acc', 'auc', 'fmeasure', 'f1', 'precision', 'recall', 'r2', 'fbeta',
                                                     'true_positives', 'true_negatives')) else 'min'
        self.mode = mode
        self.model = None

    def set_model(self, model):
        self.model = model

    def on_train_begin(self, logs=None):
        self.wait, self.best, self.best_weights, self.stopped_epoch = 0, None, None, 0

    def _better(self, cur):
        if self.best is None:
            return True
        return cur > self.best + self.min_delta if self.mode == 'max' else cur < self.best - self.min_delta

    def on_epoch_end(self, epoch, logs=None):
        logs = {k.lower(): v for k, v in (logs or {}).items()}
        cur = logs.get(self.monitor.lower())
        if cur is None:
            return
        if self._better(cur):
            self.best, self.wait = cur, 0
            if self.restore_best_weights:
                self.best_weights = {k: v.clone() for k, v in self.model.state_dict().items()}
        else:
            self.wait += 1
            if self.wait >= self.patience:
                self.stopped_epoch = epoch
                self.model.stop_training = True
                if self.restore_best_weights and self.best_weights is not None:
                    self.model.load_state_dict(self.best_weights)


class DefaultPreprocessor:
    """Minimal stand-in for the reference's DefaultPreprocessor (preprocessor.py:100-515)."""

    def __init__(self, config):
        self.config = config
        self.labels_ = None
        self.task_ = None
        self.categorical_columns = []
        self.continuous_columns = []
        self._cat_maps = {}
        self._cont_fill = {}
        self._scale = {}
        self.X_types = None

    # ---- y ------------------------------------------------------------------------------------
    def _infer_task(self, y):
        if self.config.task != consts.TASK_AUTO:
            return self.config.task
        y = pd.Series(np.asarray(y).reshape(-1))
        n = y.nunique()
        if n == 2:
            return consts.TASK_BINARY
        if y.dtype.kind in 'OUSb' or (y.dtype.kind in 'iu' and n <= 1000) or \
                (y.dtype.kind == 'f' and n <= 20 and np.allclose(y, y.round())):
            return consts.TASK_MULTICLASS
        return consts.TASK_REGRESSION

    def fit_transform(self, X, y):
        t0 = time.time()
        X = X.copy()
        if len(set(X.columns)) != len(X.columns):
            raise ValueError('Columns with duplicate names in X.')
        X.columns = [str(c) for c in X.columns]
        self.feature_names_in_ = list(X.columns)          # the fitted frame's columns, excluded ones included
        self.task_ = self._infer_task(y)
        y = np.asarray(y).reshape(-1)
        if self.task_ in (consts.TASK_BINARY, consts.TASK_MULTICLASS) and self.config.auto_encode_label:
            self.labels_ = list(pd.unique(pd.Series(y)))
            try:
                self.labels_ = sorted(self.labels_)
            except TypeError:
                pass
            if self.task_ == consts.TASK_BINARY and self.config.pos_label is not None:
                self.labels_ = [l for l in self.labels_ if l != self.config.pos_label] + [self.config.pos_label]
            lut = {l: i for i, l in enumerate(self.labels_)}
            y = np.array([lut[v] for v in y], dtype=np.int64)
        elif self.task_ == consts.TASK_REGRESSION:
            y = y.astype(np.float32)
        X = X.drop(columns=[c for c in (self.config.exclude_columns or []) if c in X.columns])
        cfg = self.config
        if cfg.apply_gbm_features:
            from .gbm import GbmLeavesEncoder
            GbmLeavesEncoder.check_names(X)
        cats, conts = [], []
        for c in X.columns:
            col = X[c]
            explicit = isinstance(cfg.categorical_columns, (list, tuple)) and c in cfg.categorical_columns
            auto = cfg.categorical_columns == 'auto' and (
                col.dtype.kind in 'OUSb' or str(col.dtype) == 'category' or
                (cfg.auto_categorize and col.nunique() < len(col) ** cfg.cat_exponent))
            if explicit or auto:
                cats.append(c)
            else:
                conts.append(c)
        if cfg.auto_discard_unique:
            for c in list(cats) + list(conts):
                if X[c].nunique(dropna=False) <= 1:
                    (cats if c in cats else conts).remove(c)
        self._cat_names, self._cont_names = cats, conts
        for c in cats:
            vals = X[c].astype(object).where(X[c].notna(), '__nan__')
            classes = sorted(pd.unique(vals), key=str)
            self._cat_maps[c] = {v: i for i, v in enumerate(classes)}
        for c in conts:
            col = pd.to_numeric(X[c], errors='coerce').astype(np.float64)
            self._cont_fill[c] = float(col.mean()) if col.notna().any() else 0.0
            if cfg.auto_scale:
                lo, hi = float(col.min()), float(col.max())
                self._scale[c] = (lo, (hi - lo) or 1.0)
        # a fixed width of 0 means the default width 4, not CategoricalColumn's fourth root (preprocessor.py:477-478)
        dim = (cfg.embeddings_output_dim if cfg.embeddings_output_dim > 0 else consts.EMBEDDING_OUT_DIM_DEFAULT) \
            if cfg.fixed_embedding_dim else 0
        self.categorical_columns = []
        for c in cats:
            vocab = len(self._cat_maps[c]) + 2            # + unseen + reserved (preprocessor.py:333)
            d = dim if cfg.fixed_embedding_dim else min(4 * int(pow(vocab, 0.25)), 20)
            self.categorical_columns.append(CategoricalColumn(c, vocab, d))
        self.continuous_columns = [ContinuousColumn('input_continuous_all', list(conts))] if conts else []
        self.gbm_encoder_ = None
        self.discretizer_ = None
        if cfg.auto_discrete and conts:
            from .discrete import MultiKBinsDiscretizer
            MultiKBinsDiscretizer.check_names(X, conts)
        Xt = self._encode(X)
        if cfg.auto_discrete and conts:
            Xt = self._fit_discretizer(Xt, dim)
        if cfg.apply_gbm_features and y is not None:
            Xt = self._fit_gbm_features(Xt, y, dim)
        self.fit_seconds_ = time.time() - t0
        return Xt, y

    def _fit_discretizer(self, Xt, dim):
        """The reference's _discretization (preprocessor.py:406-415): one quantile-bin code per continuous column,
        appended after the label-encoded categoricals as an embedded column of vocabulary n_bins + 1."""
        from .discrete import MultiKBinsDiscretizer
        disc = MultiKBinsDiscretizer(self._cont_names)
        Xt = disc.fit_transform(Xt)
        self.discretizer_ = disc
        for name, vocab in zip(disc.new_columns, disc.vocabulary_sizes):
            d = dim if self.config.fixed_embedding_dim else min(4 * int(pow(vocab, 0.25)), 20)
            self.categorical_columns.append(CategoricalColumn(name, vocab, d))
        return Xt

    def _fit_gbm_features(self, Xt, y, dim):
        """The reference's _apply_gbm_features (preprocessor.py:431-452): trees on the encoded, imputed and scaled
        columns, the discretised ones among the categorical inputs; one embedded column per tree, or one continuous
        group holding the raw leaf indices."""
        from . import gbm
        cfg = self.config
        if self.task_ == consts.TASK_MULTILABEL:
            raise NotImplementedError('apply_gbm_features on the multilabel task')
        disc = self.discretizer_
        enc = gbm.GbmLeavesEncoder(self._cat_names + (disc.new_columns if disc is not None else []), self._cont_names,
                                   self.task_, **(cfg.gbm_params or {}))
        Xt = enc.fit_transform(Xt, y, len(self.labels_) if self.labels_ else None)
        self.gbm_encoder_ = enc
        if cfg.gbm_feature_type == consts.GBM_FEATURE_TYPE_EMB:
            for name, leaves in zip(enc.new_columns, enc.trees.num_leaves):
                vocab = int(leaves)           # every leaf holds training rows: the reference's max + 1
                d = dim if cfg.fixed_embedding_dim else min(4 * int(pow(vocab, 0.25)), 20)
                self.categorical_columns.append(CategoricalColumn(name, vocab, d))
        elif enc.new_columns:
            self.continuous_columns.append(ContinuousColumn(consts.INPUT_PREFIX_NUM + 'gbm_leaves',
                                                            list(enc.new_columns)))
        return Xt

    def transform_X(self, X):
        enc = getattr(self, 'gbm_encoder_', None)
        disc = getattr(self, 'discretizer_', None)
        if enc is not None:
            enc.check_names(X)
        if disc is not None:
            disc.check_names(X, disc.columns)
        Xt = self._encode(X)
        if disc is not None:
            Xt = disc.transform(Xt)
        return enc.transform(Xt) if enc is not None else Xt

    def _encode(self, X):
        X = X.copy()
        X.columns = [str(c) for c in X.columns]
        out = {}
        for c in self._cat_names:
            m = self._cat_maps[c]
            unseen = len(m)
            vals = X[c].astype(object).where(X[c].notna(), '__nan__')
            out[c] = vals.map(lambda v, _m=m, _u=unseen: _m.get(v, _u)).astype(np.int32).values
        for c in self._cont_names:
            col = pd.to_numeric(X[c], errors='coerce').astype(np.float64)
            if self.config.auto_imputation:
                col = col.fillna(self._cont_fill[c])
            if c in self._scale:
                lo, span = self._scale[c]
                col = (col - lo) / span
            out[c] = col.astype(np.float32).values
        return pd.DataFrame(out, index=X.index)

    def transform_y(self, y):
        y = np.asarray(y).reshape(-1)
        if self.labels_ is not None:
            lut = {l: i for i, l in enumerate(self.labels_)}
            return np.array([lut[v] for v in y], dtype=np.int64)
        return y.astype(np.float32)

    def transform(self, X, y):
        return self.transform_X(X), self.transform_y(y)

    def inverse_transform_y(self, y_indicator):
        if self.labels_ is not None:
            return np.array([self.labels_[int(i)] for i in y_indicator])
        return y_indicator

    @property
    def task(self):
        return self.task_

    @property
    def pos_label(self):
        return self.labels_[-1] if (self.labels_ and self.task_ == consts.TASK_BINARY) else None

    @property
    def labels(self):
        return self.labels_

    def get_categorical_columns(self):
        return [c.name for c in self.categorical_columns]

    def get_continuous_columns(self):
        return list(self._cont_names)


_OOF_SKLEARN_NAMES = ('auc', 'roc_auc', 'accuracy', 'acc', 'f1', 'f1_score', 'logloss', 'log_loss', 'mse',
                      'mean_squared_error', 'rmse', 'mae', 'mean_absolute_error', 'r2', 'r2_score')


def _is_streaming_metric(m):
    """An ``oof_metrics`` entry that metrics.py computes: its objects, and its names that _calc_scores does not take."""
    from . import metrics as M
    return M.is_metric_object(m) or (isinstance(m, str) and m.lower() not in _OOF_SKLEARN_NAMES and M.is_metric_name(m))


def _calc_scores(y_true, y_pred, y_proba, task, metrics, pos_label, classes):
    """Scores of one fold for ``oof_metrics`` (the reference delegates to hypernets' calc_score): metric name -> value."""
    from sklearn import metrics as M
    out = {}
    for m in metrics:
        key = (m if isinstance(m, str) else getattr(m, '__name__', str(m))).lower()
        if key in ('auc', 'roc_auc'):
            out[key] = M.roc_auc_score(y_true, y_proba[:, -1]) if task == consts.TASK_BINARY else \
                M.roc_auc_score(y_true, y_proba, multi_class='ovo', labels=classes)
        elif key in ('accuracy', 'acc'):
            out[key] = M.accuracy_score(y_true, y_pred)
        elif key in ('f1', 'f1_score'):
            out[key] = M.f1_score(y_true, y_pred, pos_label=pos_label) if task == consts.TASK_BINARY else \
                M.f1_score(y_true, y_pred, average='macro')
        elif key in ('logloss', 'log_loss'):
            out[key] = M.log_loss(y_true, y_proba, labels=classes)
        elif key in ('mse', 'mean_squared_error'):
            out[key] = M.mean_squared_error(y_true, y_pred)
        elif key in ('rmse',):
            out[key] = float(np.sqrt(M.mean_squared_error(y_true, y_pred)))
        elif key in ('mae', 'mean_absolute_error'):
            out[key] = M.mean_absolute_error(y_true, y_pred)
        elif key in ('r2', 'r2_score'):
            out[key] = M.r2_score(y_true, y_pred)
        else:
            raise NotImplementedError(f'oof metric {m!r}')
    return out


class DeepTable:
    """Reference user API (deeptable.py:27-330 docstring surface)."""

    def __init__(self, config=None, preprocessor=None, cache_home=None):
        self.config = config if config is not None else ModelConfig()
        self.nets = self.config.nets
        self.output_path = self._prepare_output_dir(self.config.home_dir, self.nets)
        self.preprocessor = preprocessor if preprocessor is not None else DefaultPreprocessor(self.config)
        self.__current_model = None
        self.__modelset = {}

    @staticmethod
    def _prepare_output_dir(home_dir, nets):
        if home_dir is None:
            home_dir = 'dt_output'
        if home_dir[-1] == '/':
            home_dir = home_dir[:-1]
        running_dir = f'dt_{time.strftime("%Y%m%d%H%M%S")}_{"_".join(nets)}'[:120]
        return os.path.expanduser(f'{home_dir}/{running_dir}/')

    @property
    def task(self):
        return self.preprocessor.task

    @property
    def num_classes(self):
        return len(self.preprocessor.labels) if self.preprocessor.labels else None

    @property
    def classes_(self):
        return self.preprocessor.labels

    @property
    def pos_label(self):
        return self.config.pos_label if self.config.pos_label is not None else self.preprocessor.pos_label

    @property
    def monitor(self):
        monitor = self.config.monitor_metric
        if monitor is None and self.config.metrics:
            monitor = 'val_' + self.config.first_metric_name
        return monitor

    def fit(self, X=None, y=None, batch_size=128, epochs=1, verbose=1, callbacks=None, validation_split=0.2,
            validation_data=None, shuffle=True, class_weight=None, sample_weight=None, initial_epoch=0,
            steps_per_epoch=None, validation_steps=None, validation_freq=1, max_queue_size=10, workers=1,
            use_multiprocessing=False):
        X, y = self.preprocessor.fit_transform(X, y)
        if validation_data is not None:
            validation_data = self.preprocessor.transform(*validation_data)
        if class_weight is None and self.config.apply_class_weight and \
                self.task in (consts.TASK_BINARY, consts.TASK_MULTICLASS):
            vals, counts = np.unique(y, return_counts=True)
            class_weight = {int(v): float(len(y) / (len(vals) * c)) for v, c in zip(vals, counts)}
        callbacks = self._inject_callbacks(callbacks)
        model = deepmodel.DeepModel(self.task, self.num_classes, self.config,
                                    self.preprocessor.categorical_columns, self.preprocessor.continuous_columns)
        history = model.fit(X, y, batch_size=batch_size, epochs=epochs, verbose=verbose, callbacks=callbacks,
                            validation_split=validation_split, validation_data=validation_data, shuffle=shuffle,
                            class_weight=class_weight, sample_weight=sample_weight, initial_epoch=initial_epoch,
                            steps_per_epoch=steps_per_epoch, validation_steps=validation_steps,
                            validation_freq=validation_freq)
        name = f'{"+".join(self.nets)}'
        self.__modelset[name] = (model, history.history)
        self.__current_model = model
        return model, history

    def fit_cross_validation(self, X, y, X_eval=None, X_test=None, num_folds=5, stratified=False, iterators=None,
                             batch_size=None, epochs=1, verbose=1, callbacks=None, n_jobs=1, random_state=9527,
                             shuffle=True, class_weight=None, sample_weight=None, initial_epoch=0, steps_per_epoch=None,
                             validation_steps=None, validation_freq=1, max_queue_size=10, workers=1,
                             use_multiprocessing=False, oof_metrics=None):
        """K-fold training with out-of-fold probabilities (reference deeptable.py:373-517).  One model per fold is fitted on
        the fold's training rows with the held-out rows as validation data, scores the held-out rows (-> the out-of-fold
        matrix), X_eval and X_test (-> fold means), is saved next to the run's outputs and registered in the model set as
        ``<nets>-kfold-<n>`` (``predict(..., model_selector='all')`` averages them).  Returns
        ``(oof_proba, eval_proba_mean, test_proba_mean[, oof_scores])`` with binary probabilities as ``[1-p, p]`` columns.
        The folds run one after the other on this process' GPU (``n_jobs`` is accepted for signature parity)."""
        from sklearn.model_selection import KFold, StratifiedKFold
        self.__modelset.clear()
        X, y = self.preprocessor.fit_transform(X, y)
        if X_eval is not None:
            X_eval = self.preprocessor.transform_X(X_eval)
        if X_test is not None:
            X_test = self.preprocessor.transform_X(X_test)
        if iterators is None:
            if stratified and self.task != consts.TASK_REGRESSION:
                iterators = StratifiedKFold(n_splits=num_folds, shuffle=True, random_state=random_state)
            else:
                iterators = KFold(n_splits=num_folds, shuffle=True, random_state=random_state)
        y = np.array(y)
        n_rows = X.shape[0]
        width = self.num_classes if self.task in (consts.TASK_MULTICLASS, consts.TASK_MULTILABEL) else 1
        oof_proba = np.full((n_rows, width), np.nan)
        eval_mean = test_mean = None
        if class_weight is None and self.config.apply_class_weight and self.task == consts.TASK_BINARY:
            vals, counts = np.unique(y, return_counts=True)
            class_weight = {int(v): float(len(y) / (len(vals) * c)) for v, c in zip(vals, counts)}
        callbacks = self._inject_callbacks(callbacks)
        sw_all = None if sample_weight is None else np.asarray(sample_weight)
        oof_scores = [] if oof_metrics is not None else None
        os.makedirs(self.output_path, exist_ok=True)
        for n_fold, (train_idx, valid_idx) in enumerate(iterators.split(X, y)):
            model = deepmodel.DeepModel(self.task, self.num_classes, self.config, self.preprocessor.categorical_columns,
                                        self.preprocessor.continuous_columns)
            history = model.fit(X.iloc[train_idx], y[train_idx], batch_size=batch_size, epochs=epochs, verbose=verbose,
                                callbacks=callbacks, validation_data=(X.iloc[valid_idx], y[valid_idx]), shuffle=shuffle,
                                class_weight=class_weight, sample_weight=None if sw_all is None else sw_all[train_idx],
                                initial_epoch=initial_epoch, steps_per_epoch=steps_per_epoch,
                                validation_steps=validation_steps, validation_freq=validation_freq)
            fold_oof = model.predict(X.iloc[valid_idx])
            oof_proba[valid_idx] = fold_oof.reshape(len(valid_idx), -1)
            if X_eval is not None:
                pe = model.predict(X_eval) / num_folds
                eval_mean = pe if eval_mean is None else eval_mean + pe
            if X_test is not None:
                pt = model.predict(X_test) / num_folds
                test_mean = pt if test_mean is None else test_mean + pt
            if oof_metrics is not None:
                y_true = self.preprocessor.inverse_transform_y(y[valid_idx])
                y_proba = self._fix_softmax_proba(fold_oof.copy()) if self.task == consts.TASK_BINARY else fold_oof.copy()
                y_pred = self.proba2predict(y_proba, encode_to_label=True)
                streaming = [m for m in oof_metrics if _is_streaming_metric(m)]
                scores = _calc_scores(y_true, y_pred, y_proba, self.task,
                                      [m for m in oof_metrics if not _is_streaming_metric(m)], self.pos_label, self.classes_)
                if streaming:           # the names and objects of metrics.py, on the fold's encoded labels and raw output
                    scores.update(model.streaming_scores(streaming, y[valid_idx], fold_oof))
                oof_scores.append(scores)
            name = f'{"+".join(self.nets)}-kfold-{n_fold + 1}'
            model.save(f'{self.output_path}{"_".join(self.nets)}-kfold-{n_fold + 1}.npz')
            self.__modelset[name] = (model, history.history)
            self.__current_model = model
        nan_idx = np.argwhere(np.isnan(oof_proba).any(1)).ravel()
        if self.task == consts.TASK_BINARY:
            oof_fixed = self._fix_softmax_proba(oof_proba.copy())
            eval_fixed = self._fix_softmax_proba(eval_mean.copy()) if eval_mean is not None else None
            test_fixed = self._fix_softmax_proba(test_mean.copy()) if test_mean is not None else None
            if test_mean is not None:
                import pandas as pd
                pd.DataFrame(test_mean.reshape(-1)).to_csv(f'{self.output_path}{"_".join(self.nets)}-cv-{num_folds}.csv',
                                                           index=False)
        else:
            oof_fixed = oof_proba.reshape(n_rows) if self.task == consts.TASK_REGRESSION else oof_proba
            eval_fixed, test_fixed = eval_mean, test_mean
        if len(nan_idx) > 0:
            oof_fixed[nan_idx] = np.nan
        if oof_metrics is not None:
            return oof_fixed, eval_fixed, test_fixed, oof_scores
        return oof_fixed, eval_fixed, test_fixed

    @staticmethod
    def _fix_softmax_proba(proba):
        """(n, 1) sigmoid output -> (n, 2) columns [1-p, p] (hypernets' fix_binary_predict_proba_result)."""
        if proba is None:
            return None
        proba = proba.reshape(len(proba), -1)
        return np.hstack([1.0 - proba, proba]) if proba.shape[1] == 1 else proba

    def _inject_callbacks(self, callbacks):
        callbacks = list(callbacks or [])
        if self.monitor is None or any(isinstance(cb, EarlyStopping) for cb in callbacks):
            return callbacks
        mode = self.config.earlystopping_mode
        callbacks.append(EarlyStopping(monitor=self.monitor, min_delta=0,
                                       patience=self.config.earlystopping_patience, verbose=1, mode=mode,
                                       restore_best_weights=True))
        return callbacks

    def get_model(self, model_selector=consts.MODEL_SELECTOR_CURRENT, brevity=True):
        if model_selector in (consts.MODEL_SELECTOR_CURRENT, consts.MODEL_SELECTOR_BEST):
            return self.__current_model
        if model_selector == consts.MODEL_SELECTOR_ALL:
            return [m for m, _ in self.__modelset.values()]
        if model_selector in self.__modelset:
            return self.__modelset[model_selector][0]
        raise ValueError(f'{model_selector} does not exist.')

    @property
    def best_model(self):
        return self.__current_model

    def _predict_raw(self, X, batch_size, verbose, auto_transform_data, model_selector):
        model = self.get_model(model_selector)
        if model is None:
            raise ValueError(f'"{model_selector}" not found in modelset.')
        if auto_transform_data:
            X = self.preprocessor.transform_X(X)
        if isinstance(model, list):         # 'all': mean of the model set's probabilities (reference deeptable.py:541-552)
            if not model:
                raise ValueError('the model set is empty')
            return sum(m.predict(X, batch_size=batch_size, verbose=verbose) for m in model) / len(model)
        return model.predict(X, batch_size=batch_size, verbose=verbose)

    def predict_proba(self, X, batch_size=128, verbose=0, model_selector=consts.MODEL_SELECTOR_CURRENT,
                      auto_transform_data=True):
        proba = self._predict_raw(X, batch_size, verbose, auto_transform_data, model_selector)
        if self.task == consts.TASK_BINARY and proba.shape[-1] == 1:
            proba = np.hstack([1.0 - proba, proba])        # [1-p, p]  (reference deeptable.py:689-691)
        return proba

    def predict(self, X, encode_to_label=True, batch_size=128, verbose=0,
                model_selector=consts.MODEL_SELECTOR_CURRENT, auto_transform_data=True):
        proba = self.predict_proba(X, batch_size, verbose, model_selector, auto_transform_data)
        return self.proba2predict(proba, encode_to_label)

    def proba2predict(self, proba, encode_to_label=True):
        if self.task == consts.TASK_REGRESSION:
            return proba
        if proba is None:
            raise ValueError('[proba] can not be none.')
        if len(proba.shape) == 1:
            proba = proba.reshape((-1, 1))
        if proba.shape[-1] > 1:
            predict = proba.argmax(axis=-1)
        else:
            predict = (proba > 0.5).astype(consts.DATATYPE_PREDICT_CLASS)
        if encode_to_label:
            predict = self.preprocessor.inverse_transform_y(predict.reshape(-1))
        return predict

    def evaluate(self, X_test, y_test, batch_size=256, verbose=0, model_selector=consts.MODEL_SELECTOR_CURRENT,
                 return_dict=True):
        X_t, y_t = self.preprocessor.transform(X_test, y_test)
        model = self.get_model(model_selector)
        if model is None:
            raise ValueError(f'"{model_selector}" not found in modelset.')
        return model.evaluate(X_t, y_t, batch_size=batch_size, verbose=verbose, return_dict=return_dict)

    def apply(self, X, output_layers, concat_outputs=False, batch_size=128, verbose=0,
              model_selector=consts.MODEL_SELECTOR_CURRENT, auto_transform_data=True, transformer=None):
        model = self.get_model(model_selector)
        if auto_transform_data:
            X = self.preprocessor.transform_X(X)
        return model.apply(X, output_layers, concat_outputs, batch_size, verbose, transformer)

    def save(self, filepath, deepmodel_basename=None):
        os.makedirs(filepath, exist_ok=True)
        model = self.__current_model
        name = deepmodel_basename or 'current_model'
        if model is not None:
            model.save(os.path.join(filepath, f'{name}.npz'))
        meta = {'config': self.config._replace(distribute_strategy=None), 'preprocessor': self.preprocessor,
                'model_name': name if model is not None else None, 'step': model._step if model else 0}
        with open(os.path.join(filepath, 'dt.pkl'), 'wb') as f:
            pickle.dump(meta, f, protocol=pickle.HIGHEST_PROTOCOL)

    @staticmethod
    def load(filepath):
        with open(os.path.join(filepath, 'dt.pkl'), 'rb') as f:
            meta = pickle.load(f)
        dt = DeepTable(meta['config'], preprocessor=meta['preprocessor'])
        if meta['model_name'] is not None:
            pre = meta['preprocessor']
            model = deepmodel.DeepModel(pre.task, len(pre.labels) if pre.labels else None, meta['config'],
                                        pre.categorical_columns, pre.continuous_columns,
                                        model_file=os.path.join(filepath, f"{meta['model_name']}.npz"))
            dt._DeepTable__current_model = model      # the .npz carries the Adam step and moments (DeepModel._restore_optimizer)
        return dt


def probe_evaluate(dt, X, y, X_test, y_test, layers, score_fn={}, *, batch_size=65536):
    """How much of the label a linear model reads off each named layer (reference deeptable.py ``probe_evaluate``).

    For each name in ``layers``, in order, the layer's outputs for ``X`` (flattened to ``(rows, -1)``) fit a
    ``LogisticRegression(random_state=0)`` of scikit-learn 1.9 on ``dt.preprocessor.transform_y(y)``, computed on the
    GPU (probe.py), and the probe is scored on ``X_test`` / ``y_test``.  Returns ``{layer: {'accuracy': mean
    accuracy}}`` when ``score_fn`` is empty, else ``{layer: {name: fn(y_test, .)}}`` in ``score_fn`` order, where ``fn``
    gets ``predict_proba[:, 1]`` when it is ``sklearn.metrics.roc_auc_score`` and the predicted classes otherwise.
    ``batch_size`` rows go through each inference forward.  Binary and multiclass models only."""
    from . import probe
    return probe.probe_evaluate(dt, X, y, X_test, y_test, layers, score_fn, batch_size=batch_size)
