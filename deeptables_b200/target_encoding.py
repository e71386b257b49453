"""Target encoding on the GPU: scikit-learn's ``TargetEncoder`` and the reference's ``preprocessing.utils.target_encoding``.

Each categorical value is replaced by a smoothed mean of the target over the rows that carry it.  ``fit_transform``
cross-fits: the rows of fold f are encoded by statistics of the rows outside f, so a row's own target never reaches
its encoding.

Host work is validation, the fold ids (the scikit-learn splitter) and, for columns that are not numeric, one
``pandas.factorize``.  Numeric columns are coded on the device (sort, unique with NaN last, searchsorted).  Each column's
rows are then sorted by (category, fold, class) and the kernels of ``csrc/target_encode.cu`` turn the sorted segments
into per-fold statistics, the encoding tables of every fold's fitting rows, and the float64 output.  Every sum has one
fixed order, so a call gives the same bits run to run, whatever the tile and column-group sizes.
"""
import numbers

import numpy as np
import pandas as pd
import torch
from sklearn.base import BaseEstimator, TransformerMixin

from . import _native as N
from ._native import check, ptr, stream_ptr

TE_SMOOTH, TE_AUTO, TE_RECALLED = 0, 1, 2
_TARGET_TYPES = ('auto', 'continuous', 'binary', 'multiclass')
_TILE_ROWS = 4096
_WORKSPACE_BYTES = 1 << 30


def _device():
    return torch.device('cuda', torch.cuda.current_device())


def _is_nan(v):
    return isinstance(v, (float, np.floating)) and v != v


# ---- host: columns, codes and the target --------------------------------------------------------------------------

def split_columns(X, where='X'):
    """(columns, feature names or None, rows) of a 2-D frame or array, one column at a time as scikit-learn sees them."""
    if hasattr(X, 'iloc') and getattr(X, 'ndim', 0) == 2:
        names = [str(c) for c in X.columns] if all(isinstance(c, str) for c in X.columns) else None
        return [X.iloc[:, i] for i in range(X.shape[1])], names, X.shape[0]
    arr = np.asarray(X)
    if not hasattr(X, 'dtype') and arr.dtype.kind == 'U':
        arr = np.asarray(X, dtype=object)
    if arr.ndim != 2:
        raise ValueError(f'{where} must be 2-D (rows, columns); got shape {arr.shape}')
    return [arr[:, i] for i in range(arr.shape[1])], None, arr.shape[0]


def _numeric_values(col):
    """The column as a numpy array when the device codes it (numeric, bool, category of numbers), else None."""
    if isinstance(col, pd.Series):
        dt = col.dtype
        if isinstance(dt, pd.CategoricalDtype):
            return np.asarray(col) if dt.categories.dtype.kind in 'biuf' else None
        if not isinstance(dt, np.dtype):
            return None
        col = col.to_numpy()
    if col.dtype.kind in 'bif' or (col.dtype.kind == 'u' and col.dtype.itemsize < 8):
        return col
    return None


def _code_numeric(values, cats, missing_category):
    """Device codes (int32, -1 unknown) of a numeric column and its categories (sorted, NaN last)."""
    dev = _device()
    floating = values.dtype.kind == 'f' or (cats is not None and np.asarray(cats).dtype.kind == 'f')
    work = np.float64 if floating else np.int64
    host = np.ascontiguousarray(values, dtype=work)
    t = torch.from_numpy(host if host.flags.writeable else host.copy()).to(dev)
    if cats is None:
        srt = torch.sort(t).values
        nnan = int(torch.isnan(srt).sum()) if floating else 0
        known = torch.unique_consecutive(srt[:t.numel() - nnan])
        cats = known.cpu().numpy().astype(values.dtype)
        nan_code = -1
        if nnan and missing_category:
            nan_code = len(cats)
            cats = np.append(cats, np.array([np.nan], dtype=values.dtype))
        codes = torch.searchsorted(known, t, out_int32=True)
    else:
        cats = np.asarray(cats)
        nan_mask = np.isnan(cats) if cats.dtype.kind == 'f' else np.zeros(len(cats), dtype=bool)
        kn = cats[~nan_mask].astype(work)
        nan_code = int(np.flatnonzero(nan_mask)[0]) if nan_mask.any() and missing_category else -1
        known = torch.from_numpy(kn).to(dev)
        if len(kn) == 0:
            codes = torch.full_like(t, -1, dtype=torch.int32)
        else:
            codes = torch.searchsorted(known, t, out_int32=True)
            hit = known[codes.clamp(max=len(kn) - 1).long()] == t
            codes = torch.where(hit & (codes < len(kn)), codes, torch.full_like(codes, -1))
    if floating:
        codes = torch.where(torch.isnan(t), torch.full_like(codes, nan_code), codes)
    return codes.contiguous(), cats


def _code_host(col, cats, missing_category):
    """Codes of a column factorised by pandas on the host, remapped on the device into sorted category order."""
    fcodes, uniq = pd.factorize(col)
    uniq = np.asarray(uniq, dtype=object)
    U = len(uniq)
    na = fcodes < 0
    has_none = has_nan = False
    if na.any():
        rows = np.flatnonzero(na)
        na_vals = col.iloc[rows] if isinstance(col, pd.Series) else col[rows]
        none = np.fromiter((v is None for v in na_vals), dtype=bool, count=len(rows))
        has_none, has_nan = bool(none.any()), bool((~none).any())
        fcodes = fcodes.copy()
        fcodes[rows] = np.where(none, U, U + 1)
    remap = np.full(U + 2, -1, dtype=np.int32)
    if cats is None:
        order = np.argsort(uniq, kind='stable')          # Python's ordering, as scikit-learn's sorted(set(values))
        remap[order] = np.arange(U, dtype=np.int32)
        listed = list(uniq[order])
        if missing_category and has_none:
            remap[U] = len(listed)
            listed.append(None)
        if missing_category and has_nan:
            remap[U + 1] = len(listed)
            listed.append(np.nan)
        dtype = col.dtype if isinstance(col, np.ndarray) else np.dtype(object)
        cats = np.array(listed, dtype=dtype) if listed else np.array([], dtype=dtype)
    else:
        lut, none_pos, nan_pos = {}, -1, -1
        for i, c in enumerate(cats):
            if c is None:
                none_pos = i
            elif _is_nan(c):
                nan_pos = i
            else:
                lut.setdefault(c, i)
        remap[:U] = [lut.get(u, -1) for u in uniq]
        if missing_category:
            remap[U], remap[U + 1] = none_pos, nan_pos
    dev = _device()
    src = torch.from_numpy(np.ascontiguousarray(fcodes, dtype=np.int64)).to(dev)
    rm = torch.from_numpy(remap).to(dev)
    codes = torch.empty(src.numel(), dtype=torch.int32, device=dev)
    check(N.lib.dtb_te_remap(ptr(src), ptr(rm), src.numel(), len(remap), ptr(codes), stream_ptr()), 'dtb_te_remap')
    return codes, cats


def code_column(col, cats=None, missing_category=True):
    """(device int32 codes, categories) of one column; code -1 for values outside the given categories (and for
    missing values when they are not a category)."""
    values = _numeric_values(col)
    if values is not None and (cats is None or np.asarray(cats).dtype.kind in 'biuf'):
        return _code_numeric(values, cats, missing_category)
    return _code_host(col, cats, missing_category)


def _check_y(y, n):
    y = y.to_numpy() if hasattr(y, 'to_numpy') else np.asarray(y)
    if y.ndim == 2 and y.shape[1] == 1:
        y = y.ravel()
    if y.ndim != 1:
        raise ValueError(f'y must be 1-D: a multilabel or multi-output target (shape {y.shape}) is not supported')
    if len(y) != n:
        raise ValueError(f'X and y have different lengths: {n} rows against {len(y)} targets')
    if pd.isna(y).any():
        raise ValueError('y contains NaN or None: every row needs a target')
    return y


def _float_target(y, what):
    try:
        return np.asarray(y, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError(f'{what} must be numeric for a continuous target') from None


class _Target:
    """The target, the fold ids and the whole-target statistics on the device."""

    def __init__(self, y_cls, classes, y_float, fold, folds, formula, smooth, tile_rows, sklearn_unknowns):
        dev = _device()
        # scikit-learn fits the rows outside given categories as the first category, and its fit_transform gives every
        # such row the last fold's mean; the reference helper counts them toward no category
        self.sklearn_unknowns = sklearn_unknowns
        self.n = len(y_cls) if y_cls is not None else len(y_float)
        self.classes = max(classes, 2) if y_cls is not None else 0
        self.n_out = self.classes if self.classes > 2 else 1
        self.folds = folds
        self.groups = folds + 1 if folds > 1 else 1
        self.formula, self.smooth, self.tile_rows = formula, float(smooth), tile_rows
        self.cls = torch.from_numpy(np.ascontiguousarray(y_cls, dtype=np.int32)).to(dev) if y_cls is not None else None
        self.y = torch.from_numpy(np.ascontiguousarray(y_float, dtype=np.float64)).to(dev) if y_cls is None else None
        self.fold = torch.from_numpy(np.ascontiguousarray(fold, dtype=np.uint8)).to(dev) if fold is not None else None
        self.whole = self.stats(None, 1)

    def stats(self, codes, cats):
        """starts, sums and sums of squares of every (category, fold[, class]) slot of one column (codes None: the
        whole target as one category)."""
        dev, n, s = _device(), self.n, stream_ptr()
        keys = torch.empty(n, dtype=torch.int64, device=dev)
        unknown = 0 if self.sklearn_unknowns and cats > 0 else -1
        check(N.lib.dtb_te_keys(ptr(codes), ptr(self.fold), ptr(self.cls), n, self.folds, self.classes, unknown,
                                ptr(keys), s), 'dtb_te_keys')
        keys, perm = torch.sort(keys, stable=True)
        slots = cats * self.folds * max(self.classes, 1)
        starts = torch.empty(slots + 1, dtype=torch.int64, device=dev)
        check(N.lib.dtb_te_segment_starts(ptr(keys), n, slots, ptr(starts), s), 'dtb_te_segment_starts')
        sums = m2 = None
        if self.classes == 0:
            partial = torch.empty(n, dtype=torch.float64, device=dev)
            sums = torch.empty(slots, dtype=torch.float64, device=dev)
            check(N.lib.dtb_te_segment_stats(ptr(keys), ptr(perm), ptr(self.y), ptr(starts), None, n, self.tile_rows,
                                             ptr(partial), s), 'dtb_te_segment_stats')
            check(N.lib.dtb_te_segment_join(ptr(starts), ptr(partial), slots, ptr(sums), s), 'dtb_te_segment_join')
            if self.formula == TE_AUTO:
                m2 = torch.empty(slots, dtype=torch.float64, device=dev)
                check(N.lib.dtb_te_segment_stats(ptr(keys), ptr(perm), ptr(self.y), ptr(starts), ptr(sums), n,
                                                 self.tile_rows, ptr(partial), s), 'dtb_te_segment_stats')
                check(N.lib.dtb_te_segment_join(ptr(starts), ptr(partial), slots, ptr(m2), s), 'dtb_te_segment_join')
        return starts, sums, m2

    def encodings(self, codes, cats, prior=None):
        """The float64 table [groups, cats, n_out] of one column (and the group means into prior)."""
        starts, sums, m2 = self.stats(codes, cats)
        ps, psum, pm2 = self.whole
        table = torch.empty(self.groups * cats * self.n_out, dtype=torch.float64, device=_device())
        check(N.lib.dtb_te_encodings(ptr(starts), ptr(sums), ptr(m2), ptr(ps), ptr(psum), ptr(pm2), cats, self.folds,
                                     self.classes, self.formula, self.smooth, ptr(table), ptr(prior), stream_ptr()),
              'dtb_te_encodings')
        return table


def gather(out, col0, codes, tables, cats, prior, fold, n_out, unknown_group=-1):
    """Write the encodings of a group of columns into out[:, col0 * n_out : (col0 + len(codes)) * n_out]."""
    dev, n = _device(), out.shape[0]
    if n == 0:
        return
    block = torch.stack(codes)
    flat = torch.cat(tables)
    off = np.concatenate([[0], np.cumsum([t.numel() for t in tables])[:-1]]).astype(np.int64)
    off_t = torch.from_numpy(off).to(dev)
    cats_t = torch.tensor(cats, dtype=torch.int32, device=dev)
    base = out.data_ptr() + col0 * n_out * out.element_size()
    check(N.lib.dtb_te_gather(ptr(block), ptr(fold), ptr(flat), ptr(off_t), ptr(cats_t), ptr(prior), n, len(codes),
                              n_out, unknown_group, out.shape[1], N.c_void_p(base), stream_ptr()), 'dtb_te_gather')


def _group_bytes(n, cats, groups, n_out):
    return 4 * n + 8 * groups * cats * n_out


def cross_fit(columns, target, *, categories=None, missing_category=True, transform=True, test_columns=None,
              group_cols=None, workspace_bytes=_WORKSPACE_BYTES):
    """Encode every column: the categories, each column's group-0 table [cats, n_out] (host), the group means
    [groups, n_out] (host) and, with transform, the device output [rows, columns * n_out] in which each row takes its
    fold's group (group 0 without folds).  test_columns are coded against the learned categories and encoded by group
    0 into a second output.  Columns are processed in groups whose codes and tables fit workspace_bytes (and hold at
    most group_cols columns); the output bits do not depend on the grouping."""
    dev, n, G, n_out = _device(), target.n, target.groups, target.n_out
    F = len(columns)
    prior = torch.empty(G * n_out, dtype=torch.float64, device=dev)
    out = torch.empty((n, F * n_out), dtype=torch.float64, device=dev) if transform else None
    test_out = None
    if test_columns is not None:
        test_out = torch.empty((len(test_columns[0]) if F else 0, F * n_out), dtype=torch.float64, device=dev)
    all_cats, host_tables = [], []
    pending = []                                    # (column index, codes, table, cats, test codes)

    def flush():
        if not pending:
            return
        c0 = pending[0][0]
        tabs, ncat = [p[2] for p in pending], [len(p[3]) for p in pending]
        if transform:
            gather(out, c0, [p[1] for p in pending], tabs, ncat, prior, target.fold, n_out,
                   target.folds if target.sklearn_unknowns and target.folds > 1 else -1)
        if test_out is not None:
            gather(test_out, c0, [p[4] for p in pending], tabs, ncat, prior, None, n_out)
        pending.clear()

    for i, col in enumerate(columns):
        codes, cats = code_column(col, None if categories is None else categories[i], missing_category)
        V = len(cats)
        table = target.encodings(codes, V, prior if i == 0 else None)
        all_cats.append(cats)
        host_tables.append(table[:V * n_out].view(V, n_out).cpu().numpy())
        test_codes = code_column(test_columns[i], cats, missing_category)[0] if test_columns is not None else None
        if pending and (len(pending) == group_cols or sum(_group_bytes(n, len(p[3]), G, n_out) for p in pending)
                        + _group_bytes(n, V, G, n_out) > workspace_bytes):
            flush()
        pending.append((i, codes, table, cats, test_codes))
    flush()
    return all_cats, host_tables, prior.view(G, n_out).cpu().numpy(), out, test_out


def fold_ids(splits, n, where='cv'):
    """Fold id (uint8) of every row from the (fitting rows, held-out rows) pairs of a splitter.  The held-out rows must
    cover every row exactly once, and each fold's fitting rows must be the other rows."""
    fold = np.zeros(n, dtype=np.uint8)
    seen = np.zeros(n, dtype=np.int64)
    k = 0
    for train_idx, test_idx in splits:
        if k == 255:
            raise ValueError(f'{where}: at most 255 folds are supported')
        train_idx, test_idx = np.asarray(train_idx), np.asarray(test_idx)
        mark = np.bincount(train_idx, minlength=n) + np.bincount(test_idx, minlength=n)
        if len(mark) != n or not np.all(mark == 1):
            raise ValueError(f'{where}: the fitting rows of fold {k} are not the rows outside its validation rows')
        seen += np.bincount(test_idx, minlength=n)[:n]
        fold[test_idx] = k
        k += 1
    if k < 2:
        raise ValueError(f'{where}: cross fitting needs at least 2 folds, got {k}')
    if not np.all(seen == 1):
        raise ValueError(f'{where}: validation indices must cover each sample index exactly once with no overlap')
    return fold, k


# ---- scikit-learn's TargetEncoder --------------------------------------------------------------------------------

class TargetEncoder(TransformerMixin, BaseEstimator):
    """scikit-learn 1.9's ``TargetEncoder`` computed on the GPU: same arguments, attributes and results (to float64
    rounding).  ``shuffle`` and ``random_state`` act on an integer ``cv`` as in scikit-learn, without its deprecation
    warning."""

    def __init__(self, categories='auto', target_type='auto', smooth='auto', cv=5, shuffle=True, random_state=None):
        self.categories = categories
        self.target_type = target_type
        self.smooth = smooth
        self.cv = cv
        self.shuffle = shuffle
        self.random_state = random_state

    # -- validation (host only, before any device work)
    def _check_params(self, n_features):
        if isinstance(self.smooth, str):
            if self.smooth != 'auto':
                raise ValueError(f"smooth must be 'auto' or a non-negative float, got {self.smooth!r}")
        elif (not isinstance(self.smooth, numbers.Real) or isinstance(self.smooth, bool) or not self.smooth >= 0
              or not np.isfinite(self.smooth)):
            raise ValueError(f"smooth must be 'auto' or a non-negative float, got {self.smooth!r}")
        if self.target_type not in _TARGET_TYPES:
            raise ValueError(f'target_type must be one of {_TARGET_TYPES}, got {self.target_type!r}')
        if isinstance(self.categories, str):
            if self.categories != 'auto':
                raise ValueError(f"categories must be 'auto' or a list of arrays, got {self.categories!r}")
            return None
        if not isinstance(self.categories, list) or len(self.categories) != n_features:
            raise ValueError(f'categories must be a list with one array per feature ({n_features})')
        cats = []
        for i, c in enumerate(self.categories):
            c = np.asarray(c)
            if c.ndim != 1:
                raise ValueError(f'categories[{i}] must be 1-D')
            if c.dtype.kind in 'biuf':
                nan = np.isnan(c) if c.dtype.kind == 'f' else np.zeros(len(c), dtype=bool)
                if nan.any() and not (nan.sum() == 1 and nan[-1]):
                    raise ValueError(f'categories[{i}]: nan must be the last numerical category')
                body = c[~nan]
                if np.any(body[1:] < body[:-1]):
                    raise ValueError(f'categories[{i}]: unsorted categories are not supported for numerical categories')
            cats.append(c)
        return cats

    def _target(self, y):
        from sklearn.utils.multiclass import type_of_target
        inferred = type_of_target(y, input_name='y')
        if self.target_type == 'auto':
            if inferred not in ('binary', 'multiclass', 'continuous'):
                raise ValueError(f'y: the target type was inferred to be {inferred!r}; only binary, multiclass and '
                                 f'continuous targets are supported')
            ttype = inferred
        else:
            ttype = self.target_type
            if ttype == 'binary' and inferred != 'binary':
                raise ValueError(f"target_type='binary' does not fit y, whose type is {inferred!r}")
            if ttype == 'multiclass' and inferred != 'multiclass':
                raise ValueError(f"target_type='multiclass' does not fit y, whose type is {inferred!r}")
        if ttype == 'continuous':
            return ttype, None, None, _float_target(y, "target_type='continuous' does not fit y: y")
        from sklearn.preprocessing import LabelEncoder
        le = LabelEncoder()
        codes = le.fit_transform(y)
        return ttype, le.classes_, codes, None

    def _prepare(self, X, y):
        columns, names, n = split_columns(X)
        if not columns:
            raise ValueError('X has no columns')
        cats = self._check_params(len(columns))
        y = _check_y(y, n)
        ttype, classes, y_cls, y_float = self._target(y)
        return columns, names, n, cats, ttype, classes, y_cls, y_float, y

    def _fit_device(self, prep, fold, folds, transform, tile_rows, group_cols, workspace_bytes):
        columns, names, n, cats, ttype, classes, y_cls, y_float, _ = prep
        formula = TE_AUTO if self.smooth == 'auto' else TE_SMOOTH
        smooth = 0.0 if self.smooth == 'auto' else float(self.smooth)
        target = _Target(y_cls, 0 if classes is None else len(classes), y_float, fold, folds, formula, smooth,
                         tile_rows, True)
        all_cats, tables, prior, out, _ = cross_fit(columns, target, categories=cats, transform=transform,
                                                    group_cols=group_cols, workspace_bytes=workspace_bytes)
        self.categories_ = all_cats
        self.target_type_ = ttype
        self.classes_ = classes
        self.n_features_in_ = len(columns)
        if names is not None:
            self.feature_names_in_ = np.asarray(names, dtype=object)
        elif hasattr(self, 'feature_names_in_'):
            del self.feature_names_in_
        if ttype == 'multiclass':
            self.target_mean_ = prior[0].copy()
            self.encodings_ = [t[:, j].copy() for t in tables for j in range(len(classes))]
        else:
            self.target_mean_ = np.float64(prior[0, 0])
            self.encodings_ = [t[:, 0].copy() for t in tables]
        return out

    def fit(self, X, y, *, _tile_rows=_TILE_ROWS, _group_cols=None, _workspace_bytes=_WORKSPACE_BYTES):
        """Learn the categories and the encodings on all of X."""
        self._fit_device(self._prepare(X, y), None, 1, False, _tile_rows, _group_cols, _workspace_bytes)
        return self

    def fit_transform(self, X, y, *, _tile_rows=_TILE_ROWS, _group_cols=None, _workspace_bytes=_WORKSPACE_BYTES,
                      **split_params):
        """Fit on all of X, and encode X by cross fitting: the rows of each fold by the encodings of the other rows.
        split_params go to ``cv.split``."""
        from sklearn.model_selection import check_cv
        prep = self._prepare(X, y)
        y_raw = prep[-1]
        cv = check_cv(self.cv, y_raw, classifier=prep[4] != 'continuous', shuffle=self.shuffle,
                      random_state=self.random_state)
        fold, folds = fold_ids(cv.split(X, y_raw, **split_params), prep[2])
        out = self._fit_device(prep, fold, folds, True, _tile_rows, _group_cols, _workspace_bytes)
        return out.cpu().numpy()

    def transform(self, X, *, _group_cols=None, _workspace_bytes=_WORKSPACE_BYTES):
        """Encode X with the encodings learned on all of the fitted rows; unknown categories get ``target_mean_``."""
        if not hasattr(self, 'encodings_'):
            raise ValueError('this TargetEncoder is not fitted yet: call fit or fit_transform first')
        columns, names, n = split_columns(X)
        if len(columns) != self.n_features_in_:
            raise ValueError(f'X has {len(columns)} features, but TargetEncoder was fitted with {self.n_features_in_}')
        fitted = getattr(self, 'feature_names_in_', None)
        if fitted is not None and names is not None and list(names) != list(fitted):
            raise ValueError(f'X: the feature names {names} differ from those seen at fit {list(fitted)}')
        dev = _device()
        multi = self.target_type_ == 'multiclass'
        n_out = len(self.classes_) if multi else 1
        prior = torch.from_numpy(np.atleast_1d(np.asarray(self.target_mean_, dtype=np.float64))).to(dev)
        out = torch.empty((n, len(columns) * n_out), dtype=torch.float64, device=dev)
        pending = []

        def flush():
            if pending:
                gather(out, pending[0][0], [p[1] for p in pending], [p[2] for p in pending],
                       [len(p[3]) for p in pending], prior, None, n_out)
                pending.clear()

        for i, col in enumerate(columns):
            cats = self.categories_[i]
            codes, _ = code_column(col, cats)
            enc = np.stack(self.encodings_[i * n_out:(i + 1) * n_out], axis=1) if multi else self.encodings_[i][:, None]
            table = torch.from_numpy(np.ascontiguousarray(enc, dtype=np.float64).ravel()).to(dev)
            if pending and (len(pending) == _group_cols or sum(_group_bytes(n, len(p[3]), 1, n_out) for p in pending)
                            + _group_bytes(n, len(cats), 1, n_out) > _workspace_bytes):
                flush()
            pending.append((i, codes, table, cats))
        flush()
        return out.cpu().numpy()

    def get_feature_names_out(self, input_features=None):
        """The input names (``x0, x1, ...`` without names), each followed by ``_<class>`` on a multiclass target."""
        if not hasattr(self, 'n_features_in_'):
            raise ValueError('this TargetEncoder is not fitted yet')
        fitted = getattr(self, 'feature_names_in_', None)
        if input_features is None:
            names = list(fitted) if fitted is not None else [f'x{i}' for i in range(self.n_features_in_)]
        else:
            names = [str(f) for f in input_features]
            if len(names) != self.n_features_in_ or (fitted is not None and names != list(fitted)):
                raise ValueError('input_features do not match the fitted features')
        if self.target_type_ == 'multiclass':
            names = [f'{f}_{c}' for f in names for c in self.classes_]
        return np.asarray(names, dtype=object)


# ---- the reference's preprocessing.utils.target_encoding ---------------------------------------------------------

def target_encoding(train, target, test=None, feat_to_encode=None, smooth=0.2, random_state=9527, *,
                    _tile_rows=_TILE_ROWS, _group_cols=None):
    """The reference helper: sorts ``train`` by index in place and pops ``target`` from it, encodes each fold of
    ``StratifiedKFold(5, shuffle=True, random_state)`` by the other folds and ``test`` by all of ``train``, with
    category_encoders' formula (min_samples_leaf 20, smoothing ``smooth``; unseen and missing values get the prior).
    Returns ``(train_encoded, test_encoded, features, target)``."""
    from sklearn.model_selection import StratifiedKFold
    if not isinstance(smooth, numbers.Real) or isinstance(smooth, bool) or not smooth >= 0:
        raise ValueError(f'smooth must be a non-negative float, got {smooth!r}')
    if target not in train.columns:
        raise ValueError(f'target {target!r} is not a column of train')
    train.sort_index(inplace=True)
    y = train.pop(target)
    feats = train.columns.tolist() if feat_to_encode is None else list(feat_to_encode)
    missing = [f for f in feats if f not in train.columns]
    if not feats or missing:
        raise ValueError(f'feat_to_encode: {missing} are not columns of train')
    if test is not None and any(f not in test.columns for f in feats):
        raise ValueError(f'test lacks columns of feat_to_encode: {[f for f in feats if f not in test.columns]}')
    y_float = _float_target(y.to_numpy(), f'the target column {target!r}')
    if np.isnan(y_float).any():
        raise ValueError(f'the target column {target!r} contains NaN')
    skf = StratifiedKFold(n_splits=5, shuffle=True, random_state=random_state)
    fold, folds = fold_ids(skf.split(train, y), len(train), 'folds')
    tgt = _Target(None, 0, y_float, fold, folds, TE_RECALLED, smooth, _tile_rows, False)
    test_cols = [test[f] for f in feats] if test is not None else None
    _, _, _, out, test_out = cross_fit([train[f] for f in feats], tgt, missing_category=False,
                                       test_columns=test_cols, group_cols=_group_cols)
    enc = out.cpu().numpy()
    train_out = train.copy()
    for i, f in enumerate(feats):
        train_out[f] = enc[:, i]
    test_enc = None
    if test is not None:
        tenc = test_out.cpu().numpy()
        test_enc = test.copy()
        for i, f in enumerate(feats):
            test_enc[f] = tenc[:, i]
    return train_out, test_enc, list(train_out.columns), y
