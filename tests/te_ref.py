"""Numpy float64 restatement of target encoding (deeptables_b200/target_encoding.py).

- scikit-learn 1.9's TargetEncoder: the float-smooth and 'auto' formulas of sklearn/preprocessing/_target_encoder_fast.pyx,
  one-vs-rest indicators for multiclass targets, and the cross fitting of ``fit_transform``.  Pinned against the
  installed scikit-learn by tests/test_target_encoding_cpu.py.
- The reference helper preprocessing.utils.target_encoding, whose formula is category_encoders' TargetEncoder AS
  RECALLED (that package is not installed, so this branch is not pinned against it).
"""
import numpy as np
import pandas as pd

MIN_SAMPLES_LEAF = 20


def _is_nan(v):
    return isinstance(v, (float, np.floating)) and v != v


def codes_of(values, cats):
    """Index of each value in cats (None and NaN are values of their own), -1 when absent."""
    lut, nan_pos = {}, -1
    for i, c in enumerate(cats):
        if _is_nan(c):
            nan_pos = i
        else:
            lut.setdefault(c, i)
    return np.array([nan_pos if _is_nan(v) else lut.get(v, -1) for v in values], dtype=np.int64)


def indicators(y, target_type, classes=None):
    """[rows, n_out] float64 columns that are encoded: the class-1 indicator (binary), one indicator per class
    (multiclass) or the target (continuous)."""
    if target_type == 'continuous':
        return np.asarray(y, dtype=np.float64)[:, None]
    idx = np.searchsorted(classes, y)
    if target_type == 'binary':
        return (idx == 1).astype(np.float64)[:, None]
    return (idx[:, None] == np.arange(len(classes))[None, :]).astype(np.float64)


def encode_one(codes, y, V, smooth, prior, formula='sklearn'):
    """Encodings [V] of one column from the fitting rows (codes -1 do not count toward any category)."""
    k = codes >= 0
    c, yk = codes[k], y[k]
    n = np.bincount(c, minlength=V).astype(np.float64)
    S = np.bincount(c, weights=yk, minlength=V)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        if formula == 'recalled':
            s = 1.0 / (1.0 + np.exp(-(n - MIN_SAMPLES_LEAF) / smooth))
            return np.where(n == 0, prior, prior * (1 - s) + (S / n) * s)
        if smooth == 'auto':
            var = np.var(y)
            m = S / n
            ssd = np.bincount(c, weights=(yk - m[c]) ** 2, minlength=V)
            lam = var * n / (var * n + ssd / n)
            return np.where(np.isnan(lam), prior, lam * m + (1 - lam) * prior)
        den = smooth + n
        return np.where(den == 0, prior, (smooth * prior + S) / den)


def fit(codes, Y, Vs, smooth, formula='sklearn'):
    """encodings_ (feature-major: f0_c0, f0_c1, ...) and the target mean of all rows.  codes [rows, F], Y [rows, n_out].
    scikit-learn fits the rows outside given categories (code -1) as the first category; the recalled formula counts
    them toward none."""
    prior = Y.mean(axis=0)
    if formula == 'sklearn':
        codes = np.maximum(codes, 0)
    encs = [encode_one(codes[:, f], Y[:, j], Vs[f], smooth, prior[j], formula)
            for f in range(codes.shape[1]) for j in range(Y.shape[1])]
    return encs, prior


def transform(codes, encs, prior):
    n_out = len(prior)
    out = np.empty((codes.shape[0], codes.shape[1] * n_out))
    for f in range(codes.shape[1]):
        for j in range(n_out):
            e = encs[f * n_out + j]
            c = codes[:, f]
            out[:, f * n_out + j] = np.where(c >= 0, e[np.maximum(c, 0)], prior[j])
    return out


def cross_fit(codes, Y, Vs, fold, smooth, formula='sklearn'):
    """fit_transform's output: the rows of fold f encoded by a fit on the rows outside f.  scikit-learn then sets every
    row outside given categories, in any fold, to the mean of each fold's fitting rows in turn: the last fold's stays."""
    out = np.empty((codes.shape[0], codes.shape[1] * Y.shape[1]))
    n_out = Y.shape[1]
    for f in np.unique(fold):
        tr, te = fold != f, fold == f
        encs, prior = fit(codes[tr], Y[tr], Vs, smooth, formula)
        out[te] = transform(codes[te], encs, prior)
        if formula == 'sklearn':
            for c in range(codes.shape[1]):
                out[codes[:, c] < 0, c * n_out:(c + 1) * n_out] = prior
    return out


def fold_ids(splits, n):
    fold = np.full(n, -1, dtype=np.int64)
    for k, (_, te) in enumerate(splits):
        fold[te] = k
    return fold


def target_encoding(train, target, test=None, feat_to_encode=None, smooth=0.2, random_state=9527):
    """The reference helper with the recalled formula: missing values are no category and get the prior."""
    from sklearn.model_selection import StratifiedKFold
    train.sort_index(inplace=True)
    y_ser = train.pop(target)
    feats = train.columns.tolist() if feat_to_encode is None else list(feat_to_encode)
    y = y_ser.to_numpy(dtype=np.float64)[:, None]
    cats = [pd.unique(train[f].dropna().to_numpy()) for f in feats]
    codes = np.stack([codes_of(train[f].to_numpy(), c) for f, c in zip(feats, cats)], axis=1)
    Vs = [len(c) for c in cats]
    fold = fold_ids(StratifiedKFold(n_splits=5, shuffle=True, random_state=random_state).split(train, y_ser),
                    len(train))
    enc = cross_fit(codes, y, Vs, fold, smooth, 'recalled')
    out = train.copy()
    for i, f in enumerate(feats):
        out[f] = enc[:, i]
    test_out = None
    if test is not None:
        encs, prior = fit(codes, y, Vs, smooth, 'recalled')
        tcodes = np.stack([codes_of(test[f].to_numpy(), c) for f, c in zip(feats, cats)], axis=1)
        tenc = transform(tcodes, encs, prior)
        test_out = test.copy()
        for i, f in enumerate(feats):
            test_out[f] = tenc[:, i]
    return out, test_out, list(out.columns), y_ser
