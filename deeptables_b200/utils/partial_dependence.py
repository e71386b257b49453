"""Partial dependence (PD) and individual conditional expectation (ICE) of a fitted DeepTable, computed on the GPU.

``partial_dependence`` follows scikit-learn's ``sklearn.inspection.partial_dependence`` with ``method='brute'``
argument for argument and returns a Bunch with the same keys, shapes and order, so the result can be handed to
``PartialDependenceDisplay``.  The response is the positive class's probability on binary, one probability per class on
multiclass, one per label on multilabel, and the prediction on regression.

How it runs: X and the grid rows (one small frame with the feature columns set to each grid value) are encoded once by
the fitted preprocessor, so categories, unseen values, NaN imputation and scaling are exactly those of ``predict``.
``dtb_shap_compose`` then writes the rows of a range of grid points, row ``k*m + j`` being X row ``r0 + j`` with the
feature columns taken from grid point k; the quantile-bin and boosted-leaf columns are recomputed from the composed rows,
the inference forward runs over them in batches and ``dtb_pdp_block_sums`` reduces each grid point's outputs over fixed
blocks of ``_BLOCK_ROWS`` X rows into float64.  The host adds each grid point's blocks in index order and divides by the
sum of the weights, added in the same block order.  Chunks of rows start on block boundaries, so the result is the
same bits for any ``batch_size``.  No pandas work happens per grid point.

Data parallel: every rank calls with the same arguments; grid point g is computed on rank ``g % world``, the results
are all-gathered, and every rank returns what one process would.
"""
import numbers
import time
from collections.abc import Iterable

import numpy as np
import pandas as pd
import torch

from .. import _native as N, discrete
from .._native import check, ptr, stream_ptr
from ..analysis import Stages, check_positive_int, fitted_model, forward_rows, gather_strided, is_int, model_columns, \
    rank_share

_BLOCK_ROWS = 1024        # X rows per float64 block sum; chunks of rows start on multiples of it
_KINDS = ('average', 'individual', 'both')


def _as_frame(X, feature_names):
    if isinstance(X, pd.DataFrame):
        return X
    arr = np.asarray(X)
    if arr.ndim != 2:
        raise ValueError(f'X must be a DataFrame or a 2-D array, got an array of shape {arr.shape}')
    if feature_names is None or len(feature_names) != arr.shape[1]:
        raise ValueError('feature_names: a 2-D array X needs one name per column')
    return pd.DataFrame(arr, columns=list(feature_names)).infer_objects()


def _check_columns(dt_model, X):
    pre = dt_model.preprocessor
    got = [str(c) for c in X.columns]
    want = getattr(pre, 'feature_names_in_', None)
    if want is not None:
        if got != list(want):
            raise ValueError(f'X has columns {got}, the model was fitted on {list(want)}')
        return
    missing = [c for c in list(pre._cat_names) + list(pre._cont_names) if c not in got]
    if missing:
        raise ValueError(f'X lacks the columns {missing} the model was fitted on')


def feature_indices(columns, features):
    """Positions in ``columns`` of ``features`` (an int, a str, a bool mask, or a list of ints or of strs) and the key
    of each in ``custom_values`` (the element as given; the position for a mask)."""
    names = [str(c) for c in columns]

    def one(f):
        if is_int(f):
            if not 0 <= f < len(names):
                raise ValueError(f'features: index {f} is not in [0, {len(names) - 1}]')
            return int(f)
        if isinstance(f, str):
            if f not in names:
                raise ValueError(f'features: unknown feature name {f!r}')
            return names.index(f)
        raise ValueError(f'features: {f!r} is not an int, a str or a bool mask')

    if is_int(features) or isinstance(features, str):
        return [one(features)], [features]
    flist = list(features) if isinstance(features, Iterable) else [features]
    if not flist:
        raise ValueError('features: no feature given')
    if all(isinstance(f, (bool, np.bool_)) for f in flist):
        if len(flist) != len(names):
            raise ValueError(f'features: a bool mask needs {len(names)} entries, got {len(flist)}')
        idx = [int(i) for i in np.flatnonzero(flist)]
        if not idx:
            raise ValueError('features: the bool mask selects no feature')
        return idx, idx
    if not (all(is_int(f) for f in flist) or all(isinstance(f, str) for f in flist)):
        raise ValueError('features: a list of features holds ints or strs, not both')
    return [one(f) for f in flist], flist


def categorical_mask(columns, idx, categorical_features):
    """scikit-learn's ``is_categorical`` of the features at positions ``idx``."""
    if categorical_features is None:
        return [False] * len(idx)
    cf = np.asarray(categorical_features)
    if cf.size == 0:
        raise ValueError('categorical_features: an empty list is not supported; use None for no categorical feature')
    if cf.dtype.kind == 'b':
        if cf.size != len(columns):
            raise ValueError(f'categorical_features: a bool mask needs {len(columns)} entries, got {cf.size}')
        return [bool(cf[i]) for i in idx]
    if cf.dtype.kind in 'iOU':
        cat_idx, _ = feature_indices(columns, [int(c) if cf.dtype.kind == 'i' else c for c in cf.tolist()])
        return [i in cat_idx for i in idx]
    raise ValueError(f'categorical_features: expected bools, ints or strs, got {cf.dtype}')


def _check_percentiles(percentiles):
    if not isinstance(percentiles, Iterable) or isinstance(percentiles, str) or len(percentiles) != 2:
        raise ValueError('percentiles must be a sequence of 2 elements')
    if not all(isinstance(p, numbers.Real) and 0 <= p <= 1 for p in percentiles):
        raise ValueError('percentiles values must be in [0, 1]')
    if percentiles[0] >= percentiles[1]:
        raise ValueError('percentiles[0] must be strictly less than percentiles[1]')


def _check_grid_resolution(grid_resolution):
    if not is_int(grid_resolution) or grid_resolution <= 1:
        raise ValueError(f'grid_resolution must be an integer strictly greater than 1, got {grid_resolution!r}')


def grid_from_columns(columns, percentiles, is_categorical, grid_resolution, custom_values):
    """scikit-learn's ``_grid_from_X`` on a list of (name, Series): (grid [points, features], values per feature).

    A feature's axis is ``custom_values[i]`` if given, else the column's unique values when the feature is categorical
    or has fewer than ``grid_resolution`` of them, else ``grid_resolution`` points evenly spaced between the
    ``mquantiles`` of ``percentiles``.  Where scikit-learn fails inside ``mquantiles`` (a string column that needs the
    quantile branch) this raises ``ValueError`` naming the column."""
    from scipy.stats.mstats import mquantiles
    from sklearn.utils.extmath import cartesian
    _check_percentiles(percentiles)
    _check_grid_resolution(grid_resolution)

    def convert(v):
        return np.asarray(v, dtype=object if any(isinstance(x, str) for x in v) else None)

    custom = {k: convert(v) for k, v in custom_values.items()}
    bad = [f'Feature {k}: {v.ndim} dimensions' for k, v in custom.items() if v.ndim != 1]
    if bad:
        raise ValueError(f'custom_values: the custom grid for some features is not a one-dimensional array. '
                         f'{", ".join(bad)}')
    values = []
    for i, ((name, col), is_cat) in enumerate(zip(columns, is_categorical)):
        if i in custom:
            values.append(custom[i])
            continue
        try:
            uniques = np.unique(col)
        except TypeError as exc:
            raise ValueError(f'The column {name!r} contains mixed data types (np.nan together with str categories '
                             f'cannot be sorted into unique categories).') from exc
        if is_cat or uniques.shape[0] < grid_resolution:
            values.append(uniques)
            continue
        try:
            emp = mquantiles(col, prob=percentiles, axis=0)
        except (TypeError, ValueError) as exc:
            raise ValueError(f'The column {name!r} has {uniques.shape[0]} distinct non-numeric values, at least '
                             f'grid_resolution: list it in categorical_features') from exc
        if np.allclose(emp[0], emp[1]):
            raise ValueError('percentiles are too close to each other, unable to build the grid. Please choose '
                             'percentiles that are further apart.')
        values.append(np.linspace(emp[0], emp[1], num=grid_resolution, endpoint=True))
    return cartesian(values), values


def _check_weights(sample_weight, rows):
    if sample_weight is None:
        return None
    w = np.asarray(sample_weight, dtype=np.float64).reshape(-1)
    if len(w) != rows:
        raise ValueError(f'sample_weight has {len(w)} entries for {rows} rows of X')
    if not np.all(np.isfinite(w)) or np.any(w < 0):
        raise ValueError('sample_weight: weights must be finite and non-negative')
    if not w.sum() > 0:
        raise ValueError('sample_weight: the weights sum to 0')
    return w


def partial_dependence(dt_model, X, features, *, sample_weight=None, categorical_features=None, feature_names=None,
                       response_method='auto', percentiles=(0.05, 0.95), grid_resolution=100, custom_values=None,
                       method='auto', kind='average', batch_size=65536):
    """Partial dependence of the current model of ``dt_model`` on ``features``, over the rows of ``X``.

    ``X``: a DataFrame with the columns the model was fitted on, or a 2-D array of them with ``feature_names``.
    ``features``: an int, a str, a bool mask, or a list of ints or of strs; one call computes one PD over the joint grid
    of all of them (the cartesian product, first feature varying slowest).  The other arguments are scikit-learn's;
    ``custom_values`` is keyed by the elements of ``features`` as given (the column position for a bool mask).
    ``batch_size``: rows per forward call.

    Returns ``Bunch(grid_values=[one array per feature], average=..., individual=...)``, ``average`` of shape
    ``(n_outputs, *grid_shape)`` and ``individual`` ``(n_outputs, n_rows, *grid_shape)`` as ``kind`` asks.
    ``average`` is the weighted mean in float64 (scikit-learn gives float32 without ``sample_weight``);
    ``individual`` is float32."""
    return _partial_dependence(dt_model, X, features, sample_weight=sample_weight,
                               categorical_features=categorical_features, feature_names=feature_names,
                               response_method=response_method, percentiles=percentiles,
                               grid_resolution=grid_resolution, custom_values=custom_values, method=method, kind=kind,
                               batch_size=batch_size)


def _partial_dependence(dt_model, X, features, *, sample_weight, categorical_features, feature_names, response_method,
                        percentiles, grid_resolution, custom_values, method, kind, batch_size, stages=None):
    """``partial_dependence``; ``stages``: a dict that receives the seconds spent encoding X and the grid rows (host
    clock) and in compose, forward and reduce (CUDA events)."""
    from sklearn.utils import Bunch
    from .. import consts
    model = fitted_model(dt_model)
    regression = model.task == consts.TASK_REGRESSION
    if method == 'recursion':
        raise ValueError("method='recursion' needs a tree-based estimator; use method='brute' or 'auto'")
    if method not in ('auto', 'brute'):
        raise ValueError(f"method must be 'auto' or 'brute', got {method!r}")
    if response_method == 'decision_function':
        raise ValueError("response_method='decision_function': a DeepTable has no decision function")
    if response_method not in ('auto', 'predict_proba'):
        raise ValueError(f"response_method must be 'auto' or 'predict_proba', got {response_method!r}")
    if regression and response_method != 'auto':
        raise ValueError("response_method is ignored for regression and must be 'auto'")
    if kind not in _KINDS:
        raise ValueError(f'kind must be one of {_KINDS}, got {kind!r}')
    check_positive_int(batch_size, 'batch_size')
    if custom_values is not None and not isinstance(custom_values, dict):
        raise ValueError('custom_values must be a dict or None')
    _check_percentiles(percentiles)
    _check_grid_resolution(grid_resolution)
    X = _as_frame(X, feature_names)
    _check_columns(dt_model, X)
    if len(X) < 1:
        raise ValueError('X has no rows')
    weight = _check_weights(sample_weight, len(X))
    idx, keys = feature_indices(X.columns, features)
    is_cat = categorical_mask(X.columns, idx, categorical_features)
    for j, key, cat in zip(idx, keys, is_cat):
        if not cat and X.iloc[:, j].dtype.kind in 'iu':
            raise ValueError(f'features: the column {key!r} holds integer data; list it in categorical_features or '
                             f'convert it to float')
    custom = {i: custom_values[k] for i, k in enumerate(keys) if custom_values and k in custom_values}
    grid, values = grid_from_columns([(X.columns[j], X.iloc[:, j]) for j in idx], percentiles, is_cat,
                                     grid_resolution, custom)

    avg, ice = _device_pd(dt_model, model, X, idx, grid, weight, kind != 'average', batch_size, stages)
    shape = [len(v) for v in values]
    out = Bunch(grid_values=values)
    if kind in ('average', 'both'):
        out['average'] = avg.reshape(-1, *shape)
    if kind in ('individual', 'both'):
        out['individual'] = ice.reshape(-1, len(X), *shape)
    return out


def block_sums(pred, weight, groups, rows_per_group, out):
    """``dtb_pdp_block_sums`` of ``pred`` [groups*rows_per_group, cols] into the float64 device tensor ``out``
    (``groups * blocks * cols`` elements from its start)."""
    check(N.lib.dtb_pdp_block_sums(ptr(pred), ptr(weight), groups, rows_per_group, pred.shape[1], _BLOCK_ROWS,
                                   ptr(out), stream_ptr()), 'pdp_block_sums')


def add_blocks(sums):
    """float64 [groups, blocks, cols] -> [groups, cols]: each group's blocks added in index order."""
    acc = np.zeros((sums.shape[0], sums.shape[2]), np.float64)
    for b in range(sums.shape[1]):
        acc += sums[:, b]
    return acc


def _device_pd(dt_model, model, X, idx, grid, weight, individual, batch_size, stages):
    """(average float64 [cols, points], individual float32 [cols, rows, points] or None)."""
    dev, pre = model.device, dt_model.preprocessor
    n, G, cols = len(X), len(grid), model._output_dim()
    nb = (n + _BLOCK_ROWS - 1) // _BLOCK_ROWS
    timer = Stages(stages)
    t0 = time.perf_counter()
    model.flush_optimizer_state()       # every embedding row current: the forward needs no per-batch catch-up
    x_cat, x_cont = model._to_device_inputs(pre.transform_X(X))
    w_dev = torch.as_tensor(weight).to(dev) if weight is not None else None
    if weight is None:
        w_total = float(n)
    else:
        w_blocks = torch.empty(nb, dtype=torch.float64, device=dev)
        block_sums(torch.ones(n, 1, dtype=torch.float32, device=dev), w_dev, 1, n, w_blocks)
        w_total = float(add_blocks(w_blocks.cpu().numpy().reshape(1, nb, 1))[0, 0])

    names = {str(X.columns[j]) for j in idx}
    cat_names, cont_names = model_columns(model)
    cat_bit = [0 if c in names else -1 for c in cat_names]
    cont_bit = [0 if c in names else -1 for c in cont_names]

    if 0 not in cat_bit + cont_bit:
        # no feature column is read: every grid point's rows are X's own, so every point has X's mean
        pred = torch.empty(n, cols, dtype=torch.float32, device=dev)
        with timer.device('forward'):
            forward_rows(model, x_cat, x_cont, pred, batch_size)
        sums = torch.empty(nb * cols, dtype=torch.float64, device=dev)
        with timer.device('reduce'):
            block_sums(pred, w_dev, 1, n, sums)
        mean = add_blocks(sums.cpu().numpy().reshape(1, nb, cols))[0] / w_total
        timer.finish()
        avg = np.repeat(mean[:, None], G, axis=1)
        ice = np.repeat(pred.cpu().numpy().T[:, :, None], G, axis=2) if individual else None
        return avg, ice

    frame = X.iloc[np.zeros(G, np.intp)].reset_index(drop=True)
    for i, j in enumerate(idx):
        frame.isetitem(j, grid[:, i])
    g_cat, g_cont = model._to_device_inputs(pre.transform_X(frame))
    timer.host('encode', t0)
    cat_bit = torch.tensor(cat_bit, dtype=torch.int32, device=dev)
    cont_bit = torch.tensor(cont_bit, dtype=torch.int32, device=dev)

    mine = rank_share(G)
    cap = max(batch_size, _BLOCK_ROWS)
    if n <= cap:
        row_step, per = n, max(1, cap // n)            # all rows of X, several grid points per chunk
    else:
        row_step, per = cap // _BLOCK_ROWS * _BLOCK_ROWS, 1
    F = x_cat.shape[1] if x_cat is not None else 0
    C = x_cont.shape[1] if x_cont is not None else 0
    buf_rows = per * row_step
    out_cat = torch.empty(buf_rows, F, dtype=torch.int32, device=dev) if F else None
    out_cont = torch.empty(buf_rows, C, dtype=torch.float32, device=dev) if C else None
    pred = torch.empty(buf_rows, cols, dtype=torch.float32, device=dev)
    masks = torch.ones(per, dtype=torch.int32, device=dev)          # one mask word per grid point: bit 0
    index = torch.as_tensor(np.array(mine, np.int32)).to(dev)
    sums = torch.empty(len(mine) * nb * cols, dtype=torch.float64, device=dev)
    ice = np.empty((cols, n, len(mine)), np.float32) if individual else None

    for i0 in range(0, len(mine), per):
        k = min(per, len(mine) - i0)
        for r0 in range(0, n, row_step):
            m = min(row_step, n - r0)
            rows = k * m
            with timer.device('compose'):
                check(N.lib.dtb_shap_compose(ptr(g_cat), ptr(g_cont), ptr(x_cat[r0:] if F else None),
                                             ptr(x_cont[r0:] if C else None), ptr(masks), 1, ptr(index[i0:]),
                                             ptr(cat_bit), ptr(cont_bit), k, m, F, C, ptr(out_cat), ptr(out_cont),
                                             stream_ptr()), 'shap_compose')
                discrete.rewrite_derived(pre, out_cat[:rows] if F else None, out_cont[:rows] if C else None)
            with timer.device('forward'):
                forward_rows(model, out_cat, out_cont, pred[:rows], batch_size)
            with timer.device('reduce'):
                block_sums(pred[:rows], w_dev[r0:] if w_dev is not None else None, k, m,
                           sums[(i0 * nb + r0 // _BLOCK_ROWS) * cols:])
            if individual:
                ice[:, r0:r0 + m, i0:i0 + k] = pred[:rows].view(k, m, cols).permute(2, 1, 0).cpu().numpy()

    avg_mine = (add_blocks(sums.cpu().numpy().reshape(len(mine), nb, cols)) / w_total).T       # [cols, mine]
    timer.finish()
    return gather_strided(avg_mine, G, 1), gather_strided(ice, G, 2) if individual else None
