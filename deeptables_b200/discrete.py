"""Quantile-bin discretisation of the continuous columns (``ModelConfig.auto_discrete``; reference preprocessor.py:406-415).

The reference fits hypernets' ``MultiKBinsDiscretizer`` on every continuous column after imputation, scaling and label
encoding, and appends one ``CategoricalColumn`` per continuous column, ``<col>_discrete``, with vocabulary
``n_bins + 1``; the continuous columns stay as they are.  hypernets is not needed here, and the encoder is restated
as recalled (the ``'_discrete'`` suffix is confirmed by the reference's utils/consts.py):

- ``n_bins = max(nunique // 10, 2)`` per column, NaN excluded;
- scikit-learn's ``KBinsDiscretizer(n_bins, encode='ordinal', strategy='quantile')``: edges are
  ``np.percentile(col, linspace(0, 100, n_bins + 1), method='averaged_inverted_cdf')``, bins of width <= 1e-8 are
  removed, a constant column gets edges ``[-inf, inf]``, and the code of x is
  ``np.searchsorted(edges[1:-1], x, side='right')``;
- the vocabulary is the requested ``n_bins + 1`` even when narrow bins were removed.

The values binned are the float32 values the model reads (DefaultPreprocessor._encode), widened to float64.  Unlike the
reference, every row is used: scikit-learn's default draws a random subsample of 200 000 rows with replacement, so
above that size the reference's bins change from run to run.

The fit sorts the ``[columns, rows]`` block once on the device, counts the distinct values from it and gathers only
the order statistics the quantiles read; the interpolation is numpy's, in float64 on the host.  ``dtb_discretize``
writes the codes, for ``transform`` and for the device rewrites of permutation importance and SHAP.
"""
import numpy as np
import torch

from . import _native as N, dp
from ._native import check, ptr, stream_ptr

SUFFIX = '_discrete'


def n_bins_for(nunique):
    """hypernets' bin count of a column with ``nunique`` distinct values, as recalled."""
    return max(int(nunique) // 10, 2)


def quantile_plan(n, n_bins):
    """What ``np.percentile(v, np.linspace(0, 100, n_bins + 1), method='averaged_inverted_cdf')`` reads of ``n`` sorted
    values: (prev, next) positions in ``[0, n)`` and the weight gamma of each level, by numpy's own arithmetic
    (the virtual index ``n*q - 1``, ``_get_indexes``'s clipping, gamma 0.5 where the index is integral, else 1)."""
    q = np.true_divide(np.linspace(0, 100, n_bins + 1), np.float64(100))
    vi = n * q - 1
    prev = np.floor(vi)
    nxt = prev + 1
    above, below = vi >= n - 1, vi < 0
    prev[above] = nxt[above] = -1
    prev[below] = nxt[below] = 0
    prev, nxt = prev.astype(np.intp), nxt.astype(np.intp)
    gamma = np.where(vi - prev == 0, 0.5, 1.0)
    return prev % n, nxt % n, gamma


def lerp(a, b, gamma):
    """numpy's ``_lerp`` for gamma >= 0.5: ``b - (b - a) * (1 - gamma)``, float64."""
    return b - (b - a) * (1 - gamma)


def edges_from_order_stats(prev_values, next_values, gamma, constant):
    """The bin edges of one column after KBinsDiscretizer's width filter, from the float64 order statistics."""
    if constant:
        return np.array([-np.inf, np.inf])
    edges = lerp(np.asarray(prev_values, np.float64), np.asarray(next_values, np.float64), gamma)
    return edges[np.ediff1d(edges, to_begin=np.inf) > 1e-8]


def check_finite(finite, columns, where):
    bad = [c for c, ok in zip(columns, finite) if not ok]
    if bad:
        raise ValueError(f'auto_discrete: column(s) {bad} hold NaN or infinite values at {where}; the bins take finite '
                         f'values only (turn auto_imputation on, or clean the column)')


class MultiKBinsDiscretizer:
    """hypernets' ``MultiKBinsDiscretizer`` over the continuous columns ``columns`` of the encoded frame: one ordinal
    quantile-bin code per column, in the new column ``<col>_discrete``.  Holds only numpy arrays, so it pickles with the
    preprocessor."""

    def __init__(self, columns):
        self.columns = list(columns)
        self.new_columns = [f'{c}{SUFFIX}' for c in self.columns]
        self.n_bins = self.bin_edges = None

    @staticmethod
    def check_names(X, columns):
        """Refuse a frame that already has ``<col>_discrete`` for a continuous column ``col``."""
        stems = set(str(c) for c in columns)
        clash = [c for c in X.columns if str(c).endswith(SUFFIX) and str(c)[:-len(SUFFIX)] in stems]
        if clash:
            raise ValueError(f'auto_discrete: the frame already has discretised column names {clash}')

    @property
    def vocabulary_sizes(self):
        return [int(b) + 1 for b in self.n_bins]

    def _block(self, X, where):
        """The float32 ``[rows, columns]`` block of the encoded frame, checked finite (``where``: 'fit' or
        'transform', for the message)."""
        arr = np.require(X[self.columns].to_numpy(np.float32), requirements=['C', 'W'])
        check_finite(np.isfinite(arr).all(axis=0), self.columns, where)
        return arr

    def fit(self, X):
        if len(X) < 1:
            raise ValueError('auto_discrete: the frame has no rows')
        arr = self._block(X, 'fit')
        if dp.is_distributed():
            box = [None]
            if torch.distributed.get_rank() == 0:
                box = [self._fit(arr)]
            torch.distributed.broadcast_object_list(box, src=0)
            self.n_bins, self.bin_edges = box[0]
        else:
            self.n_bins, self.bin_edges = self._fit(arr)
        self._stage()
        return self

    def _fit(self, arr):
        rows = len(arr)
        block = torch.as_tensor(arr).cuda().t().contiguous()     # [C, rows]
        block += 0.0                                              # -0.0 -> 0.0: one value, as the comparisons see it
        s = torch.sort(block, dim=1).values
        nunique = ((s[:, 1:] != s[:, :-1]).sum(dim=1) + 1).cpu().numpy()
        n_bins = np.array([n_bins_for(u) for u in nunique], np.int64)
        plans = [quantile_plan(rows, int(b)) for b in n_bins]
        flat = np.concatenate([np.concatenate([p[0], p[1]]) + j * rows for j, p in enumerate(plans)])
        stats = s.view(-1)[torch.as_tensor(flat).to(s.device)].cpu().numpy().astype(np.float64)
        edges, at = [], 0
        for j, (prev, _, gamma) in enumerate(plans):
            k = len(prev)
            edges.append(edges_from_order_stats(stats[at:at + k], stats[at + k:at + 2 * k], gamma, nunique[j] == 1))
            at += 2 * k
        return n_bins, edges

    def _stage(self):
        """The inner edges, flat, as the kernel reads them."""
        inner = [e[1:-1] for e in self.bin_edges]
        self._edge_off = np.concatenate([[0], np.cumsum([len(e) for e in inner])]).astype(np.int64)
        self._edges = np.concatenate(inner + [np.zeros(1)]).astype(np.float64)
        self._device = None

    def _device_arrays(self, device):
        if self._device is None or self._device[0].device != device:
            self._device = tuple(torch.as_tensor(a).to(device) for a in
                                 (self._edges, self._edge_off, np.arange(len(self.columns), dtype=np.int32)))
        return self._device

    def __getstate__(self):
        state = dict(self.__dict__)
        state['_device'] = None
        return state

    def write_device(self, cat, cont, out_col):
        """``dtb_discretize``: the codes of the first ``len(columns)`` columns of the device tensor ``cont`` [rows, *]
        (the continuous columns, in order) into columns ``out_col ..`` of ``cat`` [rows, *] (int32)."""
        if cont.shape[0] == 0:
            return
        edges, edge_off, src_col = self._device_arrays(cont.device)
        check(N.lib.dtb_discretize(ptr(cont), cont.shape[1], cont.shape[0], ptr(src_col), ptr(edges), ptr(edge_off),
                                   len(self.columns), ptr(cat), cat.shape[1], out_col, stream_ptr()),
              'discretize')

    def codes(self, X):
        """int32 [rows, columns]: the bin codes of the encoded frame X."""
        cont = torch.as_tensor(self._block(X, 'transform')).cuda()
        out = torch.empty(len(X), len(self.columns), dtype=torch.int32, device=cont.device)
        self.write_device(out, cont, 0)
        return out.cpu().numpy()

    def transform(self, X):
        import pandas as pd
        extra = pd.DataFrame(self.codes(X), columns=self.new_columns, index=X.index)
        return pd.concat([X, extra], axis=1)

    def fit_transform(self, X):
        return self.fit(X).transform(X)

def rewrite_derived(preprocessor, cat, cont):
    """After an input column of the model's device inputs changed (permutation importance, SHAP coalitions): recompute
    the columns derived from the raw ones, the discretised columns first and then the gradient-boosted leaf columns,
    which may read them.  Nothing to do without either option."""
    from . import gbm
    disc = getattr(preprocessor, 'discretizer_', None)
    if disc is not None:
        disc.write_device(cat, cont, len(preprocessor._cat_names))
    gbm.rewrite_leaves(preprocessor, cat, cont)
