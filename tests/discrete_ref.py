"""The scikit-learn oracle of auto_discrete, and a host stand-in for the device parts of MultiKBinsDiscretizer so that
the preprocessor's plumbing can be tested without a GPU."""
import warnings

import numpy as np


def n_bins(col32):
    """hypernets' bin count on the float32 values the model reads (NaN excluded)."""
    v = np.asarray(col32, np.float32)
    return max(len(np.unique(v[~np.isnan(v)])) // 10, 2)


def kbins(col32, nb):
    """scikit-learn's fitted discretiser on the float64 widening of one float32 column, every row used."""
    from sklearn.preprocessing import KBinsDiscretizer
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')         # constant feature / narrow bins removed
        return KBinsDiscretizer(nb, encode='ordinal', strategy='quantile', quantile_method='averaged_inverted_cdf',
                                subsample=None).fit(np.asarray(col32, np.float32).astype(np.float64)[:, None])


def edges(col32, nb=None):
    return kbins(col32, n_bins(col32) if nb is None else nb).bin_edges_[0]


def codes(bin_edges, x32):
    """KBinsDiscretizer.transform's ordinal codes, as int32."""
    return np.searchsorted(bin_edges[1:-1], np.asarray(x32, np.float32).astype(np.float64), side='right').astype(
        np.int32)


def host_edges(col32, nb=None):
    """The discretiser's host arithmetic fed a numpy-sorted column instead of the device's sorted block."""
    from deeptables_b200 import discrete as D
    s = np.sort(np.asarray(col32, np.float32) + np.float32(0.0)).astype(np.float64)
    nunique = len(np.unique(s))
    nb = D.n_bins_for(nunique) if nb is None else nb
    prev, nxt, gamma = D.quantile_plan(len(s), nb)
    return nb, D.edges_from_order_stats(s[prev], s[nxt], gamma, nunique == 1)


def patch_host(monkeypatch):
    """Run MultiKBinsDiscretizer's fit and codes on the host (scikit-learn), for tests without a device."""
    from deeptables_b200 import discrete as D

    def _fit(self, arr):
        nbs = np.array([n_bins(arr[:, j]) for j in range(arr.shape[1])], np.int64)
        return nbs, [edges(arr[:, j], int(nb)) for j, nb in enumerate(nbs)]

    def _codes(self, X):
        arr = self._block(X, 'transform')
        return np.stack([codes(e, arr[:, j]) for j, e in enumerate(self.bin_edges)], 1).reshape(len(X), -1)

    monkeypatch.setattr(D.MultiKBinsDiscretizer, '_fit', _fit)
    monkeypatch.setattr(D.MultiKBinsDiscretizer, 'codes', _codes)
