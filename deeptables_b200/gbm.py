"""Gradient-boosted leaf features (``ModelConfig.apply_gbm_features``; reference preprocessor.py:431-452).

The reference fits hypernets' ``LgbmLeavesEncoder`` (a LightGBM model) on the encoded frame and appends each tree's
leaf index as a new column.  LightGBM is not needed here: this module grows the trees itself, on the GPU
(csrc/gbdt.cu), with LightGBM's ``gbdt`` algorithm at its sklearn defaults restated:

- bins: at most ``max_bin`` per feature, edges from at most ``subsample_for_bin`` seeded sample rows (``bin_edges``);
  a row goes left of edge e when ``x <= e``, NaN always right;
- gradients of the binary log loss, L2 or the softmax, turned into int64 fixed point with a power-of-two scale chosen
  per tree so that no sum over the rows reaches 2^62; histograms are integer sums, the larger child is the parent
  minus the smaller one;
- splits by the regularised gain in float64, leaf-wise growth up to ``num_leaves`` (ties to the lowest leaf), leaf
  numbering as LightGBM's ``pred_leaf`` (the left child keeps the parent's index, the right one takes the next);
- leaf values ``-learning_rate * T(G) / (H + lambda)`` in float32.

A given frame and set of parameters gives the same trees, bit for bit.  The trees are this project's own: they are
not claimed to be LightGBM's bits.
"""
import ctypes
import math
import numbers

import numpy as np
import torch

from . import _native as N, consts, dp
from ._native import check, ptr, stream_ptr
from .analysis import Stages, is_int

LEAF_PREFIX = 'lgbm_leaf_'       # hypernets' column naming, as recalled

_DEFAULTS = {'n_estimators': 100, 'num_leaves': 31, 'max_depth': -1, 'learning_rate': 0.1, 'min_child_samples': 20,
             'min_child_weight': 1e-3, 'reg_lambda': 0.0, 'reg_alpha': 0.0, 'min_split_gain': 0.0, 'max_bin': 255,
             'subsample_for_bin': 200000, 'random_state': None}
_ALIASES = {'num_iterations': 'n_estimators', 'min_data_in_leaf': 'min_child_samples',
            'min_sum_hessian_in_leaf': 'min_child_weight', 'lambda_l2': 'reg_lambda', 'lambda_l1': 'reg_alpha',
            'seed': 'random_state'}
_IGNORED = ('n_jobs', 'verbose', 'verbosity')
# LightGBM's defaults for options that are not built: accepted only at these values
_NEUTRAL = {'boosting_type': 'gbdt', 'boosting': 'gbdt', 'subsample': 1.0, 'bagging_fraction': 1.0,
            'subsample_freq': 0, 'bagging_freq': 0, 'colsample_bytree': 1.0, 'feature_fraction': 1.0}
MAX_LEAVES = N.GBDT_STAGE_NODES + 1


def _is_real(v):
    return isinstance(v, numbers.Real) and not isinstance(v, bool) and math.isfinite(v)


def resolve_params(gbm_params, task, num_classes=None):
    """``ModelConfig.gbm_params`` -> a dict of every parameter of ``_DEFAULTS``.  LightGBM's sklearn names and their
    aliases are accepted; ``n_jobs``, ``verbose`` and ``verbosity`` are ignored; anything else raises
    ``NotImplementedError`` naming it, and an out-of-range value ``ValueError``."""
    out, given = dict(_DEFAULTS), set()
    for key, value in dict(gbm_params or {}).items():
        if key in _IGNORED:
            continue
        if key in _NEUTRAL:
            if value != _NEUTRAL[key]:
                raise NotImplementedError(f'gbm_params[{key!r}] = {value!r}: only gbdt without bagging or feature '
                                          f'sampling is built (the default {_NEUTRAL[key]!r} is accepted)')
            continue
        name = _ALIASES.get(key, key)
        if name not in _DEFAULTS:
            raise NotImplementedError(f'gbm_params[{key!r}] is not supported by the built-in booster')
        if name in given:
            raise ValueError(f'gbm_params sets {name!r} twice (through an alias)')
        given.add(name)
        out[name] = value
    ints = {'n_estimators': 1, 'num_leaves': 2, 'min_child_samples': 0, 'subsample_for_bin': 1}
    for name, lo in ints.items():
        if not is_int(out[name]) or out[name] < lo:
            raise ValueError(f'gbm_params {name!r} must be an integer >= {lo}, got {out[name]!r}')
    if out['num_leaves'] > MAX_LEAVES:
        raise ValueError(f'gbm_params num_leaves must be at most {MAX_LEAVES}, got {out["num_leaves"]}')
    if not is_int(out['max_depth']):
        raise ValueError(f'gbm_params max_depth must be an integer (<= 0: no limit), got {out["max_depth"]!r}')
    if not is_int(out['max_bin']) or out['max_bin'] < 2:
        raise ValueError(f'gbm_params max_bin must be an integer >= 2, got {out["max_bin"]!r}')
    if out['max_bin'] > 255:
        raise NotImplementedError(f'gbm_params max_bin = {out["max_bin"]}: bins are uint8, at most 255 are built')
    if not _is_real(out['learning_rate']) or out['learning_rate'] <= 0:
        raise ValueError(f'gbm_params learning_rate must be a positive number, got {out["learning_rate"]!r}')
    for name in ('min_child_weight', 'reg_lambda', 'reg_alpha', 'min_split_gain'):
        if not _is_real(out[name]) or out[name] < 0:
            raise ValueError(f'gbm_params {name!r} must be a finite number >= 0, got {out[name]!r}')
        out[name] = float(out[name])
    out['learning_rate'] = float(out['learning_rate'])
    rs = out['random_state']
    if rs is not None and (not is_int(rs) or not 0 <= rs < 2 ** 32):
        raise ValueError(f'gbm_params random_state must be None or an integer in [0, 2**32), got {rs!r}')
    if task == consts.TASK_MULTICLASS and 'n_estimators' not in given:
        out['n_estimators'] = int(100 / num_classes) + 1      # hypernets' encoder, as recalled
    return out


def sample_rows(rows, subsample_for_bin, random_state):
    """Sorted row numbers the bin edges are computed from: all rows, or a seeded choice without replacement."""
    if rows <= subsample_for_bin:
        return np.arange(rows)
    rng = np.random.RandomState(1 if random_state is None else random_state)
    return np.sort(rng.choice(rows, subsample_for_bin, replace=False))


def _midpoints(lo, hi):
    """float32 midpoints of neighbouring distinct float32 values, set to ``lo`` where rounding reaches ``hi``."""
    e = ((lo.astype(np.float64) + hi.astype(np.float64)) / 2).astype(np.float32)
    return np.where(e >= hi, lo, e).astype(np.float32)


def bin_edges(values, max_bin):
    """Increasing float32 edges (at most ``max_bin - 1``) of one feature from its sampled float32 values.  One bin per
    distinct value when there are at most ``max_bin`` of them; otherwise edges at the gaps where the cumulative count
    first reaches each ``k / max_bin`` quantile.  NaN is ignored (it falls in the last bin)."""
    v = np.asarray(values, np.float32)
    v = v[~np.isnan(v)]
    u, counts = np.unique(v, return_counts=True)
    if len(u) <= 1:
        return np.zeros(0, np.float32)
    if len(u) <= max_bin:
        return _midpoints(u[:-1], u[1:])
    cum = np.cumsum(counts)
    targets = np.arange(1, max_bin) * (cum[-1] / max_bin)
    cut = np.unique(np.searchsorted(cum, targets, side='left'))
    cut = cut[cut < len(u) - 1]
    return _midpoints(u[cut], u[cut + 1])


def fixed_shift(max_abs, rows):
    """Power of two for the fixed point: ``rows * max_abs * 2^shift <= 2^62`` (0 when every value is 0)."""
    if not max_abs > 0:
        return 0
    _, e = math.frexp(float(max_abs))            # max_abs < 2^e
    return 62 - (int(rows) - 1).bit_length() - e


def init_scores(y, task, num_classes):
    """LightGBM's boost-from-average starting scores (float64 [K])."""
    if task == consts.TASK_REGRESSION:
        return np.array([np.mean(y.astype(np.float64))])
    if task == consts.TASK_BINARY:
        p = min(max(float(np.mean(y.astype(np.float64))), 1e-15), 1 - 1e-15)
        return np.array([math.log(p / (1 - p))])
    prior = np.bincount(y.astype(np.int64), minlength=num_classes) / len(y)
    return np.log(np.maximum(prior, 1e-15))


def leaf_value(g, h, shift_g, shift_h, p):
    """float32 leaf output from the leaf's integer sums."""
    G, H = float(g) * 2.0 ** -shift_g, float(h) * 2.0 ** -shift_h
    a = p['reg_alpha']
    t = G - a if G > a else (G + a if G < -a else 0.0)
    return np.float32(-p['learning_rate'] * (t / (H + p['reg_lambda'])))


class Trees:
    """A fitted booster as flat numpy arrays.  Tree t owns nodes ``node_off[t] .. node_off[t+1]`` and leaves
    ``leaf_off[t] .. leaf_off[t+1]``; a child >= 0 is a node of the same tree, a child < 0 the leaf ``~child``."""

    def __init__(self, node_feature, node_bin, node_threshold, node_left, node_right, node_gain, node_off, leaf_value,
                 leaf_off):
        self.node_feature = np.asarray(node_feature, np.int32)
        self.node_gain = np.asarray(node_gain, np.float64)
        self.node_bin = np.asarray(node_bin, np.int32)
        self.node_threshold = np.asarray(node_threshold, np.float32)
        self.node_left = np.asarray(node_left, np.int32)
        self.node_right = np.asarray(node_right, np.int32)
        self.node_off = np.asarray(node_off, np.int32)
        self.leaf_value = np.asarray(leaf_value, np.float32)
        self.leaf_off = np.asarray(leaf_off, np.int32)

    @property
    def n_trees(self):
        return len(self.node_off) - 1

    @property
    def num_leaves(self):
        return np.diff(self.leaf_off)

    def arrays(self):
        return {k: v for k, v in vars(self).items()}


def _trees_from_lists(trees):
    nf, nb, nt, nl, nr, ng, lv = [], [], [], [], [], [], []
    node_off, leaf_off = [0], [0]
    for t in trees:
        for key, dst in (('feature', nf), ('bin', nb), ('threshold', nt), ('left', nl), ('right', nr), ('gain', ng)):
            dst.extend(t[key])
        lv.extend(t['values'])
        node_off.append(node_off[-1] + len(t['feature']))
        leaf_off.append(leaf_off[-1] + len(t['values']))
    return Trees(nf, nb, nt, nl, nr, ng, node_off, lv, leaf_off)


class Booster:
    """Grows the trees on the device from the model's own input tensors.  ``feat_col[i]``: column c >= 0 of ``cat`` or
    ``-1 - c`` of ``cont``; ``edges[i]``: the feature's float32 bin edges."""

    def __init__(self, params, task, num_classes, feat_col, edges, device):
        self.p, self.task, self.device = params, task, device
        self.K = num_classes if task == consts.TASK_MULTICLASS else 1
        self.objective = {consts.TASK_BINARY: N.GBDT_BINARY, consts.TASK_REGRESSION: N.GBDT_L2}.get(
            task, N.GBDT_SOFTMAX)
        self.nf = len(edges)
        self.n_bins = np.array([len(e) + 1 for e in edges], np.int32)
        self.nb = int(self.n_bins.max())
        self.edges = [np.asarray(e, np.float32) for e in edges]
        off = np.concatenate([[0], np.cumsum([len(e) for e in edges])]).astype(np.int32)
        flat = np.concatenate(self.edges + [np.zeros(1, np.float32)])
        self.feat_col_d = torch.as_tensor(np.asarray(feat_col, np.int32)).to(device)
        self.edges_d = torch.as_tensor(flat).to(device)
        self.edge_off_d = torch.as_tensor(off).to(device)
        self.n_bins_d = torch.as_tensor(self.n_bins).to(device)

    def bin(self, cat, cont, rows):
        bins = torch.empty(rows, self.nf, dtype=torch.uint8, device=self.device)
        check(N.lib.dtb_gbdt_bin(ptr(cat), cat.shape[1] if cat is not None else 0, ptr(cont),
                                 cont.shape[1] if cont is not None else 0, ptr(self.feat_col_d), ptr(self.edges_d),
                                 ptr(self.edge_off_d), rows, self.nf, ptr(bins), stream_ptr()), 'gbdt_bin')
        return bins

    def fit(self, cat, cont, label, leaf_log=None, stages=None):
        """Trees fitted to ``label`` (numpy: 0/1, the target, or class codes).  ``leaf_log``: an int32 [rows, trees]
        device tensor, or None; it receives each training row's leaf from the partition, tree by tree.  ``stages``: a
        dict that receives the seconds spent in bin, grad, hist, split, partition and update (CUDA events)."""
        p, K, dev = self.p, self.K, self.device
        rows = len(label)
        if rows >= 2 ** 31:
            raise ValueError('the booster takes fewer than 2**31 rows')
        timer = Stages(stages)
        with timer.device('bin'):
            bins = self.bin(cat, cont, rows)
        y = torch.as_tensor(np.asarray(label, np.float32)).to(dev)
        scores = torch.empty(rows, K, dtype=torch.float64, device=dev)
        scores[:] = torch.as_tensor(init_scores(np.asarray(label), self.task, K), device=dev)
        g = torch.empty(K, rows, dtype=torch.float32, device=dev)
        h = torch.empty_like(g)
        gq = torch.empty(rows, dtype=torch.int64, device=dev)
        hq = torch.empty_like(gq)
        maxgh = torch.zeros(K, 2, dtype=torch.float32, device=dev)
        arange = torch.arange(rows, dtype=torch.int32, device=dev)
        index = torch.empty_like(arange)
        scratch = torch.empty(rows + 2, dtype=torch.int32, device=dev)
        L, cells = p['num_leaves'], self.nf * self.nb
        hg = torch.empty(L, cells, dtype=torch.int64, device=dev)
        hh = torch.empty_like(hg)
        hn = torch.empty(L, cells, dtype=torch.int32, device=dev)
        recs = torch.empty(2 * ctypes.sizeof(N.GbdtSplitRec), dtype=torch.uint8, device=dev)
        recs_host = torch.empty(recs.numel(), dtype=torch.uint8, pin_memory=True)
        pair = torch.empty(2, dtype=torch.int32, device=dev)
        pair_host = torch.empty(2, dtype=torch.int32, pin_memory=True)
        trees = []

        def split(leaves, sp):
            pair_host[:len(leaves)] = torch.tensor(leaves, dtype=torch.int32)
            pair[:len(leaves)].copy_(pair_host[:len(leaves)], non_blocking=True)
            with timer.device('split'):
                check(N.lib.dtb_gbdt_split(ptr(hg), ptr(hh), ptr(hn), ptr(pair), len(leaves), ptr(self.n_bins_d),
                                           self.nf, self.nb, ctypes.byref(sp), ptr(recs), stream_ptr()), 'gbdt_split')
            recs_host.copy_(recs)           # synchronises: the host picks the next leaf from these records
            raw = recs_host.numpy().tobytes()
            size = ctypes.sizeof(N.GbdtSplitRec)
            return [N.GbdtSplitRec.from_buffer_copy(raw[i * size:(i + 1) * size]) for i in range(len(leaves))]

        def hist(slot, begin, count):
            with timer.device('hist'):
                check(N.lib.dtb_gbdt_hist(ptr(bins), ptr(index), begin, count, ptr(gq), ptr(hq), self.nf, self.nb,
                                          ptr(hg[slot]), ptr(hh[slot]), ptr(hn[slot]), stream_ptr()), 'gbdt_hist')

        for it in range(p['n_estimators']):
            maxgh.zero_()
            with timer.device('grad'):
                for k in range(K):   # every class's gradient from the scores before this iteration's trees (LightGBM)
                    check(N.lib.dtb_gbdt_grad(ptr(scores), ptr(y), rows, K, k, self.objective, ptr(g[k]), ptr(h[k]),
                                              ptr(maxgh[k]), stream_ptr()), 'gbdt_grad')
            m = maxgh.cpu().numpy()
            grown = []
            for k in range(K):      # each tree updates its class's scores at once; the gradients were taken above
                tree = self._grow(k, rows, m[k], g[k], h[k], gq, hq, arange, index, scratch, hist, split, hg, hh, hn,
                                  bins, timer)
                if tree is not None:
                    self._update(tree, index, scores, k, leaf_log, len(trees) + k, timer)
                grown.append(tree)
            if all(t is None for t in grown):
                break           # no root meets the split requirements: boosting stops, as in LightGBM
            for k, tree in enumerate(grown):
                if tree is None:        # a class whose root cannot split gets a one-leaf tree of value 0
                    tree = {'feature': [], 'bin': [], 'threshold': [], 'left': [], 'right': [], 'gain': [],
                            'values': [0.0]}
                    if leaf_log is not None:
                        leaf_log[:, len(trees)] = 0
                trees.append(tree)
        timer.finish()
        return _trees_from_lists(trees)

    def _update(self, tree, index, scores, k, leaf_log, column, timer):
        dev = self.device
        values = torch.as_tensor(np.asarray(tree['values'], np.float32)).to(dev)
        seg_b = torch.as_tensor(np.asarray(tree['seg_begin'], np.int64)).to(dev)
        seg_c = torch.as_tensor(np.asarray(tree['seg_count'], np.int64)).to(dev)
        col = leaf_log[:, column] if leaf_log is not None else None
        with timer.device('update'):
            check(N.lib.dtb_gbdt_update(ptr(index), ptr(seg_b), ptr(seg_c), len(tree['values']),
                                        int(max(tree['seg_count'])), ptr(values), ptr(scores), self.K, k, ptr(col),
                                        leaf_log.shape[1] if leaf_log is not None else 0, stream_ptr()), 'gbdt_update')

    def _grow(self, k, rows, m, g, h, gq, hq, arange, index, scratch, hist, split, hg, hh, hn, bins, timer):
        p = self.p
        sg, sh = fixed_shift(m[0], rows), fixed_shift(m[1], rows)
        with timer.device('grad'):
            check(N.lib.dtb_gbdt_fixed(ptr(g), ptr(h), rows, sg, sh, ptr(gq), ptr(hq), stream_ptr()), 'gbdt_fixed')
        sp = N.GbdtSplitParams(p['reg_lambda'], p['reg_alpha'], p['min_split_gain'], p['min_child_weight'],
                               2.0 ** -sg, 2.0 ** -sh, p['min_child_samples'])
        index.copy_(arange)
        hist(0, 0, rows)
        root = split([0], sp)[0]
        if root.feature < 0:
            return None
        leaves = [{'begin': 0, 'count': rows, 'depth': 0, 'rec': root, 'parent': None}]
        feature, bin_, thr, left, right, gain = [], [], [], [], [], []
        while len(leaves) < p['num_leaves']:
            best = -1
            for i, lf in enumerate(leaves):
                r = lf['rec']
                if r.feature < 0 or (0 < p['max_depth'] <= lf['depth']):
                    continue
                if best < 0 or r.gain > leaves[best]['rec'].gain:
                    best = i
            if best < 0:
                break
            lf, new = leaves[best], len(leaves)
            r = lf['rec']
            with timer.device('partition'):
                check(N.lib.dtb_gbdt_partition(ptr(bins), self.nf, ptr(index), lf['begin'], lf['count'], r.feature,
                                               r.bin, r.left_count, ptr(scratch), stream_ptr()), 'gbdt_partition')
            node = len(feature)
            feature.append(r.feature)
            bin_.append(r.bin)
            gain.append(r.gain)
            thr.append(self.edges[r.feature][r.bin])
            left.append(~best)
            right.append(~new)
            if lf['parent'] is not None:
                pn, side = lf['parent']
                (left if side == 0 else right)[pn] = node
            lc, rc = r.left_count, lf['count'] - r.left_count
            right_leaf = {'begin': lf['begin'] + lc, 'count': rc, 'depth': lf['depth'] + 1, 'parent': (node, 1)}
            lf.update(count=lc, depth=lf['depth'] + 1, parent=(node, 0))
            leaves.append(right_leaf)
            small_is_left = lc <= rc
            small = lf if small_is_left else right_leaf
            hist(new, small['begin'], small['count'])
            with timer.device('hist'):
                check(N.lib.dtb_gbdt_hist_sub(ptr(hg[best]), ptr(hh[best]), ptr(hn[best]), ptr(hg[new]), ptr(hh[new]),
                                              ptr(hn[new]), hg.shape[1], int(small_is_left), stream_ptr()),
                      'gbdt_hist_sub')
            lf['rec'], right_leaf['rec'] = split([best, new], sp)
        values = [leaf_value(lf['rec'].g, lf['rec'].h, sg, sh, p) for lf in leaves]
        return {'feature': feature, 'bin': bin_, 'threshold': thr, 'left': left, 'right': right, 'gain': gain,
                'values': values,
                'seg_begin': [lf['begin'] for lf in leaves], 'seg_count': [lf['count'] for lf in leaves]}


def write_leaves(trees, feat_col, cat, cont, rows, out_cat=None, out_cont=None, out_col=0):
    """``dtb_gbdt_leaves``: the leaf of every row of ``cat`` / ``cont`` in every tree, into columns ``out_col ..`` of
    ``out_cat`` (int32) or ``out_cont`` (float32)."""
    if trees.n_trees == 0 or rows == 0:
        return
    dev = (out_cat if out_cat is not None else out_cont).device
    d = {k: torch.as_tensor(v).to(dev) for k, v in trees.arrays().items() if k.startswith('node_')}
    fc = torch.as_tensor(np.asarray(feat_col, np.int32)).to(dev)
    out = out_cat if out_cat is not None else out_cont
    check(N.lib.dtb_gbdt_leaves(ptr(cat), cat.shape[1] if cat is not None else 0, ptr(cont),
                                cont.shape[1] if cont is not None else 0, ptr(fc), ptr(d['node_feature']),
                                ptr(d['node_threshold']), ptr(d['node_left']), ptr(d['node_right']),
                                ptr(d['node_off']), trees.n_trees, int(np.diff(trees.node_off).max()), rows,
                                ptr(out_cat), ptr(out_cont), out.shape[1], out_col, stream_ptr()), 'gbdt_leaves')


class GbmLeavesEncoder:
    """hypernets' ``LgbmLeavesEncoder`` on the built-in booster: fits trees on the encoded columns ``cat_vars`` (int32
    codes) and ``cont_vars`` (float32) and appends one column per tree, ``lgbm_leaf_<i>``, holding each row's leaf.
    Holds only numpy arrays, so it pickles with the preprocessor."""

    def __init__(self, cat_vars, cont_vars, task, **gbm_params):
        self.cat_vars, self.cont_vars, self.task = list(cat_vars), list(cont_vars), task
        self.gbm_params = dict(gbm_params)
        self.edges = self.trees = None
        self.new_columns = []

    @property
    def feat_col(self):
        """Input column of each booster feature in the model's own layout: categorical codes first, then continuous."""
        return list(range(len(self.cat_vars))) + [-1 - c for c in range(len(self.cont_vars))]

    def _arrays(self, X):
        cat = np.ascontiguousarray(X[self.cat_vars].to_numpy(np.int32)) if self.cat_vars else None
        cont = np.ascontiguousarray(X[self.cont_vars].to_numpy(np.float32)) if self.cont_vars else None
        return cat, cont

    @staticmethod
    def _device(arr):
        return torch.as_tensor(arr).cuda() if arr is not None else None

    @staticmethod
    def check_names(X):
        clash = [c for c in X.columns if str(c).startswith(LEAF_PREFIX)]
        if clash:
            raise ValueError(f'apply_gbm_features: the frame already has leaf column names {clash}')

    def fit(self, X, y, num_classes=None):
        self.check_names(X)
        y = np.asarray(y).reshape(-1)
        if self.task == consts.TASK_MULTILABEL:
            raise NotImplementedError('apply_gbm_features on the multilabel task')
        if not self.cat_vars and not self.cont_vars:
            raise ValueError('apply_gbm_features: the frame has no encoded columns to fit trees on')
        if self.task == consts.TASK_REGRESSION:
            label = y.astype(np.float32)
        else:
            classes, label = np.unique(y, return_inverse=True)
            num_classes = max(num_classes or 0, len(classes))
        params = resolve_params(self.gbm_params, self.task, num_classes)
        if dp.is_distributed():
            box = [None]
            if torch.distributed.get_rank() == 0:
                box = [self._fit(X, label, params, num_classes)]
            torch.distributed.broadcast_object_list(box, src=0)
            self.edges, self.trees = box[0]
        else:
            self.edges, self.trees = self._fit(X, label, params, num_classes)
        self.new_columns = [f'{LEAF_PREFIX}{i}' for i in range(self.trees.n_trees)]
        return self

    def _fit(self, X, label, params, num_classes):
        cat, cont = self._arrays(X)
        rows = sample_rows(len(X), params['subsample_for_bin'], params['random_state'])
        cols = ([cat[rows, j].astype(np.float32) for j in range(cat.shape[1])] if cat is not None else []) + \
               ([cont[rows, j] for j in range(cont.shape[1])] if cont is not None else [])
        edges = [bin_edges(v, params['max_bin']) for v in cols]
        dev = torch.device('cuda', torch.cuda.current_device())
        booster = Booster(params, self.task, num_classes, self.feat_col, edges, dev)
        trees = booster.fit(self._device(cat), self._device(cont), label)
        return edges, trees

    def leaves(self, X):
        """int32 [rows, trees]: the leaf of each row of the encoded frame X in every tree."""
        cat, cont = self._arrays(X)
        out = torch.zeros(len(X), max(self.trees.n_trees, 1), dtype=torch.int32, device='cuda')
        write_leaves(self.trees, self.feat_col, self._device(cat), self._device(cont), len(X), out_cat=out)
        return out[:, :self.trees.n_trees].cpu().numpy()

    def transform(self, X):
        self.check_names(X)
        import pandas as pd
        leaves = self.leaves(X)
        extra = pd.DataFrame(leaves, columns=self.new_columns, index=X.index)
        return pd.concat([X, extra], axis=1)

    def fit_transform(self, X, y, num_classes=None):
        return self.fit(X, y, num_classes).transform(X)

    def write_device(self, cat, cont, embedding):
        """Rewrite the leaf columns of the model's device inputs from their raw columns: the columns after the raw
        categorical ones (``embedding``) or after the raw continuous ones."""
        rows = (cat if cat is not None else cont).shape[0]
        if embedding:
            write_leaves(self.trees, self.feat_col, cat, cont, rows, out_cat=cat, out_col=len(self.cat_vars))
        else:
            write_leaves(self.trees, self.feat_col, cat, cont, rows, out_cont=cont, out_col=len(self.cont_vars))


def rewrite_leaves(preprocessor, cat, cont):
    """After an input column of the model's device inputs changed (permutation importance, SHAP coalitions): recompute
    their leaf columns.  Nothing to do without leaf features."""
    enc = getattr(preprocessor, 'gbm_encoder_', None)
    if enc is not None and enc.trees.n_trees:
        enc.write_device(cat, cont, preprocessor.config.gbm_feature_type == consts.GBM_FEATURE_TYPE_EMB)
