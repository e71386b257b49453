"""float64 numpy restatement of the booster of deeptables_b200/gbm.py and csrc/gbdt.cu: binning, gradients, fixed
point, histograms, split search, leaf-wise growth, leaf values and traversal.  Written from the rules the header
states, without the device's data layout; the tests compare the device against it."""
import math

import numpy as np


def bins(X, edges):
    """uint8 [rows, features]: the number of edges below x; NaN in the last bin."""
    out = np.empty(X.shape, np.uint8)
    for j, e in enumerate(edges):
        b = np.searchsorted(e, X[:, j], side='left')
        b[np.isnan(X[:, j])] = len(e)
        out[:, j] = b
    return out


def grad_hess(scores, y, objective, K):
    """float32 [K, rows] gradients and hessians of float64 scores [rows, K]."""
    rows = len(y)
    g, h = np.empty((K, rows), np.float32), np.empty((K, rows), np.float32)
    if objective == 'binary':
        p = 1.0 / (1.0 + np.exp(-scores[:, 0]))
        g[0], h[0] = p - y, p * (1.0 - p)
    elif objective == 'regression':
        g[0], h[0] = scores[:, 0] - y, 1.0
    else:
        m = scores.max(axis=1)
        s = np.zeros(rows)
        for j in range(K):
            s = s + np.exp(scores[:, j] - m)
        for k in range(K):
            p = np.exp(scores[:, k] - m) / s
            g[k] = p - (y.astype(np.int64) == k)
            h[k] = (K / (K - 1)) * (p * (1.0 - p))
    return g, h


def shift(max_abs, rows):
    if not max_abs > 0:
        return 0
    return 62 - (rows - 1).bit_length() - math.frexp(float(max_abs))[1]


def fixed(v, s):
    return np.rint(v.astype(np.float64) * 2.0 ** s).astype(np.int64)


def histogram(B, rows, gq, hq, nb):
    """int64 sums of gq, hq and counts per (feature, bin) over the given rows."""
    nf = B.shape[1]
    G, H, C = np.zeros((nf, nb), np.int64), np.zeros((nf, nb), np.int64), np.zeros((nf, nb), np.int64)
    for f in range(nf):
        b = B[rows, f].astype(np.int64)
        np.add.at(G[f], b, gq[rows])
        np.add.at(H[f], b, hq[rows])
        C[f] = np.bincount(b, minlength=nb)
    return G, H, C


def _T(G, a):
    return np.where(G > a, G - a, np.where(G < -a, G + a, 0.0))


def _term(G, H, p):
    t = _T(G, p['reg_alpha'])
    return (t * t) / (H + p['reg_lambda'])


def best_split(G, H, C, n_bins, p, sg, sh):
    """(gain, feature, bin, left_count) of the best candidate, or None; ties to the lowest feature, then bin."""
    Gi, Hi, Ni = int(G[0].sum()), int(H[0].sum()), int(C[0].sum())
    parent = _term(np.float64(Gi) * sg, np.float64(Hi) * sh, p)
    best = None
    for f in range(len(n_bins)):
        k = n_bins[f] - 1
        if k < 1:
            continue
        gl, hl, nl = np.cumsum(G[f, :k]), np.cumsum(H[f, :k]), np.cumsum(C[f, :k])
        GL, HL = gl.astype(np.float64) * sg, hl.astype(np.float64) * sh
        GR, HR = (Gi - gl).astype(np.float64) * sg, (Hi - hl).astype(np.float64) * sh
        with np.errstate(invalid='ignore', divide='ignore'):
            gain = ((_term(GL, HL, p) + _term(GR, HR, p)) - parent) - p['min_split_gain']
        ok = (nl >= p['min_child_samples']) & (Ni - nl >= p['min_child_samples']) & \
             (HL >= p['min_child_weight']) & (HR >= p['min_child_weight']) & (gain > 0)
        if not ok.any():
            continue
        t = int(np.flatnonzero(ok)[np.argmax(gain[ok])])
        if best is None or gain[t] > best[0]:
            best = (float(gain[t]), f, t, int(nl[t]))
    return best


def leaf_value(Gi, Hi, sg, sh, p):
    G, H = float(Gi) * sg, float(Hi) * sh
    a = p['reg_alpha']
    t = G - a if G > a else (G + a if G < -a else 0.0)
    return np.float32(-p['learning_rate'] * (t / (H + p['reg_lambda'])))


def grow(B, gq, hq, n_bins, p, sg, sh):
    """One tree: dict of node lists, leaf values and each row's leaf (None when the root cannot split)."""
    rows = len(gq)
    nb = int(max(n_bins))
    members = [np.arange(rows)]
    depth = [0]
    parent = [None]
    hist = [histogram(B, members[0], gq, hq, nb)]
    rec = [best_split(*hist[0], n_bins, p, sg, sh)]
    if rec[0] is None:
        return None
    tree = {'feature': [], 'bin': [], 'left': [], 'right': [], 'gain': []}
    while len(members) < p['num_leaves']:
        cand = [i for i in range(len(members)) if rec[i] is not None and not (0 < p['max_depth'] <= depth[i])]
        if not cand:
            break
        best = max(cand, key=lambda i: (rec[i][0], -i))
        gain, f, t, _ = rec[best]
        new = len(members)
        node = len(tree['feature'])
        for key, v in (('feature', f), ('bin', t), ('left', ~best), ('right', ~new), ('gain', gain)):
            tree[key].append(v)
        if parent[best] is not None:
            pn, side = parent[best]
            tree['left' if side == 0 else 'right'][pn] = node
        m = members[best]
        go_left = B[m, f] <= t
        members[best] = m[go_left]
        members.append(m[~go_left])
        depth[best] += 1
        depth.append(depth[best])
        parent[best] = (node, 0)
        parent.append((node, 1))
        for i in (best, new):
            hist_i = histogram(B, members[i], gq, hq, nb)
            if len(hist) <= i:
                hist.append(hist_i)
            else:
                hist[i] = hist_i
            r = best_split(*hist_i, n_bins, p, sg, sh)
            if len(rec) <= i:
                rec.append(r)
            else:
                rec[i] = r
    leaf = np.empty(rows, np.int32)
    tree['values'] = []
    for i, m in enumerate(members):
        leaf[m] = i
        tree['values'].append(leaf_value(gq[m].sum(), hq[m].sum(), sg, sh, p))
    tree['leaf'] = leaf
    return tree


def fit(X, y, task, K, p, edges):
    """The booster on raw float32 features X [rows, nf]: a list of trees (dict of node lists and leaf values)."""
    objective = task
    B = bins(X, edges)
    n_bins = [len(e) + 1 for e in edges]
    rows = len(y)
    if task == 'regression':
        init = np.array([np.mean(y.astype(np.float64))])
    elif task == 'binary':
        q = min(max(float(np.mean(y.astype(np.float64))), 1e-15), 1 - 1e-15)
        init = np.array([math.log(q / (1 - q))])
    else:
        init = np.log(np.maximum(np.bincount(y.astype(np.int64), minlength=K) / rows, 1e-15))
    scores = np.tile(init, (rows, 1))
    trees = []
    for _ in range(p['n_estimators']):
        g, h = grad_hess(scores, y, objective, K)
        grown = []
        for k in range(K):
            sg, sh = shift(np.abs(g[k]).max(), rows), shift(h[k].max(), rows)
            t = grow(B, fixed(g[k], sg), fixed(h[k], sh), n_bins, p, 2.0 ** -sg, 2.0 ** -sh)
            if t is not None:
                scores[:, k] += np.asarray(t['values'], np.float32).astype(np.float64)[t['leaf']]
            grown.append(t)
        if all(t is None for t in grown):
            break
        for t in grown:
            trees.append(t if t is not None else {'feature': [], 'bin': [], 'left': [], 'right': [], 'gain': [],
                                                  'values': [np.float32(0)], 'leaf': np.zeros(rows, np.int32)})
    return trees


def traverse(tree, X, edges):
    """Leaf of each row of raw features X: x <= threshold goes left, NaN right."""
    rows = len(X)
    if not tree['feature']:
        return np.zeros(rows, np.int32)
    node = np.zeros(rows, np.int64)
    out = np.empty(rows, np.int32)
    live = np.arange(rows)
    while len(live):
        n = node[live]
        f = np.asarray(tree['feature'])[n]
        thr = np.array([edges[ff][bb] for ff, bb in zip(f, np.asarray(tree['bin'])[n])], np.float32)
        x = X[live, f]
        nxt = np.where(x <= thr, np.asarray(tree['left'])[n], np.asarray(tree['right'])[n])
        done = nxt < 0
        out[live[done]] = ~nxt[done]
        node[live[~done]] = nxt[~done]
        live = live[~done]
    return out
