"""numpy float64 restatement of the linear-probe objective (deeptables_b200/probe.py, csrc/probe.cu): scikit-learn's
lbfgs LogisticRegression objective, its row sums and the estimator driven by them on the host."""
import numpy as np
from scipy.special import expit, logsumexp, softmax


def loss_grad_sums(X, codes, W, fit_intercept):
    """(sum of the row losses, their gradient [K, d + 1]) at W [K, d + 1] -- what dtb_probe_loss_grad and
    dtb_probe_join give.  codes: binary (K = 1) 0 / 1, multinomial the class index."""
    X = np.asarray(X, np.float64)
    codes = np.asarray(codes).astype(np.int64)
    n, d = X.shape
    K = W.shape[0]
    Z = X @ W[:, :d].T
    if fit_intercept:
        Z = Z + W[:, d]
    if K == 1:
        z, yv = Z[:, 0], codes.astype(np.float64)
        loss = np.logaddexp(0.0, z) - yv * z
        R = (expit(z) - yv)[:, None]
    else:
        loss = logsumexp(Z, axis=1) - Z[np.arange(n), codes]
        R = softmax(Z, axis=1)
        R[np.arange(n), codes] -= 1.0
    G = np.zeros_like(W, dtype=np.float64)
    G[:, :d] = R.T @ X
    if fit_intercept:
        G[:, d] = R.sum(axis=0)
    return float(loss.sum()), G


def objective(X, codes, w, K, C, fit_intercept):
    """(1/n) sum l_i + (1/(2 C n)) ||coef||^2 and its gradient at the flat w [K * (d + fit_intercept)]."""
    n, d = np.shape(X)
    cols = d + 1 if fit_intercept else d
    W = np.zeros((K, d + 1))
    W[:, :cols] = np.reshape(w, (K, cols))
    loss, G = loss_grad_sums(X, codes, W, fit_intercept)
    l2 = 1.0 / (C * n)
    coef = W[:, :d]
    g = G[:, :cols] / n
    g[:, :d] += l2 * coef
    return loss / n + 0.5 * l2 * float((coef * coef).sum()), g.ravel()


class HostObjective:
    """Stands in for probe.DeviceObjective: the same call, computed by loss_grad_sums."""

    def __init__(self, X, codes, K, fit_intercept, tile_rows=0):
        self.X = np.asarray(X.cpu().numpy() if hasattr(X, 'cpu') else X, np.float32)
        self.codes = np.asarray(codes.cpu().numpy() if hasattr(codes, 'cpu') else codes)
        self.fit_intercept = fit_intercept

    def __call__(self, W):
        return loss_grad_sums(self.X, self.codes, W, self.fit_intercept)


def hessian(X, codes, w, K, C, fit_intercept):
    """The Hessian of ``objective`` at the flat w, float64 [K * cols, K * cols] (cols = d + fit_intercept).  For the
    multinomial with an intercept the objective is flat along "add t to every class's intercept" (softmax ignores it,
    and the intercept is not penalised); that direction changes no class margin, so it gets curvature 1 here to make
    the matrix invertible without changing any bound on margins."""
    X = np.asarray(X, np.float64)
    n, d = X.shape
    cols = d + 1 if fit_intercept else d
    Xt = np.c_[X, np.ones(n)] if fit_intercept else X
    W = np.reshape(w, (K, cols))
    Z = Xt @ W.T
    pen = np.full(cols, 1.0 / (C * n))
    if fit_intercept:
        pen[d] = 0.0
    if K == 1:
        p = expit(Z[:, 0])
        return (Xt.T * (p * (1 - p))) @ Xt / n + np.diag(pen)
    P = softmax(Z, axis=1)
    H = np.zeros((K * cols, K * cols))
    for a in range(K):
        for b in range(a, K):
            s = P[:, a] * ((a == b) - P[:, b])
            blk = (Xt.T * s) @ Xt / n
            H[a * cols:(a + 1) * cols, b * cols:(b + 1) * cols] = blk
            H[b * cols:(b + 1) * cols, a * cols:(a + 1) * cols] = blk
    H += np.diag(np.tile(pen, K))
    if fit_intercept:
        v = np.zeros(K * cols)
        v[d::cols] = 1.0 / np.sqrt(K)
        H += np.outer(v, v)
    return H


def margin_bounds(X, w_probe, H_inv, radius, K, fit_intercept):
    """For each row, with w within ``radius`` of w_probe in the H metric (sqrt(dw' H dw) <= radius): the most any
    logit difference z_a - z_b the probe's decision rests on can move, radius * sqrt(u' H^-1 u) with u the gradient of
    that difference in w (Cauchy-Schwarz in the H metric).  Binary: the logit itself; multinomial: the probe's top
    class against each other class, the smallest margin-to-bound ratio kept.  Returns (margins, bounds) per row."""
    X = np.asarray(X, np.float64)
    n, d = X.shape
    cols = d + 1 if fit_intercept else d
    Xt = np.c_[X, np.ones(n)] if fit_intercept else X
    W = np.reshape(w_probe, (K, cols))
    Z = Xt @ W.T
    if K == 1:
        q = np.einsum('ij,jk,ik->i', Xt, H_inv, Xt)
        return np.abs(Z[:, 0]), radius * np.sqrt(np.maximum(q, 0.0))
    top = np.argmax(Z, axis=1)
    margins = np.full(n, np.inf)
    bounds = np.zeros(n)
    B = lambda a, b: H_inv[a * cols:(a + 1) * cols, b * cols:(b + 1) * cols]
    for a in range(K):
        rows = top == a
        for b in range(K):
            if b == a or not rows.any():
                continue
            M = B(a, a) - B(a, b) - B(b, a) + B(b, b)
            x = Xt[rows]
            q = radius * np.sqrt(np.maximum(np.einsum('ij,jk,ik->i', x, M, x), 0.0))
            m = Z[rows, a] - Z[rows, b]
            worse = m - q < margins[rows] - bounds[rows]
            idx = np.flatnonzero(rows)[worse]
            margins[idx], bounds[idx] = m[worse], q[worse]
    return margins, bounds


def newton_decrement(X, codes, w, K, C, fit_intercept, H_inv):
    """sqrt(g' H^-1 g) of ``objective`` at w: near the optimum w*, the H-metric distance from w to w*."""
    g = objective(X, codes, w, K, C, fit_intercept)[1]
    return float(np.sqrt(max(g @ H_inv @ g, 0.0)))
