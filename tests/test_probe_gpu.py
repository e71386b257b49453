"""Linear probes on the GPU: dtb_probe_loss_grad / join / predict / correct against the numpy restatement across
classes, widths (past one gradient column group), rows (block edges, several million) and intercepts; the same bits
across calls, tile heights and batch sizes; the device estimator on real layer features against scikit-learn's
float64 optimum; probe_evaluate against the reference's own computation; and the model left as it was."""
import numpy as np
import pandas as pd
import pytest
import torch

import probe_ref

pytestmark = pytest.mark.gpu

ROWS, TEST_ROWS = 4000, 2000


def _case(n, d, K, seed, scale=0.3):
    g = np.random.default_rng(seed)
    X = g.normal(size=(n, d)).astype(np.float32)
    codes = g.integers(0, 2 if K == 1 else K, n).astype(np.int32)
    W = g.normal(scale=scale, size=(K, d + 1))
    return X, codes, W


def _device_sums(X, codes, W, fit_intercept, tile_rows=0):
    from deeptables_b200 import probe
    obj = probe.DeviceObjective(torch.tensor(X).cuda(), torch.tensor(codes).cuda(), W.shape[0], fit_intercept,
                                tile_rows)
    return obj(W)


def _check_sums(got, want):
    (f, g), (wf, wg) = got, want
    assert abs(f - wf) <= 1e-12 * abs(wf), (f, wf)
    assert np.abs(g - wg).max() <= 1e-12 * np.abs(wg).max(), np.abs(g - wg).max() / np.abs(wg).max()


SHAPES = [(K, d) for K in (1, 3, 10) for d in (1, 7, 64, 429, 1079)] + [(10, 2000), (3, 5000), (1, 14000)]


@pytest.mark.parametrize('K, d', SHAPES)
@pytest.mark.parametrize('fit_intercept', [True, False])
def test_loss_grad_matches_numpy_across_classes_and_widths(K, d, fit_intercept):
    X, codes, W = _case(1025, d, K, K * 7919 + d, scale=1.0 / np.sqrt(d))
    _check_sums(_device_sums(X, codes, W, fit_intercept), probe_ref.loss_grad_sums(X, codes, W, fit_intercept))


@pytest.mark.parametrize('n', [1, 1023, 1024, 1025, 65537])
@pytest.mark.parametrize('K', [1, 3, 10])
def test_loss_grad_matches_numpy_at_block_edges(n, K):
    X, codes, W = _case(n, 64, K, n + K)
    for fit_intercept in (True, False):
        _check_sums(_device_sums(X, codes, W, fit_intercept), probe_ref.loss_grad_sums(X, codes, W, fit_intercept))


def test_loss_grad_matches_numpy_on_millions_of_rows():
    X, codes, W = _case(3_000_001, 16, 3, 11)
    _check_sums(_device_sums(X, codes, W, True), probe_ref.loss_grad_sums(X, codes, W, True))


def test_strided_and_unaligned_rows():
    """A column slice of a wider matrix (row stride != d, rows not 16-byte aligned) reads the same values."""
    from deeptables_b200 import probe
    X, codes, W = _case(3000, 13, 3, 5)
    wide = torch.zeros(3000, 20, dtype=torch.float32, device='cuda')
    wide[:, 1:14] = torch.tensor(X).cuda()
    obj = probe.DeviceObjective(wide[:, 1:14], torch.tensor(codes).cuda(), 3, True)
    _check_sums(obj(W), probe_ref.loss_grad_sums(X, codes, W, True))


@pytest.mark.parametrize('K, d', [(1, 429), (10, 1079), (10, 2000)])
def test_same_bits_across_calls_and_tile_heights(K, d):
    from deeptables_b200 import _native as N
    X, codes, W = _case(5000, d, K, 3)
    first = _device_sums(X, codes, W, True)
    most = N.lib.dtb_probe_tile_rows(d, K)
    for tile_rows in (0, 1, 5, most):
        f, g = _device_sums(X, codes, W, True, tile_rows)
        assert f == first[0] and np.array_equal(g, first[1])


@pytest.mark.parametrize('K', [1, 4])
@pytest.mark.parametrize('fit_intercept', [True, False])
def test_predict_and_correct_count_match_numpy(K, fit_intercept):
    from scipy.special import expit, softmax
    from deeptables_b200 import probe
    X, codes, W = _case(70_001, 33, K, 9)
    clf = probe.LogisticProbe(fit_intercept=fit_intercept)
    clf._W = W if fit_intercept else np.concatenate([W[:, :-1], np.zeros((K, 1))], 1)
    clf.classes_ = np.arange(max(K, 2))
    proba, pred = clf._predict(torch.tensor(X).cuda())
    Z = X.astype(np.float64) @ clf._W[:, :-1].T + clf._W[:, -1]
    if K == 1:
        want_p = np.stack([1 - expit(Z[:, 0]), expit(Z[:, 0])], 1)
        want_c = (Z[:, 0] > 0).astype(np.int32)
    else:
        want_p, want_c = softmax(Z, axis=1), np.argmax(Z, axis=1).astype(np.int32)
    np.testing.assert_allclose(proba.cpu().numpy(), want_p, rtol=1e-12, atol=1e-15)
    np.testing.assert_array_equal(pred.cpu().numpy(), want_c)
    assert probe.count_correct(pred, torch.tensor(codes).cuda()) == int((want_c == codes).sum())


def _frame(rows, seed):
    g = np.random.default_rng(seed)
    X = pd.DataFrame({f'c{i}': g.choice(list('abcdef')[:3 + i % 4], rows) for i in range(4)})
    for i in range(4):
        X[f'n{i}'] = g.normal(size=rows)
    lead = (X['c0'] == 'a') * 2.0 + X['n0'] + 0.5 * X['n1'] * (X['c1'] == 'b') + 0.3 * g.normal(size=rows)
    return X, lead


_CACHE = {}


def _fitted(task):
    if task not in _CACHE:
        from deeptables_b200 import deepnets, deeptable
        X, lead = _frame(ROWS + TEST_ROWS, 4)
        y = np.where(lead > 0.8, 'yes', 'no') if task == 'binary' else \
            np.array(['lo', 'mid', 'hi'])[np.digitize(lead, [0.0, 1.5])]
        conf = deeptable.ModelConfig(nets=deepnets.DeepFM, metrics=['AUC'] if task == 'binary' else ['accuracy'],
                                     embeddings_output_dim=4, auto_categorize=True)
        dt = deeptable.DeepTable(config=conf)
        y = pd.Series(y)
        dt.fit(X.iloc[:ROWS], y.iloc[:ROWS], epochs=2, batch_size=128, verbose=0)
        _CACHE[task] = (dt, X.iloc[:ROWS], y.iloc[:ROWS].to_numpy(), X.iloc[ROWS:], y.iloc[ROWS:].to_numpy())
    return _CACHE[task]


LAYERS = ['flatten_embeddings', 'dnn_dense_1', 'dnn_dense_2']


def _certified(X, codes, w_probe, w_other, K, C):
    """Newton-decrement radii of two solutions of the same problem and the per-coordinate bound on their difference.
    Near the optimum w*, sqrt((w - w*)' H (w - w*)) is the Newton decrement delta(w) = sqrt(g' H^-1 g) to first order;
    a factor 2 covers the change of H over the tiny ball, so |w_probe - w_other|_j <= 2 (delta_p + delta_o)
    sqrt(H^-1_jj) whichever stopping rule of L-BFGS-B fired."""
    H_inv = np.linalg.inv(probe_ref.hessian(X, codes, w_probe, K, C, True))
    d_p = probe_ref.newton_decrement(X, codes, w_probe, K, C, True, H_inv)
    d_o = probe_ref.newton_decrement(X, codes, w_other, K, C, True, H_inv)
    return H_inv, d_p, d_o, 2 * (d_p + d_o) * np.sqrt(np.diag(H_inv))


@pytest.mark.parametrize('K', [1, 3])
def test_estimator_meets_the_float64_optimum_where_both_solvers_stop_on_gtol(K):
    """A well-conditioned problem (Gaussian features) on which both solvers stop on the gradient test at tol = 1e-8:
    ours by its stop message, scikit-learn's by its float64 gradient.  The per-coordinate gap is then bounded by the
    Newton decrements (``_certified``); for the binary problem that bound is below 1e-6 * max(1, |c|)."""
    from sklearn.linear_model import LogisticRegression
    from deeptables_b200 import probe
    g = np.random.default_rng(20 + K)
    n, d = 20_000, 64
    X = g.normal(size=(n, d)).astype(np.float32)
    w = 0.3 * g.normal(size=(d, max(K, 2)))
    y = (X @ w[:, 0] + g.logistic(size=n) > 0).astype(int) if K == 1 else np.argmax(X @ w + g.gumbel(size=(n, K)), 1)
    clf = probe.LogisticProbe(tol=1e-8, max_iter=10_000).fit(torch.tensor(X).cuda(), y)
    ref = LogisticRegression(tol=1e-8, max_iter=10_000).fit(X.astype(np.float64), y)
    assert 'PROJECTED GRADIENT' in clf.stop_message_, clf.stop_message_
    w_o, w_r = np.c_[clf.coef_, clf.intercept_].ravel(), np.c_[ref.coef_, ref.intercept_].ravel()
    assert np.abs(probe_ref.objective(X, y, w_r, K, 1.0, True)[1]).max() <= 1e-8
    _, _, _, bound = _certified(X, y, w_o, w_r, K, 1.0)
    assert np.all(np.abs(w_o - w_r) <= bound)
    if K == 1:
        scale = max(1.0, np.abs(w_r).max())
        assert bound.max() <= 1e-6 * scale
        np.testing.assert_allclose(w_o, w_r, rtol=0, atol=1e-6 * scale)


@pytest.mark.parametrize('task', ['binary', 'multiclass'])
def test_estimator_on_layer_features_agrees_with_float64_sklearn_within_the_certified_bound(task):
    """On relu layer features both solvers stop on the relative-reduction test (ftol = 64 eps) before the gradient
    reaches 1e-10, at a distance from the optimum set by the features' conditioning.  The assertion is the bound that
    follows from the gradients actually reached (``_certified``), so it holds for any trained model."""
    from sklearn.linear_model import LogisticRegression
    from deeptables_b200 import probe
    dt, X, y, _, _ = _fitted(task)
    yt = dt.preprocessor.transform_y(y)
    for layer in LAYERS:
        feats = dt.apply(X, output_layers=[layer])
        clf = probe.LogisticProbe(tol=1e-10, max_iter=10_000).fit(torch.tensor(feats).cuda(), yt)
        ref = LogisticRegression(tol=1e-10, max_iter=10_000).fit(feats.astype(np.float64), yt)
        K = clf.coef_.shape[0]
        codes = np.searchsorted(clf.classes_, yt)
        w_o, w_r = np.c_[clf.coef_, clf.intercept_].ravel(), np.c_[ref.coef_, ref.intercept_].ravel()
        _, d_o, d_r, bound = _certified(feats, codes, w_o, w_r, K, 1.0)
        print(f'{task} {layer}: {clf.stop_message_}; decrements {d_o:.2e} / {d_r:.2e}; certified gap '
              f'{bound.max():.2e}, actual {np.abs(w_o - w_r).max():.2e}')
        assert d_o <= 1e-4 and d_r <= 1e-4            # both inside the region where the quadratic model holds
        assert np.all(np.abs(w_o - w_r) <= bound), layer


def _uncertain(f_train, codes, f_test, w_probe, w_ref, K):
    """Test rows whose predicted class can differ between two solutions of the training objective, and the bound per
    row of each decision value's move: a row is certain when its margin under w_probe exceeds the bound
    (``probe_ref.margin_bounds``), the radius being twice the sum of the two Newton decrements."""
    H_inv = np.linalg.inv(probe_ref.hessian(f_train, codes, w_probe, K, 1.0, True))
    radius = 2 * sum(probe_ref.newton_decrement(f_train, codes, w, K, 1.0, True, H_inv) for w in (w_probe, w_ref))
    margins, bounds = probe_ref.margin_bounds(f_test, w_probe, H_inv, radius, K, True)
    return margins <= bounds, bounds


@pytest.mark.parametrize('task', ['binary', 'multiclass'])
def test_probe_evaluate_matches_the_reference_computation(task):
    """probe_evaluate against the reference's computation (scikit-learn on the float32 apply output, default
    settings).  scikit-learn minimises the float32 objective and stops at gtol = 1e-4, so its solution w_r sits at a
    Newton decrement delta_r from the float64 optimum, and ours (gtol = 1e-4 in float64) at delta_p.  A test row's
    decision value moves by at most 2 (delta_p + delta_r) sqrt(u' H^-1 u) between them, so only rows whose margin is
    below that bound can change class, and only positive-negative pairs closer than the sum of their bounds can change
    order.  Those counts bound the accuracy and AUC gaps; they are computed from the solutions reached, not fixed."""
    from sklearn.linear_model import LogisticRegression
    from sklearn.metrics import f1_score, mean_squared_error, roc_auc_score
    from deeptables_b200 import deeptable, probe
    dt, X, y, Xt, yt = _fitted(task)
    got = deeptable.probe_evaluate(dt, X, y, Xt, yt, layers=LAYERS)
    assert list(got) == LAYERS and all(list(v) == ['accuracy'] for v in got.values())
    fns = {'AUC': roc_auc_score, 'F1': f1_score, 'MSE': mean_squared_error}
    got_fns = None if task == 'multiclass' else deeptable.probe_evaluate(dt, X, y, Xt, yt, LAYERS, score_fn=fns)
    y_c, yt_c = dt.preprocessor.transform_y(y), dt.preprocessor.transform_y(yt)
    for layer in LAYERS:
        f_tr, f_te = dt.apply(X, output_layers=[layer]), dt.apply(Xt, output_layers=[layer])
        mine = probe.LogisticProbe().fit(torch.tensor(f_tr).cuda(), y_c)           # what probe_evaluate fits
        ref = LogisticRegression(random_state=0).fit(f_tr, y_c)
        pred = mine.classes_[mine._predict(torch.tensor(f_te).cuda())[1].cpu().numpy()]
        assert got[layer]['accuracy'] == float(np.mean(pred == yt_c))               # the same probe, exactly
        K = mine.coef_.shape[0]
        codes = np.searchsorted(mine.classes_, y_c)
        w_p = np.c_[mine.coef_, mine.intercept_].ravel()
        w_r = np.c_[ref.coef_, ref.intercept_].ravel().astype(np.float64)
        uncertain, bounds = _uncertain(f_tr, codes, f_te, w_p, w_r, K)
        want = ref.score(f_te, yt_c)
        moved = pred != ref.predict(f_te)
        assert not np.any(moved & ~uncertain), layer
        acc_bound = uncertain.mean()
        print(f'{task} {layer}: accuracy {got[layer]["accuracy"]:.6f} vs {want:.6f}, certified bound {acc_bound:.2e}')
        assert abs(got[layer]['accuracy'] - want) <= acc_bound
        if got_fns is None:
            continue
        z = np.c_[f_te.astype(np.float64), np.ones(len(f_te))] @ w_p                 # our probe's logits
        pos, neg = yt_c == 1, yt_c == 0
        close = np.abs(z[pos][:, None] - z[neg][None, :]) <= bounds[pos][:, None] + bounds[neg][None, :]
        auc_bound = close.mean()
        want_auc = roc_auc_score(yt_c, ref.predict_proba(f_te)[:, 1])
        print(f'{task} {layer}: AUC {got_fns[layer]["AUC"]:.6f} vs {want_auc:.6f}, certified bound {auc_bound:.2e}')
        assert abs(got_fns[layer]['AUC'] - want_auc) <= auc_bound
    if task == 'multiclass':
        with pytest.raises(ValueError):
            deeptable.probe_evaluate(dt, X, y, Xt, yt, layers=LAYERS[:1], score_fn=fns)
    else:
        assert list(got_fns) == LAYERS and all(list(v) == ['AUC', 'F1', 'MSE'] for v in got_fns.values())


def test_same_result_across_calls_and_batch_sizes():
    from deeptables_b200 import deeptable
    from sklearn.metrics import roc_auc_score
    dt, X, y, Xt, yt = _fitted('binary')
    runs = [deeptable.probe_evaluate(dt, X, y, Xt, yt, LAYERS, {'AUC': roc_auc_score}, batch_size=bs)
            for bs in (1000, 65536, 65536)]
    assert runs[0] == runs[1] == runs[2]


def test_model_state_keeps_its_bits():
    from test_gradshap_gpu import _train_state
    from deeptables_b200 import deeptable
    dt, X, y, Xt, yt = _fitted('multiclass')
    m = dt.get_model()
    m.flush_optimizer_state()
    before = _train_state(m)
    deeptable.probe_evaluate(dt, X, y, Xt, yt, LAYERS)
    after = _train_state(m)
    assert before.keys() == after.keys()
    assert [k for k in before if before[k] != after[k]] == []
