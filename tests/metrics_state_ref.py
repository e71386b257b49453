"""Numpy restatement of the state ``dtb_metrics_update`` builds (layout in include/deeptables_b200.h), from whole arrays
of labels and predictions.  Built on metrics_ref.py's row formulas; takes a ``metrics.Plan`` only for its sizes."""
import numpy as np

import metrics_ref as MR

_SUM_KINDS = ('mse', 'mae', 'mape', 'msle', 'logcosh', 'bce', 'cce')


def state_of(plan, y, p):
    """uint64 [plan.words]: what the device state holds after updates with rows ``y``, ``p`` (float32 [rows, cols])."""
    y = np.asarray(y, np.float32).reshape(-1, plan.cols)
    p = np.asarray(p, np.float32).reshape(-1, plan.cols)
    cols = plan.cols
    sums = np.zeros(8 + 3 * cols, np.float64)
    for bit, kind in enumerate(_SUM_KINDS):
        if plan.sums & (1 << bit) and len(y):
            sums[bit] = MR.row_values(kind, y, p).sum()
    if plan.sums & 128:
        y64, p64 = y.astype(np.float64), p.astype(np.float64)
        sums[8 + 0::3], sums[8 + 1::3], sums[8 + 2::3] = y64.sum(0), (y64 ** 2).sum(0), ((y64 - p64) ** 2).sum(0)
    cnt = np.zeros(plan.words - plan.counters, np.uint64)
    cnt[0] = len(y)
    label = y != 0
    if plan.argmax and len(y):
        with np.errstate(invalid='ignore'):
            pred = (p >= np.nanmax(np.where(np.isnan(p), -np.inf, p), -1, keepdims=True)) & (np.abs(p) > 1e-9)
            target = np.take_along_axis(p, y.argmax(-1)[:, None], -1)
            above = (p > target).sum(-1)
        first_max = np.where(np.isnan(p), -np.inf, p).argmax(-1)
        cnt[1] = (first_max == y.argmax(-1)).sum()
        cnt[2] = (np.isfinite(target[:, 0]) & (above < plan.top_k)).sum()
        cnt[3:3 + cols] = (pred & label).sum(0)
        cnt[3 + cols:3 + 2 * cols] = (pred & ~label).sum(0)
        cnt[3 + 2 * cols:3 + 3 * cols] = (~pred & label).sum(0)
    for li, thresholds in enumerate(plan.lists):
        t = np.asarray(thresholds, np.float32)
        # thresholds strictly below p (the list is ascending); NaN: none
        bucket = np.where(np.isnan(p), 0, np.searchsorted(t, p, side='left'))
        hist = np.zeros((cols, 2, len(t) + 1), np.uint64)
        for c in range(cols):
            for lab in (0, 1):
                hist[c, lab] = np.bincount(bucket[label[:, c] == bool(lab), c], minlength=len(t) + 1)
        cnt[plan.hist_off[li]:plan.hist_off[li] + hist.size] = hist.reshape(-1)
    return np.concatenate([sums.view(np.uint64), cnt])
