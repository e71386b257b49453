"""Permutation feature importance (reference deeptables/utils/feature_importance.py over eli5's
get_score_importances), computed on the GPU by deeptables_b200.importance.

Differences from the reference: the result is sorted by the numeric importance (the reference sorts the strings), and
nothing is printed per pass.  The aliases 'roc_auc' and 'logloss' score probabilities, as 'auc' and 'log_loss' do.
"""
import numpy as np

from .. import importance


def get_score_importances(dt_model, X, y, metric, n_iter=5, mode='min', *, random_state=None, batch_size=65536):
    """Mean decrease of the score over ``n_iter`` random permutations of each column of ``X``.

    The score of a pass is ``metric`` on the current model's predictions, negated when ``mode == 'min'``.  ``metric``
    is one of the scikit-learn names ``fit_cross_validation(oof_metrics=)`` takes ('auc', 'log_loss', 'accuracy',
    'f1', 'mse', 'rmse', 'mae', 'r2' and their aliases) or a streaming metric of ``deeptables_b200.metrics`` (object
    or name).  ``random_state``: an int in [0, 2**32) or None (a seed drawn from numpy's global generator).
    ``batch_size``: rows per forward call.  Returns a ``(n_columns, 2)`` string array of ``[column, importance]``
    rows, sorted by importance, highest first."""
    res = importance.score_decreases(dt_model, X, y, metric.lower() if isinstance(metric, str) else metric,
                                     n_iter=n_iter, mode=mode, random_state=random_state, batch_size=batch_size)
    feature_importances = np.stack([res.columns, np.mean(res.decreases, axis=0)], axis=1)
    return np.array(sorted(feature_importances, key=lambda fi: float(fi[1]), reverse=True))


def select_features(feature_importances, threshold=0.):
    """Column names split at ``float(importance) > threshold``: (selected, discarded)."""
    selected_columns = [fi[0] for fi in feature_importances if float(fi[1]) > threshold]
    discard_columns = [fi[0] for fi in feature_importances if float(fi[1]) <= threshold]
    return selected_columns, discard_columns
