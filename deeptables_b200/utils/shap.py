"""Kernel SHAP explanations of a fitted DeepTable (reference deeptables/utils/shap.py over shap.KernelExplainer),
computed on the GPU by deeptables_b200.explain.

The explained quantity is the reference's model function, ``predict(X, encode_to_label=False)``: the prediction on
regression, the class code on the classification tasks.  Differences from shap: no L1 feature selection when the
coalitions are sampled, the identity link only, one output only, and the random coalitions are drawn from a generator
seeded per explained row (``random_state``), not from numpy's global one.
"""
import numbers

import numpy as np
import pandas as pd

from .. import explain, importance


class KernelExplainer:
    """What the reference reads of its ``shap.KernelExplainer``: ``expected_value``, the mean of the model function
    over the background rows (float64)."""

    def __init__(self, expected_value):
        self.expected_value = np.float64(expected_value)


class DeepTablesExplainer:
    def __init__(self, dt_model, X, num_samples=50, *, random_state=None, batch_size=65536):
        """Kernel SHAP against a background of ``num_samples`` rows of ``X`` drawn without replacement (shap.sample's
        rule: ``sklearn.utils.resample(X, n_samples=num_samples, random_state=0, replace=False)``), or all of ``X``
        when ``num_samples`` is None or at least ``len(X)``.

        ``random_state``: an int in [0, 2**32) seeding the random coalitions, or None for a seed drawn from numpy's
        global generator at each ``get_shap_values`` call (rank 0's under data parallel).  ``batch_size``: rows per
        forward call."""
        if random_state is not None:
            importance.draw_seed(random_state)                  # validates it
        if isinstance(batch_size, bool) or not isinstance(batch_size, numbers.Integral) or batch_size < 1:
            raise ValueError(f'batch_size must be a positive integer, got {batch_size!r}')
        if num_samples is not None and (isinstance(num_samples, bool) or not isinstance(num_samples, numbers.Integral)
                                        or num_samples < 1):
            raise ValueError(f'num_samples must be None or a positive integer, got {num_samples!r}')
        self.dt_model = dt_model
        self.num_samples = num_samples
        self.feature_names = X.columns.to_list()
        self.random_state = random_state
        self.batch_size = int(batch_size)
        if num_samples is not None and num_samples < len(X):
            from sklearn.utils import resample
            samples = resample(X, n_samples=num_samples, random_state=0, replace=False)
        else:
            samples = X
        self._background = explain.Background(dt_model, samples, self.batch_size)
        self.explainer = KernelExplainer(self._background.expected)

    def model_fn(self, data_asarray):
        """The explained function on the host (pandas and ``predict``): one value per row of ``data_asarray``."""
        data_asframe = pd.DataFrame(data_asarray, columns=self.feature_names)
        return self.dt_model.predict(data_asframe, encode_to_label=False)

    def get_shap_values(self, X_to_explain, nsamples='auto'):
        """float64 ``(n_rows, n_columns)`` SHAP values of the model function at each row of ``X_to_explain`` (a
        DataFrame with the explainer's columns, or a 2-D array of them).  Each row plus ``explainer.expected_value``
        sums to the model function at that row.  ``nsamples``: coalitions per row, ``'auto'`` (2M + 2048 for M varying
        columns) or a positive int, at most 2^M - 2 when M <= 30."""
        explain.check_nsamples(nsamples)
        if not isinstance(X_to_explain, pd.DataFrame):
            X_to_explain = pd.DataFrame(np.asarray(X_to_explain, dtype=object).reshape(-1, len(self.feature_names)),
                                        columns=self.feature_names)
        seed = importance.draw_seed(self.random_state)
        return explain.shap_values(self._background, X_to_explain, nsamples, seed, self.batch_size)
