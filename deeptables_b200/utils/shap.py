"""Kernel SHAP explanations of a fitted DeepTable (reference deeptables/utils/shap.py over shap.KernelExplainer),
computed on the GPU by deeptables_b200.explain, and expected gradients (shap.GradientExplainer's method) of its output
layer (``DeepTablesGradientExplainer``).

The explained quantity is the reference's model function, ``predict(X, encode_to_label=False)``: the prediction on
regression, the class code on the classification tasks.  Differences from shap: no L1 feature selection when the
coalitions are sampled, the identity link only, one output only, and the random coalitions are drawn from a generator
seeded per explained row (``random_state``), not from numpy's global one.
"""
import numpy as np
import pandas as pd

from .. import explain
from ..analysis import check_positive_int, draw_seed, is_int


class KernelExplainer:
    """What the reference reads of its ``shap.KernelExplainer``: ``expected_value``, the mean of the model function
    over the background rows (float64)."""

    def __init__(self, expected_value):
        self.expected_value = np.float64(expected_value)


def _background_rows(X, num_samples):
    """shap.sample's rule: ``num_samples`` rows of X drawn without replacement with random_state 0, or all of X."""
    if num_samples is not None and num_samples < len(X):
        from sklearn.utils import resample
        return resample(X, n_samples=num_samples, random_state=0, replace=False)
    return X


def _init_explainer(ex, dt_model, X, num_samples, random_state, batch_size):
    """What both explainers check and set up: the arguments, the attributes and the background."""
    if random_state is not None:
        draw_seed(random_state)                             # validates it
    check_positive_int(batch_size, 'batch_size')
    if num_samples is not None and (not is_int(num_samples) or num_samples < 1):
        raise ValueError(f'num_samples must be None or a positive integer, got {num_samples!r}')
    ex.dt_model = dt_model
    ex.num_samples = num_samples
    ex.feature_names = X.columns.to_list()
    ex.random_state = random_state
    ex.batch_size = int(batch_size)
    ex._background = explain.Background(dt_model, _background_rows(X, num_samples), ex.batch_size)


def _as_frame(X, feature_names):
    if isinstance(X, pd.DataFrame):
        return X
    return pd.DataFrame(np.asarray(X, dtype=object).reshape(-1, len(feature_names)), columns=feature_names)


class DeepTablesExplainer:
    def __init__(self, dt_model, X, num_samples=50, *, random_state=None, batch_size=65536):
        """Kernel SHAP against a background of ``num_samples`` rows of ``X`` drawn without replacement (shap.sample's
        rule: ``sklearn.utils.resample(X, n_samples=num_samples, random_state=0, replace=False)``), or all of ``X``
        when ``num_samples`` is None or at least ``len(X)``.

        ``random_state``: an int in [0, 2**32) seeding the random coalitions, or None for a seed drawn from numpy's
        global generator at each ``get_shap_values`` call (rank 0's under data parallel).  ``batch_size``: rows per
        forward call."""
        _init_explainer(self, dt_model, X, num_samples, random_state, batch_size)
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
        X_to_explain = _as_frame(X_to_explain, self.feature_names)
        seed = draw_seed(self.random_state)
        return explain.shap_values(self._background, X_to_explain, nsamples, seed, self.batch_size)


class DeepTablesGradientExplainer:
    def __init__(self, dt_model, X, num_samples=50, *, random_state=None, batch_size=65536):
        """Expected gradients (shap.GradientExplainer's method with ``local_smoothing=0``) of the model's output layer
        against a background of ``num_samples`` rows of ``X``, chosen as ``DeepTablesExplainer`` chooses them.

        The explained output is the output layer, not ``predict``'s class code (a class code has no gradient): the
        sigmoid probability (binary), the prediction (regression), every output column (multiclass: the softmax,
        multilabel: the sigmoids).  For explained row x and each of ``nsamples`` samples, a background row b is drawn
        uniformly with replacement and alpha uniformly on [0, 1); the model's inputs are interpolated at
        b + alpha * (x - b) -- a categorical column on its embedding, a continuous column on the encoded, scaled value
        the model reads -- and the column's value of the sample is the gradient there times x - b (summed over the
        embedding coordinates).  A column's attribution is the mean over the samples.  The method is restated from
        shap's description; shap itself is not a dependency, and the draws (from ``np.random.RandomState([seed, i])``
        for row i) are not shap's.  Columns the model does not read get exactly 0.  ``apply_gbm_features`` and
        ``auto_discrete`` models are refused (NotImplementedError): their derived columns are step functions of the
        continuous inputs, whose jumps a gradient cannot attribute.

        ``random_state``: an int in [0, 2**32) seeding the draws, or None for a seed drawn from numpy's global generator
        at each call (rank 0's under data parallel).  ``batch_size``: interpolated rows per forward and backward.

        Attributes: ``dt_model``, ``num_samples``, ``feature_names`` and, beyond shap's, ``expected_value``: the float64
        mean of the explained output over the background (a scalar, or one value per output column)."""
        explain.check_gradient_options(dt_model)
        _init_explainer(self, dt_model, X, num_samples, random_state, batch_size)
        bg = self._background
        means = explain.output_means(bg, bg.cat, bg.cont, bg.rows, self.batch_size)
        self.expected_value = np.float64(means[0]) if bg.cols == 1 else means

    def get_shap_values(self, X_to_explain, nsamples=200):
        """Expected gradients at each row of ``X_to_explain`` (a DataFrame with the explainer's columns, or a 2-D array
        of them), float64: ``(n_rows, n_columns)`` on binary and regression models, ``(n_rows, n_columns,
        n_outputs)`` on multiclass and multilabel ones (output column last; shap's own layout for several outputs
        differs between its versions).  ``nsamples``: samples per row, a positive int.  Each row sums to about the
        output at that row minus ``expected_value``; the error shrinks as ``nsamples`` grows."""
        check_positive_int(nsamples, 'nsamples')
        X_to_explain = _as_frame(X_to_explain, self.feature_names)
        if X_to_explain.columns.to_list() != self._background.columns:
            raise ValueError(f'X_to_explain has columns {X_to_explain.columns.to_list()}, the explainer '
                             f'{self._background.columns}')
        seed = draw_seed(self.random_state)
        phi = explain.gradient_values(self._background, X_to_explain, nsamples, seed, self.batch_size)
        return phi[:, :, 0] if self._background.cols == 1 else phi
