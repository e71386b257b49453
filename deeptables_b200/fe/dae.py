"""Denoising auto-encoder features (reference deeptables/fe/dae.py), trained on the GPU by deeptables_b200.dae.

``DAE(...).fit_transform(X)`` trains the reference's ``build_dae`` auto-encoder on X and returns its ``feature_layer``
activations.  Differences from the reference: every epoch reshuffles the rows (the reference's noise generator does not
when the batch size divides N), NaN or infinite inputs are refused, each ``fit`` starts a fresh optimiser,
``random_state`` seeds the weights, permutations and noise, and nothing is printed.
"""
from ..dae import AutoEncoder, DAE

__all__ = ['AutoEncoder', 'DAE']
