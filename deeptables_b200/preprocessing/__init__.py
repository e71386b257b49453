"""Preprocessing helpers computed on the GPU.  ``TargetEncoder`` is scikit-learn 1.9's target encoder; the module
``utils`` holds the reference's ``target_encoding`` helper.  Both live in deeptables_b200.target_encoding."""
from ..target_encoding import TargetEncoder

__all__ = ['TargetEncoder']
