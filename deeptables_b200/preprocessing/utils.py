"""The reference's deeptables/preprocessing/utils.py ``target_encoding``, computed on the GPU by
deeptables_b200.target_encoding.

Differences from the reference: nothing is printed, it runs on pandas 2 and later (the reference calls the removed
``DataFrame.append``), and it needs no category_encoders: the formula is restated from memory of that package (see the
README).  ``target_rate_encodeing`` is not ported: the reference returns its input frame without the columns it
computes.
"""
from ..target_encoding import target_encoding

__all__ = ['target_encoding']
