"""Utilities over a fitted DeepTable (reference deeptables/utils)."""
