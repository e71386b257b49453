"""Feature engineering over numeric data (reference deeptables/fe)."""
