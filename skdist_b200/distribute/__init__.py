"""H100-native counterparts of ``skdist.distribute`` (reference skdist/distribute/__init__.py)."""
__all__ = ["search", "multiclass", "ensemble", "predict", "eliminate"]
