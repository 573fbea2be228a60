"""Drop-in alias: ``import skdist`` resolves to the H100-native implementation
(package ``skdist_b200``), keeping the reference's import paths
(``skdist.distribute.search.DistGridSearchCV`` ...)."""
__version__ = "0.1.9+b200"
__all__ = ["distribute"]
