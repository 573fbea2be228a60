"""Validation helpers (host side); mirrors /root/reference/skdist/distribute/validation.py
for the functions the hot path calls: ``_check_estimator`` (validation.py:14-20) and
``_check_is_fitted`` (validation.py:23-29)."""
from sklearn.utils.validation import check_is_fitted


def _check_estimator(estimator, verbose=False):
    """Print backend awareness (ref validation.py:14-20: spark vs local).  Here the
    backend is always the H100 engine; ``sc`` is accepted and ignored."""
    if verbose:
        from .. import parallel
        rank, world, _ = parallel.dist_info()
        if rank == 0:
            print("skdist_b200: running on %d H100 process(es); sc=%s is ignored"
                  % (world, "None" if getattr(estimator, "sc", None) is None else "given"))


def _check_is_fitted(estimator, attributes=None):
    return check_is_fitted(estimator)


def _validate_models(models, clf):
    """Validate the `models` argument of DistMultiModelSearch (ref validation.py:43-96): a list of
    (name, estimator, param_set) tuples with unique string names that do not clash with the
    constructor arguments and do not contain '__'."""
    try:
        iter(models)
    except TypeError:
        raise TypeError("Input argument 'models' is not iterable.")
    if not isinstance(models[0], (tuple, list)):
        models = [models]
    names, estimators, param_sets = zip(*models)
    if len(set(names)) != len(names):
        raise ValueError("Names provided are not unique: {0!r}".format(list(names)))
    bad = [name for name in names if not isinstance(name, str)]
    if bad:
        raise ValueError("Estimator names must be strings: got {0!r}".format(bad))
    bad = set(names).intersection(clf.get_params(deep=False))
    if bad:
        raise ValueError("Estimator names conflict with constructor arguments: {0!r}".format(sorted(bad)))
    bad = [name for name in names if "__" in name]
    if bad:
        raise ValueError("Estimator names must not contain __: got {0!r}".format(bad))
    bad = [type(e) for e in estimators if not (hasattr(e, "fit") and hasattr(e, "predict"))]
    if bad:
        raise ValueError("Estimators must be sklearn estimators: got {0!r}".format(bad))
    bad = [p for p in param_sets if not isinstance(p, dict)]
    if bad:
        raise ValueError("Parameter sets must be dictionaries: got {0!r}".format(bad))
    return models


def _check_n_iter(n_iter, param_distributions):
    """min(n_iter, grid size) when every distribution is a list (ref validation.py:99-111)."""
    import numpy as np
    from sklearn.model_selection import ParameterGrid
    if np.all([not hasattr(v, "rvs") for v in param_distributions.values()]):
        return min(len(ParameterGrid(param_distributions)), n_iter)
    return n_iter
