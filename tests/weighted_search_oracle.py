"""The reference's search fan-out with fit_params -- TEST INFRASTRUCTURE ONLY.

oracle/search_oracle.py restates DistBaseSearchCV.fit and _fit_and_score with fit_params={}; this module adds
the fit_params the reference routes (ref search.py:180-288, 315-571):
  * fit_and_score()  indexes every fit param by the task's training rows        search.py:208-211
                     (_index_param_value: arrays of n_samples entries only), fits with them; the scorer
                     stays unweighted: scorer(est, X_test, y_test)              search.py:264
  * search_cv()      oracle.search_oracle.search_cv with that task, and the refit
                     on (X, y) with the full arrays                             search.py:543-550
scikit-learn's own GridSearchCV also passes sample_weight to the scorer, so its cv_results_ differ from these."""
from functools import partial

import numpy as np
from sklearn.base import clone
from sklearn.utils import _safe_indexing
from sklearn.utils.validation import _is_arraylike, _num_samples

from oracle import search_oracle


def index_param_value(X, v, indices):
    """ref search.py _index_param_value: a fit param with one entry per sample, restricted to `indices`."""
    if not _is_arraylike(v) or _num_samples(v) != _num_samples(X):
        return v
    return _safe_indexing(v, indices)


def fit_and_score(estimator, X, y, scorer, train, test, parameters, fit_params=None):
    """oracle.search_oracle.fit_and_score with the fit params of the task's training rows."""
    fp = {k: index_param_value(X, v, train) for k, v in (fit_params or {}).items()}
    est = clone(estimator)
    if parameters is not None:
        est.set_params(**parameters)
    est.fit(X[train], y[train], **fp)
    test_score = scorer(est, X[test], y[test])
    if hasattr(test_score, "item"):
        test_score = test_score.item()
    return [{"score": test_score}, len(test), 0.0, 0.0]


def search_cv(estimator, candidate_params, X, y, cv=5, scoring=None, iid=True, refit=True, fit_params=None,
              task_fn=None):
    """oracle.search_oracle.search_cv with fit_params: each task fits with the params of its training rows,
    the refit with the full ones.  task_fn as in search_oracle.search_cv (fit_params are the caller's then)."""
    fit_params = fit_params or {}
    if task_fn is None:
        task_fn = partial(fit_and_score, fit_params=fit_params)
    res = search_oracle.search_cv(estimator, candidate_params, X, y, cv=cv, scoring=scoring, iid=iid, refit=False,
                                  task_fn=task_fn)
    if refit:
        res["best_estimator_"] = clone(estimator).set_params(**res["best_params_"]).fit(X, y, **fit_params)
    return res


def sample_weight_case(n_classes):
    """(X, y, sample_weight, candidates, cv) of the fixture tests/golden/sample_weight_pins.npz records."""
    from sklearn.model_selection import ParameterGrid, StratifiedKFold
    from skdist_b200.datasets import make_g1_classification
    X, y = make_g1_classification(900, 7, seed=41 + n_classes)
    rng = np.random.default_rng(5 + n_classes)
    if n_classes > 2:
        y = np.minimum(rng.integers(0, n_classes + 2, len(y)), n_classes - 1)
    w = np.exp(rng.normal(0.0, 1.0, len(y)))
    w[rng.random(len(y)) < 0.1] = 0.0
    cw3 = {c: 1.0 + 0.5 * c for c in range(n_classes)}
    cands = list(ParameterGrid({"C": [0.03, 1.0], "class_weight": [None, "balanced", cw3]}))
    return X, y, w, cands, StratifiedKFold(3)
