"""What the search families do with a column's fit status, host side (no GPU).

An engine double forces chosen statuses (and, for SGD, epoch counts) on the columns fitted with chosen C / alpha
values.  Per family this pins which columns' test scores become NaN (the search then applies error_score),
whether their train scores do too, and which convergence warnings a search raises:

  binary logistic   status 5 masks test and train scores; one warning per launch with a status 3 or 4 column
  multinomial       nothing is masked; no warning
  SGD               a diverged class column masks test and train scores; one warning per fold layout when a
                    non-diverged column ran max_iter epochs with tol set
  Ridge             status != 1 masks test scores only; no warning"""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import LogisticRegression, Ridge, SGDClassifier

from skdist.distribute.search import DistGridSearchCV
from skdist_b200 import engine
from skdist_b200.datasets import make_g1_classification, make_multiclass
from skdist_b200.distribute.sgd_family import _SGDFamily
from skdist_b200.distribute.utils import _check_multimetric_scoring
from tests.sgd_fake_engine import SGDFakeEngine
from tests.weighted_fake_engine import WeightedFakeEngine

CV = 3
ERROR = -1.0
LBFGS_MSG = "lbfgs failed to converge within max_iter=%d for %d of %d (candidate, fold) fits"
SGD_MSG = "Maximum number of iteration reached before convergence. Consider increasing max_iter to improve the fit."


class _ForcedEngine(WeightedFakeEngine, SGDFakeEngine):
    """Fits as its bases do, then reports status[v][k] (and, for SGD, n_iter[v][k]) for engine column k of
    every fit whose C / alpha is v (k: class column within an SGD fit, 0 otherwise)."""

    def __init__(self, status, n_iter):
        super().__init__()
        self.force_status, self.force_iter = status, n_iter

    def _force(self, res, values):
        for key, force in (("status", self.force_status), ("n_iter", self.force_iter)):
            for j, v in enumerate(values):
                if float(v) in force:
                    f = force[float(v)]
                    res[key][j] = f[j % len(f)]
        return res

    def logreg_fit_batch(self, C, *args, **kw):
        return self._force(super().logreg_fit_batch(C, *args, **kw), C)

    def logreg_multinomial_fit_batch(self, C, *args, **kw):
        return self._force(super().logreg_multinomial_fit_batch(C, *args, **kw), C)

    def ridge_fit_batch(self, alpha, *args, **kw):
        return self._force(super().ridge_fit_batch(alpha, *args, **kw), alpha)

    def sgd_fit_groups(self, params, col_pos, col_group, col_alpha, group_rows, group_seeds):
        return self._force(super().sgd_fit_groups(params, col_pos, col_group, col_alpha, group_rows, group_seeds),
                           col_alpha)


@pytest.fixture
def forced():
    """Dict {"status": {value: [status per class column]}, "n_iter": {...}} the engine reads at creation."""
    cfg = {"status": {}, "n_iter": {}}
    engine.set_engine_factory(lambda: _ForcedEngine(cfg["status"], cfg["n_iter"]))
    yield cfg
    engine.set_engine_factory(None)


def _search(est, grid, X, y, scoring=None):
    """(cv_results_, ConvergenceWarning messages) of a grid search with train scores and error_score=ERROR."""
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        gs = DistGridSearchCV(est, grid, cv=CV, scoring=scoring, refit=False, error_score=ERROR,
                              return_train_score=True).fit(X, y)
    return gs.cv_results_, [str(w.message) for w in rec if issubclass(w.category, ConvergenceWarning)]


def _splits(res, kind, name="score"):
    return np.stack([res["split%d_%s_%s" % (i, kind, name)] for i in range(CV)], axis=1)


def _check_masks(res, bad, train_masked, name="score"):
    """Candidates `bad` carry error_score in every test split and NaN (train_masked) or a finite value in
    every train split; every other candidate is finite everywhere."""
    test, train = _splits(res, "test", name), _splits(res, "train", name)
    bad = np.asarray(bad, bool)
    assert np.all(test[bad] == ERROR) and np.all(np.isfinite(test[~bad])) and not np.any(test[~bad] == ERROR)
    assert np.all(np.isnan(train[bad]) if train_masked else np.isfinite(train[bad]))
    assert np.all(np.isfinite(train[~bad]))


def test_binary_logreg_masks_status_5_and_warns_once_per_launch(forced):
    forced["status"].update({1.0: [3], 2.0: [4], 10.0: [5]})
    X, y = make_g1_classification(300, 5, seed=1)
    grid = [{"C": [0.1, 1.0, 2.0, 10.0], "tol": [1e-4]},      # one launch: statuses 1, 3, 4, 5
            {"C": [0.1, 10.0], "tol": [1e-3]},                # one launch: statuses 1 and 5 only
            {"C": [2.0], "max_iter": [50]}]                   # one launch: status 4 only
    res, msgs = _search(LogisticRegression(), grid, X, y)
    _check_masks(res, [False, False, False, True, False, True, False], train_masked=True)
    assert msgs == [LBFGS_MSG % (100, 2 * CV, 4 * CV), LBFGS_MSG % (50, CV, CV)]


def test_multinomial_masks_nothing_and_never_warns(forced):
    forced["status"].update({1.0: [3], 10.0: [5]})
    X, y = make_multiclass(300, 5, 3, seed=2)
    res, msgs = _search(LogisticRegression(max_iter=50), {"C": [0.1, 1.0, 10.0]}, X, y, scoring="f1_macro")
    _check_masks(res, [False, False, False], train_masked=False)
    assert msgs == []


def test_ridge_masks_test_scores_only_and_never_warns(forced):
    forced["status"].update({1.0: [4], 10.0: [2]})
    X, _ = make_g1_classification(300, 5, seed=3)
    y = X @ np.arange(1.0, 6.0) + np.random.default_rng(3).normal(size=300)
    for scoring in (None, "neg_mean_squared_error", "neg_root_mean_squared_error"):
        res, msgs = _search(Ridge(), {"alpha": [0.1, 1.0, 10.0]}, X, y, scoring=scoring)
        _check_masks(res, [False, True, True], train_masked=False)
        assert msgs == []


ALPHAS = [1e-4, 1e-3, 1e-2]


@pytest.mark.parametrize("loss", ["hinge", "log_loss"])
def test_binary_sgd_masks_diverged_columns(forced, loss):
    forced["status"].update({1e-3: [5]})
    X, y = make_g1_classification(300, 5, seed=4)
    res, _ = _search(SGDClassifier(loss=loss, random_state=0, max_iter=5, tol=None), {"alpha": ALPHAS}, X, y)
    _check_masks(res, [False, True, False], train_masked=True)


def test_multiclass_sgd_masks_a_fit_with_one_diverged_class(forced):
    forced["status"].update({1e-2: [1, 5, 1]})
    X, y = make_multiclass(300, 5, 3, seed=5)
    res, _ = _search(SGDClassifier(random_state=0, max_iter=5, tol=None), {"alpha": ALPHAS}, X, y,
                     scoring="accuracy")
    _check_masks(res, [False, False, True], train_masked=True)


@pytest.mark.parametrize("case, n_warn", [
    ("hit_in_two_launches", 1),         # one warning per fold layout, not per launch
    ("hit_only_when_diverged", 0),      # a diverged column's epoch count does not warn
    ("hit_with_tol_none", 0),           # without tol every fit runs max_iter epochs
])
def test_sgd_warns_once_when_a_live_column_hits_max_iter(forced, case, n_warn):
    X, y = make_g1_classification(300, 5, seed=6)
    tol = None if case == "hit_with_tol_none" else 1e-3
    grid = {"alpha": ALPHAS, "fit_intercept": [True, False]}
    if case == "hit_only_when_diverged":
        forced["status"].update({1e-2: [5]})
        forced["n_iter"].update({1e-2: [1000]})
    else:
        forced["n_iter"].update({1e-3: [1000]})
    res, msgs = _search(SGDClassifier(random_state=0, max_iter=1000, tol=tol), grid, X, y)
    assert msgs == [SGD_MSG] * n_warn


def test_sgd_status_and_n_iter_reduce_over_class_columns(forced):
    """A fit's status: SGD_DIVERGED when any class column diverged, else the least class status; its n_iter:
    the most epochs of its class columns."""
    forced["status"].update({1e-4: [3, 1, 3], 1e-3: [1, 5, 3], 1e-2: [3, 3, 3]})
    forced["n_iter"].update({1e-4: [2, 4, 3], 1e-3: [1, 1, 6]})
    X, y = make_multiclass(300, 5, 3, seed=7)
    est = SGDClassifier(random_state=0, max_iter=6, tol=1e-3)
    scorers, _ = _check_multimetric_scoring(est, scoring="accuracy")
    family = _SGDFamily(est, [{"alpha": a} for a in ALPHAS], X, y, scorers)
    eng = engine.get_engine()
    fold = np.arange(len(y)) % CV
    family.stage(eng, X, fold, CV)
    family.set_train_rows([None] * CV)
    cols = np.arange(len(ALPHAS) * CV)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", ConvergenceWarning)
        out = family.run_columns(eng, cols, CV, True)
    np.testing.assert_array_equal(out["status"], np.repeat([1, 5, 3], CV))
    np.testing.assert_array_equal(out["n_iter"][:2 * CV], np.repeat([4, 6], CV))
    assert np.isnan(out["test_score"][CV:2 * CV]).all() and np.isnan(out["train_score"][CV:2 * CV]).all()
    assert np.isfinite(out["test_score"][:CV]).all() and np.isfinite(out["test_score"][2 * CV:]).all()
