"""SGDClassifier cross-validation on the device (run with -m gpu on an H100).

Engine level: `Engine.sgd_fit_groups` runs (alpha, fold) columns in order groups, each group walking its fold's
training rows in its own shuffled order.  Hinge fits must equal `SGDClassifier(alpha=a, ...).fit(X[train],
y[train])` bit for bit (coef_, intercept_, n_iter_, t_).  log_loss goes through CUDA's exp / log, so it is
compared within 1e-5 of the coefficient scale under small constant / invscaling steps, as tests/test_sgd_gpu.py
does for one-vs-rest.

Public API: DistGridSearchCV(SGDClassifier) refits bit for bit, and its split scores equal scikit-learn's except
for test rows whose device decision value lies within fp32 rounding of 0 (the scoring kernels form the decision
in fp32, scikit-learn adds the float64 intercept)."""
import warnings

import numpy as np
import pytest
from sklearn.datasets import load_digits
from sklearn.linear_model import SGDClassifier
from sklearn.model_selection import GridSearchCV, check_cv

from skdist_b200.datasets import make_g1_classification, make_multiclass
from skdist_b200.distribute.sgd_family import sgd_class_seeds

pytestmark = pytest.mark.gpu

ALPHAS = np.logspace(-6, -1, 8)
LOG_STEPS = {"constant": {"learning_rate": "constant", "eta0": 1e-3},
             "invscaling": {"learning_rate": "invscaling", "eta0": 0.01}}


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _folds(n, seed):
    """Training rows of 3 folds of unequal size; the second in a permuted order (as ShuffleSplit gives them)."""
    rs = np.random.RandomState(seed)
    cuts = [0, n // 5, n // 5 + n // 3, n]
    rows = []
    for f in range(3):
        test = np.arange(cuts[f], cuts[f + 1])
        train = np.setdiff1d(np.arange(n), test)
        rows.append(rs.permutation(train) if f == 1 else train)
    return rows


def _params(**kw):
    p = SGDClassifier(random_state=5).get_params()
    p.update(kw)
    return p


def _fit_groups(eng, X, y, params, rows, n_classes=2):
    """Every (alpha, fold[, class]) column in one call; returns the result and the column layout."""
    eng.stage_x(X)
    eng.stage_labels(y)
    Kc = 1 if n_classes == 2 else n_classes
    seeds = sgd_class_seeds(params["random_state"], n_classes)
    group_rows, group_seeds, cols = [], [], []
    for f, r in enumerate(rows):
        for k in range(Kc):
            group_rows.append(r)
            group_seeds.append(seeds[k])
    for a in ALPHAS:
        for f in range(len(rows)):
            for k in range(Kc):
                cols.append((a, f, k))
    col_pos = np.array([k if Kc > 1 else 1 for _, _, k in cols], np.int32)
    col_group = np.array([f * Kc + k for _, f, k in cols], np.int32)
    col_alpha = np.array([a for a, _, _ in cols])
    res = eng.sgd_fit_groups(params, col_pos, col_group, col_alpha, group_rows, np.array(group_seeds, np.uint32))
    return res, cols


def _reference(X, y, params, alpha, train):
    p = dict(params, alpha=alpha)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return SGDClassifier(**p).fit(X[train], y[train])


@pytest.mark.parametrize("d", [12, 300])
@pytest.mark.parametrize("shuffle", [True, False])
@pytest.mark.parametrize("lr", ["optimal", "constant", "invscaling"])
def test_hinge_groups_bit_identical(eng, d, shuffle, lr):
    n = 1500
    X, y = make_g1_classification(n, d, seed=d)
    params = _params(loss="hinge", shuffle=shuffle, learning_rate=lr, eta0=0.01, max_iter=60)
    rows = _folds(n, d)
    res, cols = _fit_groups(eng, X, y.astype(np.int32), params, rows)
    for j, (a, f, _) in enumerate(cols):
        ref = _reference(X, y, params, a, rows[f])
        np.testing.assert_array_equal(res["coef32"][j], ref.coef_[0], err_msg=str((a, f)))
        assert res["intercept"][j] == ref.intercept_[0], (a, f)
        assert res["n_iter"][j] == ref.n_iter_ and res["t"][j] == ref.t_, (a, f)


@pytest.mark.parametrize("d", [12, 300])
@pytest.mark.parametrize("step", sorted(LOG_STEPS))
def test_log_loss_groups_within_envelope(eng, d, step):
    n = 1500
    X, y = make_g1_classification(n, d, seed=d + 1)
    params = _params(loss="log_loss", max_iter=40, **LOG_STEPS[step])
    rows = _folds(n, d + 1)
    res, cols = _fit_groups(eng, X, y.astype(np.int32), params, rows)
    for j, (a, f, _) in enumerate(cols):
        ref = _reference(X, y, params, a, rows[f])
        scale = max(np.abs(ref.coef_).max(), 1e-30)
        assert res["n_iter"][j] == ref.n_iter_ and res["t"][j] == ref.t_, (a, f)
        assert np.abs(res["coef32"][j] - ref.coef_[0]).max() <= 1e-5 * scale, (a, f)
        assert abs(res["intercept"][j] - ref.intercept_[0]) <= 1e-5 * max(scale, abs(ref.intercept_[0])), (a, f)


def test_four_classes_per_class_seeds(eng):
    n, d, K = 1200, 20, 4
    X, y = make_multiclass(n, d, K, seed=3)
    params = _params(loss="hinge", random_state=17)
    rows = _folds(n, 4)
    res, cols = _fit_groups(eng, X, y.astype(np.int32), params, rows, n_classes=K)
    for a in ALPHAS[::3]:
        for f in range(3):
            ref = _reference(X, y, params, a, rows[f])
            js = [j for j, c in enumerate(cols) if c[0] == a and c[1] == f]
            np.testing.assert_array_equal(res["coef32"][js], ref.coef_)
            np.testing.assert_array_equal(res["intercept"][js].astype(np.float32), ref.intercept_)
            assert res["n_iter"][js].max() == ref.n_iter_
            assert 1.0 + res["n_iter"][js].max() * len(rows[f]) == ref.t_


def test_large_groups_stay_on_the_warp_kernels(eng, monkeypatch, capfd):
    """n >= 2 ST_T rows, where the one-vs-rest entry takes the tensor-core path: the group entry runs the warp
    kernels and is bit-identical."""
    n, d = 2 * 2048 + 700, 40
    X, y = make_g1_classification(n, d, seed=21)
    monkeypatch.setenv("SKDIST_B200_TRACE", "2")
    params = _params(loss="hinge", max_iter=12)
    rows = [np.arange(n), np.arange(n // 3, n)]
    eng.stage_x(X)
    eng.stage_labels(y.astype(np.int32))
    seed = sgd_class_seeds(params["random_state"], 2)[0]
    alphas = np.array([1e-5, 1e-4, 1e-3, 1e-5])
    res = eng.sgd_fit_groups(params, np.ones(4, np.int32), np.array([0, 0, 0, 1], np.int32), alphas, rows,
                             np.array([seed, seed], np.uint32))
    err = capfd.readouterr().err
    assert "[skd trace] sgd epoch" in err and "sgd-tc" not in err
    for j, g in enumerate([0, 0, 0, 1]):
        ref = _reference(X, y, params, alphas[j], rows[g])
        np.testing.assert_array_equal(res["coef32"][j], ref.coef_[0])
        assert res["intercept"][j] == ref.intercept_[0] and res["n_iter"][j] == ref.n_iter_


def test_bad_arguments_are_refused(eng):
    from skdist_b200._lib import SkdError
    X, y = make_g1_classification(200, 5, seed=1)
    eng.stage_x(X)
    eng.stage_labels(y.astype(np.int32))
    p = _params()
    one = np.ones(1, np.int32)
    with pytest.raises(SkdError, match="alpha <= 0"):
        eng.sgd_fit_groups(p, one, np.zeros(1, np.int32), np.zeros(1), [np.arange(200)], np.ones(1, np.uint32))
    with pytest.raises(SkdError, match="not in \\[0, G\\)"):
        eng.sgd_fit_groups(p, one, np.ones(1, np.int32), np.ones(1), [np.arange(200)], np.ones(1, np.uint32))
    with pytest.raises(SkdError, match="is empty"):
        eng.sgd_fit_groups(p, one, np.zeros(1, np.int32), np.ones(1), [np.arange(0)], np.ones(1, np.uint32))


# ---------------------------------------------------------------------------------------------------------------
# public API
# ---------------------------------------------------------------------------------------------------------------
def _near_zero_rows(est, X, test):
    """Test rows whose fp32 decision value (what the scoring kernels form) lies within fp32 rounding of 0."""
    coef = est.coef_.astype(np.float32)
    z = X[test] @ coef.T + est.intercept_.astype(np.float32)
    scale = np.abs(X[test]) @ np.abs(coef.T) + np.abs(est.intercept_)
    return int(np.sum(np.any(np.abs(z) <= 4 * np.finfo(np.float32).eps * scale, axis=1)))


@pytest.mark.parametrize("dataset", ["g1", "digits"])
def test_grid_search_matches_scikit_learn(dataset):
    if dataset == "g1":
        X, y = make_g1_classification(20000, 32, seed=4)
        scoring, grid = "accuracy", {"alpha": [1e-5, 1e-4, 1e-3, 1e-2]}
    else:
        X, y = load_digits(return_X_y=True)
        X = (X / 16.0).astype(np.float32)
        scoring, grid = "f1_weighted", {"alpha": [1e-4, 1e-3, 1e-2]}
    est = SGDClassifier(random_state=0)
    from skdist.distribute.search import DistGridSearchCV
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = DistGridSearchCV(est, grid, cv=5, scoring=scoring).fit(X, y)
        ref = GridSearchCV(est, grid, cv=5, scoring=scoring).fit(X, y)
    np.testing.assert_array_equal(ours.best_estimator_.coef_, ref.best_estimator_.coef_)
    np.testing.assert_array_equal(ours.best_estimator_.intercept_, ref.best_estimator_.intercept_)
    assert ours.best_estimator_.n_iter_ == ref.best_estimator_.n_iter_ and ours.best_estimator_.t_ == ref.best_estimator_.t_
    folds = list(check_cv(5, y, classifier=True).split(X, y))
    for ci, p in enumerate(ref.cv_results_["params"]):
        for s, (train, test) in enumerate(folds):
            a, b = ours.cv_results_["split%d_test_score" % s][ci], ref.cv_results_["split%d_test_score" % s][ci]
            if a != b:
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore")
                    fitted = SGDClassifier(random_state=0, **p).fit(X[train], y[train])
                near = _near_zero_rows(fitted, X, test)
                assert abs(a - b) <= near / len(test) + 1e-12, (p, s, a, b, near)


def test_diverging_column_gives_error_score():
    X, y = make_g1_classification(2000, 8, seed=7)
    X = X * 1e3
    from skdist.distribute.search import DistGridSearchCV
    est = SGDClassifier(learning_rate="constant", eta0=1e36, random_state=0, max_iter=5, tol=None)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = DistGridSearchCV(est, {"alpha": [1e-4, 1e-3]}, cv=3, error_score=np.nan, refit=False).fit(X, y)
    for s in range(3):
        assert np.all(np.isnan(ours.cv_results_["split%d_test_score" % s]))
