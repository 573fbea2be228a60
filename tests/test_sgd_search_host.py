"""Host logic of the SGDClassifier search family (no GPU): training rows in the splitter's order, seeds,
order groups, scoring assembly and refit, on an engine double that runs scikit-learn's own SGD loop per
column (tests/sgd_fake_engine.py).  cv_results_ must equal scikit-learn's GridSearchCV split for split."""
import warnings

import numpy as np
import pytest
from scipy.stats import loguniform
from sklearn.datasets import load_digits
from sklearn.linear_model import LogisticRegression, SGDClassifier
from sklearn.model_selection import GridSearchCV, RandomizedSearchCV, ShuffleSplit

from skdist.distribute.search import DistGridSearchCV, DistMultiModelSearch, DistRandomizedSearchCV
from skdist_b200.datasets import make_g1_classification
from skdist_b200.distribute.sgd_family import sgd_class_seeds
from skdist_b200.engine import sgd_seed

ALPHAS = [1e-4, 1e-3, 1e-2]


@pytest.fixture
def sgd_engine():
    from skdist_b200 import engine
    from tests.sgd_fake_engine import SGDFakeEngine
    engine.set_engine_factory(SGDFakeEngine)
    yield engine
    engine.set_engine_factory(None)


def _digits():
    X, y = load_digits(return_X_y=True)
    return (X / 16.0).astype(np.float32)[:900], y[:900]


def _same_results(ours, ref, names, train=False):
    n = ref.n_splits_
    for m in names:
        keys = ["split%d_test_%s" % (i, m) for i in range(n)] + ["rank_test_%s" % m]
        if train:
            keys += ["split%d_train_%s" % (i, m) for i in range(n)]
        for k in keys:
            np.testing.assert_array_equal(ours.cv_results_[k], ref.cv_results_[k], err_msg=k)
        # (mean_test_* is the reference's test-size weighted average, scikit-learn's a plain one)


def _same_estimator(a, b):
    np.testing.assert_array_equal(a.coef_, b.coef_)
    np.testing.assert_array_equal(a.intercept_, b.intercept_)
    assert a.coef_.dtype == b.coef_.dtype and a.intercept_.dtype == b.intercept_.dtype
    assert a.n_iter_ == b.n_iter_ and a.t_ == b.t_
    np.testing.assert_array_equal(a.classes_, b.classes_)


@pytest.mark.parametrize("loss", ["hinge", "log_loss"])
def test_binary_grid_matches_scikit_learn(sgd_engine, loss):
    X, y = make_g1_classification(900, 10, seed=3)
    est = SGDClassifier(loss=loss, random_state=0)
    scoring = {"score": "accuracy", "auc": "roc_auc"}
    if loss == "log_loss":
        scoring["nll"] = "neg_log_loss"
    ours = DistGridSearchCV(est, {"alpha": ALPHAS}, cv=3, scoring=scoring, refit="score").fit(X, y)
    ref = GridSearchCV(est, {"alpha": ALPHAS}, cv=3, scoring=scoring, refit="score").fit(X, y)
    _same_results(ours, ref, ["score", "auc"])
    if loss == "log_loss":      # the scoring kernels form the probabilities from fp32 decision values
        for i in range(3):
            np.testing.assert_allclose(ours.cv_results_["split%d_test_nll" % i], ref.cv_results_["split%d_test_nll" % i],
                                       rtol=1e-6)
    assert ours.best_params_ == ref.best_params_
    _same_estimator(ours.best_estimator_, ref.best_estimator_)
    np.testing.assert_array_equal(ours.predict(X), ref.predict(X))
    # one launch holds every (candidate, fold) column: 3 alphas x 3 folds in 3 order groups, then the refit
    calls = [c for c in sgd_engine.get_engine().calls if c[0] == "sgd_fit_groups"]
    assert calls == [("sgd_fit_groups", 9, 3), ("sgd_fit_groups", 1, 1)]


def test_multiclass_digits_f1_weighted(sgd_engine):
    X, y = _digits()
    est = SGDClassifier(random_state=0, max_iter=30, tol=None)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = DistGridSearchCV(est, {"alpha": [1e-3, 1e-2]}, cv=3, scoring="f1_weighted").fit(X, y)
        ref = GridSearchCV(est, {"alpha": [1e-3, 1e-2]}, cv=3, scoring="f1_weighted").fit(X, y)
    _same_results(ours, ref, ["score"])
    _same_estimator(ours.best_estimator_, ref.best_estimator_)
    np.testing.assert_array_equal(ours.predict(X), ref.predict(X))
    calls = [c for c in sgd_engine.get_engine().calls if c[0] == "sgd_fit_groups"]
    assert calls[0] == ("sgd_fit_groups", 2 * 3 * 10, 3 * 10)        # (candidate, fold, class); (fold, class seed)


def test_multimetric_refit_by_name_and_train_scores(sgd_engine):
    X, y = make_g1_classification(600, 8, seed=4)
    est = SGDClassifier(random_state=2)
    grid = {"alpha": ALPHAS, "loss": ["hinge", "log_loss"]}
    scoring = {"acc": "accuracy", "f1": "f1", "bal": "balanced_accuracy", "prec": "precision_macro"}
    ours = DistGridSearchCV(est, grid, cv=3, scoring=scoring, refit="f1", return_train_score=True).fit(X, y)
    ref = GridSearchCV(est, grid, cv=3, scoring=scoring, refit="f1", return_train_score=True).fit(X, y)
    _same_results(ours, ref, list(scoring), train=True)
    assert ours.best_params_ == ref.best_params_
    _same_estimator(ours.best_estimator_, ref.best_estimator_)


def test_randomized_loguniform(sgd_engine):
    X, y = make_g1_classification(700, 6, seed=5)
    est = SGDClassifier(loss="log_loss", random_state=7)
    dist = {"alpha": loguniform(1e-6, 1e-2)}
    ours = DistRandomizedSearchCV(est, dist, n_iter=5, cv=3, random_state=1).fit(X, y)
    ref = RandomizedSearchCV(est, dist, n_iter=5, cv=3, random_state=1).fit(X, y)
    _same_results(ours, ref, ["score"])
    _same_estimator(ours.best_estimator_, ref.best_estimator_)


def test_shuffle_split_walks_the_permuted_train_order(sgd_engine):
    X, y = make_g1_classification(500, 6, seed=6)
    est = SGDClassifier(random_state=3, learning_rate="invscaling", eta0=0.05)
    cv = ShuffleSplit(n_splits=3, test_size=0.3, random_state=0)
    ours = DistGridSearchCV(est, {"alpha": ALPHAS}, cv=cv).fit(X, y)
    ref = GridSearchCV(est, {"alpha": ALPHAS}, cv=cv).fit(X, y)
    _same_results(ours, ref, ["score"])
    # with shuffle off the permutation alone sets the order; still scikit-learn's
    est = SGDClassifier(random_state=3, shuffle=False)
    ours = DistGridSearchCV(est, {"alpha": ALPHAS}, cv=cv).fit(X, y)
    ref = GridSearchCV(est, {"alpha": ALPHAS}, cv=cv).fit(X, y)
    _same_results(ours, ref, ["score"])


def test_multi_model_search_entry(sgd_engine):
    X, y = make_g1_classification(600, 6, seed=8)
    models = [("sgd", SGDClassifier(random_state=0), {"alpha": [1e-4, 1e-3, 1e-2]}),
              ("lr", LogisticRegression(), {"C": [0.1, 1.0]})]
    mm = DistMultiModelSearch(models, n=3, cv=3, random_state=0).fit(X, y)
    sgd_rows = [i for i, name in enumerate(mm.cv_results_["model_name"]) if name == "sgd"]
    for i in sgd_rows:
        p = mm.cv_results_["params"][i]
        ref = GridSearchCV(SGDClassifier(random_state=0), {"alpha": [p["alpha"]]}, cv=3).fit(X, y)
        splits = [ref.cv_results_["split%d_test_score" % k][0] for k in range(3)]
        assert mm.cv_results_["mean_test_score"][i] == pytest.approx(np.mean(splits), rel=1e-12)
    if mm.best_model_name_ == "sgd":
        _same_estimator(mm.best_estimator_, SGDClassifier(random_state=0, **mm.best_params_).fit(X, y))


def test_seed_derivation_matches_scikit_learn():
    from sklearn.linear_model._stochastic_gradient import MAX_INT
    from sklearn.utils import check_random_state
    for rs in (0, 7, 123456):
        want = check_random_state(rs)
        want.randint(1, MAX_INT)
        assert sgd_class_seeds(rs, 2) == [int(want.randint(MAX_INT))]
        draws = np.random.RandomState(rs).randint(MAX_INT, size=5)      # _fit_multiclass's per-class draws
        assert sgd_class_seeds(rs, 5) == [sgd_seed(int(s)) for s in draws]
    state = np.random.RandomState(11)
    assert sgd_class_seeds(state, 4) == sgd_class_seeds(np.random.RandomState(11), 4)    # a clone's copy, not consumed
    assert sgd_class_seeds(state, 4) == sgd_class_seeds(11, 4)


def test_diverged_fit_gives_error_score(sgd_engine):
    X, y = make_g1_classification(400, 6, seed=9)
    X = X * 1e3
    est = SGDClassifier(learning_rate="constant", eta0=1e36, random_state=0, max_iter=5, tol=None)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ours = DistGridSearchCV(est, {"alpha": [1e-4, 1e-3]}, cv=3, error_score=np.nan, refit=False).fit(X, y)
    assert np.all(np.isnan(ours.cv_results_["split0_test_score"]))


@pytest.mark.parametrize("make", [
    lambda: (SGDClassifier(loss="modified_huber"), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(penalty="l1"), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(penalty="elasticnet"), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(learning_rate="adaptive", eta0=0.1), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(average=True), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(early_stopping=True), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(warm_start=True), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(class_weight="balanced"), {"alpha": [1e-3]}, None),
    lambda: (SGDClassifier(), {"alpha": [1e-3], "l1_ratio": [0.2]}, None),
    lambda: (SGDClassifier(), {"alpha": [1e-3], "penalty": ["l2", "l1"]}, None),
    lambda: (SGDClassifier(), {"alpha": [0.0]}, None),
    lambda: (SGDClassifier(), {"alpha": [1e-3]}, "neg_log_loss"),      # hinge has no predict_proba
    lambda: (SGDClassifier(), {"alpha": [1e-3]}, "average_precision"),
    lambda: (SGDClassifier(), {"alpha": [1e-3]}, "neg_brier_score"),
])
def test_rejected_configurations_make_no_fit(sgd_engine, make):
    X, y = make_g1_classification(300, 5, seed=10)
    est, grid, scoring = make()
    with pytest.raises(NotImplementedError):
        DistGridSearchCV(est, grid, cv=3, scoring=scoring).fit(X, y)
    assert not [c for c in sgd_engine.get_engine().calls if c[0] == "sgd_fit_groups"]


@pytest.mark.parametrize("scoring", ["neg_log_loss", "roc_auc_ovr", "f1", "precision"])
def test_rejected_multiclass_scorers_make_no_fit(sgd_engine, scoring):
    X, y = _digits()
    with pytest.raises(NotImplementedError):
        DistGridSearchCV(SGDClassifier(loss="log_loss"), {"alpha": [1e-3]}, cv=3, scoring=scoring).fit(X, y)
    assert not [c for c in sgd_engine.get_engine().calls if c[0] == "sgd_fit_groups"]


def test_preds_rejected_before_any_fit(sgd_engine):
    X, y = make_g1_classification(300, 5, seed=11)
    with pytest.raises(NotImplementedError):
        DistGridSearchCV(SGDClassifier(), {"alpha": [1e-3]}, cv=3, preds=True).fit(X, y)
    assert not [c for c in sgd_engine.get_engine().calls if c[0] == "sgd_fit_groups"]
