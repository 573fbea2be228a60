"""Ranking scorers on the host (no GPU): roc_auc_ovr / roc_auc_ovo [_weighted] and average_precision.

(a) tests/ranking_reference.py (float64 / integer per-segment counts) equals scikit-learn's roc_auc_score and
    average_precision_score on random, heavily tied and saturated-probability data, and so does the search's
    own averaging (logreg_family._rank_average) of those counts;
(b) every named scorer maps to its (kind, averaging) and score, other variants raise NotImplementedError;
(c) through the engine double, DistGridSearchCV reproduces GridSearchCV's cv_results_ for every new scorer on a
    binary and a 10-class target (multi-metric with refit and return_train_score), SGDClassifier included;
(d) scikit-learn's errors: a fold missing a class, labels {1, 2}, string labels, hinge SGD;
(e) DistFeatureEliminator scores with f1_weighted and roc_auc_ovr on a multiclass target as the reference's
    _fit_and_score_one does."""
import warnings

import numpy as np
import pytest
from sklearn.linear_model import LogisticRegression, SGDClassifier
from sklearn.metrics import average_precision_score, get_scorer, make_scorer, roc_auc_score
from sklearn.model_selection import GridSearchCV, StratifiedKFold

from skdist.distribute.eliminate import DistFeatureEliminator
from skdist.distribute.search import DistGridSearchCV
from skdist_b200.datasets import make_g1_classification
from skdist_b200.distribute import logreg_family as lf
from tests import ranking_reference as rr
from tests.ranking_fake_engine import RankingFakeEngine
from tests.sgd_fake_engine import SGDFakeEngine

NEW = ["roc_auc_ovr", "roc_auc_ovr_weighted", "roc_auc_ovo", "roc_auc_ovo_weighted", "average_precision"]
KIND = {"roc_auc_ovr": ("roc_auc_ovr", "macro"), "roc_auc_ovr_weighted": ("roc_auc_ovr", "weighted"),
        "roc_auc_ovo": ("roc_auc_ovo", "macro"), "roc_auc_ovo_weighted": ("roc_auc_ovo", "weighted"),
        "average_precision": ("average_precision", None)}


class _RankSGDEngine(RankingFakeEngine, SGDFakeEngine):
    pass


@pytest.fixture
def rank_engine():
    from skdist_b200 import engine
    engine.set_engine_factory(_RankSGDEngine)
    yield engine
    engine.set_engine_factory(None)


def _sk(name, y, S):
    kind, average = KIND[name]
    if kind == "average_precision":
        return average_precision_score(y, S)
    return roc_auc_score(y, S, multi_class=kind[-3:], average=average)


def _cases(K, rng):
    """(name, y, float32 scores) on random, heavily tied and saturated data."""
    n = 400
    y = rng.integers(0, max(K, 2), n)
    y[:max(K, 2)] = np.arange(max(K, 2))
    Zr = rng.normal(size=(n, K)).astype(np.float32)
    Zt = rng.integers(-2, 3, size=(n, K)).astype(np.float32)            # few distinct values: ties everywhere
    Zs = (rng.normal(size=(n, K)) * 40).astype(np.float32)               # probabilities saturate to 0 / 1
    for name, Z in (("random", Zr), ("tied", Zt), ("saturated", Zs)):
        yield name, y, (Z[:, 0] if K == 1 else Z)


@pytest.mark.parametrize("K", [1, 3, 4, 10])
def test_reference_and_averaging_equal_sklearn(K):
    rng = np.random.default_rng(K)
    for case, y, Z in _cases(K, rng):
        P = rr.f32_proba(Z)
        for name in NEW:
            kind, average = KIND[name]
            S = Z if kind == "average_precision" else P
            if K == 1:
                want = average_precision_score(y, S) if kind == "average_precision" else roc_auc_score(y, S)
            else:
                want = _sk(name, y, S)
            got = rr.score(kind, average, y, S, K)
            assert got == pytest.approx(want, rel=1e-12, abs=1e-15), (case, name)
            seg = rr.rank_counts(S, y, K, kind == "roc_auc_ovo")
            r = {k: v[None, :] for k, v in seg.items()}
            prod = lf._rank_average(kind, average, r, K)[0]
            assert prod == pytest.approx(want, rel=1e-12, abs=1e-15), (case, name)
        if case == "saturated":
            assert np.sum(P == 1.0) > 20                    # saturation really produced tied probabilities


def test_missing_class_and_empty_segments():
    rng = np.random.default_rng(3)
    y = rng.integers(0, 3, 200)
    y[y == 2] = 0                                          # class 2 absent
    Z = rng.normal(size=(200, 3)).astype(np.float32)
    for name in NEW:
        kind, average = KIND[name]
        with pytest.raises(ValueError):
            _sk(name, y, rr.f32_proba(Z) if kind != "average_precision" else Z)
        r = {k: v[None, :] for k, v in rr.rank_counts(Z, y, 3, kind == "roc_auc_ovo").items()}
        assert np.isnan(lf._rank_average(kind, average, r, 3)[0])
    # binary segment without positives: average precision 0 as scikit-learn gives it
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert average_precision_score(np.zeros(5, int), np.arange(5.0)) == 0.0
    assert rr.segment_counts(np.arange(5.0), np.zeros(5, bool))[3] == 0.0


def test_scorer_mapping():
    for name in NEW:
        m = lf._count_metric(get_scorer(name))
        assert m == KIND[name], name
        assert lf._RANK_SCORE[m[0]] == ("decision" if name == "average_precision" else "proba")
    assert lf._count_metric(get_scorer("roc_auc")) == ("roc_auc", None)
    rejected = [
        make_scorer(roc_auc_score, response_method="predict_proba", multi_class="ovr", average=None),
        make_scorer(roc_auc_score, response_method="predict_proba", multi_class="ovr", average="micro"),
        make_scorer(roc_auc_score, response_method="predict_proba", multi_class="ovo", max_fpr=0.5),
        make_scorer(roc_auc_score, response_method="decision_function", multi_class="ovr"),
        make_scorer(average_precision_score, response_method=("decision_function", "predict_proba"),
                    average="micro"),
        make_scorer(average_precision_score, response_method="predict_proba"),
        make_scorer(average_precision_score, response_method=("decision_function", "predict_proba"),
                    pos_label=2),
    ]
    X, y = make_g1_classification(200, 4, seed=1)
    for sc in rejected:
        assert lf._count_metric(sc) is None
        with pytest.raises(NotImplementedError, match="roc_auc_ovo_weighted"):
            lf._LogRegFamily(LogisticRegression(), [{}], X, y, {"score": sc})


def _same(ours, ref, names, train=True, atol=1e-12):
    n = ref.n_splits_
    for m in names:
        keys = ["split%d_test_%s" % (i, m) for i in range(n)] + ["mean_test_%s" % m, "rank_test_%s" % m]
        if train:
            keys += ["split%d_train_%s" % (i, m) for i in range(n)]
        for k in keys:
            np.testing.assert_allclose(ours.cv_results_[k], ref.cv_results_[k], rtol=0, atol=atol, err_msg=k)


def _digits():
    from sklearn.datasets import load_digits
    X, y = load_digits(return_X_y=True)
    return (X / 16.0).astype(np.float32)[:600], y[:600]


@pytest.mark.filterwarnings("ignore")
def test_multimetric_scoring_matches_sklearn(rank_engine):
    """Binary target: every count-based scorer and every new ranking scorer in one multi-metric search with
    refit=<name> and return_train_score, against scikit-learn's GridSearchCV."""
    X, y = make_g1_classification(600, 6, seed=5)
    scoring = ["accuracy", "f1", "precision", "recall", "balanced_accuracy"] + NEW
    grid = {"C": [0.001, 0.05, 1.0]}
    ours = DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring=scoring, refit="average_precision",
                            return_train_score=True).fit(X, y)
    ref = GridSearchCV(LogisticRegression(), grid, cv=3, scoring=scoring, refit="average_precision",
                       return_train_score=True).fit(X, y)
    _same(ours, ref, scoring)
    assert ours.best_params_ == ref.best_params_ and set(ours.scorer_) == set(scoring)
    assert ours.best_score_ == pytest.approx(ref.best_score_, abs=1e-12)
    calls = [c for c in rank_engine.get_engine().calls if c[0] == "rank"]
    # one rank call per (score, fold codes): proba for the four roc_auc_ov*, decision for average_precision
    assert {c[2] for c in calls} == {"proba", "decision"} and not any(c[3] for c in calls)
    with pytest.raises(ValueError):      # multi-metric needs refit=<scorer name> or False
        DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring=scoring).fit(X, y)


@pytest.mark.filterwarnings("ignore")
@pytest.mark.parametrize("name", NEW)
def test_single_scorer_binary_matches_sklearn(rank_engine, name):
    X, y = make_g1_classification(500, 5, seed=7)
    grid = {"C": [0.01, 1.0]}
    ours = DistGridSearchCV(LogisticRegression(), grid, None, cv=4, scoring=name, return_train_score=True).fit(X, y)
    ref = GridSearchCV(LogisticRegression(), grid, cv=4, scoring=name, return_train_score=True).fit(X, y)
    _same(ours, ref, ["score"])


@pytest.mark.filterwarnings("ignore")
def test_digits_multiclass_matches_sklearn(rank_engine):
    """10-class target (multinomial lbfgs): the five scorers plus f1_weighted in one search with refit and
    return_train_score, and each scorer alone."""
    X, y = _digits()
    grid = {"C": [0.05, 1.0]}
    scoring = NEW + ["f1_weighted"]
    ours = DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring=scoring, refit="roc_auc_ovo",
                            return_train_score=True).fit(X, y)
    ref = GridSearchCV(LogisticRegression(), grid, cv=3, scoring=scoring, refit="roc_auc_ovo",
                       return_train_score=True).fit(X, y)
    _same(ours, ref, scoring)
    assert ours.best_params_ == ref.best_params_
    calls = [c for c in rank_engine.get_engine().calls if c[0] == "rank"]
    assert ("proba", True) in {(c[2], c[3]) for c in calls}
    for name in ("roc_auc_ovr_weighted", "average_precision"):
        ours = DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring=name).fit(X, y)
        ref = GridSearchCV(LogisticRegression(), grid, cv=3, scoring=name).fit(X, y)
        _same(ours, ref, ["score"], train=False)


@pytest.mark.filterwarnings("ignore")
def test_multi_model_search(rank_engine):
    from skdist.distribute.search import DistMultiModelSearch
    X, y = _digits()
    models = [("lr", LogisticRegression(), {"C": [0.05, 1.0]})]
    ms = DistMultiModelSearch(models, n=2, cv=3, scoring="roc_auc_ovr").fit(X, y)
    for i, params in enumerate(ms.cv_results_["params"]):
        ref = GridSearchCV(LogisticRegression(), {k: [v] for k, v in params.items()}, cv=3,
                           scoring="roc_auc_ovr").fit(X, y)
        assert ms.cv_results_["mean_test_score"][i] == pytest.approx(ref.cv_results_["mean_test_score"][0],
                                                                     abs=1e-12)


@pytest.mark.filterwarnings("ignore")
def test_fold_missing_a_class_gives_error_score(rank_engine):
    X, y = _digits()
    y = y.copy()
    cv = [(np.arange(200, 600), np.arange(0, 200)), (np.arange(0, 400), np.arange(400, 600))]
    te = np.arange(0, 200)
    y[te[y[te] == 3]] = 4                                  # class 3 absent from the first test fold
    for name in NEW:
        ours = DistGridSearchCV(LogisticRegression(), {"C": [1.0]}, None, cv=cv, scoring=name,
                                error_score=np.nan).fit(X, y)
        ref = GridSearchCV(LogisticRegression(), {"C": [1.0]}, cv=cv, scoring=name, error_score=np.nan).fit(X, y)
        assert np.isnan(ref.cv_results_["split0_test_score"][0]) and np.isnan(ours.cv_results_["split0_test_score"][0])
        assert ours.cv_results_["split1_test_score"][0] == pytest.approx(ref.cv_results_["split1_test_score"][0],
                                                                          abs=1e-12)
        with pytest.raises(ValueError):
            DistGridSearchCV(LogisticRegression(), {"C": [1.0]}, None, cv=cv, scoring=name,
                             error_score="raise").fit(X, y)


@pytest.mark.filterwarnings("ignore")
def test_pos_label_of_average_precision(rank_engine):
    X, y01 = make_g1_classification(300, 5, seed=9)      # equal folds: the iid mean is the plain mean
    grid = {"C": [0.01, 1.0]}
    y12 = y01 + 1                                          # label 1 is classes_[0]: decision values negated
    ours = DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring="average_precision",
                            return_train_score=True).fit(X, y12)
    ref = GridSearchCV(LogisticRegression(), grid, cv=3, scoring="average_precision",
                       return_train_score=True).fit(X, y12)
    _same(ours, ref, ["score"])
    plain = GridSearchCV(LogisticRegression(), grid, cv=3, scoring=make_scorer(
        average_precision_score, response_method="decision_function", pos_label=2)).fit(X, y12)
    assert not np.allclose(plain.cv_results_["mean_test_score"], ref.cv_results_["mean_test_score"])
    calls = [c for c in rank_engine.get_engine().calls if c[0] == "rank"]
    assert calls and all(c[2] == "neg_decision" for c in calls[-6:])
    ys = np.where(y01 == 1, "yes", "no")                   # label 1 absent: scikit-learn raises
    ref = GridSearchCV(LogisticRegression(), grid, cv=3, scoring="average_precision", error_score=np.nan).fit(X, ys)
    ours = DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring="average_precision",
                            error_score=np.nan).fit(X, ys)
    assert np.all(np.isnan(ref.cv_results_["mean_test_score"])) and np.all(np.isnan(ours.cv_results_["mean_test_score"]))
    with pytest.raises(ValueError):
        DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring="average_precision",
                         error_score="raise").fit(X, ys)


@pytest.mark.filterwarnings("ignore")
def test_sgd_binary_ranking_scorers(rank_engine):
    X, y = make_g1_classification(300, 5, seed=12)
    grid = {"alpha": [1e-4, 1e-2]}
    for est, names in ((SGDClassifier(random_state=0), ["average_precision"]),
                       (SGDClassifier(loss="log_loss", random_state=0), NEW)):
        ours = DistGridSearchCV(est, grid, None, cv=3, scoring=names, refit=names[0],
                                return_train_score=True).fit(X, y)
        ref = GridSearchCV(est, grid, cv=3, scoring=names, refit=names[0], return_train_score=True).fit(X, y)
        _same(ours, ref, names, atol=1e-9)
    with pytest.raises(NotImplementedError):               # hinge has no predict_proba
        DistGridSearchCV(SGDClassifier(), grid, cv=3, scoring="roc_auc_ovr").fit(X, y)
    Xd, yd = _digits()
    for name in NEW:                                       # multiclass SGD normalises one-vs-rest probabilities
        with pytest.raises(NotImplementedError):
            DistGridSearchCV(SGDClassifier(loss="log_loss"), grid, cv=3, scoring=name).fit(Xd, yd)


def _covtype_like(n=900, d=10, K=7, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    W = rng.normal(size=(K, d))
    y = np.argmax(X[:, :4] @ W[:, :4].T + rng.normal(scale=1.5, size=(n, K)), axis=1)
    return X, y


@pytest.mark.filterwarnings("ignore")
@pytest.mark.parametrize("scoring", ["f1_weighted", "roc_auc_ovr"])
def test_eliminator_multiclass_scorers(rank_engine, scoring):
    """The reference's _fit_and_score_one (eliminate.py:29-38): scorer(clone.fit(X[train][:, keep], y[train]),
    X[test][:, keep], y[test]) per (feature set, fold), averaged over the folds."""
    X, y = _covtype_like()
    fe = DistFeatureEliminator(LogisticRegression(), None, step=3, cv=3, min_features_to_select=4,
                               scoring=scoring).fit(X, y)
    d = X.shape[1]
    ranks = np.argsort((LogisticRegression().fit(X, y).coef_.astype(np.float64) ** 2).sum(axis=0))[: d - 4]
    sets, k = [np.array([], int)], 0
    while k < d - 4:
        k += 3
        sets.append(ranks[:k])
    sc = get_scorer(scoring)
    exp = []
    for rm in sets:
        keep = np.setdiff1d(np.arange(d), rm)
        exp.append(np.mean([sc(LogisticRegression().fit(X[tr][:, keep], y[tr]), X[te][:, keep], y[te])
                            for tr, te in StratifiedKFold(3).split(X, y)]))
    np.testing.assert_allclose(fe.scores_, exp, atol=1e-9)
    assert fe.n_features_ == d - len(sets[int(np.argmax(exp))])
    with pytest.raises(NotImplementedError):
        DistFeatureEliminator(LogisticRegression(), None, cv=3, scoring="roc_auc").fit(X, y)


@pytest.mark.filterwarnings("ignore")
def test_config1_digits_multinomial_matches_oracle(rank_engine):
    """BASELINE config 1 (digits, 4 C x 3 folds, multinomial lbfgs): the host logic on the engine double
    reproduces the reference's driver loop (oracle/search_oracle.py), and the same search scored by
    roc_auc_ovr reproduces scikit-learn's GridSearchCV."""
    from sklearn.datasets import load_digits
    from sklearn.model_selection import ParameterGrid
    from oracle import search_oracle
    dg = load_digits()
    X, y = (dg.data / 16).astype(np.float32), dg.target
    grid = {"C": [0.01, 0.1, 1.0, 10.0]}
    est = LogisticRegression(max_iter=30)
    gs = DistGridSearchCV(est, grid, None, cv=3, return_train_score=True, preds=True).fit(X, y)
    ora = search_oracle.search_cv(est, ParameterGrid(grid), X, y, cv=3, iid=True, return_train_score=True)
    for k in ["split0_test_score", "split1_test_score", "split2_test_score", "mean_test_score",
              "std_test_score", "rank_test_score", "mean_train_score"]:
        np.testing.assert_array_equal(gs.cv_results_[k], ora["cv_results_"][k], err_msg=k)
    assert gs.best_params_ == ora["best_params_"] and gs.best_index_ == ora["best_index_"]
    be = gs.best_estimator_
    assert be.coef_.shape == (10, 64) and be.intercept_.shape == (10,) and be.n_iter_.shape == (1,)
    np.testing.assert_array_equal(be.coef_, ora["best_estimator_"].coef_)
    np.testing.assert_array_equal(gs.predict(X[:200]), ora["best_estimator_"].predict(X[:200]))
    assert gs.get_preds().shape == (len(y), 10)
    ours = DistGridSearchCV(est, grid, None, cv=3, scoring="roc_auc_ovr").fit(X, y)
    ref = GridSearchCV(est, grid, cv=3, scoring="roc_auc_ovr").fit(X, y)
    for s in range(3):
        np.testing.assert_allclose(ours.cv_results_["split%d_test_score" % s], ref.cv_results_["split%d_test_score" % s],
                                   rtol=0, atol=1e-12)


@pytest.mark.filterwarnings("ignore")
def test_multimetric_refit_false_and_regressors(rank_engine):
    """The rest of the multi-metric contract: refit=False leaves no best_*; regressor scorers from (SSE, n)."""
    from sklearn.linear_model import Ridge
    from skdist_b200.datasets import make_g1_regression
    X, y = make_g1_classification(600, 6, seed=5)
    nr = DistGridSearchCV(LogisticRegression(), {"C": [0.05, 1.0]}, None, cv=3, scoring=NEW, refit=False).fit(X, y)
    assert not hasattr(nr, "best_index_")
    Xr, yr = make_g1_regression(500, 5, seed=2)
    rs = ["r2", "neg_mean_squared_error", "neg_root_mean_squared_error"]
    ours = DistGridSearchCV(Ridge(), {"alpha": [0.1, 10.0]}, None, cv=3, scoring=rs, refit="r2").fit(Xr, yr)
    ref = GridSearchCV(Ridge(), {"alpha": [0.1, 10.0]}, cv=3, scoring=rs, refit="r2").fit(Xr, yr)
    for m in rs:
        for k in ("split0_test_%s" % m, "split1_test_%s" % m, "split2_test_%s" % m):
            np.testing.assert_allclose(ours.cv_results_[k], ref.cv_results_[k], rtol=2e-5, atol=1e-6, err_msg=k)


def test_engine_without_rank_entry_refuses_before_any_fit(fake_engine):
    """An engine that does not provide linear_rank_batch has no device path for the ranking scorers: the search
    and the eliminator raise NotImplementedError before any fit (no CPU fallback)."""
    from skdist_b200 import engine
    X, y = make_g1_classification(300, 5, seed=3)
    for name in NEW:
        with pytest.raises(NotImplementedError, match="linear_rank_batch"):
            DistGridSearchCV(LogisticRegression(), {"C": [1.0]}, None, cv=3, scoring=name).fit(X, y)
        assert not [c for c in engine.get_engine().calls if c[0] == "fit"]
    with pytest.raises(NotImplementedError, match="linear_rank_batch"):
        DistFeatureEliminator(LogisticRegression(), None, cv=3, scoring="average_precision").fit(X, y)
