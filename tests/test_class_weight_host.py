"""LogisticRegression(class_weight=...) in the searches, host side (no GPU): the per-column class weights
and sums of weights the families hand to the engine are scikit-learn's, and with an engine double that
fits exactly as scikit-learn does (tests/weighted_oracle.py) the searches reproduce GridSearchCV."""
import numpy as np
import pytest
from sklearn.linear_model import LogisticRegression
from sklearn.model_selection import GridSearchCV, KFold, ShuffleSplit, StratifiedKFold

from skdist.distribute.search import DistGridSearchCV
from skdist_b200 import engine
from skdist_b200.datasets import make_g1_classification
from tests import weighted_oracle as wo
from tests.weighted_fake_engine import WeightedFakeEngine

CW_GRID = [None, "balanced", {0: 1, 1: 5}]


@pytest.fixture
def weighted_engine():
    holder = {}

    def factory():
        holder["eng"] = WeightedFakeEngine()
        return holder["eng"]
    engine.set_engine_factory(factory)
    yield holder
    engine.set_engine_factory(None)


def _imbalanced(n, d, seed, n_classes=2):
    X, y = make_g1_classification(n, d, seed=seed)
    rng = np.random.default_rng(seed)
    if n_classes == 2:
        y = np.where(rng.random(n) < 0.25, y, 0)       # about 1 positive in 8
    else:
        y = np.minimum(rng.integers(0, 8, n), n_classes - 1)    # the last class takes half the rows
    return X, y


@pytest.mark.parametrize("n_classes", [2, 4])
@pytest.mark.parametrize("cv", ["kfold", "strat"])
def test_weighted_oracle_matches_scikit_learn(n_classes, cv):
    """The weighted oracle is bit-identical to LogisticRegression(class_weight=...).fit."""
    X, y = _imbalanced(700, 6, 3 + n_classes, n_classes)
    splitter = KFold(3) if cv == "kfold" else StratifiedKFold(3)
    train, _ = next(splitter.split(X, y))
    Xt, yt = X[train], y[train]
    for cw in CW_GRID + [{c: 0.5 + c for c in range(n_classes)}]:
        if isinstance(cw, dict) and set(cw) != set(range(n_classes)) and n_classes > 2:
            continue
        ref = LogisticRegression(C=0.3, class_weight=cw).fit(Xt, yt)
        sw, _ = wo.row_weights(cw, yt)
        if n_classes == 2:
            w, b, it = wo.fit_binary_lbfgs(Xt, yt.astype(np.float32), sw, C=0.3)
            np.testing.assert_array_equal(w, ref.coef_[0])
            assert b == ref.intercept_[0] and it == ref.n_iter_[0]
        else:
            W, b, it = wo.fit_multinomial_lbfgs(Xt, yt, sw, n_classes, C=0.3)
            np.testing.assert_array_equal(W, ref.coef_)
            np.testing.assert_array_equal(b, ref.intercept_)
            assert it == ref.n_iter_[0]


def _sklearn_weights(cw, y_train, classes):
    """What _logistic_regression_path forms for one fit: weight per class id of `classes`, sw_sum."""
    sw, sw_sum = wo.row_weights(cw, y_train)
    w = np.zeros(len(classes), np.float32)
    present = np.unique(y_train)
    w[np.searchsorted(classes, present)] = [sw[np.flatnonzero(y_train == c)[0]] for c in present]
    return w, sw_sum


@pytest.mark.parametrize("n_classes", [2, 4])
@pytest.mark.parametrize("cvname", ["kfold", "strat", "shuffle"])
def test_staged_weights_are_scikit_learns(weighted_engine, n_classes, cvname):
    """Every weighted column's staged class weights and sum of weights equal what scikit-learn forms for
    that fit, sw_sum summed in the splitter's own training-row order (ShuffleSplit's is not ascending)."""
    X, y = _imbalanced(997, 5, 11 + n_classes, n_classes)
    y = y * 3 + 1          # labels that are not class ids
    cv = {"kfold": KFold(4), "strat": StratifiedKFold(5),
          "shuffle": ShuffleSplit(n_splits=3, test_size=0.3, random_state=4)}[cvname]
    grid = {"C": [0.1, 1.0], "class_weight": CW_GRID[:2] + [{c: 1.0 + 0.37 * i for i, c in enumerate(np.unique(y))}]}
    gs = DistGridSearchCV(LogisticRegression(), grid, None, cv=cv, refit=False).fit(X, y)
    eng = weighted_engine["eng"]
    classes = np.unique(y)
    # the double does not see which split a column holds out: every staged column must be scikit-learn's
    # weights of one (split, class_weight), and every (split, class_weight) must have been staged
    options = [_sklearn_weights(cw, y[tr], classes) for tr, _ in cv.split(X, y) for cw in grid["class_weight"]]
    found = set()
    for w, sw_sum, _ in eng.staged:
        for j in range(len(sw_sum)):
            hit = [i for i, o in enumerate(options) if np.array_equal(w[j], o[0]) and sw_sum[j] == o[1]]
            assert hit, (j, w[j], sw_sum[j])
            found.update(hit)
    assert found == set(range(len(options)))
    assert len(gs.cv_results_["params"]) == 6


@pytest.mark.parametrize("n_classes", [2, 4])
@pytest.mark.parametrize("cvname", ["kfold", "strat"])
def test_search_matches_grid_search_cv(weighted_engine, n_classes, cvname):
    """cv_results_, best_params_ and the refitted coefficients of a search over class_weight are
    bit-identical to scikit-learn's GridSearchCV."""
    X, y = _imbalanced(800, 6, 21 + n_classes, n_classes)
    cv = KFold(3) if cvname == "kfold" else StratifiedKFold(3)
    cw3 = {0: 1, 1: 5} if n_classes == 2 else {0: 1, 1: 5, 2: 2, 3: 0.5}
    grid = {"C": [0.05, 1.0], "class_weight": [None, "balanced", cw3]}
    scoring = "accuracy" if n_classes == 2 else "f1_macro"
    gs = DistGridSearchCV(LogisticRegression(), grid, None, cv=cv, scoring=scoring).fit(X, y)
    ref = GridSearchCV(LogisticRegression(), grid, cv=cv, scoring=scoring).fit(X, y)
    for i in range(3):
        np.testing.assert_array_equal(gs.cv_results_["split%d_test_score" % i], ref.cv_results_["split%d_test_score" % i])
    assert gs.best_params_ == ref.best_params_
    np.testing.assert_array_equal(gs.best_estimator_.coef_, ref.best_estimator_.coef_)
    np.testing.assert_array_equal(gs.best_estimator_.intercept_, ref.best_estimator_.intercept_)
    assert gs.best_estimator_.class_weight == ref.best_estimator_.class_weight


def test_shuffle_split_matches_grid_search_cv(weighted_engine):
    X, y = _imbalanced(900, 6, 31)
    cv = ShuffleSplit(n_splits=4, test_size=0.3, random_state=2)
    grid = {"C": [0.1, 1.0], "class_weight": CW_GRID}
    gs = DistGridSearchCV(LogisticRegression(), grid, None, cv=cv).fit(X, y)
    ref = GridSearchCV(LogisticRegression(), grid, cv=cv).fit(X, y)
    for i in range(4):
        np.testing.assert_allclose(gs.cv_results_["split%d_test_score" % i], ref.cv_results_["split%d_test_score" % i],
                                   rtol=0, atol=1e-12)
    assert gs.best_params_ == ref.best_params_


def test_invalid_class_weight_raises_scikit_learns_error(weighted_engine):
    X, y = _imbalanced(300, 4, 41)
    with pytest.raises(ValueError) as ours:
        DistGridSearchCV(LogisticRegression(), {"class_weight": [{0: 1, 7: 2}]}, None, cv=3).fit(X, y)
    with pytest.raises(ValueError) as theirs:
        LogisticRegression(class_weight={0: 1, 7: 2}).fit(X, y)
    assert str(ours.value) == str(theirs.value)


def test_unweighted_searches_stage_nothing(weighted_engine):
    X, y = _imbalanced(300, 4, 51)
    DistGridSearchCV(LogisticRegression(), {"C": [0.1, 1.0]}, None, cv=3).fit(X, y)
    assert weighted_engine["eng"].staged == []


# ---- one-vs-rest, one-vs-one, feature elimination ------------------------------------------------------------
def _ovr_case(kind):
    X, y = _imbalanced(600, 5, 71, 4)
    if kind == "multilabel":
        rng = np.random.default_rng(3)
        return X, (rng.random((600, 3)) < [0.1, 0.3, 0.5]).astype(int)
    return X, y


@pytest.mark.parametrize("cw", ["balanced", {0: 1, 1: 4}])
@pytest.mark.parametrize("kind", ["multiclass", "multilabel", "max_negatives"])
def test_one_vs_rest_matches_scikit_learn(weighted_engine, kind, cw):
    """Every column's staged weights are scikit-learn's for the 0/1 column on its training rows, and the
    estimators are bit-identical to scikit-learn fits on those rows."""
    from sklearn.multiclass import OneVsRestClassifier
    from skdist.distribute.multiclass import DistOneVsRestClassifier
    X, y = _ovr_case(kind)
    kw = dict(max_negatives=0.5, random_state=2) if kind == "max_negatives" else {}
    lr = LogisticRegression(class_weight=cw)
    est = DistOneVsRestClassifier(lr, **kw).fit(X, y)
    eng = weighted_engine["eng"]
    (w, sw_sum, _), = eng.staged
    if kind == "max_negatives":
        from skdist_b200.distribute.multiclass import _negatives_rows
        cls = np.unique(y)
        cols = [(y == c) for c in cls]
        rows = [_negatives_rows(c, 0.5, 2, "ratio") for c in cols]
        for k in range(len(cls)):
            y01 = cols[k][rows[k]].astype(int)
            want = _sklearn_weights(cw, y01, np.array([0, 1]))
            assert np.array_equal(w[k], want[0]) and sw_sum[k] == want[1]
            ref = LogisticRegression(class_weight=cw).fit(X[rows[k]], y01)
            np.testing.assert_array_equal(est.estimators_[k].coef_, ref.coef_)
        return
    ref = OneVsRestClassifier(lr).fit(X, y)
    Y = y if kind == "multilabel" else (y[:, None] == np.unique(y)[None, :]).astype(int)
    for k in range(Y.shape[1]):
        want = _sklearn_weights(cw, Y[:, k], np.array([0, 1]))
        assert np.array_equal(w[k], want[0]) and sw_sum[k] == want[1]
        np.testing.assert_array_equal(est.estimators_[k].coef_, ref.estimators_[k].coef_)
        np.testing.assert_array_equal(est.estimators_[k].intercept_, ref.estimators_[k].intercept_)
    np.testing.assert_array_equal(est.predict(X), ref.predict(X))


def test_one_vs_one_matches_scikit_learn(weighted_engine):
    from sklearn.multiclass import OneVsOneClassifier
    from skdist.distribute.multiclass import DistOneVsOneClassifier
    X, y = _imbalanced(600, 5, 81, 4)
    lr = LogisticRegression(class_weight="balanced")
    est = DistOneVsOneClassifier(lr).fit(X, y)
    ref = OneVsOneClassifier(lr).fit(X, y)
    (w, sw_sum, _), = weighted_engine["eng"].staged
    pairs = [(i, j) for i in range(4) for j in range(i + 1, 4)]
    for k, (i, j) in enumerate(pairs):
        yp = y[(y == i) | (y == j)]
        want = _sklearn_weights("balanced", (yp == j).astype(int), np.array([0, 1]))
        assert np.array_equal(w[k], want[0]) and sw_sum[k] == want[1]
        np.testing.assert_array_equal(est.estimators_[k].coef_, ref.estimators_[k].coef_)
    np.testing.assert_array_equal(est.predict(X), ref.predict(X))


@pytest.mark.parametrize("n_classes", [2, 3])
def test_feature_eliminator_weights(weighted_engine, n_classes):
    """The eliminator's fits carry scikit-learn's weights of their folds; the final estimator is
    scikit-learn's weighted fit on the selected features, bit for bit."""
    from skdist.distribute.eliminate import DistFeatureEliminator
    X, y = _imbalanced(500, 6, 91, n_classes)
    cv = StratifiedKFold(3)
    fe = DistFeatureEliminator(LogisticRegression(class_weight="balanced"), cv=cv, step=2).fit(X, y)
    classes = np.unique(y)
    options = [_sklearn_weights("balanced", y[tr], classes) for tr, _ in cv.split(X, y)]
    options.append(_sklearn_weights("balanced", y, classes))
    for w, sw_sum, _ in weighted_engine["eng"].staged:
        for j in range(len(sw_sum)):
            assert any(np.array_equal(w[j], o[0]) and sw_sum[j] == o[1] for o in options)
    keep = np.asarray(fe.best_features_)
    ref = LogisticRegression(class_weight="balanced").fit(np.ascontiguousarray(X[:, keep]), y)
    np.testing.assert_array_equal(fe.best_estimator_.coef_, ref.coef_)


# ---- two ranks ------------------------------------------------------------------------------------------
def _rank_worker(rank, world, port, out_dir):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from skdist_b200 import engine as eng_mod
    from tests.weighted_fake_engine import WeightedFakeEngine as W
    eng_mod.set_engine_factory(W)
    res = _weighted_search()
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **res)
    dist.destroy_process_group()


def _weighted_search():
    X, y = _imbalanced(700, 6, 101)
    gs = DistGridSearchCV(LogisticRegression(), {"C": [0.05, 1.0], "class_weight": CW_GRID}, None,
                          cv=ShuffleSplit(3, test_size=0.3, random_state=1)).fit(X, y)
    return {"mean": gs.cv_results_["mean_test_score"], "s0": gs.cv_results_["split0_test_score"],
            "coef": gs.best_estimator_.coef_}


def test_two_rank_weighted_search_matches_one_rank(tmp_path):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_rank_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    engine.set_engine_factory(WeightedFakeEngine)
    try:
        one = _weighted_search()
    finally:
        engine.set_engine_factory(None)
    for r in (0, 1):
        got = np.load(tmp_path / ("rank%d.npz" % r))
        for k in one:
            np.testing.assert_array_equal(got[k], one[k], err_msg=k)
