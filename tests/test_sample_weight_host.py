"""LogisticRegression fits with sample_weight in the searches and one-vs-rest, host side (no GPU).

  * the per-column class weights, sums of weights and per-row weights handed to the engine are the ones
    scikit-learn's _logistic_regression_path forms for the same training rows (captured from its solver call);
  * tests/weighted_search_oracle.py (fit params indexed by each task's training rows, unweighted scores) is
    pinned against the reference's own _fit_and_score (tests/golden/sample_weight_pins.npz);
  * with an engine double that fits as scikit-learn does (tests/weighted_oracle.py with the combined
    per-row weights), the searches reproduce that oracle and one-vs-rest reproduces scikit-learn;
  * every refusal raises the stated exception."""
import os
import warnings

import numpy as np
import pytest
from sklearn.linear_model import LogisticRegression, Ridge, SGDClassifier
from sklearn.model_selection import ShuffleSplit, StratifiedKFold

from skdist.distribute.eliminate import DistFeatureEliminator
from skdist.distribute.multiclass import DistOneVsOneClassifier, DistOneVsRestClassifier
from skdist.distribute.search import DistGridSearchCV, DistMultiModelSearch, DistRandomizedSearchCV
from skdist_b200 import engine
from skdist_b200.datasets import make_g1_classification
from tests import weighted_oracle as wo
from tests import weighted_search_oracle as wso
from tests.weighted_fake_engine import WeightedFakeEngine

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class SampleWeightFakeEngine(WeightedFakeEngine):
    """WeightedFakeEngine plus the sample-weight staging call: a weighted fit's rows weigh
    float32(sample weight * class weight of the row's label), as scikit-learn forms them."""

    def __init__(self, device=0):
        super().__init__(device)
        self._sw = None
        self.staged_sw = []         # the sample weights of every weighted fit (None: none), aligned with `staged`

    def stage_sample_weights(self, w):
        self._sw = None if w is None else np.asarray(w, np.float32).copy()
        assert self._sw is None or self._sw.shape == (self.n,)

    def _take_sw(self, B, K, col_fold):
        sw, self._sw = self._sw, None
        cw = self._take(B, K, col_fold)
        if sw is not None:
            assert cw is not None, "sample weights need class weights staged for the same fit"
        if cw is not None:
            self.staged_sw.append(sw)
        return cw, sw

    def logreg_fit_batch(self, C, col_fold, col_pos, fit_intercept=True, tol=1e-4, max_iter=100, col_neg=None):
        cw, sw = self._take_sw(len(C), 2, col_fold)
        if cw is None:
            return super(WeightedFakeEngine, self).logreg_fit_batch(C, col_fold, col_pos, fit_intercept, tol,
                                                                    max_iter, col_neg)
        ybits, mbits = getattr(self, "_ybits", None), getattr(self, "_mbits", None)
        self._ybits = self._mbits = self._fmask = None
        B = len(C)
        coef = np.zeros((B, self.d + 1), np.float32)
        n_iter = np.zeros(B, np.int32)
        for j in range(B):
            m = self._train_mask(int(col_fold[j]))
            if col_neg is not None and col_neg[j] >= 0:
                m = m & ((self.y == col_pos[j]) | (self.y == col_neg[j]))
            if mbits is not None:
                m = m & mbits[j]
            yb = ((self.y[m] == col_pos[j]) if ybits is None else ybits[j][m]).astype(np.intp)
            rw = cw[0][j][yb] if sw is None else sw[m] * cw[0][j][yb]
            w, b, it = wo.fit_binary_lbfgs(np.ascontiguousarray(self.X[m]), yb.astype(np.float32), rw, C=float(C[j]),
                                           tol=tol, max_iter=max_iter, fit_intercept=fit_intercept)
            coef[j, :self.d], coef[j, self.d], n_iter[j] = w, b, it
        return {"coef": coef, "n_iter": n_iter, "status": np.ones(B, np.int32), "loss": np.zeros(B),
                "n_evals": n_iter + 1, "gpu_seconds": 0.0}

    def logreg_multinomial_fit_batch(self, C, col_fold, n_classes, fit_intercept=True, tol=1e-4, max_iter=100):
        cw, sw = self._take_sw(len(C), n_classes, col_fold)
        if cw is None:
            return super(WeightedFakeEngine, self).logreg_multinomial_fit_batch(C, col_fold, n_classes, fit_intercept,
                                                                                tol, max_iter)
        self._fmask = None
        B = len(C)
        coef = np.zeros((B, n_classes, self.d + 1), np.float32)
        n_iter = np.zeros(B, np.int32)
        for j in range(B):
            m = self._train_mask(int(col_fold[j]))
            rw = cw[0][j][self.y[m]] if sw is None else sw[m] * cw[0][j][self.y[m]]
            W, b, it = wo.fit_multinomial_lbfgs(np.ascontiguousarray(self.X[m]), self.y[m], rw, n_classes,
                                                C=float(C[j]), tol=tol, max_iter=max_iter, fit_intercept=fit_intercept)
            coef[j, :, :self.d], coef[j, :, self.d], n_iter[j] = W, b, it
        return {"coef": coef, "n_iter": n_iter, "status": np.ones(B, np.int32), "loss": np.zeros(B),
                "n_evals": n_iter + 1, "gpu_seconds": 0.0}


@pytest.fixture
def sw_engine():
    holder = {}

    def factory():
        holder["eng"] = SampleWeightFakeEngine()
        return holder["eng"]
    engine.set_engine_factory(factory)
    yield holder
    engine.set_engine_factory(None)


def _data(n, d, seed, n_classes=2, kind="lognormal"):
    X, y = make_g1_classification(n, d, seed=seed)
    rng = np.random.default_rng(seed)
    if n_classes > 2:
        y = np.minimum(rng.integers(0, n_classes + 2, n), n_classes - 1)
    if kind == "lognormal":
        w = np.exp(rng.normal(0.0, 1.5, n))
        w[rng.random(n) < 0.1] = 0.0
    else:               # frequency weights
        w = rng.integers(0, 4, n).astype(np.float64)
    return X, y, w


def _assert_same_fit(est, ref):
    """The double's fit (tests/weighted_oracle.py) against scikit-learn's: with arbitrary float sample weights the
    restated objective can differ from scikit-learn's in the last bits of a float32 sum, so the coefficients agree
    to a few float32 ulps of the optimum and the iteration counts to one."""
    np.testing.assert_allclose(est.coef_, ref.coef_, rtol=0, atol=2e-5)
    np.testing.assert_allclose(est.intercept_, ref.intercept_, rtol=0, atol=2e-5)
    assert abs(int(est.n_iter_[0]) - int(ref.n_iter_[0])) <= 1


class _Captured(Exception):
    pass


def _sklearn_path_weights(X, y, sw, cw):
    """(per-row weights, sw_sum) that _logistic_regression_path hands to its lbfgs solve for
    LogisticRegression(class_weight=cw).fit(X, y, sample_weight=sw), captured at the solver call."""
    import sklearn.linear_model._logistic as lg
    seen = {}

    class _Opt:
        @staticmethod
        def minimize(fun, x0, args=(), **kw):
            seen["sw"] = np.array(args[2], copy=True)
            raise _Captured

    real = lg.optimize
    lg.optimize = _Opt
    try:
        LogisticRegression(class_weight=cw).fit(X, y, sample_weight=sw)
    except _Captured:
        pass
    finally:
        lg.optimize = real
    return seen["sw"], float(np.sum(seen["sw"]))


@pytest.mark.parametrize("n_classes", [2, 4])
@pytest.mark.parametrize("cvname", ["strat", "shuffle"])
def test_staged_weights_are_scikit_learns(sw_engine, n_classes, cvname):
    """Every staged column's per-row weights (staged sample weight x staged class weight of the row's label,
    float32) and sw_sum equal what scikit-learn forms for one (split, class_weight) fit on that split's
    training rows in the splitter's order, bit for bit, for None, "balanced" and a dict; every
    (split, class_weight) was staged, and every fit staged the full float32 sample weights."""
    X, y, w = _data(797, 5, 13 + n_classes, n_classes)
    y = y * 3 + 1          # labels that are not class ids
    classes = np.unique(y)
    ids = np.searchsorted(classes, y)
    cv = {"strat": StratifiedKFold(4), "shuffle": ShuffleSplit(n_splits=3, test_size=0.3, random_state=4)}[cvname]
    cws = [None, "balanced", {c: 1.0 + 0.37 * i for i, c in enumerate(classes)}]
    DistGridSearchCV(LogisticRegression(), {"C": [0.1, 1.0], "class_weight": cws}, None, cv=cv,
                     refit=False).fit(X, y, sample_weight=w)
    eng = sw_engine["eng"]
    splits = list(cv.split(X, y))
    options = [(tr, *_sklearn_path_weights(X[tr], y[tr], w[tr], cw)) for tr, _ in splits for cw in cws]
    found = set()
    assert len(eng.staged) == len(eng.staged_sw) > 0
    for (cwt, sw_sum, _), sw in zip(eng.staged, eng.staged_sw):
        np.testing.assert_array_equal(sw, w.astype(np.float32))
        for j in range(len(sw_sum)):
            hit = [i for i, (tr, rows, s) in enumerate(options)
                   if s == sw_sum[j] and np.array_equal(sw[tr] * cwt[j][ids[tr]], rows)]
            assert hit, (j, sw_sum[j])
            found.update(hit)
    assert found == set(range(len(options)))


@pytest.mark.parametrize("n_classes", [2, 4])
def test_oracle_task_equals_reference_task(n_classes):
    """Pin: the reference's _fit_and_score with fit_params={"sample_weight": w} (recorded by
    tests/golden/make_sample_weight_pins.py) vs tests/weighted_search_oracle.py."""
    pins = np.load(os.path.join(GOLD, "sample_weight_pins.npz"))
    X, y, w, cands, cv = wso.sample_weight_case(n_classes)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        b = wso.search_cv(LogisticRegression(), cands, X, y, cv=cv, fit_params={"sample_weight": w}, refit=False)
    for i in range(3):
        np.testing.assert_array_equal(pins["k%d_split%d_test_score" % (n_classes, i)],
                                      b["cv_results_"]["split%d_test_score" % i])
    np.testing.assert_array_equal(pins["k%d_mean_test_score" % n_classes], b["cv_results_"]["mean_test_score"])
    assert int(pins["k%d_best_index" % n_classes]) == b["best_index_"]


@pytest.mark.parametrize("n_classes", [2, 4])
@pytest.mark.parametrize("cvname", ["strat", "shuffle"])
@pytest.mark.parametrize("kind", ["lognormal", "frequency"])
@pytest.mark.filterwarnings("ignore")
def test_search_matches_oracle(sw_engine, n_classes, cvname, kind):
    """cv_results_ and best_params_ of a weighted search equal the reference's (the oracle: weighted fits,
    unweighted scores); the refit's coefficients are LogisticRegression(**best_params_).fit(X, y, sample_weight=w)'s."""
    X, y, w = _data(700, 6, 23 + n_classes, n_classes, kind)
    cv = StratifiedKFold(3) if cvname == "strat" else ShuffleSplit(n_splits=3, test_size=0.3, random_state=7)
    cw3 = {c: 1.0 + 0.5 * c for c in range(n_classes)}
    grid = {"C": [0.05, 1.0], "class_weight": [None, "balanced", cw3]}
    gs = DistGridSearchCV(LogisticRegression(), grid, None, cv=cv).fit(X, y, sample_weight=w)
    cands = list(gs.cv_results_["params"])
    ref = wso.search_cv(LogisticRegression(), cands, X, y, cv=cv, fit_params={"sample_weight": w})
    for i in range(3):
        # ShuffleSplit's training rows are not ascending: the double sums in ascending order
        np.testing.assert_allclose(gs.cv_results_["split%d_test_score" % i],
                                   ref["cv_results_"]["split%d_test_score" % i], rtol=0, atol=1e-12)
    assert gs.best_params_ == ref["best_params_"]
    best = ref["best_estimator_"]
    _assert_same_fit(gs.best_estimator_, best)


@pytest.mark.filterwarnings("ignore")
def test_randomized_search_and_fold_proba(sw_engine):
    """DistRandomizedSearchCV takes sample_weight too; preds=True refits each fold with its training rows'
    weights (the staged weights of those fits are the folds' own)."""
    from scipy.stats import loguniform
    X, y, w = _data(600, 5, 51)
    rs = DistRandomizedSearchCV(LogisticRegression(), {"C": loguniform(0.01, 10)}, None, n_iter=3, cv=3,
                                random_state=0, preds=True).fit(X, y, sample_weight=w)
    ref = wso.search_cv(LogisticRegression(), rs.cv_results_["params"], X, y, cv=3, fit_params={"sample_weight": w})
    np.testing.assert_array_equal(rs.cv_results_["mean_test_score"], ref["cv_results_"]["mean_test_score"])
    _assert_same_fit(rs.best_estimator_, ref["best_estimator_"])
    eng = sw_engine["eng"]
    cw, sw_sum, folds = eng.staged[-1]
    assert list(folds) == [0, 1, 2]
    for k, (tr, _) in enumerate(StratifiedKFold(3).split(X, y)):
        assert sw_sum[k] == float(np.sum(w[tr].astype(np.float32)))
    assert rs.preds_.shape == (len(y), 2)


@pytest.mark.parametrize("target", ["binary", "multiclass", "multilabel"])
@pytest.mark.filterwarnings("ignore")
def test_one_vs_rest_matches_scikit_learn(sw_engine, target):
    """Every label column fits all rows with the full sample_weight (ref multiclass.py:145-151): its
    coefficients are LogisticRegression().fit(X, y == c, sample_weight=w)'s."""
    X, y, w = _data(500, 5, 61, 2 if target == "binary" else 4)
    if target == "multilabel":
        rng = np.random.default_rng(3)
        y = (rng.random((len(y), 3)) < np.array([0.2, 0.5, 0.7])).astype(int)
    for cw in (None, "balanced"):
        ovr = DistOneVsRestClassifier(LogisticRegression(C=0.5, class_weight=cw)).fit(X, y, sample_weight=w)
        cols = y.T if target == "multilabel" else ([y == 1] if target == "binary" else [y == c for c in range(4)])
        assert len(ovr.estimators_) == len(cols)
        for est, yc in zip(ovr.estimators_, cols):
            ref = LogisticRegression(C=0.5, class_weight=cw).fit(X, yc.astype(int), sample_weight=w)
            _assert_same_fit(est, ref)


def test_refusals(sw_engine):
    X, y, w = _data(300, 4, 71)
    grid = {"C": [0.1, 1.0]}
    gs = DistGridSearchCV(LogisticRegression(), grid, None, cv=3)
    with pytest.raises(TypeError, match="unexpected keyword argument 'foo'"):
        gs.fit(X, y, sample_weight=w, foo=1)
    for base, g in ((Ridge(), {"alpha": [1.0]}), (SGDClassifier(), {"alpha": [1e-4]})):
        with pytest.raises(NotImplementedError, match="sample_weight"):
            DistGridSearchCV(base, g, None, cv=3).fit(X, y, sample_weight=w)
    with pytest.raises(ValueError, match="shape"):
        gs.fit(X, y, sample_weight=w[:-1])
    for bad in (-1.0, np.nan, np.inf):
        w2 = w.copy()
        w2[5] = bad
        with pytest.raises(ValueError):
            gs.fit(X, y, sample_weight=w2)
    w0 = w.copy()       # every training row of the fold holding out the rows from 100 on weighs 0
    w0[:100] = 0.0
    from sklearn.model_selection import PredefinedSplit
    with pytest.raises(ValueError, match="sum"):
        gs.set_params(cv=PredefinedSplit(np.r_[np.full(100, -1), np.zeros(200, int)])).fit(X, y, sample_weight=w0)
    ovr_y = np.minimum(np.random.default_rng(0).integers(0, 4, len(y)), 2)
    with pytest.raises(ValueError):
        DistOneVsRestClassifier(LogisticRegression(), max_negatives=0.3).fit(X, ovr_y, sample_weight=w)
    with pytest.raises(NotImplementedError, match="sample_weight"):
        DistOneVsRestClassifier(SGDClassifier()).fit(X, ovr_y, sample_weight=w)
    with pytest.raises(TypeError):
        DistOneVsRestClassifier(LogisticRegression()).fit(X, ovr_y, sample_weight=w, bar=2)
    # entry points whose reference fits row subsets with the unindexed full-length array keep refusing
    with pytest.raises(NotImplementedError):
        DistOneVsOneClassifier(LogisticRegression()).fit(X, ovr_y, sample_weight=w)
    with pytest.raises(NotImplementedError):
        DistMultiModelSearch([("a", LogisticRegression(), {"C": [0.1, 1.0]})], n=2, cv=3).fit(X, y, sample_weight=w)
    with pytest.raises(NotImplementedError):
        DistFeatureEliminator(LogisticRegression(), cv=3).fit(X, y, sample_weight=w)
    from skdist.distribute.ensemble import DistRandomForestClassifier
    with pytest.raises(NotImplementedError):
        DistRandomForestClassifier(n_estimators=2).fit(X, y, sample_weight=w)


def test_unweighted_searches_stage_nothing_new(sw_engine):
    """Without sample_weight nothing changes: no sample weights are staged and an unweighted search stages
    no class weights either (the unweighted kernels run)."""
    X, y, _ = _data(300, 4, 81)
    DistGridSearchCV(LogisticRegression(), {"C": [0.1, 1.0]}, None, cv=3).fit(X, y)
    DistGridSearchCV(LogisticRegression(), {"C": [0.1, 1.0]}, None, cv=3).fit(X, y, sample_weight=None)
    assert sw_engine["eng"].staged == [] and sw_engine["eng"].staged_sw == []


@pytest.mark.filterwarnings("ignore")
def test_refused_one_vs_rest_leaves_nothing_staged(sw_engine):
    """A one-vs-rest fit refused after its row sets were formed (max_negatives with sample_weight: fewer rows
    than weights; a multilabel column whose weights sum to 0) leaves no staged input
    behind: the next fit on the same engine, with as many columns and no row sets of its own, equals the fit
    on a fresh engine."""
    X, y, w = _data(400, 5, 91, 3)
    ym = (np.random.default_rng(1).random((len(y), 3)) < np.array([0.3, 0.5, 0.6])).astype(int)

    def good():
        est = DistOneVsRestClassifier(LogisticRegression(C=0.7)).fit(X, y, sample_weight=w)
        return np.stack([e.coef_.ravel() for e in est.estimators_])

    with pytest.raises(ValueError):
        DistOneVsRestClassifier(LogisticRegression(), max_negatives=0.3, random_state=0).fit(X, y, sample_weight=w)
    after_negatives = good()
    # the first label column's positive rows weigh 0 and class_weight gives its negatives weight 0
    w0 = (ym[:, 0] == 0).astype(np.float64)
    with pytest.raises(ValueError, match="sum"):
        DistOneVsRestClassifier(LogisticRegression(class_weight={0: 0.0, 1: 1.0})).fit(X, ym, sample_weight=w0)
    after_multilabel = good()
    eng = sw_engine["eng"]
    assert getattr(eng, "_ybits", None) is None and getattr(eng, "_mbits", None) is None
    assert eng._cw is None and eng._sw is None
    engine.reset_engine()           # a fresh engine from the same factory
    fresh = good()
    assert sw_engine["eng"] is not eng
    np.testing.assert_array_equal(after_negatives, fresh)
    np.testing.assert_array_equal(after_multilabel, fresh)
