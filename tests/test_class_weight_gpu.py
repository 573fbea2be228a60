"""LogisticRegression(class_weight=...) on the device: the weighted variants of the tensor-core kernel
(TC_FIT_W, TC_FIT_UNI_W), the CUDA-core path and the multinomial path.

  * identity: unit weights (and "balanced" on equal class counts) give the unweighted results byte for
    byte; weights times 2^k with C times 2^-k (the same objective up to the factor 2^k) give the same
    bytes as well, which checks the power-of-two normalisation of the tensor-core epilogue;
  * exact tier: at W = 0 on integer data with power-of-two weights the gradient is formed exactly up to
    the approximate exp / reciprocal, for every NCHUNK, both fit modes and on SIMT;
  * float tier: loss and gradient at random points against a float64 weighted reference;
  * fits stop where the float64 gradient of their own weighted objective is below the tolerance;
  * the public search against scikit-learn's GridSearchCV.
"""
import warnings

import numpy as np
import pytest
from sklearn.linear_model import LogisticRegression
from sklearn.model_selection import GridSearchCV, ShuffleSplit, StratifiedKFold

from tests import weighted_oracle as wo

pytestmark = pytest.mark.gpu

# (NCHUNK, mode) of the weighted tensor-core variants run by the loss/gradient tests of this module: the
# columns of a call share one held-out fold per group and have either one positive class (TC_FIT_UNI_W,
# "uni_w") or several (TC_FIT_W, "fit_w"), so the mode follows from the call as in test_tc_eval_gpu.py
RAN = set()


def _nchunk(d):
    return (d + 63) // 64


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _data(n, d, seed, n_classes=2, integer=False):
    rng = np.random.default_rng(seed)
    if integer:
        e = rng.integers(-6, 7, d)
        X = (rng.integers(-7, 8, (n, d)) * np.exp2(e)).astype(np.float32)
    else:
        X = rng.standard_normal((n, d)).astype(np.float32)
    w = rng.standard_normal((n_classes, d))
    y = np.argmax(X.astype(np.float64) @ w.T + rng.standard_normal((n, n_classes)), axis=1).astype(np.int32)
    return X, y


def _stage(eng, X, y, nf=5, kernel=0):
    fold = (np.arange(len(y)) % nf).astype(np.int8)
    eng.set_kernel(kernel)
    eng.stage_x(X)
    eng.stage_labels(y)
    eng.stage_folds(fold, nf)
    return fold


def _binary_weights(fold, y, cf, wpair):
    """[B, 2] weights and the float32 sum over every column's training rows (ascending order)."""
    W = np.tile(np.asarray(wpair, np.float32), (len(cf), 1))
    sw = np.array([float(np.sum(W[j][y[(fold != f) | (f < 0)]])) for j, f in enumerate(cf)])
    return W, sw


PATHS = [("tc_fit", 2, False), ("tc_uni", 2, True), ("simt", 1, True)]


@pytest.mark.parametrize("path,kernel,uniform", PATHS, ids=[p[0] for p in PATHS])
def test_identity_binary(eng, path, kernel, uniform):
    X, y = _data(6000, 40, 1)
    fold = _stage(eng, X, y, kernel=kernel)
    cf = np.repeat(np.arange(5, dtype=np.int32), 3)
    B = len(cf)
    pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 2).astype(np.int32)
    C = np.tile([0.01, 0.3, 10.0], 5)
    base = eng.logreg_fit_batch(C, cf, pos)
    W, sw = _binary_weights(fold, y, cf, (1.0, 1.0))
    eng.stage_class_weights(W, sw)
    ones = eng.logreg_fit_batch(C, cf, pos)
    for k in ("coef", "n_iter", "loss"):
        assert np.array_equal(base[k], ones[k]), k
    # weights {0: 1/4, 1: 4}, then the same times 2^k with C times 2^-k
    W, sw = _binary_weights(fold, y, cf, (0.25, 4.0))
    eng.stage_class_weights(W, sw)
    a = eng.logreg_fit_batch(C, cf, pos)
    assert not np.array_equal(a["coef"], base["coef"])       # the weighted variant ran
    for k in (-7, 5):
        eng.stage_class_weights(W * np.float32(2.0 ** k), sw * 2.0 ** k)
        b = eng.logreg_fit_batch(C * 2.0 ** -k, cf, pos)
        for key in ("coef", "n_iter", "loss"):
            assert np.array_equal(a[key], b[key]), (k, key)


def test_identity_balanced_equal_counts(eng):
    """'balanced' on training rows with exactly equal class counts is all ones."""
    X, _ = _data(4000, 20, 2)
    y = (np.arange(4000) // 5 % 2).astype(np.int32)       # every fold (i % 5) holds 400 rows of each class
    fold = _stage(eng, X, y, kernel=2)
    cf = np.arange(5, dtype=np.int32)
    from skdist_b200.distribute.logreg_family import _ClassWeights
    cw = _ClassWeights(np.array([0, 1]), y)
    cw.set_folds(fold)
    cols = [cw.column("balanced", f) for f in cf]
    assert all(np.array_equal(c[0], [1.0, 1.0]) for c in cols)
    C = np.ones(5)
    base = eng.logreg_fit_batch(C, cf, np.ones(5, np.int32))
    eng.stage_class_weights(np.stack([c[0] for c in cols]), [c[1] for c in cols])
    bal = eng.logreg_fit_batch(C, cf, np.ones(5, np.int32))
    for k in ("coef", "n_iter", "loss"):
        assert np.array_equal(base[k], bal[k]), k


def test_identity_multinomial(eng):
    X, y = _data(5000, 24, 3, n_classes=4)
    fold = _stage(eng, X, y)
    cf = np.arange(5, dtype=np.int32)
    C = np.array([0.05, 0.5, 1.0, 5.0, 50.0])
    base = eng.logreg_multinomial_fit_batch(C, cf, 4)
    sw = np.array([float((fold != f).sum()) for f in cf])
    eng.stage_class_weights(np.ones((5, 4), np.float32), sw)
    ones = eng.logreg_multinomial_fit_batch(C, cf, 4)
    for k in ("coef", "n_iter", "loss"):
        assert np.array_equal(base[k], ones[k]), k
    Wc = np.tile(np.array([0.5, 2.0, 1.0, 4.0], np.float32), (5, 1))
    swc = np.array([float(np.sum(Wc[0][y[fold != f]])) for f in cf])
    eng.stage_class_weights(Wc, swc)
    a = eng.logreg_multinomial_fit_batch(C, cf, 4)
    assert not np.array_equal(a["coef"], base["coef"])


def test_stage_mismatch_fails(eng):
    from skdist_b200._lib import SkdError
    X, y = _data(500, 8, 4)
    _stage(eng, X, y)
    eng.stage_class_weights(np.ones((3, 2), np.float32), np.full(3, 400.0))
    with pytest.raises(SkdError, match="class weights"):
        eng.logreg_fit_batch(np.ones(2), np.zeros(2, np.int32), np.ones(2, np.int32))
    eng.stage_class_weights(np.ones((2, 3), np.float32), np.full(2, 400.0))
    with pytest.raises(SkdError, match="class weights"):
        eng.logreg_multinomial_fit_batch(np.ones(2), np.zeros(2, np.int32), 2)
    with pytest.raises(SkdError, match="finite"):
        eng.stage_class_weights(np.array([[1.0, -1.0]], np.float32), np.array([1.0]))


# ---- exact tier: W = 0 -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel,uniform", [(2, True), (2, False), (1, True)], ids=["tc_uni", "tc_fit", "simt"])
@pytest.mark.parametrize("d", [17, 100, 160, 256])
def test_exact_gradient_at_zero(eng, d, kernel, uniform):
    """At W = 0 every training row has sigma = 1/2: the gradient is sum_train w_y (1/2 - y) x / sw_sum,
    formed exactly on integer data with power-of-two weights up to the approximate exp / reciprocal."""
    X, y3 = _data(7001, d, 10 + d, n_classes=3, integer=True)
    fold = _stage(eng, X, y3, kernel=kernel)
    cf = np.repeat(np.arange(5, dtype=np.int32), 2)
    B = len(cf)
    pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 3).astype(np.int32)
    wpair = np.array([[0.25, 4.0], [1.0, 0.125]], np.float32)[np.arange(B) % 2]
    sw = np.array([float(np.sum(wpair[j][(y3[fold != cf[j]] == pos[j]).astype(int)])) for j in range(B)])
    eng.stage_class_weights(wpair, sw)
    f, g = eng.logreg_loss_grad(np.zeros((B, d + 1)), np.ones(B), cf, pos)
    if kernel == 2:
        RAN.add((_nchunk(d), "uni_w" if uniform else "fit_w"))
    X64 = X.astype(np.float64)
    for j in range(B):
        m = fold != cf[j]
        yb = (y3[m] == pos[j]).astype(np.float64)
        s = wpair[j][yb.astype(int)].astype(np.float64)
        want = ((s * (0.5 - yb)) @ X64[m]) / sw[j]
        bound = 2.0 ** -20 * (s @ np.abs(X64[m])) / sw[j]
        assert np.all(np.abs(g[j, :d] - want) <= bound), (j, np.max(np.abs(g[j, :d] - want) / bound))
        assert abs(g[j, d] - (s @ (0.5 - yb)) / sw[j]) <= 2.0 ** -20 * s.sum() / sw[j]
        assert abs(f[j] - np.log(2.0) * s.sum() / sw[j]) <= 2.0 ** -16


# ---- float tier and fits -----------------------------------------------------------------------------------
def _weighted_ref(X, yb, S, M, W, C, sw):
    """float64 objective, gradient and the tier-(b) error terms of test_tc_eval_gpu._bounds with every
    training row weighted: Mf = the row's weight, n_train = sw_sum."""
    from tests.test_tc_eval_gpu import EPS_Z
    d = X.shape[1]
    X64 = X.astype(np.float64)
    W32 = W.astype(np.float32).astype(np.float64)
    Z = X64 @ W32[:, :d].T + W32[:, d]
    Mf = M * S
    l2 = 1.0 / (C * sw)
    R = 1.0 / (1.0 + np.exp(-Z)) - yb
    L = np.logaddexp(0.0, Z) - yb * Z
    f = (L * Mf).sum(0) / sw + 0.5 * l2 * (W[:, :d] ** 2).sum(1)
    g = np.empty_like(W)
    g[:, :d] = (X64.T @ (R * Mf)).T / sw[:, None] + l2[:, None] * W[:, :d]
    g[:, d] = (R * Mf).sum(0) / sw
    dz = EPS_Z * (np.abs(X64) @ np.abs(W32[:, :d]).T + np.abs(W32[:, d]))
    pen = np.zeros_like(W)
    pen[:, :d] = l2[:, None] * W[:, :d]
    return dict(f=f, g=g, pen=pen, R=R, Mf=Mf, ntr=sw, dz=dz, Xa=np.abs(X64))


@pytest.mark.parametrize("kernel,uniform", [(2, True), (2, False), (1, True)], ids=["tc_uni", "tc_fit", "simt"])
@pytest.mark.parametrize("ratio", [1e-3, 1e3, 2.0 ** -30])
def test_float_tier_random_points(eng, kernel, uniform, ratio):
    """Loss and gradient at random points against float64 within the tier-(b) bound of
    test_tc_eval_gpu.py with |x| -> sw |x| and n -> sw_sum (weights 1 and `ratio`; 2^-30 lies below the fp16
    normal range after the normalisation).  A reference with one wrong weight (a row of median influence in
    the heavier class, weight doubled) violates the bound in every column."""
    from tests.test_tc_eval_gpu import EPS_ACC, EPS_ACC_SIMT, _bounds, _float_data, _float_points
    rng = np.random.default_rng(int(ratio * 7) % 1000 + 11)
    n, d = 4999, 100
    X, scale = _float_data(rng, n, d)
    ycls = rng.integers(0, 3, n).astype(np.int32)
    fold = _stage(eng, X, ycls, kernel=kernel)
    cf = np.repeat(np.arange(5, dtype=np.int32), 4)
    B = len(cf)
    pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 3).astype(np.int32)
    W = _float_points(rng, B, d, scale)
    C = np.exp(rng.uniform(np.log(1e-2), np.log(1e2), B))
    wp = np.array([1.0, ratio], np.float32)
    yb = (ycls[:, None] == pos[None, :]).astype(np.float64)
    M = (fold[:, None] != cf[None, :]).astype(np.float64)
    S32 = wp[yb.astype(int)]
    sw = np.array([float(np.sum(S32[M[:, j] > 0, j])) for j in range(B)])
    eng.stage_class_weights(np.tile(wp, (B, 1)), sw)
    f, g = eng.logreg_loss_grad(W, C, cf, pos)
    if kernel == 2:
        RAN.add((_nchunk(d), "fit_w" if not uniform else "uni_w"))
    ref = _weighted_ref(X, yb, S32.astype(np.float64), M, W, C, sw)
    bf, bg = _bounds(ref, EPS_ACC if kernel == 2 else EPS_ACC_SIMT)
    assert np.all(np.abs(f - ref["f"]) <= bf), np.max(np.abs(f - ref["f"]) / bf)
    assert np.all(np.abs(g - ref["g"]) <= bg), np.max(np.abs(g - ref["g"]) / np.maximum(bg, 1e-300))
    for j in range(B):
        # a row of the class that carries the larger weight (at 1000 : 1 a light row's whole contribution
        # lies below fp32 resolution of the sums), of median influence |w r| among those rows; the wrong
        # reference doubles its weight, sw_sum included
        heavy = ref["Mf"][:, j] == ref["Mf"][:, j].max()
        rows = np.flatnonzero(heavy & (ref["Mf"][:, j] > 0))
        infl = np.abs(ref["Mf"][rows, j] * ref["R"][rows, j])
        i = rows[np.argsort(infl)[len(rows) // 2]]
        s_i = ref["Mf"][i, j]
        xi = np.append(X[i].astype(np.float64), 1.0)
        data = ref["g"][j] - ref["pen"][j]
        wrong = (data * sw[j] + s_i * ref["R"][i, j] * xi) / (sw[j] + s_i) + ref["pen"][j]
        assert np.any(np.abs(wrong - ref["g"][j]) > bg[j]), ("bound cannot see one wrong weight", j)


def _binary_optimum(X, y01, s, C, sw, w):
    d = X.shape[1]
    z = X.astype(np.float64) @ w[:d] + w[d]
    l2 = 1.0 / (C * sw)
    obj = (s @ (np.logaddexp(0, z) - y01 * z)) / sw + 0.5 * l2 * (w[:d] @ w[:d])
    r = s * (1.0 / (1.0 + np.exp(-z)) - y01)
    grad = np.concatenate([(r @ X.astype(np.float64)) / sw + l2 * w[:d], [r.sum() / sw]])
    return obj, grad


@pytest.mark.parametrize("kernel,uniform", [(2, True), (2, False), (1, True)], ids=["tc_uni", "tc_fit", "simt"])
def test_weighted_fits_stop_at_their_own_optimum(eng, kernel, uniform):
    """Every weighted column (5 and 40 folds) stops where the float64 gradient of its own weighted objective
    is <= 2 tol, and reports that objective to 1e-6."""
    X, y = _data(20000, 30, 30, n_classes=3)
    _stage(eng, X, y, kernel=kernel)
    tol = 1e-4
    for nf in (5, 40):
        fold = (np.arange(len(y)) % nf).astype(np.int8)
        eng.stage_folds(fold, nf)
        cf = np.arange(nf, dtype=np.int32)
        pos = np.ones(nf, np.int32) if uniform else (np.arange(nf) % 3).astype(np.int32)
        wp = np.array([1.0, 3.0], np.float32)
        sw = np.array([float(np.sum(wp[(y[fold != f] == p).astype(int)])) for f, p in zip(cf, pos)])
        eng.stage_class_weights(np.tile(wp, (nf, 1)), sw)
        C = np.full(nf, 0.5)
        res = eng.logreg_fit_batch(C, cf, pos, tol=tol, max_iter=500)
        for j in range(nf):
            m = fold != cf[j]
            y01 = (y[m] == pos[j]).astype(np.float64)
            obj, grad = _binary_optimum(X[m], y01, wp[y01.astype(int)].astype(np.float64), C[j], sw[j],
                                        res["coef"][j].astype(np.float64))
            assert np.abs(grad).max() <= 2 * tol, (nf, j, np.abs(grad).max())
            assert abs(res["loss"][j] - obj) <= 1e-6, (nf, j, res["loss"][j], obj)


def test_weighted_multinomial_fits_stop_at_their_own_optimum(eng):
    """Multinomial columns at 5 and 40 folds: the float64 gradient of the weighted objective
    sum_train w_y (logsumexp(z) - z_y) / sw_sum + l2 / 2 ||W||^2 at the returned point is <= 2 tol and the
    reported loss is that objective to 1e-6."""
    from scipy.special import logsumexp, softmax
    K, d, tol = 4, 20, 1e-4
    X, y = _data(12000, d, 33, n_classes=K)
    _stage(eng, X, y)
    wk = np.array([0.5, 2.0, 1.0, 3.0], np.float32)
    for nf in (5, 40):
        fold = (np.arange(len(y)) % nf).astype(np.int8)
        eng.stage_folds(fold, nf)
        cf = np.arange(nf, dtype=np.int32)
        sw = np.array([float(np.sum(wk[y[fold != f]])) for f in cf])
        eng.stage_class_weights(np.tile(wk, (nf, 1)), sw)
        C = np.full(nf, 0.7)
        res = eng.logreg_multinomial_fit_batch(C, cf, K, tol=tol, max_iter=500)
        for j in range(nf):
            m = fold != cf[j]
            Xm = X[m].astype(np.float64)
            s = wk[y[m]].astype(np.float64)
            Wc = res["coef"][j].astype(np.float64)          # [K, d + 1]
            Z = Xm @ Wc[:, :d].T + Wc[:, d]
            l2 = 1.0 / (C[j] * sw[j])
            obj = (s @ (logsumexp(Z, axis=1) - Z[np.arange(len(Z)), y[m]])) / sw[j] + 0.5 * l2 * (Wc[:, :d] ** 2).sum()
            G = softmax(Z, axis=1)
            G[np.arange(len(Z)), y[m]] -= 1.0
            G *= s[:, None]
            grad = np.concatenate([(G.T @ Xm) / sw[j] + l2 * Wc[:, :d], G.sum(0)[:, None] / sw[j]], axis=1)
            assert np.abs(grad).max() <= 2 * tol, (nf, j, np.abs(grad).max())
            assert abs(res["loss"][j] - obj) <= 1e-6, (nf, j, res["loss"][j], obj)


# ---- public API ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_classes", [2, 4])
@pytest.mark.parametrize("cvname", ["strat", "shuffle"])
def test_search_against_scikit_learn(n_classes, cvname):
    from skdist.distribute.search import DistGridSearchCV
    X, y = _data(3000, 12, 40 + n_classes, n_classes=n_classes)
    if n_classes == 2:
        y = np.where(np.random.default_rng(1).random(len(y)) < 0.35, y, 0)
        cw3 = {0: 1, 1: 5}
        scoring = ["accuracy", "f1_macro", "roc_auc", "neg_log_loss"]
    else:
        cw3 = {0: 1, 1: 5, 2: 2, 3: 1}
        scoring = ["accuracy", "f1_macro", "neg_log_loss"]
    cv = StratifiedKFold(5) if cvname == "strat" else ShuffleSplit(4, test_size=0.25, random_state=3)
    grid = {"C": [0.1, 1.0], "class_weight": [None, "balanced", cw3]}
    for sc in scoring:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gs = DistGridSearchCV(LogisticRegression(max_iter=1000), grid, None, cv=cv, scoring=sc).fit(X, y)
            ref = GridSearchCV(LogisticRegression(max_iter=1000), grid, cv=cv, scoring=sc).fit(X, y)
        assert gs.best_params_ == ref.best_params_, sc
        np.testing.assert_allclose(gs.cv_results_["mean_test_score"], ref.cv_results_["mean_test_score"],
                                   rtol=0, atol=2e-3 if sc != "neg_log_loss" else 1e-4, err_msg=sc)
        np.testing.assert_allclose(gs.best_estimator_.coef_, ref.best_estimator_.coef_, rtol=0,
                                   atol=2e-3 * np.abs(ref.best_estimator_.coef_).max())


# ---- one-vs-rest, one-vs-one, feature elimination ------------------------------------------------------------
@pytest.mark.parametrize("which", ["ovr", "ovr_multilabel", "ovr_max_negatives", "ovo", "eliminator2", "eliminator4"])
def test_entry_points_against_scikit_learn(which):
    """class_weight="balanced" through the other entry points: predictions equal to scikit-learn's
    counterparts, n_iter within 1."""
    from sklearn.multiclass import OneVsOneClassifier, OneVsRestClassifier
    from skdist.distribute.eliminate import DistFeatureEliminator
    from skdist.distribute.multiclass import DistOneVsOneClassifier, DistOneVsRestClassifier
    lr = LogisticRegression(class_weight="balanced", max_iter=1000)
    X, y = _data(3000, 10, 50, n_classes=2 if which == "eliminator2" else 4)
    if which == "ovr_multilabel":
        y = (np.random.default_rng(2).random((3000, 3)) < [0.1, 0.3, 0.5]).astype(int)
        y[:, 0] |= (X[:, 0] > 1.0)
    if which.startswith("ovr"):
        kw = dict(max_negatives=0.5, random_state=2) if which == "ovr_max_negatives" else {}
        est = DistOneVsRestClassifier(lr, **kw).fit(X, y)
        if kw:
            from skdist_b200.distribute.multiclass import _negatives_rows
            for k, c in enumerate(np.unique(y)):
                rows = _negatives_rows(y == c, 0.5, 2, "ratio")
                ref = LogisticRegression(class_weight="balanced", max_iter=1000).fit(X[rows], (y[rows] == c).astype(int))
                assert np.array_equal(est.estimators_[k].predict(X), ref.predict(X))
                assert abs(int(est.estimators_[k].n_iter_[0]) - int(ref.n_iter_[0])) <= 1
            return
        ref = OneVsRestClassifier(lr).fit(X, y)
        pairs = zip(est.estimators_, ref.estimators_)
    elif which == "ovo":
        est = DistOneVsOneClassifier(lr).fit(X, y)
        ref = OneVsOneClassifier(lr).fit(X, y)
        pairs = zip(est.estimators_, ref.estimators_)
    else:
        est = DistFeatureEliminator(lr, cv=StratifiedKFold(3), step=3).fit(X, y)
        keep = np.asarray(est.best_features_)
        ref = LogisticRegression(class_weight="balanced", max_iter=1000).fit(X[:, keep], y)
        pairs = [(est.best_estimator_, ref)]
        np.testing.assert_array_equal(est.predict(X), ref.predict(X[:, keep]))
    for a, b in pairs:
        assert abs(int(a.n_iter_[0]) - int(b.n_iter_[0])) <= 1
    if which != "eliminator2" and which != "eliminator4":
        np.testing.assert_array_equal(est.predict(X), ref.predict(X))


def test_every_weighted_variant_ran():
    want = {(c, m) for c in (1, 2, 3, 4) for m in ("fit_w", "uni_w")}
    assert RAN == want, sorted(want - RAN)
