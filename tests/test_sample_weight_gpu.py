"""LogisticRegression with sample_weight on the device: per-row weights in the weighted variants of the
tensor-core kernel (TC_FIT_W, TC_FIT_UNI_W), the CUDA-core path and the multinomial path.

  * identity: all-ones sample weights give the bytes of the fits without them on every path; sample weights
    times 2^k with C times 2^-k give the same bytes (checks the per-column power-of-two normalisation over
    the column's training rows);
  * exact tier: at W = 0 on integer data with power-of-two sample and class weights the gradient is exact up
    to the approximate exp / reciprocal, for every NCHUNK, both fit modes and on SIMT;
  * float tier: loss and gradient at random points against float64 with weights drawn log-uniform over
    2^-30..1, zeros, and one fold 2^-20 times lighter than the rest; the bound rejects one doubled weight;
  * weighted fits stop at their own float64 optimum; frequency weights fit like the repeated rows;
  * the public search against the reference's semantics (tests/weighted_search_oracle.py) and one-vs-rest
    against scikit-learn.
"""
import warnings

import numpy as np
import pytest
from sklearn.linear_model import LogisticRegression
from sklearn.model_selection import StratifiedKFold

from tests import weighted_search_oracle as wso
from tests.test_class_weight_gpu import _binary_optimum, _data, _nchunk, _stage, _weighted_ref

pytestmark = pytest.mark.gpu

RAN = set()     # (NCHUNK, mode) of the weighted tensor-core variants run here with row weights staged


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _stage_weights(eng, fold, y, cf, pos, wpair, rw):
    """Stage sample weights rw [n] and class weights wpair [B, 2] (label 0, label 1) for binary columns
    (held-out fold cf, positive class pos); returns the float32 per-row weights [n, B] of every column
    (0 outside its training rows) and sw_sum (float32 sums in ascending row order)."""
    wpair = np.asarray(wpair, np.float32).reshape(-1, 2)
    wpair = np.broadcast_to(wpair, (len(cf), 2))
    rw = np.asarray(rw, np.float32)
    S = np.zeros((len(y), len(cf)), np.float32)
    sw = np.zeros(len(cf))
    for j, (f, p) in enumerate(zip(cf, pos)):
        m = (fold != f) | (f < 0)
        S[m, j] = rw[m] * wpair[j][(y[m] == p).astype(int)]
        sw[j] = float(np.sum(S[m, j]))
    eng.stage_class_weights(np.ascontiguousarray(wpair), sw)
    eng.stage_sample_weights(rw)
    return S, sw


PATHS = [("tc_fit", 2, False), ("tc_uni", 2, True), ("simt", 1, True)]


@pytest.mark.parametrize("path,kernel,uniform", PATHS, ids=[p[0] for p in PATHS])
def test_identity_binary(eng, path, kernel, uniform):
    X, y = _data(6000, 40, 1)
    fold = _stage(eng, X, y, kernel=kernel)
    cf = np.repeat(np.arange(5, dtype=np.int32), 3)
    B = len(cf)
    pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 2).astype(np.int32)
    C = np.tile([0.01, 0.3, 10.0], 5)
    wp = np.array([0.25, 4.0], np.float32)
    _stage_weights(eng, fold, y, cf, pos, np.ones(2), np.ones(len(y)))
    ones = eng.logreg_fit_batch(C, cf, pos)
    base = eng.logreg_fit_batch(C, cf, pos)
    for k in ("coef", "n_iter", "loss"):
        assert np.array_equal(base[k], ones[k]), k
    _stage_weights(eng, fold, y, cf, pos, wp, np.ones(len(y)))
    cw_only = eng.logreg_fit_batch(C, cf, pos)
    _stage_weights(eng, fold, y, cf, pos, wp, np.ones(len(y)))
    eng.stage_sample_weights(None)          # the class weights alone
    cw_alone = eng.logreg_fit_batch(C, cf, pos)
    for k in ("coef", "n_iter", "loss"):
        assert np.array_equal(cw_only[k], cw_alone[k]), k
    rw = np.exp2(np.random.default_rng(2).integers(-3, 3, len(y))).astype(np.float32)
    rw[::17] = 0.0
    _stage_weights(eng, fold, y, cf, pos, wp, rw)
    a = eng.logreg_fit_batch(C, cf, pos)
    if kernel == 2:
        RAN.add((_nchunk(40), "uni_w" if uniform else "fit_w"))
    assert not np.array_equal(a["coef"], cw_only["coef"])       # the row weights took part
    for k in (-20, 9):
        _stage_weights(eng, fold, y, cf, pos, wp, rw * np.float32(2.0 ** k))
        b = eng.logreg_fit_batch(C * 2.0 ** -k, cf, pos)
        for key in ("coef", "n_iter", "loss"):
            assert np.array_equal(a[key], b[key]), (k, key)


def test_identity_multinomial(eng):
    X, y = _data(5000, 24, 3, n_classes=4)
    fold = _stage(eng, X, y)
    cf = np.arange(5, dtype=np.int32)
    C = np.array([0.05, 0.5, 1.0, 5.0, 50.0])
    wk = np.array([0.5, 2.0, 1.0, 4.0], np.float32)
    sw = np.array([float(np.sum(wk[y[fold != f]])) for f in cf])
    eng.stage_class_weights(np.tile(wk, (5, 1)), sw)
    base = eng.logreg_multinomial_fit_batch(C, cf, 4)
    eng.stage_class_weights(np.tile(wk, (5, 1)), sw)
    eng.stage_sample_weights(np.ones(len(y), np.float32))
    ones = eng.logreg_multinomial_fit_batch(C, cf, 4)
    for k in ("coef", "n_iter", "loss"):
        assert np.array_equal(base[k], ones[k]), k
    rw = np.exp2(np.random.default_rng(4).integers(-2, 3, len(y))).astype(np.float32)
    out = []
    for k in (0, -12, 7):
        r = rw * np.float32(2.0 ** k)
        eng.stage_class_weights(np.tile(wk, (5, 1)), [float(np.sum(r[fold != f] * wk[y[fold != f]])) for f in cf])
        eng.stage_sample_weights(r)
        out.append(eng.logreg_multinomial_fit_batch(C * 2.0 ** -k, cf, 4))
    assert not np.array_equal(out[0]["coef"], base["coef"])
    for o in out[1:]:
        for key in ("coef", "n_iter", "loss"):
            assert np.array_equal(out[0][key], o[key]), key


def test_staging_errors(eng):
    from skdist_b200._lib import SkdError
    X, y = _data(500, 8, 4)
    _stage(eng, X, y)
    with pytest.raises(SkdError, match="n does not match"):
        eng.stage_sample_weights(np.ones(499, np.float32))
    with pytest.raises(SkdError, match="finite"):
        eng.stage_sample_weights(np.r_[np.ones(499), -1.0].astype(np.float32))
    eng.stage_sample_weights(np.ones(500, np.float32))
    with pytest.raises(SkdError, match="class weights"):
        eng.logreg_fit_batch(np.ones(2), np.zeros(2, np.int32), np.ones(2, np.int32))
    # one-shot: the failed call consumed them, the next fit runs without
    eng.logreg_fit_batch(np.ones(2), np.zeros(2, np.int32), np.ones(2, np.int32))


# ---- exact tier: W = 0 -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel,uniform", [(2, True), (2, False), (1, True)], ids=["tc_uni", "tc_fit", "simt"])
@pytest.mark.parametrize("d", [17, 100, 160, 256])
def test_exact_gradient_at_zero(eng, d, kernel, uniform):
    """At W = 0 every training row has sigma = 1/2: the gradient is sum_train s_i (1/2 - y) x / sw_sum with
    s_i = sample weight x class weight, exact on integer data with power-of-two weights."""
    X, y3 = _data(7001, d, 10 + d, n_classes=3, integer=True)
    fold = _stage(eng, X, y3, kernel=kernel)
    cf = np.repeat(np.arange(5, dtype=np.int32), 2)
    B = len(cf)
    pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 3).astype(np.int32)
    wpair = np.array([[0.25, 4.0], [1.0, 0.125]], np.float32)[np.arange(B) % 2]
    rw = np.exp2(np.random.default_rng(d).integers(-8, 5, len(y3))).astype(np.float32)
    rw[::11] = 0.0
    S, sw = _stage_weights(eng, fold, y3, cf, pos, wpair, rw)
    f, g = eng.logreg_loss_grad(np.zeros((B, d + 1)), np.ones(B), cf, pos)
    if kernel == 2:
        RAN.add((_nchunk(d), "uni_w" if uniform else "fit_w"))
    X64 = X.astype(np.float64)
    for j in range(B):
        m = fold != cf[j]
        yb = (y3[m] == pos[j]).astype(np.float64)
        s = S[m, j].astype(np.float64)
        want = ((s * (0.5 - yb)) @ X64[m]) / sw[j]
        bound = 2.0 ** -20 * (s @ np.abs(X64[m])) / sw[j]
        assert np.all(np.abs(g[j, :d] - want) <= bound), (j, np.max(np.abs(g[j, :d] - want) / bound))
        assert abs(g[j, d] - (s @ (0.5 - yb)) / sw[j]) <= 2.0 ** -20 * s.sum() / sw[j]
        assert abs(f[j] - np.log(2.0) * s.sum() / sw[j]) <= 2.0 ** -16


# ---- float tier and fits -----------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel,uniform", [(2, True), (2, False), (1, True)], ids=["tc_uni", "tc_fit", "simt"])
@pytest.mark.parametrize("d", [100, 256])
def test_float_tier_random_points(eng, kernel, uniform, d):
    """Loss and gradient at random points against float64 within the tier-(b) bound of test_tc_eval_gpu.py
    (|x| -> s |x|, n -> sw_sum), with sample weights log-uniform over 2^-30..1, one in ten 0, and every row
    outside fold 3 a further 2^-20 lighter: the columns holding out fold 3 train on those light rows alone.  A reference with one row's weight doubled violates the bound in every column."""
    from tests.test_tc_eval_gpu import EPS_ACC, EPS_ACC_SIMT, _bounds, _float_data, _float_points
    rng = np.random.default_rng(d + kernel + int(uniform))
    n = 4999
    X, scale = _float_data(rng, n, d)
    ycls = rng.integers(0, 3, n).astype(np.int32)
    fold = _stage(eng, X, ycls, kernel=kernel)
    rw = np.exp2(rng.uniform(-30, 0, n)).astype(np.float32)
    rw[rng.random(n) < 0.1] = 0.0
    rw[fold != 3] *= np.float32(2.0 ** -20)
    cf = np.repeat(np.arange(5, dtype=np.int32), 4)
    B = len(cf)
    pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 3).astype(np.int32)
    W = _float_points(rng, B, d, scale)
    C = np.exp(rng.uniform(np.log(1e-2), np.log(1e2), B))
    S, sw = _stage_weights(eng, fold, ycls, cf, pos, [1.0, 3.0], rw)
    f, g = eng.logreg_loss_grad(W, C, cf, pos)
    if kernel == 2:
        RAN.add((_nchunk(d), "fit_w" if not uniform else "uni_w"))
    yb = (ycls[:, None] == pos[None, :]).astype(np.float64)
    M = (fold[:, None] != cf[None, :]).astype(np.float64)
    ref = _weighted_ref(X, yb, S.astype(np.float64), M, W, C, sw)
    bf, bg = _bounds(ref, EPS_ACC if kernel == 2 else EPS_ACC_SIMT)
    assert np.all(np.abs(f - ref["f"]) <= bf), np.max(np.abs(f - ref["f"]) / bf)
    assert np.all(np.abs(g - ref["g"]) <= bg), np.max(np.abs(g - ref["g"]) / np.maximum(bg, 1e-300))
    for j in range(B):
        # the training row of largest influence |s r| among the heavier tenth: doubling its weight (sw_sum
        # included) must move the gradient past the bound
        rows = np.flatnonzero(ref["Mf"][:, j] > 0)
        infl = np.abs(ref["Mf"][rows, j] * ref["R"][rows, j])
        i = rows[np.argsort(infl)[int(len(rows) * 0.95)]]
        s_i = ref["Mf"][i, j]
        xi = np.append(X[i].astype(np.float64), 1.0)
        data = ref["g"][j] - ref["pen"][j]
        wrong = (data * sw[j] + s_i * ref["R"][i, j] * xi) / (sw[j] + s_i) + ref["pen"][j]
        assert np.any(np.abs(wrong - ref["g"][j]) > bg[j]), ("bound cannot see one wrong weight", j)


def _check_optimum(X, y01, s, C, sw, coef, loss, tol):
    obj, grad = _binary_optimum(X, y01, s, C, sw, coef.astype(np.float64))
    assert np.abs(grad).max() <= 2 * tol, np.abs(grad).max()
    assert abs(loss - obj) <= 1e-6, (loss, obj)


@pytest.mark.parametrize("kernel,uniform", [(2, True), (2, False), (1, True)], ids=["tc_uni", "tc_fit", "simt"])
def test_weighted_fits_stop_at_their_own_optimum(eng, kernel, uniform):
    """Every column (5 and 40 folds) with log-normal sample weights and class weights {1, 3} stops where the
    float64 gradient of its own weighted objective is <= 2 tol, and reports that objective to 1e-6."""
    X, y = _data(20000, 30, 30, n_classes=3)
    _stage(eng, X, y, kernel=kernel)
    rw = np.exp(np.random.default_rng(7).normal(0.0, 1.0, len(y))).astype(np.float32)
    rw[::13] = 0.0
    tol = 1e-4
    for nf in (5, 40):
        fold = (np.arange(len(y)) % nf).astype(np.int8)
        eng.stage_folds(fold, nf)
        cf = np.arange(nf, dtype=np.int32)
        pos = np.ones(nf, np.int32) if uniform else (np.arange(nf) % 3).astype(np.int32)
        S, sw = _stage_weights(eng, fold, y, cf, pos, [1.0, 3.0], rw)
        C = np.full(nf, 0.5)
        res = eng.logreg_fit_batch(C, cf, pos, tol=tol, max_iter=500)
        for j in range(nf):
            m = fold != cf[j]
            _check_optimum(X[m], (y[m] == pos[j]).astype(np.float64), S[m, j].astype(np.float64), C[j], sw[j],
                           res["coef"][j], res["loss"][j], tol)


def test_weighted_multinomial_fits_stop_at_their_own_optimum(eng):
    from scipy.special import logsumexp, softmax
    K, d, tol = 4, 20, 1e-4
    X, y = _data(12000, d, 33, n_classes=K)
    _stage(eng, X, y)
    wk = np.array([0.5, 2.0, 1.0, 3.0], np.float32)
    rw = np.exp(np.random.default_rng(8).normal(0.0, 1.0, len(y))).astype(np.float32)
    rw[::9] = 0.0
    for nf in (5, 40):
        fold = (np.arange(len(y)) % nf).astype(np.int8)
        eng.stage_folds(fold, nf)
        cf = np.arange(nf, dtype=np.int32)
        sw = np.array([float(np.sum(rw[fold != f] * wk[y[fold != f]])) for f in cf])
        eng.stage_class_weights(np.tile(wk, (nf, 1)), sw)
        eng.stage_sample_weights(rw)
        C = np.full(nf, 0.7)
        res = eng.logreg_multinomial_fit_batch(C, cf, K, tol=tol, max_iter=500)
        for j in range(nf):
            m = fold != cf[j]
            Xm = X[m].astype(np.float64)
            s = (rw[m] * wk[y[m]]).astype(np.float64)
            Wc = res["coef"][j].astype(np.float64)
            Z = Xm @ Wc[:, :d].T + Wc[:, d]
            l2 = 1.0 / (C[j] * sw[j])
            obj = (s @ (logsumexp(Z, axis=1) - Z[np.arange(len(Z)), y[m]])) / sw[j] + 0.5 * l2 * (Wc[:, :d] ** 2).sum()
            G = softmax(Z, axis=1)
            G[np.arange(len(Z)), y[m]] -= 1.0
            G *= s[:, None]
            grad = np.concatenate([(G.T @ Xm) / sw[j] + l2 * Wc[:, :d], G.sum(0)[:, None] / sw[j]], axis=1)
            assert np.abs(grad).max() <= 2 * tol, (nf, j, np.abs(grad).max())
            assert abs(res["loss"][j] - obj) <= 1e-6, (nf, j, res["loss"][j], obj)


@pytest.mark.parametrize("kernel", [2, 1], ids=["tc", "simt"])
def test_frequency_weights_fit_like_repeated_rows(eng, kernel):
    """Integer weights 0..3 and the matrix with every row repeated that many times: both device fits meet the
    optimum criterion of the same float64 objective, and predict the same labels on X."""
    X, y = _data(8000, 24, 60)
    rw = np.random.default_rng(9).integers(0, 4, len(y)).astype(np.float32)
    Xr, yr = np.repeat(X, rw.astype(int), axis=0), np.repeat(y, rw.astype(int))
    C, tol = np.array([0.3]), 1e-4
    out = []
    for Xf, yf, w in ((X, y, rw), (Xr, yr, None)):
        eng.set_kernel(kernel)
        eng.stage_x(Xf)
        eng.stage_labels(yf)
        eng.stage_folds(None, 0)
        if w is not None:
            _stage_weights(eng, np.zeros(len(yf), np.int8), yf, np.array([-1]), np.array([1]), [1.0, 1.0], w)
        out.append(eng.logreg_fit_batch(C, np.array([-1], np.int32), np.array([1], np.int32), tol=tol, max_iter=500))
    sw = float(np.sum(rw))
    for res in out:
        _check_optimum(X, (y == 1).astype(np.float64), rw.astype(np.float64), C[0], sw, res["coef"][0],
                       res["loss"][0], tol)
    dec = [X.astype(np.float64) @ r["coef"][0, :-1].astype(np.float64) + r["coef"][0, -1] for r in out]
    np.testing.assert_array_equal(dec[0] > 0, dec[1] > 0)


# ---- public API ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_classes", [2, 4])
def test_search_against_reference_semantics(n_classes):
    """DistGridSearchCV(..., scoring=...).fit(X, y, sample_weight=w) against the reference's search with the same
    fit_params (weighted fits, unweighted scores): equal best_params_, mean_test_score within the tolerances of
    test_class_weight_gpu.test_search_against_scikit_learn, the refit close to LogisticRegression.fit with w."""
    from skdist.distribute.search import DistGridSearchCV
    X, y = _data(3000, 12, 70 + n_classes, n_classes=n_classes)
    w = np.exp(np.random.default_rng(n_classes).normal(0.0, 1.0, len(y)))
    w[::10] = 0.0
    cw3 = {c: 1.0 + 0.5 * c for c in range(n_classes)}
    grid = {"C": [0.1, 1.0], "class_weight": [None, "balanced", cw3]}
    cv = StratifiedKFold(5)
    for sc in (["accuracy", "f1_macro", "roc_auc", "neg_log_loss"] if n_classes == 2
               else ["accuracy", "f1_macro", "neg_log_loss"]):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gs = DistGridSearchCV(LogisticRegression(max_iter=1000), grid, None, cv=cv, scoring=sc).fit(
                X, y, sample_weight=w)
            cands = list(gs.cv_results_["params"])
            ref = wso.search_cv(LogisticRegression(max_iter=1000), cands, X, y, cv=cv, scoring=sc,
                                fit_params={"sample_weight": w})
        assert gs.best_params_ == ref["best_params_"], sc
        np.testing.assert_allclose(gs.cv_results_["mean_test_score"], ref["cv_results_"]["mean_test_score"],
                                   rtol=0, atol=2e-3 if sc != "neg_log_loss" else 1e-4, err_msg=sc)
        best = ref["best_estimator_"]
        np.testing.assert_allclose(gs.best_estimator_.coef_, best.coef_, rtol=0, atol=2e-3 * np.abs(best.coef_).max())


@pytest.mark.parametrize("target", ["multiclass", "multilabel"])
def test_one_vs_rest_against_scikit_learn(target):
    """Every label column against LogisticRegression().fit(X, y == c, sample_weight=w): equal predictions,
    n_iter within 1."""
    from skdist.distribute.multiclass import DistOneVsRestClassifier
    X, y = _data(3000, 10, 80, n_classes=4)
    if target == "multilabel":
        y = (np.random.default_rng(2).random((3000, 3)) < [0.1, 0.3, 0.5]).astype(int)
        y[:, 0] |= (X[:, 0] > 1.0)
    w = np.exp(np.random.default_rng(5).normal(0.0, 1.0, len(X)))
    w[::7] = 0.0
    lr = LogisticRegression(class_weight="balanced", max_iter=1000)
    est = DistOneVsRestClassifier(lr).fit(X, y, sample_weight=w)
    cols = y.T if target == "multilabel" else [y == c for c in range(4)]
    for e, yc in zip(est.estimators_, cols):
        ref = LogisticRegression(class_weight="balanced", max_iter=1000).fit(X, yc.astype(int), sample_weight=w)
        np.testing.assert_array_equal(e.predict(X), ref.predict(X))
        assert abs(int(e.n_iter_[0]) - int(ref.n_iter_[0])) <= 1


def test_every_weighted_variant_ran_with_row_weights():
    want = {(c, m) for c in (1, 2, 3, 4) for m in ("fit_w", "uni_w")}
    assert RAN == want, sorted(want - RAN)
