"""The references of tests/scoring_reference.py against scikit-learn, without a GPU: the GPU tests of the scoring and
inference kernels (tests/test_scoring_inference_gpu.py) are only as good as these."""
import warnings

import numpy as np
import pytest
from scipy.special import expit
from sklearn.ensemble import ExtraTreesClassifier, ExtraTreesRegressor, RandomForestClassifier, RandomForestRegressor
from sklearn.metrics import accuracy_score, log_loss, r2_score, roc_auc_score

from skdist_b200.distribute.predict import _forest_arrays
from tests import scoring_reference as sr


def _codes_and_folds(rng, n, nf, B):
    fold = rng.integers(0, nf, n).astype(np.int8)
    code = rng.choice(np.r_[np.arange(nf), -2, -3 - np.arange(nf)], B).astype(np.int32)
    return fold, code


def test_select_matches_the_scoring_codes():
    fold = np.array([0, 1, 2, 0, 1, 2, 2])
    M = sr.select(np.array([0, 2, -2, -3, -5]), fold, 7)
    assert np.array_equal(M[:, 0], fold == 0) and np.array_equal(M[:, 1], fold == 2)
    assert M[:, 2].all()
    assert np.array_equal(M[:, 3], fold != 0) and np.array_equal(M[:, 4], fold != 2)
    assert np.array_equal(sr.select(np.array([-2]), None, 4), np.ones((4, 1), bool))


@pytest.mark.parametrize("seed", range(4))
def test_auc_counts_match_roc_auc_score(seed):
    """Ties within and across classes, -0.0 next to +0.0, and a selection with one class only."""
    rng = np.random.default_rng(seed)
    n = 3000
    z = rng.integers(-6, 7, n).astype(np.float64) * 0.25     # 49 distinct values: long tie groups
    z[z == 0] = np.where(rng.random((z == 0).sum()) < 0.5, -0.0, 0.0)
    y = rng.random(n) < 0.3
    u2, npos, nneg = sr.auc_counts(z, y)
    assert (npos, nneg) == (y.sum(), (~y).sum())
    assert u2 / (2.0 * npos * nneg) == pytest.approx(roc_auc_score(y, z), rel=1e-13)
    u2, npos, nneg = sr.auc_counts(np.zeros(n), y)            # every row tied
    assert 2 * u2 == 2 * npos * nneg
    assert sr.auc_counts(z, np.zeros(n, bool))[1] == 0 and sr.auc_counts(z, np.ones(n, bool))[2] == 0
    # pair counts above 2^31 stay exact
    u2, npos, nneg = sr.auc_counts(np.arange(120_000.0), np.arange(120_000) % 2 == 0)
    assert npos * nneg > 2 ** 31 and u2 == 2 * sum(range(60_000))


def test_counts_and_sse_match_sklearn_metrics():
    rng = np.random.default_rng(5)
    n, B, nf = 2000, 12, 5
    Z = rng.integers(-3, 4, (n, B)).astype(np.float64)          # many z == 0 rows: predicted negative
    ycls = rng.integers(0, 3, n)
    pos = rng.integers(0, 3, B)
    fold, code = _codes_and_folds(rng, n, nf, B)
    yreal = rng.standard_normal(n).astype(np.float32)
    correct, count = sr.accuracy_counts(Z, ycls, pos, code, fold)
    s, cnt = sr.sse(Z, yreal, code, fold)
    M = sr.select(code, fold, n)
    for j in range(B):
        m = M[:, j]
        yb = ycls[m] == pos[j]
        assert count[j] == m.sum() == cnt[j]
        assert correct[j] == round(accuracy_score(yb, Z[m, j] > 0) * m.sum())
        y64 = yreal[m].astype(np.float64)
        r2 = 1.0 - s[j] / ((y64 - y64.mean()) ** 2).sum()
        assert r2 == pytest.approx(r2_score(y64, Z[m, j]), rel=1e-12, abs=1e-12)
        u2, npos, nneg = sr.auc_counts(Z[m, j], yb)
        assert u2 / (2.0 * npos * nneg) == pytest.approx(roc_auc_score(yb, Z[m, j]), rel=1e-13)


def test_binary_logloss_matches_sklearn():
    """The reference's float32 probabilities are scikit-learn's (expit on float32 decision values) to one
    float32 ulp of p1, and the per-row bound covers the difference of the summed losses."""
    rng = np.random.default_rng(6)
    n = 20000
    z32 = (rng.standard_normal(n) * 6).astype(np.float32)
    z32[:50] = np.float32(40.0)                               # saturated rows: p clipped to 1 - eps
    z32[50:100] = np.float32(-40.0)
    y = rng.random(n) < expit(z32)
    p1 = sr.binary_proba32(z32)
    p1_sk = expit(z32)                                         # scikit-learn's _predict_proba_lr on float32
    assert p1_sk.dtype == np.float32
    assert np.all(np.abs(p1 - p1_sk) <= np.spacing(p1_sk))
    ours = sr.binary_logloss(z32, y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sk = log_loss(y, np.column_stack([1 - p1_sk, p1_sk]), normalize=False)
    bound = sr.binary_logloss_bound(z32, y, np.zeros(n)).sum() + 1e-6 * ours.sum()   # + log in float32
    assert abs(ours.sum() - sk) <= bound
    # the bound in dz is first order: a decision error of dz moves the loss by at most (1 - p_true) dz
    dz = np.full(n, 1e-3)
    moved = sr.binary_logloss(z32 + np.where(y, -1e-3, 1e-3).astype(np.float32), y)
    assert np.all(np.abs(moved - ours) <= sr.binary_logloss_bound(z32, y, 1.5 * dz))


def test_decision_bound_discriminates():
    """The float-tier bound holds for a numpy restatement of both kernels' summation orders, and a reference that
    drops one feature's term of median magnitude violates it in every column (d <= 1000)."""
    rng = np.random.default_rng(7)
    for d in (17, 300, 1000):
        n, B = 300, 5
        X = rng.standard_normal((n, d)).astype(np.float32)
        coef = (rng.standard_normal((B, d + 1)) / np.sqrt(d)).astype(np.float32)
        Z = sr.decision(X, coef)
        A = sr.decision_abs(X, coef)
        # fwd_kernel: sequential fp32 FMA chain (emulated exactly in float64: one product + one add rounded once)
        acc = np.zeros((n, B), np.float32)
        for k in range(d):
            acc = (acc.astype(np.float64) + X[:, k:k + 1].astype(np.float64) * coef[None, :, k]).astype(np.float32)
        z_fwd = (acc + coef[:, d]).astype(np.float64)
        assert np.all(np.abs(z_fwd - Z) <= sr.gamma(sr.depth_fwd(d)) * A)
        # predict_kernel: 32 lane chains over float4 quads, a shuffle tree, + b
        ldx = sr.round_up(d, 4)
        Xp = np.zeros((n, ldx), np.float32); Xp[:, :d] = X
        Wp = np.zeros((B, ldx), np.float32); Wp[:, :d] = coef[:, :d]
        lanes = np.zeros((32, n, B), np.float32)
        for q in range(ldx // 4):
            for c in (3, 2, 1, 0):
                k = 4 * q + c
                lanes[q % 32] = (lanes[q % 32].astype(np.float64) + Xp[:, k:k + 1].astype(np.float64) * Wp[None, :, k]).astype(np.float32)
        for o in (16, 8, 4, 2, 1):
            lanes = (lanes + lanes[np.arange(32) ^ o]).astype(np.float32)
        z_pred = (lanes[0] + coef[:, d]).astype(np.float64)
        assert np.all(np.abs(z_pred - Z) <= sr.gamma(sr.depth_predict(ldx)) * A)
        bound = sr.gamma(sr.depth_fwd(d)) * A
        for j in range(B):
            terms = np.abs(X.astype(np.float64) * coef[j, :d].astype(np.float64))
            k = np.argsort(terms.mean(0))[d // 2]
            wrong = Z[:, j] - X[:, k].astype(np.float64) * coef[j, k]
            assert np.any(np.abs(wrong - z_fwd[:, j]) > bound[:, j]), (d, j)


def _forest_case(cls, C, n_trees, seed, **kw):
    rng = np.random.default_rng(seed)
    X = np.round(rng.standard_normal((600, 6)) * 4).astype(np.float32) / 4      # ties, representable midpoints
    if C == 1:
        y = X[:, 0] * 2 + rng.standard_normal(600)
    else:
        y = rng.integers(0, C, 600)
    model = cls(n_estimators=n_trees, random_state=seed, n_jobs=1, **kw).fit(X, y)
    return model, X


@pytest.mark.parametrize("cls,C,n_trees", [
    (RandomForestClassifier, 2, 3), (ExtraTreesClassifier, 9, 5), (RandomForestClassifier, 33, 2),
    (RandomForestRegressor, 1, 4), (ExtraTreesRegressor, 1, 3)])
def test_forest_walk_matches_sklearn(cls, C, n_trees):
    model, X = _forest_case(cls, C, n_trees, 10 + C)
    arrays = _forest_arrays(model.estimators_)
    thr = arrays[4][arrays[1] != -1]
    feat = arrays[3][arrays[1] != -1]
    rng = np.random.default_rng(0)
    Xt = X[rng.integers(0, len(X), 3 * len(thr))].copy()
    t32 = thr.astype(np.float32)
    vals = np.concatenate([t32, np.nextafter(t32, np.float32(np.inf)), np.nextafter(t32, np.float32(-np.inf))])
    Xt[np.arange(len(vals)), np.tile(feat, 3)] = vals
    got = sr.forest_walk(Xt, *arrays)
    if C == 1:
        assert np.array_equal(got[:, 0], model.predict(Xt))
    else:
        assert np.array_equal(got, model.predict_proba(Xt))
        assert np.array_equal(model.classes_.take(np.argmax(got, 1)), model.predict(Xt))
