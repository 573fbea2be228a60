"""csrc/ridge.cu against float64, column by column (run with -m gpu on an H100).

Reference: float64 statistics of the same float32 X and y (tests/ridge_reference.py: per-fold block sums, the
training statistics of each held-out fold, centred by the training mean), w64 = (A_h + alpha I)^-1 b_h.

Per column:
  a. normwise backward error  eta = |(A_h + alpha I) w - b_h|_inf / (|A_h + alpha I|_inf |w|_inf + |b_h|_inf)
     <= 1e-6.  It does not depend on the condition number; correct fp32 arithmetic reaches a few 1e-8 (see
     tests/test_ridge_accumulation_host.py), a lost or misplaced Gram tile or an uncentred target does not
     (test_the_bound_bites).
  b. forward error  |w - w64|_inf <= E_w = 3 |w_sk - w64|_inf + 2e-5 |w64|_inf, w_sk = scikit-learn's own
     float32 solve of the column (oracle/ridge_oracle.fit_ridge), on a few alphas per shape.
  c. intercept  b = fl32(ybar) - fl32 dot(fl32(xbar), w)  against  b64 = ybar - xbar . w64:
        |b - b64| <= |xbar|_1 E_w                          (xbar . (w - w64), from b.)
                   + (d + 2) 2^-24 sum_i |xbar_i w_i|       (xbar rounded to fp32, d-term fp32 dot product)
                   + 2^-23 (|ybar| + |b64| + std(y_train))  (ybar and the target shift in fp32, last subtraction)
  d. status == 1 for every alpha > 0.

Features are made to couple the 64-wide tiles of the Gram matrix (columns j, j + 64, j + 128, ... share one
strong component), so that a lost, transposed or misplaced off-diagonal tile moves the solution.
"""
import numpy as np
import pytest

from oracle import ridge_oracle as ro
from skdist_b200.datasets import make_g1_regression
from tests.ridge_reference import ETA_BOUND, RidgeRef, cholesky_solve32, emulate_statistics, eta

pytestmark = pytest.mark.gpu
U = 2.0 ** -24


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine, set_engine_factory
    e = Engine(0)
    set_engine_factory(lambda: e)
    yield e
    set_engine_factory(None)
    e.close()


def coupled(n, d, seed, y_offset=0.0):
    """G1 features under a component shared by every 64th column; y = X w + N(0, 1) (+ y_offset * std y)."""
    G, _ = make_g1_regression(n, d, seed=seed)
    rng = np.random.default_rng(seed + 1000)
    Z = rng.standard_normal((n, 64), dtype=np.float32)
    X = np.ascontiguousarray(Z[:, np.arange(d) % 64] + np.float32(0.3) * G, dtype=np.float32)
    w = rng.standard_normal(d) / np.sqrt(d)
    y = X.astype(np.float64) @ w + rng.standard_normal(n)
    return X, (y + y_offset * y.std()).astype(np.float32)


def log_alphas(k, seed, lo=1e-6, hi=1e6):
    return np.exp(np.random.default_rng(seed).uniform(np.log(lo), np.log(hi), k))


def check(eng, X, y, fold, n_folds, alphas, holds, fit_intercept=True, fwd=3, label="", ref=None):
    """Stage, fit the columns (alphas[j], holds[j]) and assert a.-d.; returns (result, max eta / bound,
    max forward error / E_w)."""
    d = X.shape[1]
    alphas = np.asarray(alphas, np.float64)
    holds = np.asarray(holds, np.int32)
    eng.stage_x(X)
    eng.stage_targets(y)
    eng.stage_folds(fold, n_folds)
    res = eng.ridge_fit_batch(alphas, holds, fit_intercept=fit_intercept)
    ref = ref or RidgeRef(X, y, fold, n_folds, fit_intercept)
    W, icpt = res["coef"][:, :d].astype(np.float64), res["coef"][:, d].astype(np.float64)
    assert np.all(res["status"][alphas > 0] == 1), (label, res["status"])
    assert np.all(np.isfinite(res["coef"]))
    worst = 0.0
    for h in np.unique(holds):
        m = holds == h
        A, b, _, _ = ref.stats(max(int(h), -1))
        e = eta(A, b, alphas[m], W[m])
        worst = max(worst, e.max() / ETA_BOUND)
        assert np.all(e <= ETA_BOUND), (label, int(h), e.max(), alphas[m][e.argmax()])
    fwd_ratio = 0.0
    picks = np.unique(np.linspace(0, len(alphas) - 1, fwd).round().astype(int)) if fwd else []
    for j in picks:
        h, a = int(holds[j]), float(alphas[j])
        w64, b64 = ref.solve(h, [a])
        w64, b64 = w64[0], b64[0]
        tr = np.ones(len(y), bool) if (fold is None or h < 0) else np.asarray(fold) != h
        w_sk, _ = ro.fit_ridge(X[tr], y[tr], a, fit_intercept)
        Ew = 3 * np.abs(w_sk - w64).max() + 2e-5 * np.abs(w64).max()
        err = np.abs(W[j] - w64).max()
        fwd_ratio = max(fwd_ratio, err / Ew)
        assert err <= Ew, (label, j, a, err, Ew)
        if fit_intercept:
            _, _, xbar, ybar = ref.stats(h)
            bound = (np.abs(xbar).sum() * Ew + (d + 2) * U * np.abs(xbar * W[j]).sum()
                     + 2 * U * (abs(ybar) + abs(b64) + y[tr].astype(np.float64).std()))
            assert abs(icpt[j] - b64) <= bound, (label, j, icpt[j], b64, bound)
        else:
            assert icpt[j] == 0.0
    print("ridge %-32s d=%3d columns=%5d  max eta/bound %.3g  max fwd err/E_w %.3g"
          % (label, d, len(alphas), worst, fwd_ratio))
    return res, worst, fwd_ratio


def grid_columns(alphas, holds):
    """Every (alpha, hold) pair, the holds of consecutive columns interleaved (held-out codes mixed with -1)."""
    A, H = np.meshgrid(alphas, holds, indexing="ij")
    return A.ravel(), H.ravel().astype(np.int32)


# every tile count 1..6; 155 / 156: the last / first d past 48 KB of dynamic shared memory; 338: the largest d
DIMS = [1, 2, 15, 16, 17, 63, 64, 65, 80, 127, 128, 129, 155, 156, 192, 193, 256, 257, 320, 338]


@pytest.mark.parametrize("d", DIMS)
def test_every_tile_count(eng, d):
    """Uneven folds of 2049, 1500, 1 and 2050 rows (chunk boundaries inside folds, a one-row fold), randomly
    interleaved rows, alpha log-uniform in [1e-6, 1e6], every fold held out and none."""
    sizes = [2049, 1500, 1, 2050]
    X, y = coupled(sum(sizes), d, seed=100 + d)
    fold = np.random.default_rng(d).permutation(np.repeat(np.arange(4), sizes)).astype(np.int8)
    alphas, holds = grid_columns(log_alphas(6, d), [0, -1, 1, 2, 3])
    check(eng, X, y, fold, 4, alphas, holds, label="tiles", fwd=4)


def test_the_bound_bites(eng):
    """d = 130 (three tiles): the device passes; on the host, the float64 solve with one off-diagonal 64 x 64
    block of A_h zeroed and the emulated kernel without the target shift both fail the same bound."""
    X, y = coupled(6000, 130, seed=7, y_offset=1e4)
    fold = np.repeat(np.arange(3), 2000).astype(np.int8)
    alphas = np.array([1e-3, 1e-1, 10.0, 1e3])
    ref = RidgeRef(X, y, fold, 3)
    check(eng, X, y, fold, 3, *grid_columns(alphas, [0, -1]), label="bound bites, y + 1e4 std", ref=ref)
    A, b, _, _ = ref.stats(0)
    Abad = A.copy()
    Abad[:64, 64:128] = 0.0
    Abad[64:128, :64] = 0.0
    for a in alphas:
        w = np.linalg.solve(Abad + a * np.eye(130), b)
        assert eta(A, b, [a], w)[0] > ETA_BOUND, ("zeroed tile", a)
    A32, b32, _, _ = emulate_statistics(X, y, fold, 3, 0, shift_y=False)
    for a in alphas[:2]:
        w, _ = cholesky_solve32(A32, b32, a)
        assert eta(A, b, [a], w)[0] > ETA_BOUND, ("uncentred y", a)


def test_fold_sizes_across_chunk_boundaries(eng):
    """Folds of 1, 2047, 2048, 2049 and 4097 rows: one row, one short of a chunk, exactly one, one over, two
    chunks and a row."""
    sizes = [1, 2047, 2048, 2049, 4097]
    X, y = coupled(sum(sizes), 130, seed=11)
    fold = np.random.default_rng(3).permutation(np.repeat(np.arange(5), sizes)).astype(np.int8)
    check(eng, X, y, fold, 5, *grid_columns(log_alphas(4, 3), [-1, 0, 1, 2, 3, 4]), label="fold sizes", fwd=6)


@pytest.mark.parametrize("n_folds", [40, 127])
def test_many_uneven_folds(eng, n_folds):
    """127 is the most folds skd_stage_folds accepts; rows are dealt at random, so fold sizes differ."""
    X, y = coupled(9000, 70, seed=n_folds)
    fold = np.random.default_rng(n_folds).integers(0, n_folds, len(y)).astype(np.int8)
    holds = np.concatenate([np.arange(n_folds), np.arange(n_folds), [-1, -1]]).astype(np.int32)
    alphas = log_alphas(len(holds), n_folds, 1e-3, 1e3)
    check(eng, X, y, fold, n_folds, alphas, holds, label="%d folds" % n_folds, fwd=3)


def test_empty_fold_and_no_folds(eng):
    """A staged fold id without rows: holding it out is the all-rows fit, bit for bit.  Then the same rows with no
    folds staged (other chunks, so other roundings: held to a.-d. like any column)."""
    X, y = coupled(7000, 100, seed=5)
    fold = np.random.default_rng(5).integers(0, 3, len(y)).astype(np.int8)   # fold 3 of 4 is empty
    alphas = np.array([1e-2, 1.0, 100.0] * 2)
    holds = np.array([3, 3, 3, -1, -1, -1], np.int32)
    res, _, _ = check(eng, X, y, fold, 4, alphas, holds, label="empty fold")
    assert np.array_equal(res["coef"][:3], res["coef"][3:])
    check(eng, X, y, None, 0, alphas[:3], [-1, -1, -1], label="no folds staged")


def test_fewer_training_rows_than_features(eng):
    """n_train < d: A_h is singular, alpha > 0 makes the system positive definite."""
    X, y = coupled(150, 200, seed=9)
    fold = np.arange(150).astype(np.int8) % 3
    check(eng, X, y, fold, 3, *grid_columns(log_alphas(5, 9, 1e-3, 1e3), [0, 1, 2, -1]), label="n < d", fwd=4)


@pytest.mark.parametrize("c", [0.0, 1e2, 1e4, 1e6])
def test_target_offsets(eng, c):
    """y + c * std(y): the statistics must carry the spread of y, not its offset."""
    X, y = coupled(12000, 130, seed=13, y_offset=c)
    fold = np.repeat(np.arange(5), 2400).astype(np.int8)
    check(eng, X, y, fold, 5, *grid_columns(log_alphas(5, 13), [0, -1, 2, 4]), label="y + %g std" % c, fwd=4)


def test_feature_offsets_and_no_intercept(eng):
    """Features + 1e3 with an intercept; fit_intercept=False on centred data."""
    X, y = coupled(8000, 90, seed=17)
    fold = np.repeat(np.arange(4), 2000).astype(np.int8)
    cols = grid_columns(log_alphas(5, 17), [1, -1, 3])
    check(eng, (X + np.float32(1e3)).astype(np.float32), y, fold, 4, *cols, label="x + 1e3", fwd=4)
    Xc = (X - X.mean(0)).astype(np.float32)
    yc = (y - y.mean()).astype(np.float32)
    check(eng, Xc, yc, fold, 4, *cols, fit_intercept=False, label="no intercept, centred", fwd=4)


def test_config5_shape_every_column_and_bits(eng):
    """200 000 x 256 (config 5 at 1/5 of its rows), 5 folds, 2048 log-uniform alphas = 10 240 columns: eta on
    every column; a column's bits do not depend on the batch around it, its place in it, or the call."""
    X, y = make_g1_regression(200000, 256, seed=0)
    fold = np.repeat(np.arange(5), 40000).astype(np.int8)
    alphas, holds = grid_columns(log_alphas(2048, 5, 1e-3, 1e3), np.arange(5))
    res, _, _ = check(eng, X, y, fold, 5, alphas, holds, label="config 5 shape", fwd=3)
    again = eng.ridge_fit_batch(alphas, holds)
    assert np.array_equal(again["coef"], res["coef"])
    rev = eng.ridge_fit_batch(alphas[::-1].copy(), holds[::-1].copy())
    assert np.array_equal(rev["coef"][::-1], res["coef"])
    for j in (0, 4097, len(alphas) - 1):
        alone = eng.ridge_fit_batch(alphas[j:j + 1], holds[j:j + 1])
        assert np.array_equal(alone["coef"][0], res["coef"][j]), j


def test_pivot_breakdown(eng):
    """alpha = 0 with an exactly constant integer column and an intercept: the centred column is zero, the
    pivot is 0 and the column reports status 4.  The alpha > 0 columns of the batch are unaffected, bit for
    bit.  (No parity claim: scikit-learn's float32 centring leaves 1e-8 residues there.)"""
    X, y = coupled(5000, 40, seed=19)
    X[:, 7] = 3.0
    fold = np.repeat(np.arange(2), 2500).astype(np.int8)
    eng.stage_x(X); eng.stage_targets(y); eng.stage_folds(fold, 2)
    alphas = np.array([0.0, 0.5, 0.0, 20.0])
    holds = np.array([0, 0, -1, 1], np.int32)
    res = eng.ridge_fit_batch(alphas, holds)
    assert list(res["status"]) == [4, 1, 4, 1]
    for j in (1, 3):
        alone = eng.ridge_fit_batch(alphas[j:j + 1], holds[j:j + 1])
        assert alone["status"][0] == 1
        assert np.array_equal(alone["coef"][0], res["coef"][j])


def test_too_many_features_fails_cleanly(eng):
    """d = 339 is past the shared-memory bound: an error that states the bound, and the context stays usable."""
    X, y = coupled(500, 339, seed=23)
    eng.stage_x(X); eng.stage_targets(y); eng.stage_folds(None, 0)
    with pytest.raises(Exception, match="d <= 338"):
        eng.ridge_fit_batch(np.array([1.0]), np.array([-1], np.int32))
    X, y = coupled(3000, 20, seed=24)
    check(eng, X, y, None, 0, [0.1, 10.0], [-1, -1], label="after d = 339", fwd=2)


@pytest.mark.parametrize("kernel", [1, 2], ids=["simt", "tc"])
@pytest.mark.parametrize("c", [0.0, 1e4])
def test_grid_search_matches_scikit_learn(eng, kernel, c):
    """DistGridSearchCV(Ridge) against GridSearchCV(Ridge) on tile-coupled d = 200, y + c * std(y), with the
    r2 scores from the fp32 CUDA-core (1) and the tensor-core (2) epilogue."""
    from sklearn.linear_model import Ridge
    from sklearn.model_selection import GridSearchCV
    from skdist.distribute.search import DistGridSearchCV
    X, y = coupled(20000, 200, seed=29, y_offset=c)
    grid = {"alpha": [1e-2, 1.0, 30.0, 300.0, 3e3, 3e4]}
    prev = eng.set_kernel(kernel)
    try:
        ours = DistGridSearchCV(Ridge(), grid, None, cv=5).fit(X, y)
    finally:
        eng.set_kernel(prev)
    ref = GridSearchCV(Ridge(), grid, cv=5).fit(X, y)
    # float64 scores of the float64 fits (KFold(5): contiguous folds of 4000 rows).  Far from zero, y loses its
    # last digits to the fp32 predictions of both sides: the tolerance is 1e-5 plus scikit-learn's own distance
    # from these scores (below 1e-6 at c = 0)
    fold = np.repeat(np.arange(5), 4000)
    rr = RidgeRef(X, y, fold, 5)
    X64, y64 = X.astype(np.float64), y.astype(np.float64)
    s64 = np.zeros((len(grid["alpha"]), 5))
    for k in range(5):
        W, b = rr.solve(k, grid["alpha"])
        t = y64[fold == k]
        s64[:, k] = 1 - ((X64[fold == k] @ W.T + b - t[:, None]) ** 2).sum(0) / ((t - t.mean()) ** 2).sum()
    s64 = s64.mean(1)
    sk = ref.cv_results_["mean_test_score"]
    rtol = 1e-5 + np.max(np.abs(sk - s64) / np.abs(s64))
    print("ridge grid search y + %g std, kernel %d: max rel distance from float64 scores: ours %.3g, scikit-learn %.3g"
          % (c, kernel, np.max(np.abs(ours.cv_results_["mean_test_score"] - s64) / np.abs(s64)), rtol - 1e-5))
    np.testing.assert_allclose(ours.cv_results_["mean_test_score"], sk, rtol=rtol)
    assert ours.best_params_ == ref.best_params_
    w64, _ = RidgeRef(X, y, None, 1).solve(-1, [ours.best_params_["alpha"]])
    Ew = 3 * np.abs(ref.best_estimator_.coef_ - w64[0]).max() + 2e-5 * np.abs(w64).max()
    assert np.abs(ours.best_estimator_.coef_ - w64[0]).max() <= Ew
