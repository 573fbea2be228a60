"""The tensor-core logistic kernel (csrc/logreg_tc.cu, tc_eval_kernel) against float64, variant by variant.

The kernel has 16 instantiations: NCHUNK = ceil(d / 64) in 1..4 times the modes TC_FIT (fold decoded per
element), TC_FIT_UNI (per-fold sign arrays), TC_SCORE and TC_R2.  Every test body below runs the same
shape matrix, which reaches each NCHUNK with

  * d with and without column padding (1, 17, 63, 64, 65, 100, 128, 129, 160, 192, 193, 255, 256),
  * fewer 64-row tiles than the 132 row chunks (empty chunks), one to two tiles per chunk, and many
    sub-tiles per chunk, with n not a multiple of 32 (padding rows in the last sub-tile),
  * contiguous folds with boundaries inside a tile, shuffled stratified folds and 40 folds (more than
    the 32 folds for which per-fold tile lists and sign arrays exist),
  * 1, 64, 65, 128 and 129 columns per fold (groups of 128 slots that do not divide the 132 SMs).

Three tiers:

(a) exact: integer data on power-of-two grids, so every product the kernel forms and every sum is exact;
    accuracy counts and squared-error sums must equal the float64 reference, and the gradient at W = 0
    must match it to the error of the approximate exp / reciprocal alone.
(b) float: loss and gradient at random points against a float64 reference, per component, within a bound
    derived from the kernel's arithmetic (constants below), and the bound is shown to fail for a reference
    that is wrong by one training row.
(c) end to end: fits on the production path stop where the float64 gradient of each column's own
    objective is below the tolerance, and the public search matches scikit-learn.
"""
import warnings

import numpy as np
import pytest
from scipy.special import expit
from sklearn.model_selection import StratifiedKFold

pytestmark = pytest.mark.gpu

# error model of the tensor-core evaluation (tier b), fixed once for every variant:
EPS_ACC = 2.0 ** -15    # fp32 accumulation of the tensor cores (round toward zero), relative to sum |x r|
EPS_Z = 2.0 ** -20      # z = x.w from fp16 hi/lo splits, relative to sum |x w| + |b|
EPS_SIG = 2.0 ** -20    # sigma from ex2.approx / rcp.approx, absolute
EPS_ACC_SIMT = 2.0 ** -20
EPS_F = 2.0 ** -18      # the loss, relative

MODES = ("fit", "uni", "score", "r2")
RAN = set()             # (NCHUNK, mode) pairs run by the tests of this module

N_SIZES = {"S": 2000, "M": 12345, "L": 70001}   # 32 tiles < 132 chunks; 1-2 tiles per chunk; ~8 tiles per chunk
N_FLOAT_MAX = 4999                               # tier (b): n <= 5000 keeps the float64 bound tight enough to bite

# (d, n size, folds, columns per fold): every NCHUNK meets every n size and every fold layout
SHAPES = [
    (1, "S", "kfold", 1),
    (17, "M", "strat", 64),
    (63, "L", "f40", 1),
    (64, "S", "strat", 129),
    (65, "M", "kfold", 65),
    (100, "L", "strat", 128),
    (128, "S", "f40", 64),
    (129, "M", "kfold", 129),
    (160, "L", "f40", 1),
    (192, "S", "strat", 65),
    (193, "M", "f40", 1),
    (255, "L", "kfold", 64),
    (256, "S", "strat", 128),
]
SHAPE_IDS = ["d%d-%s-%s-c%d" % s for s in SHAPES]
# W = 0 gradients are cheap to reference: there the matrix gains a case of 160 groups (> 132 SMs)
SHAPES_W0 = SHAPES + [(33, "S", "f40", 385)]
SHAPE_W0_IDS = SHAPE_IDS + ["d33-S-f40-c385"]


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    e.set_kernel(2)
    yield e
    e.close()


def _nchunk(d):
    return (d + 63) // 64


def _fit_mode(n_folds, uniform):
    """The kernel variant a loss/gradient evaluation runs: the per-fold sign arrays need one list per fold."""
    return "uni" if uniform and n_folds <= 32 else "fit"


def _folds(kind, n, y, seed):
    if kind == "kfold":     # contiguous, boundaries inside a tile (n / 5 is not a multiple of 64)
        return (np.arange(n) * 5 // n).astype(np.int8), 5
    if kind == "strat":     # interleaved: every tile holds rows of every fold
        fold = np.zeros(n, np.int8)
        for k, (_, te) in enumerate(StratifiedKFold(5, shuffle=True, random_state=seed).split(np.zeros(n), y)):
            fold[te] = k
        return fold, 5
    return np.random.default_rng(seed).permutation(np.arange(n) % 40).astype(np.int8), 40


def _columns(n_folds, cpf):
    """Held-out fold of every column: cpf columns per fold, interleaved (the fits sort them by fold)."""
    return np.tile(np.arange(n_folds, dtype=np.int32), cpf)


def _train_mask(fold, cf):
    """[n, B] training rows of every column (col_fold < 0: every row)."""
    return (fold[:, None] != cf[None, :]) | (cf[None, :] < 0)


def _int_data(rng, n, d):
    """Integer entries in [-7, 7], column k times 2^e_k, e_k in [-20, 20]; every column non-zero."""
    e = rng.integers(-20, 21, d)
    Xi = rng.integers(-7, 8, (n, d))
    Xi[0] = 7
    return (Xi * np.exp2(e)).astype(np.float32), e


# ---- (a) exact tier -------------------------------------------------------------------------------------
def _exact_setup(eng, shape, seed):
    d, nk, fk, cpf = shape
    n = N_SIZES[nk]
    rng = np.random.default_rng(seed)
    X, e = _int_data(rng, n, d)
    ycls = rng.integers(0, 3, n).astype(np.int32)
    fold, nf = _folds(fk, n, ycls, seed)
    eng.stage_x(X)
    eng.stage_labels(ycls)
    eng.stage_folds(fold, nf)
    return rng, X, e, ycls, fold, nf


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_exact_score_and_r2(eng, shape):
    d, _, _, cpf = shape
    rng, X, e, ycls, fold, nf = _exact_setup(eng, shape, 100 + d)
    n = X.shape[0]
    ftrain = _columns(nf, cpf)
    B = ftrain.shape[0]
    # every scoring code: the rows of fold f, every row (-2), the rows outside fold f (-3 - f)
    code = np.select([np.arange(B) % 3 == 0, np.arange(B) % 3 == 1], [ftrain, -2], -3 - ftrain).astype(np.int32)
    pos = (np.arange(B) % 3).astype(np.int32)
    coef = np.zeros((B, d + 1), np.float32)
    coef[:, :d] = rng.integers(-2, 3, (B, d)) * np.exp2(-e)
    coef[:, d] = rng.integers(-100, 101, B)
    yreal = rng.integers(-100, 101, n).astype(np.float32)
    eng.stage_targets(yreal)

    Z = X.astype(np.float64) @ coef[:, :d].T.astype(np.float64) + coef[:, d].astype(np.float64)   # exact
    M = np.where(code[None, :] == -2, True,
                 np.where(code[None, :] >= 0, fold[:, None] == code[None, :], fold[:, None] != (-3 - code)[None, :]))
    want_count = M.sum(0)
    want_correct = (M & ((Z > 0) == (ycls[:, None] == pos[None, :]))).sum(0)
    R = yreal.astype(np.float64)[:, None] - Z
    want_sse = (M * R * R).sum(0)

    correct, count = eng.linear_score_batch(coef, code, pos)
    RAN.add((_nchunk(d), "score"))
    assert np.array_equal(count, want_count)
    bad = np.flatnonzero(correct != want_correct)
    assert bad.size == 0, ("accuracy counts differ", bad[:10], correct[bad[:10]], want_correct[bad[:10]])
    sse, count = eng.linear_r2_batch(coef, code)
    RAN.add((_nchunk(d), "r2"))
    assert np.array_equal(count, want_count)
    bad = np.flatnonzero(sse != want_sse)
    assert bad.size == 0, ("squared-error sums differ", bad[:10], sse[bad[:10]], want_sse[bad[:10]])


@pytest.mark.parametrize("uniform", [True, False], ids=["uniform_pos", "mixed_pos"])
@pytest.mark.parametrize("shape", SHAPES_W0, ids=SHAPE_W0_IDS)
def test_exact_gradient_at_zero(eng, shape, uniform):
    """At W = 0, z = 0 and sigma = 1/2 on every row: the gradient is sum_train (1/2 - y_i) x_i / n_train, which
    the kernel forms exactly up to the approximate exp / reciprocal.  A row counted in the wrong fold, a
    skipped tile or a slot written to the wrong column moves a component by |x_ik| / (2 n_train), far above
    the bound."""
    d, _, _, cpf = shape
    rng, X, e, ycls, fold, nf = _exact_setup(eng, shape, 200 + d)
    cf = _columns(nf, cpf)
    B = cf.shape[0]
    pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 3).astype(np.int32)
    C = np.full(B, 1.0)
    f, g = eng.logreg_loss_grad(np.zeros((B, d + 1)), C, cf, pos)
    RAN.add((_nchunk(d), _fit_mode(nf, uniform)))

    X64 = np.abs(X.astype(np.float64))
    Xs = X.astype(np.float64)
    # per (fold, class): sums over the rows of that fold and class, then per column the training rows
    S = np.zeros((nf, 3, d)); A = np.zeros((nf, 3, d)); N = np.zeros((nf, 3))
    for k in range(nf):
        for c in range(3):
            m = (fold == k) & (ycls == c)
            S[k, c] = Xs[m].sum(0); A[k, c] = X64[m].sum(0); N[k, c] = m.sum()
    Sc, Ac, Nc = S.sum(0), A.sum(0), N.sum(0)            # per class over every fold
    St, At, Nt = Sc - S, Ac - A, Nc - N                 # per (held-out fold, class): the training rows
    for j in range(B):
        k, p = cf[j], pos[j]
        ntr = Nt[k].sum()
        # (1/2 - y) x summed over training rows: 1/2 sum x - sum over the positive class
        want = (0.5 * St[k].sum(0) - St[k, p]) / ntr
        bound = 2.0 ** -20 * At[k].sum(0) / ntr
        err = np.abs(g[j, :d] - want)
        assert np.all(err <= bound), (j, k, p, np.argmax(err / np.maximum(bound, 1e-300)), (err / bound).max())
        want_b = (0.5 * ntr - Nt[k, p]) / ntr
        assert abs(g[j, d] - want_b) <= 2.0 ** -20, (j, g[j, d], want_b)
    assert np.all(np.isfinite(f))


# ---- (b) float tier -------------------------------------------------------------------------------------
def _float_data(rng, n, d):
    scale = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), d))
    X = (rng.standard_normal((n, d)) * scale).astype(np.float32)
    return X, scale


def _float_points(rng, B, d, scale):
    """Random points with, in the first three columns, W = 0, a one-hot weight vector and a saturated
    column (|z| up to ~40)."""
    W = np.empty((B, d + 1))
    W[:, :d] = rng.standard_normal((B, d)) / (scale * np.sqrt(d))
    W[:, d] = rng.standard_normal(B)
    W[0] = 0.0
    if B > 1:
        W[1] = 0.0
        k = rng.integers(0, d)
        W[1, k] = 3.0 / scale[k]
        W[1, d] = 0.5
    if B > 2:
        W[2, :d] *= 13.0
        W[2, d] = 2.0
    return W


def _ref_loss_grad(X, yb, M, W, C):
    """float64 objective and gradient of every column on its training rows, with the error bound of the
    kernel's arithmetic.  yb: [n, B] 0/1 labels, M: [n, B] training rows, W: [B, d + 1] float64 points:
    the weights enter the products rounded to fp32 (as scikit-learn casts them) and the penalty as float64."""
    d = X.shape[1]
    X64 = X.astype(np.float64)
    W32 = W.astype(np.float32).astype(np.float64)
    Z = X64 @ W32[:, :d].T + W32[:, d]
    Mf = M.astype(np.float64)
    ntr = Mf.sum(0)
    l2 = 1.0 / (C * ntr)
    R = expit(Z) - yb
    L = np.logaddexp(0.0, Z) - yb * Z
    f = (L * Mf).sum(0) / ntr + 0.5 * l2 * (W[:, :d] ** 2).sum(1)
    g = np.empty_like(W)
    g[:, :d] = (X64.T @ (R * Mf)).T / ntr[:, None] + l2[:, None] * W[:, :d]
    g[:, d] = (R * Mf).sum(0) / ntr
    dz = EPS_Z * (np.abs(X64) @ np.abs(W32[:, :d]).T + np.abs(W32[:, d]))
    pen = np.zeros_like(W)
    pen[:, :d] = l2[:, None] * W[:, :d]
    return dict(f=f, g=g, pen=pen, R=R, Mf=Mf, ntr=ntr, dz=dz, Xa=np.abs(X64))


def _bounds(ref, eps_acc):
    Q = (eps_acc * np.abs(ref["R"]) + 0.25 * ref["dz"] + EPS_SIG) * ref["Mf"]
    bg = np.empty((Q.shape[1], ref["Xa"].shape[1] + 1))
    bg[:, :-1] = (ref["Xa"].T @ Q).T / ref["ntr"][:, None]
    bg[:, -1] = Q.sum(0) / ref["ntr"]
    bf = EPS_F * np.abs(ref["f"]) + (np.abs(ref["R"]) * ref["dz"] * ref["Mf"]).sum(0) / ref["ntr"]
    return bf, bg


def _check_float(X, ref, f, g, eps_acc, label):
    bf, bg = _bounds(ref, eps_acc)
    assert np.all(np.isfinite(f)) and np.all(np.isfinite(g)), label
    def ratio(err, bound):          # error / bound; a zero bound (an all-zero feature) allows no error
        return np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)
    rf = ratio(np.abs(f - ref["f"]), bf)
    rg = ratio(np.abs(g - ref["g"]), bg)
    print("%s: max error / bound  loss %.3f  gradient %.3f" % (label, rf.max(), rg.max()))
    j, k = np.unravel_index(np.argmax(rg), rg.shape)
    assert rg.max() <= 1.0, (label, "gradient", j, k, g[j, k], ref["g"][j, k], bg[j, k])
    assert rf.max() <= 1.0, (label, "loss", np.argmax(rf), rf.max())
    # the bound discriminates: a reference missing one training row (of median |r|) violates it in every column
    for j in range(g.shape[0]):
        rows = np.flatnonzero(ref["Mf"][:, j])
        r = ref["R"][rows, j]
        i = rows[np.argsort(np.abs(r))[len(r) // 2]]
        ntr = ref["ntr"][j]
        data = ref["g"][j] - ref["pen"][j]
        xi = np.append(X[i].astype(np.float64), 1.0)
        moved = (data * ntr - ref["R"][i, j] * xi) / (ntr - 1) + ref["pen"][j]
        assert np.any(np.abs(moved - ref["g"][j]) > bg[j]), (label, "bound cannot see one row", j)


def _float_case(eng, shape, seed, n_max):
    d, nk, fk, cpf = shape
    n = min(N_SIZES[nk], n_max)
    rng = np.random.default_rng(seed)
    X, scale = _float_data(rng, n, d)
    ycls = rng.integers(0, 3, n).astype(np.int32)
    fold, nf = _folds(fk, n, ycls, seed)
    eng.stage_x(X)
    eng.stage_labels(ycls)
    eng.stage_folds(fold, nf)
    cf = _columns(nf, cpf)
    W = _float_points(rng, cf.shape[0], d, scale)
    C = np.exp(rng.uniform(np.log(1e-2), np.log(1e2), cf.shape[0]))
    return X, ycls, fold, nf, cf, W, C


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_float_loss_grad(eng, shape):
    d = shape[0]
    X, ycls, fold, nf, cf, W, C = _float_case(eng, shape, 300 + d, N_FLOAT_MAX)
    B = cf.shape[0]
    M = _train_mask(fold, cf)
    for uniform in (True, False):
        pos = np.ones(B, np.int32) if uniform else (np.arange(B) % 3).astype(np.int32)
        yb = (ycls[:, None] == pos[None, :]).astype(np.float64)
        ref = _ref_loss_grad(X, yb, M, W, C)
        f, g = eng.logreg_loss_grad(W, C, cf, pos)
        mode = _fit_mode(nf, uniform)
        RAN.add((_nchunk(d), mode))
        _check_float(X, ref, f, g, EPS_ACC, "TC <%d, %s> %s" % (_nchunk(d), mode, "-".join(map(str, shape))))


@pytest.mark.parametrize("d", [40, 300])
def test_float_loss_grad_simt(eng, d):
    """The fp32 CUDA-core kernel under the same assertions (d = 300 is beyond the tensor-core path).  At
    d = 40 (6000 rows, 4 stratified folds, nine columns from C = 1e-3 to 1e3, one without a held-out fold)
    the tensor cores run the same case."""
    rng = np.random.default_rng(400 + d)
    n = 4999 if d == 300 else 6000
    X, scale = _float_data(rng, n, d)
    ycls = rng.integers(0, 2, n).astype(np.int32)
    fold = np.zeros(n, np.int8)
    for k, (_, te) in enumerate(StratifiedKFold(4).split(np.zeros(n), ycls)):
        fold[te] = k
    eng.stage_x(X); eng.stage_labels(ycls); eng.stage_folds(fold, 4)
    cf = np.array([-1, 0, 1, 2, 3, 0, 1, 2, 3], np.int32)
    B = cf.shape[0]
    W = _float_points(rng, B, d, scale)
    C = np.logspace(-3, 3, B)
    pos = np.ones(B, np.int32)
    ref = _ref_loss_grad(X, (ycls[:, None] == 1).astype(np.float64) * np.ones((1, B)), _train_mask(fold, cf), W, C)
    prev = eng.set_kernel(1)
    try:
        f, g = eng.logreg_loss_grad(W, C, cf, pos)
    finally:
        eng.set_kernel(prev)
    _check_float(X, ref, f, g, EPS_ACC_SIMT, "SIMT d=%d" % d)
    if d <= 256:        # the same case on the tensor cores
        f, g = eng.logreg_loss_grad(W, C, cf, pos)
        RAN.add((_nchunk(d), "uni"))
        _check_float(X, ref, f, g, EPS_ACC, "TC d=%d" % d)


# ---- (c) end to end -------------------------------------------------------------------------------------
def _e2e_data(seed, n, d):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    V = rng.standard_normal((d, 3)) * (2.0 / np.sqrt(d))
    ycls = np.argmax(X @ V + rng.gumbel(size=(n, 3)), 1).astype(np.int32)
    return rng, X, ycls


def _check_fit(X, yb, M, C, res, tol, max_iter, label):
    """Every converged column stops where the float64 gradient of its own objective is below 2 tol, and
    reports that objective."""
    coef = res["coef"].astype(np.float64)
    ref = _ref_loss_grad(X, yb, M, coef, C)
    ok = (res["n_iter"] < max_iter) & (res["status"] == 1)
    assert ok.sum() >= 0.5 * len(C), (label, res["status"], res["n_iter"])
    gmax = np.abs(ref["g"]).max(1)
    assert np.all(gmax[ok] <= 2 * tol), (label, np.flatnonzero(gmax[ok] > 2 * tol), gmax[ok].max())
    good = (res["n_iter"] < max_iter) & ((res["status"] == 1) | (res["status"] == 2))
    rel = np.abs(res["loss"] - ref["f"]) / ref["f"]
    assert np.all(rel[good] <= 1e-6), (label, rel[good].max())
    print("%s: %d of %d columns converged, max |g| %.2e, max loss rel. error %.2e"
          % (label, ok.sum(), len(C), gmax[ok].max(), rel[good].max()))


@pytest.mark.parametrize("d", [100, 160, 256])
def test_fits_stop_at_float64_optimum(eng, d):
    n, tol, max_iter = 6000, 1e-4, 100
    rng, X, ycls = _e2e_data(500 + d, n, d)
    eng.stage_x(X); eng.stage_labels(ycls)
    for nf in (5, 40):       # one-vs-rest, every column positive class 1 (the per-fold sign arrays below 33 folds)
        fold = np.random.default_rng(nf).permutation(np.arange(n) % nf).astype(np.int8)
        eng.stage_folds(fold, nf)
        cf = np.tile(np.arange(nf, dtype=np.int32), 2)
        C = np.repeat([0.1, 1.0], nf)
        res = eng.logreg_fit_batch(C, cf, np.ones(len(C), np.int32), tol=tol, max_iter=max_iter)
        yb = (ycls[:, None] == 1) * np.ones((1, len(C)))
        _check_fit(X, yb, _train_mask(fold, cf), C, res, tol, max_iter, "d=%d %d folds" % (d, nf))
    fold = (np.arange(n) * 5 // n).astype(np.int8)
    eng.stage_folds(fold, 5)
    # one-vs-rest with a positive class per column
    cf = np.repeat(np.arange(5, dtype=np.int32), 3)
    pos = np.tile(np.arange(3, dtype=np.int32), 5)
    C = np.full(len(cf), 0.5)
    res = eng.logreg_fit_batch(C, cf, pos, tol=tol, max_iter=max_iter)
    yb = (ycls[:, None] == pos[None, :]).astype(np.float64)
    _check_fit(X, yb, _train_mask(fold, cf), C, res, tol, max_iter, "d=%d one-vs-rest" % d)
    # one-vs-one pairs: only the rows of the pair's two classes train
    pairs = np.array([(0, 1), (0, 2), (1, 2)], np.int32)
    cf = np.repeat(np.arange(5, dtype=np.int32), 3)
    pos, neg = np.tile(pairs[:, 0], 5), np.tile(pairs[:, 1], 5)
    res = eng.logreg_fit_batch(C, cf, pos, col_neg=neg, tol=tol, max_iter=max_iter)
    M = _train_mask(fold, cf) & ((ycls[:, None] == pos[None, :]) | (ycls[:, None] == neg[None, :]))
    yb = (ycls[:, None] == pos[None, :]).astype(np.float64)
    _check_fit(X, yb, M, C, res, tol, max_iter, "d=%d one-vs-one" % d)
    # staged row bits: per-column labels and training rows
    eng.stage_folds(None, 0)
    B = 6
    lab = rng.random((B, n)) < expit((X @ rng.standard_normal((d, B)) / np.sqrt(d)).T)
    tr = rng.random((B, n)) < 0.7
    eng.stage_row_bits(labels=lab, train=tr)
    C = np.full(B, 1.0)
    res = eng.logreg_fit_batch(C, np.full(B, -1, np.int32), np.ones(B, np.int32), tol=tol, max_iter=max_iter)
    _check_fit(X, lab.T.astype(np.float64), tr.T, C, res, tol, max_iter, "d=%d row bits" % d)


def _split_scores(search, cv):
    return np.array([search.cv_results_["split%d_test_score" % k] for k in range(cv)])   # [fold, candidate]


def _search(eng, kernel, X, y, Cs, cv):
    from skdist.distribute.search import DistGridSearchCV
    from skdist_b200.engine import set_engine_factory
    from sklearn.linear_model import LogisticRegression
    prev = eng.set_kernel(kernel)
    set_engine_factory(lambda: eng)
    try:
        return DistGridSearchCV(LogisticRegression(), {"C": Cs}, None, cv=cv).fit(X, y)
    finally:
        set_engine_factory(None)
        eng.set_kernel(prev)


def _sk_search(X, y, Cs, cv):
    from sklearn.linear_model import LogisticRegression
    from sklearn.model_selection import GridSearchCV
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return GridSearchCV(LogisticRegression(), {"C": Cs}, cv=cv).fit(X, y)


def _assert_flips(a, b, y, cv, label):
    test_sizes = np.array([len(te) for _, te in StratifiedKFold(cv).split(np.zeros(len(y)), y)])
    flips = np.rint(np.abs(a - b) * test_sizes[:, None])
    assert flips.max() <= 2, (label, flips.max(axis=1))


def test_search_40_folds_matches_sklearn(eng):
    """40 folds: beyond the per-fold sign arrays, so the fits run the per-element fold decode."""
    _, X, ycls = _e2e_data(600, 4000, 100)
    y = (ycls == 1).astype(np.int64)
    Cs, cv = [0.01, 0.1, 1.0], 40
    ours = _search(eng, 2, X, y, Cs, cv)
    RAN.add((_nchunk(100), "fit"))
    ref = _sk_search(X, y, Cs, cv)
    _assert_flips(_split_scores(ours, cv), _split_scores(ref, cv), y, cv, "40 folds")


def test_tiny_feature(eng):
    """A feature with max |x| = 1e-36 (below 2^-114, where the power-of-two scale of 2^13 / max |x| is not a
    finite float) next to an all-zero feature: the search matches scikit-learn and the fp32 CUDA-core
    kernel, and the loss / gradient stay within the float bound."""
    rng, X, ycls = _e2e_data(700, 3000, 50)
    X[:, 3] *= np.float32(1e-36) / np.abs(X[:, 3]).max()
    X[:, 7] = 0.0
    assert np.abs(X[:, 3]).max() < 2.0 ** -114
    y = (ycls == 1).astype(np.int64)
    Cs, cv = [0.1, 1.0], 5
    tc = _split_scores(_search(eng, 2, X, y, Cs, cv), cv)
    simt = _split_scores(_search(eng, 1, X, y, Cs, cv), cv)
    ref = _split_scores(_sk_search(X, y, Cs, cv), cv)
    assert np.all(np.isfinite(tc))
    _assert_flips(tc, ref, y, cv, "tensor cores vs scikit-learn")
    _assert_flips(tc, simt, y, cv, "tensor cores vs SIMT")

    fold = (np.arange(len(y)) * 5 // len(y)).astype(np.int8)
    eng.stage_x(X); eng.stage_labels(y.astype(np.int32)); eng.stage_folds(fold, 5)
    cf = _columns(5, 2)
    B = len(cf)
    W = _float_points(rng, B, 50, np.ones(50))
    W[3:, 3] = 1e3          # weight on the tiny feature
    W[-1] = 0.0             # a point whose only weight is on the tiny feature
    W[-1, 3], W[-1, 50] = 1.0, 0.3
    C = np.full(B, 1.0)
    pos = np.ones(B, np.int32)
    ref = _ref_loss_grad(X, (y[:, None] == 1) * np.ones((1, B)), _train_mask(fold, cf), W, C)
    f, g = eng.logreg_loss_grad(W, C, cf, pos)
    _check_float(X, ref, f, g, EPS_ACC, "TC tiny feature")
    prev = eng.set_kernel(1)
    try:
        fs, gs = eng.logreg_loss_grad(W, C, cf, pos)
    finally:
        eng.set_kernel(prev)
    _check_float(X, ref, fs, gs, EPS_ACC_SIMT, "SIMT tiny feature")


def test_every_variant_ran():
    """Every (NCHUNK, mode) instantiation of the kernel was run by the tests above."""
    want = {(c, m) for c in range(1, 5) for m in MODES}
    assert RAN == want, sorted(want - RAN)
