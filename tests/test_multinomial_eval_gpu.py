"""The multinomial evaluation (csrc/logreg_multi.cu, gather_fg / lb_step_kernel in csrc/lbfgs_dev.cu) against
float64, through skd_logreg_multinomial_loss_grad, which runs the passes, buffers and kernels of one round of the
multinomial fit.

Every test body runs one shape matrix (K, d, n, fold layout, candidates B) that reaches

  * K = 2 .. 128: candidates whose K class slots straddle 64-slot tiles (K = 3, 5, 33, 65), tiles filled
    exactly (K = 64, 128), and K >= 111, where the K x K confusion counts no longer fit 48 KB of shared memory
    and mn_confusion_kernel<0> counts in global memory;
  * d = 1, 15, 16, 17, 64, 65, 100, 255, 300: padded rows of X and a partial last 64-column block of bwd_kernel;
  * the row chunks of multi_chunks: one partial chunk (n < 64), 64 chunks of 64 rows (4096), 33 chunks of 128
    (4097), 40 chunks of 128 (5000) and 61 chunks of 1152 (70001);
  * no folds, contiguous KFold with boundaries inside a tile, shuffled stratified folds and 40 folds;
  * B * K slot totals below, at and above multiples of 64;
  * class weights, column masks and fit_intercept, each on and off.

Tiers:

(a) exact: integer data on power-of-two grids (_int_data).  At W = 0 with K a power of two, p = 1/K and
    g = 1/K - [y = k] are exact in fp32, and so are the products and the fp32 chunk sums: every gradient entry
    equals sum_train (1/K - [y = k]) x / n_train within 2 ulp of float64 and the loss equals float32(ln K).
    Class weights 1/2, 1, 2 keep this exact (n_train becomes the sum of the weights).  With integer W, Z is exact
    for any K, so confusion counts and accuracy counts equal the float64 arg-max for every scoring code, ties
    (duplicated class rows) going to the first maximum.
(b) float (n <= 5000): loss and gradient at random points, W of mixed scale with saturated rows, per component
    within the first-order bound of tests/multinomial_reference.py (U = 2^-24; forward U times the partial sums of
    the FMA chain, at most (d + 2) U (sum |x w| + |b|), softmax and pointwise 2 max|dz| + 4 U relative to p plus
    U |g|, backward (rpc + 1) U sum |g x|); a reference missing one training
    row must violate it in every candidate.  The multiclass log loss at K = 3, 65, 128 against scikit-learn's
    log_loss of the softmax of exact Z.
(c) end to end: fits over C = 1e-3 .. 1e3 stop where the float64 gradient of each candidate's own objective is
    <= 2 tol, report that objective within 1e-6 relative, and refit alone bit for bit.
(d) pass split: n = 200,000, d = 16, K = 128 puts 58 candidates in a 6 GB pass, so B = 60 runs two passes; every
    result must equal the same candidates run in slices of at most 58, bit for bit.
"""
import warnings

import numpy as np
import pytest
from sklearn.metrics import log_loss
from sklearn.model_selection import StratifiedKFold

from tests import multinomial_reference as mr

pytestmark = pytest.mark.gpu

N_FLOAT_MAX = 5000
SMEM_LIMIT = 48 * 1024

# (K, d, n, folds, B)
SHAPES = [
    (2, 1, 50, "none", 32),
    (3, 15, 4096, "kfold", 21),
    (4, 16, 4097, "strat", 17),
    (5, 17, 5000, "f40", 13),
    (8, 64, 70001, "kfold", 8),
    (10, 65, 50, "strat", 7),
    (16, 100, 4096, "none", 4),
    (33, 255, 4097, "kfold", 2),
    (64, 300, 5000, "strat", 1),
    (65, 1, 70001, "f40", 3),
    (111, 16, 5000, "kfold", 2),
    (128, 17, 4097, "none", 1),
    (128, 64, 50, "f40", 2),
    (3, 300, 70001, "strat", 22),
]
SHAPE_IDS = ["K%d-d%d-n%d-%s-B%d" % s for s in SHAPES]
OPTIONS = {s: (i % 2 == 1, i % 4 >= 2, i % 3 != 2) for i, s in enumerate(SHAPES)}   # class weights, masks, intercept

RAN = set()


def k_regime(K):
    if K % 64 == 0:
        return "fills tiles"
    if 64 % K == 0:
        return "divides a tile"
    return "straddles tiles"


def chunk_regime(n):
    nz, rpc = mr.multi_chunks(n)
    return "%d x %d" % (nz, rpc)


def conf_path(K):
    return "shared" if K * K * 4 <= SMEM_LIMIT else "global"


def _record(K, n, passes=1):
    RAN.add((k_regime(K), chunk_regime(n), conf_path(K), passes))


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _folds(kind, n, y, seed):
    if kind == "none":
        return None, 0
    if kind == "kfold":     # contiguous, boundaries inside a tile (n / 5 is not a multiple of 64)
        return (np.arange(n) * 5 // n).astype(np.int8), 5
    if kind == "strat":
        fold = np.zeros(n, np.int8)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")     # classes with fewer members than folds at n = 50
            for k, (_, te) in enumerate(StratifiedKFold(5, shuffle=True, random_state=seed).split(np.zeros(n), y)):
                fold[te] = k
        return fold, 5
    return np.random.default_rng(seed).permutation(np.arange(n) % 40).astype(np.int8), 40


def _columns(nf, B):
    """Held-out fold of every candidate, interleaved; the last one of several holds nothing out."""
    if nf == 0:
        return np.full(B, -1, np.int32)
    cf = (np.arange(B) % nf).astype(np.int32)
    if B > 1:
        cf[-1] = -1
    return cf


def _int_data(rng, n, d):
    """Integer entries in [-7, 7], column k times 2^e_k, e_k in [-20, 20]; every column non-zero."""
    e = rng.integers(-20, 21, d)
    Xi = rng.integers(-7, 8, (n, d))
    Xi[0] = 7
    return (Xi * np.exp2(e)).astype(np.float32), e


def _float_data(rng, n, d):
    scale = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), d))
    return (rng.standard_normal((n, d)) * scale).astype(np.float32), scale


def _stage(eng, X, y, fold, nf):
    eng.stage_x(X)
    eng.stage_labels(y)
    eng.stage_folds(fold, nf)


def _options(eng, rng, shape, y, M, dyadic):
    """Stage the case's class weights and masks (one-shot); returns (cw, fmask)."""
    K, d, _, _, B = shape
    use_cw, use_mask, _ = OPTIONS[shape]
    cw = fmask = None
    if use_cw:
        if dyadic:
            cw = np.exp2(rng.integers(-1, 2, (B, K))).astype(np.float32)
        else:
            cw = rng.uniform(0.2, 3.0, (B, K)).astype(np.float32)
        sw = np.array([(M[:, b] * cw[b, y].astype(np.float64)).sum() for b in range(B)])
        eng.stage_class_weights(cw, sw)
    if use_mask:
        fmask = (rng.random((B, d)) < 0.7).astype(np.uint8)
        fmask[:, 0] = 1
        eng.stage_column_masks(fmask)
    return cw, fmask


# ---- (a) exact tier -------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_exact_gradient_at_zero(eng, shape):
    K, d, n, fk, B = shape
    fi = OPTIONS[shape][2]
    rng = np.random.default_rng(K * 1000 + d)
    X, _ = _int_data(rng, n, d)
    y = rng.integers(0, K, n).astype(np.int32)
    fold, nf = _folds(fk, n, y, K + d)
    _stage(eng, X, y, fold, nf)
    cf = _columns(nf, B)
    M = mr.row_mask(n, fold, cf)
    cw, fmask = _options(eng, rng, shape, y, M, dyadic=True)
    C = np.full(B, 1.0)
    f, g = eng.logreg_multinomial_loss_grad(np.zeros((B, K, d + 1)), C, cf, fit_intercept=fi)
    _record(K, n)
    want, ntr = mr.grad_at_zero(X, y, M, K, cw, fi)
    if fmask is not None:
        want[:, :, :d] *= fmask[:, None, :]
    if K & (K - 1) == 0:
        err = np.abs(g - want)
        tol = 2 * np.spacing(np.abs(want))
        bad = np.argwhere(err > tol)
        assert bad.size == 0, ("gradient at W = 0 not exact", bad[:5], g[tuple(bad[0])], want[tuple(bad[0])])
        lnK = float(np.float32(np.log(K)))
        assert np.all(np.abs(f - lnK) <= 2 * np.spacing(lnK)), (f, lnK)
    else:
        ref = mr.loss_grad(X, y, M, np.zeros((B, K, d + 1)), C, cw, fmask, fi)
        mr.check_float(X, ref, f, g, "W = 0 %s" % "-".join(map(str, shape)), fi)


def _int_points(rng, B, K, d, e, ties=True):
    coef = np.zeros((B, K, d + 1), np.float32)
    coef[:, :, :d] = rng.integers(-2, 3, (B, K, d)) * np.exp2(-e)
    coef[:, :, d] = rng.integers(-3, 4, (B, K))
    if ties and K > 2:
        coef[::2, 1] = coef[::2, 0]          # duplicated class rows: the first maximum wins
        coef[1::2, K - 1] = coef[1::2, K - 2]
    return coef


def _score_codes(cf, nf):
    B = len(cf)
    if nf == 0:
        return np.full(B, -2, np.int32)
    f = np.where(cf >= 0, cf, np.arange(B) % nf).astype(np.int32)
    return np.select([np.arange(B) % 3 == 0, np.arange(B) % 3 == 1], [f, -2], -3 - f).astype(np.int32)


def _selected(fold, code):
    """[n, B] rows each scoring code selects (fold f, every row, or the rows outside fold f)."""
    return np.where(code[None, :] == -2, True,
                    np.where(code[None, :] >= 0, fold[:, None] == code[None, :], fold[:, None] != (-3 - code)[None, :]))


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_exact_confusion_and_accuracy(eng, shape):
    K, d, n, fk, B = shape
    rng = np.random.default_rng(K * 1000 + d + 1)
    X, e = _int_data(rng, n, d)
    y = rng.integers(0, K, n).astype(np.int32)
    fold, nf = _folds(fk, n, y, K + d)
    _stage(eng, X, y, fold, nf)
    code = _score_codes(_columns(nf, B), nf)
    coef = _int_points(rng, B, K, d, e)
    conf = eng.multinomial_confusion_batch(coef, code)
    correct, count = eng.multinomial_score_batch(coef, code)
    _record(K, n)
    X64 = X.astype(np.float64)
    sel = np.ones((n, B), bool) if fold is None else _selected(fold, code)
    for b in range(B):
        Z = X64 @ coef[b, :, :d].T.astype(np.float64) + coef[b, :, d].astype(np.float64)    # exact
        pred = np.argmax(Z, 1)
        m = sel[:, b]
        want = np.bincount(y[m] * K + pred[m], minlength=K * K).reshape(K, K)
        bad = np.argwhere(conf[b] != want)
        assert bad.size == 0, ("confusion counts differ", b, bad[:5])
        assert correct[b] == np.trace(want) and count[b] == m.sum(), (b, correct[b], np.trace(want))


# ---- (b) float tier -------------------------------------------------------------------------------------
def _float_points(rng, B, K, d, scale, fi):
    W = np.empty((B, K, d + 1))
    W[:, :, :d] = rng.standard_normal((B, K, d)) / (scale * np.sqrt(d))
    W[:, :, d] = rng.standard_normal((B, K)) if fi else 0.0
    W[0] = 0.0
    if B > 1:                        # saturated rows: |z| of tens from the last feature alone
        W[1, :, :d] = 0.0
        W[1, :, d - 1] = rng.choice([-12.0, 12.0], K) * rng.uniform(0.5, 1.0, K) / scale[d - 1]
    if B > 2:
        W[2, :, :d] *= 1e-3
    if B > 3:
        W[3, :, :d] *= 4.0
    return W


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_float_loss_grad(eng, shape):
    K, d, n, fk, B = shape
    n = min(n, N_FLOAT_MAX)
    fi = OPTIONS[shape][2]
    rng = np.random.default_rng(K * 1000 + d + 2)
    X, scale = _float_data(rng, n, d)
    y = rng.integers(0, K, n).astype(np.int32)
    fold, nf = _folds(fk, n, y, K + d)
    _stage(eng, X, y, fold, nf)
    cf = _columns(nf, B)
    M = mr.row_mask(n, fold, cf)
    cw, fmask = _options(eng, rng, shape, y, M, dyadic=False)
    W = _float_points(rng, B, K, d, scale, fi)
    C = np.exp(rng.uniform(np.log(1e-2), np.log(1e2), B))
    f, g = eng.logreg_multinomial_loss_grad(W, C, cf, fit_intercept=fi)
    _record(K, n)
    ref = mr.loss_grad(X, y, M, W, C, cw, fmask, fi)
    mr.check_float(X, ref, f, g, "K=%d d=%d n=%d %s B=%d cw=%d mask=%d fi=%d"
                   % (K, d, n, fk, B, cw is not None, fmask is not None, fi), fi)


@pytest.mark.parametrize("K", [3, 65, 128])
def test_logloss_matches_sklearn(eng, K):
    n, d = 4097, 17
    rng = np.random.default_rng(900 + K)
    X, e = _int_data(rng, n, d)
    y = rng.integers(0, K, n).astype(np.int32)
    fold, nf = _folds("strat", n, y, K)
    _stage(eng, X, y, fold, nf)
    B = 3
    code = _score_codes(np.arange(B, dtype=np.int32), nf)
    coef = _int_points(rng, B, K, d, e, ties=False)
    coef[1] *= 64            # saturated rows: probabilities below float32 epsilon are clipped
    mean, count = eng.linear_logloss_batch(coef, code)
    _record(K, n)
    sel = _selected(fold, code)
    X64 = X.astype(np.float64)
    for b in range(B):
        m = sel[:, b]
        Z = X64[m] @ coef[b, :, :d].T.astype(np.float64) + coef[b, :, d].astype(np.float64)
        P = np.exp(Z - Z.max(1, keepdims=True))
        P = (P / P.sum(1, keepdims=True)).astype(np.float32)          # predict_proba is float32
        eps = np.finfo(np.float32).eps
        mine = -np.log(np.clip(P[np.arange(m.sum()), y[m]].astype(np.float64), eps, 1 - eps)).mean()
        assert count[b] == m.sum()
        assert abs(mean[b] - mine) <= 1e-6 * mine, (K, b, mean[b], mine)
        sk = log_loss(y[m], P, labels=np.arange(K))
        assert abs(mean[b] - sk) <= 1e-5 * sk, (K, b, mean[b], sk)
        if b == 1:
            assert np.any(P[np.arange(m.sum()), y[m]] < eps), "no saturated row"


# ---- (c) end to end -------------------------------------------------------------------------------------
@pytest.mark.parametrize("weighted", [False, True], ids=["unweighted", "class_weight"])
def test_fits_stop_at_float64_optimum(eng, weighted):
    n, d, K, tol, max_iter = 3000, 20, 5, 1e-4, 300
    rng = np.random.default_rng(1100 + weighted)
    X = rng.standard_normal((n, d)).astype(np.float32)
    V = rng.standard_normal((d, K)) * (2.0 / np.sqrt(d))
    y = np.argmax(X @ V + rng.gumbel(size=(n, K)), 1).astype(np.int32)
    fold = np.random.default_rng(7).permutation(np.arange(n) % 5).astype(np.int8)
    _stage(eng, X, y, fold, 5)
    C = np.logspace(-3, 3, 10)
    cf = (np.arange(10) % 5).astype(np.int32)
    cf[-1] = -1
    M = mr.row_mask(n, fold, cf)
    cw = None

    def stage(idx):
        if cw is not None:
            eng.stage_class_weights(cw[idx], np.array([(M[:, b] * cw[b, y]).sum() for b in idx]))

    if weighted:
        cw = rng.uniform(0.5, 2.0, (10, K)).astype(np.float32)
    stage(np.arange(10))
    res = eng.logreg_multinomial_fit_batch(C, cf, K, tol=tol, max_iter=max_iter)
    coef = res["coef"].astype(np.float64)
    ref = mr.loss_grad(X, y, M, coef, C, cw, bounds=False)
    ok = (res["n_iter"] < max_iter) & (res["status"] == 1)
    assert ok.sum() >= 5, (res["status"], res["n_iter"])
    assert len(set(res["n_iter"][ok])) > 1, "every candidate stopped in the same round"
    gmax = np.abs(ref["g"]).reshape(10, -1).max(1)
    assert np.all(gmax[ok] <= 2 * tol), (np.flatnonzero(gmax[ok] > 2 * tol), gmax[ok].max())
    good = (res["n_iter"] < max_iter) & ((res["status"] == 1) | (res["status"] == 2))
    rel = np.abs(res["loss"] - ref["f"]) / ref["f"]
    assert np.all(rel[good] <= 1e-6), rel[good].max()
    print("weighted=%d: %d of 10 converged, n_iter %s, max |g| %.2e, max loss rel. error %.2e"
          % (weighted, ok.sum(), res["n_iter"].tolist(), gmax[ok].max(), rel[good].max()))
    for b in (0, 4, 9):       # a candidate alone: the same bits as inside the batch
        stage(np.array([b]))
        one = eng.logreg_multinomial_fit_batch(C[b:b + 1], cf[b:b + 1], K, tol=tol, max_iter=max_iter)
        assert np.array_equal(one["coef"][0], res["coef"][b]), b
        assert one["n_iter"][0] == res["n_iter"][b] and one["loss"][0] == res["loss"][b], b
    _record(K, n)


# ---- (d) pass split -------------------------------------------------------------------------------------
def _free_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def test_pass_split_matches_slices(eng):
    n, d, K, B = 200_000, 16, 128, 60
    nz, rpc = mr.multi_chunks(n)
    per_pass = mr.candidates_per_pass(n, d, K, nz)
    assert per_pass == 58 and mr.candidates_per_pass(n, d, K, 0) == 58
    if _free_bytes() < 10e9:
        pytest.skip("the two-pass case needs about 6 GB of device memory; less than 10 GB is free")
    rng = np.random.default_rng(1300)
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = rng.integers(0, K, n).astype(np.int32)
    fold = (np.arange(n) * 5 // n).astype(np.int8)
    _stage(eng, X, y, fold, 5)
    cf = (np.arange(B) % 5).astype(np.int32)
    C = np.logspace(-2, 2, B)
    cw = rng.uniform(0.5, 2.0, (B, K)).astype(np.float32)           # distinct per candidate: a wrong b0 shows
    sw = np.array([(cw[b, y] * (fold != cf[b])).astype(np.float64).sum() for b in range(B)])
    fmask = (rng.random((B, d)) < 0.8).astype(np.uint8)
    fmask[:, 0] = 1
    W = rng.standard_normal((B, K, d + 1)) * 0.1
    coef = W.astype(np.float32)
    code = _score_codes(cf, 5)
    slices = [np.arange(0, 30), np.arange(30, 60)]

    def staged(idx):
        eng.stage_class_weights(cw[idx], sw[idx])
        eng.stage_column_masks(fmask[idx])

    l0 = eng.counters()["launches"]
    staged(np.arange(B))
    f, g = eng.logreg_multinomial_loss_grad(W, C, cf)
    l1 = eng.counters()["launches"]
    parts = []
    for idx in slices:
        staged(idx)
        parts.append(eng.logreg_multinomial_loss_grad(W[idx], C[idx], cf[idx]))
    l2 = eng.counters()["launches"]
    assert l1 - l0 == l2 - l1, ("the batch of 60 must run two passes, as many launches as two slices",
                                l1 - l0, l2 - l1)
    assert np.array_equal(f, np.concatenate([p[0] for p in parts]))
    assert np.array_equal(g, np.concatenate([p[1] for p in parts]))

    conf = eng.multinomial_confusion_batch(coef, code)
    mean, count = eng.linear_logloss_batch(coef, code)
    for idx in slices:
        assert np.array_equal(conf[idx], eng.multinomial_confusion_batch(coef[idx], code[idx]))
        m2, c2 = eng.linear_logloss_batch(coef[idx], code[idx])
        assert np.array_equal(mean[idx], m2) and np.array_equal(count[idx], c2)

    staged(np.arange(B))
    res = eng.logreg_multinomial_fit_batch(C, cf, K, max_iter=3)
    for idx in slices:
        staged(idx)
        one = eng.logreg_multinomial_fit_batch(C[idx], cf[idx], K, max_iter=3)
        for key in ("coef", "n_iter", "status", "loss", "n_evals"):
            assert np.array_equal(res[key][idx], one[key]), key
    RAN.add((k_regime(K), chunk_regime(n), conf_path(K), 2))


def test_every_regime_ran():
    """Every planned (K regime, row-chunk regime, confusion path, passes) combination ran above."""
    want = {(k_regime(s[0]), chunk_regime(s[2]), conf_path(s[0]), 1) for s in SHAPES}
    want |= {(k_regime(s[0]), chunk_regime(min(s[2], N_FLOAT_MAX)), conf_path(s[0]), 1) for s in SHAPES}
    want |= {(k_regime(K), chunk_regime(4097), conf_path(K), 1) for K in (3, 65, 128)}
    want |= {(k_regime(5), chunk_regime(3000), conf_path(5), 1)}
    want |= {(k_regime(128), chunk_regime(200_000), conf_path(128), 2)}
    assert {w[0] for w in want} == {"fills tiles", "divides a tile", "straddles tiles"}
    assert {w[1] for w in want} >= {chunk_regime(n) for n in (50, 4096, 4097, 5000, 70001)}
    assert {w[2] for w in want} == {"shared", "global"} and {w[3] for w in want} == {1, 2}
    assert RAN == want, sorted(want - RAN)
