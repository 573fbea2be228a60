"""The scoring and inference kernels against float64 and integer references (tests/scoring_reference.py).

Entries and the kernels they run:

  skd_linear_decision      predict_kernel<NB> (B <= 16 and 8 rows of pitch ldx in the 48 KB weight cache), otherwise
                           fwd_kernel<MODE_DECISION> (simt_decision)
  skd_predict_linear       stream_rows (row chunks, direct / threaded-bounce / page-locked staging) and
                           predict_kernel<NB, cached> with NB = 8/4/2/1, or <NB, uncached> for rows wider than the cache
  skd_linear_score_batch,  fwd_kernel<MODE_SCORE>, <MODE_R2> on the CUDA cores: d > 256, or skd_set_kernel(1)
  skd_linear_r2_batch
  skd_linear_auc_batch     simt_decision, auc_key_kernel, radix sort, auc_count_kernel; columns in blocks of <= 4096
  skd_linear_logloss_batch mn_logloss_kernel, binary columns (K = 1)
  skd_forest_predict       forest_predict_kernel<CMAX> for C <= 2 / 8 / 32, and <0> (zeroed output, in-place sums)

Tiers:

(a) exact: X holds integers in [-7, 7] times 2^e_k and the weights integers in [-2, 2] times 2^-e_k, intercepts are
    integers.  Every product is an integer and every partial sum an integer below 2^24, so every decision value is
    its float64 value in any summation order, and decision values, accuracy counts, squared-error sums and AUC pair
    counts must be equal.  Forest outputs must equal the float64 walk and scikit-learn bit for bit.
(b) float: random float32 data; decision values within gamma_h (sum |x w| + |b|) of float64 with h the summation depth
    of the kernel (shown to reject a reference missing one median term), accuracy counts equal outside that band,
    and the binary log loss within one float32 ulp of p per row plus the effect of the decision error.
(c) public path: batch_predict / get_prediction_udf against scikit-learn's predict / predict_proba, and a roc_auc
    grid search against GridSearchCV.

The last test asserts that every planned (entry, kernel variant, regime) ran.
"""
import ctypes
import warnings

import numpy as np
import pytest

from tests import scoring_reference as sr

pytestmark = pytest.mark.gpu

CACHE_BYTES = 48 * 1024
CHUNK_BYTES = 256 << 20          # stream_rows: input and output of one row chunk
BOUNCE_BYTES = 8 << 20           # stage_rows_h2d: pinned bounce block, and the size below which it copies directly

D_EXACT = [1, 3, 4, 5, 15, 16, 17, 63, 64, 65, 256, 257, 300, 1000, 1536, 1537, 3000, 12288, 12289, 20000]
B_EXACT = [1, 2, 3, 5, 7, 8, 9, 15, 16, 17, 63, 64, 65, 129]

RAN = set()


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _launches(eng):
    return eng.counters()["launches"]


def _int_data(rng, n, d, e=None):
    """Integers in [-7, 7] times 2^e_k, e_k in [-20, 20] (or given); a zero row, so some decision values equal b."""
    if e is None:
        e = rng.integers(-20, 21, d)
    Xi = rng.integers(-7, 8, (n, d))
    Xi[0] = 7
    if n > 2:
        Xi[1] = 0
    return (Xi * np.exp2(e)).astype(np.float32), e


def _int_coef(rng, B, d, e, b_range=100):
    coef = np.zeros((B, d + 1), np.float32)
    coef[:, :d] = rng.integers(-2, 3, (B, d)) * np.exp2(-e)
    coef[:, d] = rng.integers(-b_range, b_range + 1, B)
    return coef


def _decision_route(d, B):
    """skd_linear_decision's kernel for a staged X of row pitch round_up(d, 16)."""
    ldx = sr.round_up(d, 16)
    return "predict" if B <= 16 and min(8, CACHE_BYTES // (4 * ldx)) == 8 else "simt"


def _predict_passes(ldx, B):
    """(NB, cached) of every pass of predict_device over B models of pitch ldx."""
    rows = min(8, CACHE_BYTES // (4 * ldx))
    out, b0 = [], 0
    while b0 < B:
        cap = min(B - b0, rows if rows > 0 else 8)
        nb = 8 if cap >= 8 else 4 if cap >= 4 else 2 if cap >= 2 else 1
        out.append((nb, rows > 0))
        b0 += nb
    return out


def _chunk_rows(d, out_row_bytes):
    return max(1, CHUNK_BYTES // max(4 * sr.round_up(d, 4), out_row_bytes))


def _n_for(d, i):
    """n < 64, n not a multiple of 64, and n with many pick_chunks chunks, in turn; X stays below 2e7 entries."""
    n = (37, 1000, 4099)[i % 3]
    return max(37, min(n, int(2e7 // d)))


# ---- (a) exact tier: decision values --------------------------------------------------------------------
@pytest.mark.parametrize("d", D_EXACT)
def test_exact_decision_and_predict(eng, d):
    i = D_EXACT.index(d)
    rng = np.random.default_rng(1000 + d)
    n = _n_for(d, i)
    X, e = _int_data(rng, n, d)
    eng.stage_x(X)
    ldx4 = sr.round_up(d, 4)
    for B in B_EXACT:
        coef = _int_coef(rng, B, d, e)
        want = sr.decision(X, coef)
        route = _decision_route(d, B)
        got = eng.linear_decision(coef)
        bad = np.argwhere(got != want)
        assert bad.size == 0, ("decision", route, d, B, bad[:5])
        RAN.add(("decision", route))
        l0 = _launches(eng)
        got = eng.predict_linear(X, coef)
        passes = _predict_passes(ldx4, B)
        assert _launches(eng) - l0 == len(passes), (d, B)
        bad = np.argwhere(got != want)
        assert bad.size == 0, ("predict", d, B, passes, bad[:5])
        RAN.update(("predict", p) for p in passes)


def _predict_exact(eng, X, coef, want_chunks, ld=None):
    """skd_predict_linear of the first d columns of X (row pitch ld, default d) through the C-ABI, checked exactly
    and for the number of chunks it ran."""
    m, d = X.shape[0], coef.shape[1] - 1
    ld = ld or d
    B = coef.shape[0]
    out = np.empty((m, B), np.float32)
    secs = ctypes.c_double()
    l0 = _launches(eng)
    from skdist_b200._lib import check, ptr
    check(eng._lib.skd_predict_linear(eng._h, ptr(X), m, d, ld, B, ptr(coef), ptr(out), ctypes.byref(secs)), eng._h)
    passes = _predict_passes(sr.round_up(d, 4), B)
    assert _launches(eng) - l0 == want_chunks * len(passes), ("chunks", want_chunks)
    for r0 in range(0, m, 1 << 18):                 # the reference in blocks of rows
        bad = np.argwhere(out[r0:r0 + (1 << 18)] != sr.decision(X[r0:r0 + (1 << 18), :d], coef))
        assert bad.size == 0, ("predict rows", r0, bad[:5])
    return out


def test_exact_predict_streaming(eng):
    """The staging routes of stream_rows and its row chunks, each counted by the kernel launches."""
    rng = np.random.default_rng(7)
    # (i) below 8 MiB: one direct copy
    X, e = _int_data(rng, 5000, 300)
    _predict_exact(eng, X, _int_coef(rng, 3, 300, e), 1)
    RAN.add(("stream", "direct"))
    # (ii) pageable rows through the threaded bounce, last bounce block short (6990 rows per 8 MiB block)
    d = 300
    per_blk = BOUNCE_BYTES // (4 * d)
    X, e = _int_data(rng, 5 * per_blk + 123, d)
    assert X.nbytes > BOUNCE_BYTES and X.shape[0] % per_blk != 0
    _predict_exact(eng, X, _int_coef(rng, 9, d, e), 1)
    RAN.add(("stream", "bounce"))
    # (iii) a page-locked source goes straight to the copy engine
    import torch
    Xp = torch.empty((30000, d), dtype=torch.float32, pin_memory=True).numpy()
    Xp[:] = X[:30000]
    assert Xp.nbytes > BOUNCE_BYTES
    _predict_exact(eng, Xp, _int_coef(rng, 5, d, e), 1)
    RAN.add(("stream", "pinned"))
    # (iv) a row-strided source, ld > d: direct (small) and through the bounce (large)
    for m in (1000, 3 * per_blk + 7):
        big, e2 = _int_data(rng, m, d + 13)
        coef = _int_coef(rng, 4, d, e2[:d])
        _predict_exact(eng, np.ascontiguousarray(big), coef, 1, ld=d + 13)
    RAN.add(("stream", "strided"))
    # (v) two full 256 MiB chunks and a short third
    d = 1024
    rows = _chunk_rows(d, 3 * 4)
    X, e = _int_data(rng, 2 * rows + 77, d)
    _predict_exact(eng, X, _int_coef(rng, 3, d, e), 3)
    RAN.add(("stream", "chunks"))
    # narrow rows, wide output: the chunk is bounded by the output (129 x 4 bytes per row against 16 of input)
    d, B = 4, 129
    rows = _chunk_rows(d, 4 * B)
    assert rows < CHUNK_BYTES // 16
    X, e = _int_data(rng, rows + 100, d)
    _predict_exact(eng, X, _int_coef(rng, B, d, e), 2)
    RAN.add(("stream", "output-bound"))


# ---- (a) exact tier: accuracy and R^2 on the CUDA cores -------------------------------------------------
# (d, n, folds, kernel choice): d > 256 picks fwd_kernel by itself, d <= 256 under skd_set_kernel(1)
SIMT_SHAPES = [
    (257, 4097, 5, 0), (300, 63, 40, 0), (1000, 20001, 40, 0),
    (1, 64, 5, 1), (17, 65, 40, 1), (64, 129, 0, 1), (256, 4096, 5, 1),
]
B_SIMT = [1, 63, 64, 65, 129]


def _folds(rng, n, nf):
    if nf == 0:
        return None
    if nf == 5:                                     # contiguous, boundaries inside a 64-row tile
        return (np.arange(n) * 5 // n).astype(np.int8)
    return rng.permutation(np.arange(n) % nf).astype(np.int8)


def _codes(rng, nf, B):
    pool = np.array([-2]) if nf == 0 else np.r_[np.arange(nf), -2, -3 - np.arange(nf)]
    code = rng.choice(pool, B).astype(np.int32)
    code[:min(B, len(pool))] = pool[:min(B, len(pool))]          # every code at least once where B allows
    return code


def _stage(eng, X, ycls, fold, nf, yreal=None):
    eng.stage_x(X)
    eng.stage_labels(ycls)
    eng.stage_folds(fold, nf) if fold is not None else eng.stage_folds(None, 0)
    if yreal is not None:
        eng.stage_targets(yreal)


@pytest.mark.parametrize("shape", SIMT_SHAPES, ids=["d%d-n%d-f%d-k%d" % s for s in SIMT_SHAPES])
def test_exact_score_and_r2_simt(eng, shape):
    d, n, nf, kernel = shape
    rng = np.random.default_rng(2000 + d)
    X, e = _int_data(rng, n, d)
    ycls = rng.integers(0, 3, n).astype(np.int32)
    fold = _folds(rng, n, nf)
    yreal = rng.integers(-100, 101, n).astype(np.float32)
    _stage(eng, X, ycls, fold, nf, yreal)
    prev = eng.set_kernel(kernel)
    try:
        for B in B_SIMT:
            coef = _int_coef(rng, B, d, e, b_range=3)       # small intercepts: many rows with z == 0 exactly
            coef[0, :] = 0.0                                # z == 0 on every row: predicted negative
            code = _codes(rng, nf, B)
            pos = rng.integers(0, 3, B).astype(np.int32)
            Z = sr.decision(X, coef)
            assert (Z == 0).any()
            want_c, want_n = sr.accuracy_counts(Z, ycls, pos, code, fold)
            correct, count = eng.linear_score_batch(coef, code, pos)
            assert np.array_equal(count, want_n), (B, np.flatnonzero(count != want_n)[:5])
            bad = np.flatnonzero(correct != want_c)
            assert bad.size == 0, ("accuracy", B, bad[:5], correct[bad[:5]], want_c[bad[:5]])
            want_s, _ = sr.sse(Z, yreal, code, fold)
            s, count = eng.linear_r2_batch(coef, code)
            assert np.array_equal(count, want_n)
            bad = np.flatnonzero(s != want_s)
            assert bad.size == 0, ("sse", B, bad[:5], s[bad[:5]], want_s[bad[:5]])
            regime = "auto" if kernel == 0 else "forced"
            RAN.add(("score", regime))
            RAN.add(("r2", regime))
    finally:
        eng.set_kernel(prev)


# ---- (a) exact tier: ROC-AUC pair counts ----------------------------------------------------------------
def _auc_raw(eng, coef, code, pos):
    from skdist_b200._lib import check, ptr
    B = coef.shape[0]
    coef = np.ascontiguousarray(coef, np.float32)
    code = np.ascontiguousarray(code, np.int32)
    pos = np.ascontiguousarray(pos, np.int32)
    out = np.empty((3, B), np.int64)
    check(eng._lib.skd_linear_auc_batch(eng._h, B, ptr(coef), ptr(code), ptr(pos), ptr(out[0]), ptr(out[1]),
                                        ptr(out[2])), eng._h)
    return out


def _check_auc(eng, X, ycls, fold, coef, code, pos, label):
    got = _auc_raw(eng, coef, code, pos)
    want = sr.auc_counts_batch(sr.decision(X, coef), ycls, pos, code, fold)
    bad = np.flatnonzero((got != want).any(0))
    assert bad.size == 0, (label, bad[:5], got[:, bad[:5]], want[:, bad[:5]])
    return got


def test_exact_auc_ties_and_empty_classes(eng):
    """Tie groups of thousands of rows, every row tied, selections without positives or without negatives, every
    scoring code, B = 1 and a block of many columns."""
    rng = np.random.default_rng(3)
    n, d, nf = 50000, 17, 5
    X, e = _int_data(rng, n, d)
    ycls = rng.integers(0, 3, n).astype(np.int32)
    fold = rng.permutation(np.arange(n) % nf).astype(np.int8)
    ycls[fold == 0] = 1                              # fold 0 holds class 1 only
    _stage(eng, X, ycls, fold, nf)
    code = _codes(rng, nf, 40)
    pos = rng.integers(0, 3, 40).astype(np.int32)
    coef = _int_coef(rng, 40, d, e, b_range=3)
    coef[:20, :d] = 0.0
    coef[:20, 3] = rng.integers(1, 3, 20) * np.exp2(-e[3])     # z takes at most 15 values: ~3000 rows a group
    coef[20:23] = 0.0                                           # every row tied: 2U = n_pos n_neg
    code[23:26] = 0                                             # fold 0: class 1 only
    pos[23], pos[24], pos[25] = 1, 2, 5                         # no negatives / no positives / class absent
    got = _check_auc(eng, X, ycls, fold, coef, code, pos, "ties")
    assert np.array_equal(got[0, 20:23], got[1, 20:23] * got[2, 20:23])
    assert got[2, 23] == 0 and got[1, 24] == 0 and got[1, 25] == 0
    sizes = np.array([np.unique(sr.decision(X, coef[j:j + 1])[:, 0], return_counts=True)[1].max() for j in range(20)])
    assert sizes.min() > 2 * (n // 256 + 1)                     # groups span several per-thread runs
    RAN.add(("auc", "ties"))
    for j in (0, 23, 24):                                       # B = 1
        _check_auc(eng, X, ycls, fold, coef[j:j + 1], code[j:j + 1], pos[j:j + 1], "B=1")
    RAN.add(("auc", "B=1"))


def test_exact_auc_column_blocks(eng):
    """B > 4096: auc_batch runs two column blocks, each with several selection lists."""
    rng = np.random.default_rng(4)
    n, d, nf = 3000, 5, 5
    X, e = _int_data(rng, n, d)
    ycls = rng.integers(0, 2, n).astype(np.int32)
    fold = _folds(rng, n, nf)
    _stage(eng, X, ycls, fold, nf)
    B = 4096 + 37
    code = _codes(rng, nf, B)
    pos = rng.integers(0, 2, B).astype(np.int32)
    coef = _int_coef(rng, B, d, e, b_range=3)
    l0 = _launches(eng)
    _check_auc(eng, X, ycls, fold, coef, code, pos, "blocks")
    # per block of 4096 columns: the decision values, one key launch per selection list, the sort and the count
    lists = [len(np.unique(code[b0:b0 + 4096])) for b0 in (0, 4096)]
    assert min(lists) > 1 and _launches(eng) - l0 == sum(3 + k for k in lists), (lists, _launches(eng) - l0)
    RAN.add(("auc", "blocks"))


def test_exact_auc_pair_counts_beyond_int32(eng):
    """n_pos n_neg > 2^31 on the every-row code."""
    rng = np.random.default_rng(5)
    n, d = 120_000, 300
    X, e = _int_data(rng, n, d)
    ycls = (np.arange(n) % 2).astype(np.int32)
    _stage(eng, X, ycls, None, 0)
    coef = _int_coef(rng, 3, d, e, b_range=3)
    got = _check_auc(eng, X, ycls, None, coef, np.full(3, -2, np.int32), np.array([1, 0, 1], np.int32), "2^31")
    assert np.all(got[1] * got[2] > 2 ** 31)
    RAN.add(("auc", "beyond int32"))


# ---- (a) exact tier: forest inference -------------------------------------------------------------------
def _forest(C, n_trees, seed, depth=None, d=6, n=800):
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier, RandomForestRegressor
    rng = np.random.default_rng(seed)
    X = (np.round(rng.standard_normal((n, d)) * 4) / 4).astype(np.float32)   # repeated values, float32 midpoints
    if C == 1:
        y = X[:, 0] * 3 + rng.standard_normal(n)
        model = RandomForestRegressor(n_estimators=n_trees, max_depth=depth, random_state=seed, n_jobs=1)
    else:
        y = rng.integers(0, C, n)
        y[:C] = np.arange(C)
        cls = ExtraTreesClassifier if seed % 2 else RandomForestClassifier
        model = cls(n_estimators=n_trees, max_depth=depth, random_state=seed, n_jobs=1)
    return model.fit(X, y), X


def _threshold_rows(X, arrays, rng, cap=30000):
    """Rows of X with one feature set to float32(t) and its two float32 neighbours, for the thresholds t."""
    inner = np.flatnonzero(arrays[1] != -1)
    if len(inner) * 3 > cap:
        inner = rng.choice(inner, cap // 3, replace=False)
    t32 = arrays[4][inner].astype(np.float32)
    vals = np.concatenate([t32, np.nextafter(t32, np.float32(np.inf)), np.nextafter(t32, np.float32(-np.inf))])
    Xt = X[rng.integers(0, len(X), len(vals))].copy()
    Xt[np.arange(len(vals)), np.tile(arrays[3][inner], 3)] = vals
    return Xt


def _cmax(C):
    return 2 if C <= 2 else 8 if C <= 8 else 32 if C <= 32 else 0


FOREST_CASES = [(1, 3, None), (2, 257, None), (3, 1, None), (8, 3, 6), (9, 257, 8), (32, 1, None), (33, 3, None),
                (100, 257, 10)]


@pytest.mark.parametrize("case", FOREST_CASES, ids=["C%d-t%d" % c[:2] for c in FOREST_CASES])
def test_exact_forest_predict(eng, case):
    from skdist_b200.distribute.predict import _forest_arrays
    C, n_trees, depth = case
    model, X = _forest(C, n_trees, 40 + C, depth)
    arrays = _forest_arrays(model.estimators_)
    Xt = _threshold_rows(X, arrays, np.random.default_rng(C))
    got = eng.forest_predict(Xt, *arrays)
    want = sr.forest_walk(Xt, *arrays)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    if C == 1:
        assert np.array_equal(got[:, 0], model.predict(Xt))
    else:
        assert np.array_equal(got, model.predict_proba(Xt))
    RAN.add(("forest", _cmax(C)))


def test_exact_forest_threshold_equality(eng):
    """Hand-built trees with thresholds exact in float32: x == t goes left, nextafter(t, +inf) right."""
    t = np.array([0.5, -2.0, 3.0], np.float64)
    # tree 0: root on feature 1 at 0.5, left leaf, right node on feature 0 at -2.0 with two leaves
    # tree 1: a lone leaf; tree 2: root on feature 2 at 3.0 with two leaves
    off = np.array([0, 5, 6, 9], np.int64)
    left = np.array([1, -1, 3, -1, -1, -1, 1, -1, -1], np.int32)
    right = np.array([2, -1, 4, -1, -1, -1, 2, -1, -1], np.int32)
    feature = np.array([1, 0, 0, 0, 0, 0, 2, 0, 0], np.int32)
    thr = np.array([t[0], -2, t[1], -2, -2, -2, t[2], -2, -2], np.float64)
    C = 3
    value = np.random.default_rng(0).random((9, C))
    xs = []
    for f, tv in ((1, t[0]), (0, t[1]), (2, t[2])):
        for v in (np.float32(tv), np.nextafter(np.float32(tv), np.float32(np.inf)),
                  np.nextafter(np.float32(tv), np.float32(-np.inf))):
            for base in (-5.0, 0.5, 5.0):
                row = np.full(3, base, np.float32)
                row[f] = v
                xs.append(row)
    Xt = np.array(xs, np.float32)
    got = eng.forest_predict(Xt, off, left, right, feature, thr, value)
    want = sr.forest_walk(Xt, off, left, right, feature, thr, value)
    assert np.array_equal(got, want)
    # the reference itself: x == t takes the left child, the next float32 above it the right one
    for f, k, leaf_left, leaf_right in ((1, 0, 1, None), (2, 6, 7, 8)):
        for v, leaf in ((np.float32(thr[k]), leaf_left), (np.nextafter(np.float32(thr[k]), np.float32(np.inf)), leaf_right)):
            if leaf is None:
                continue
            row = np.full((1, 3), -5.0, np.float32)
            row[0, f] = v
            t0 = 0 if k < 5 else 2
            one = sr.forest_walk(row, off[t0:t0 + 2] - off[t0], left[off[t0]:off[t0 + 1]], right[off[t0]:off[t0 + 1]],
                                 feature[off[t0]:off[t0 + 1]], thr[off[t0]:off[t0 + 1]], value[off[t0]:off[t0 + 1]])
            assert np.array_equal(one[0], value[leaf])
    RAN.add(("forest", "equality"))


def test_exact_forest_chunks(eng):
    """More rows than one chunk; and narrow rows with C = 40, whose chunk is bounded by the 320-byte output rows."""
    from skdist_b200.distribute.predict import _forest_arrays
    rng = np.random.default_rng(9)
    for C, d, trees in ((100, 6, 3), (40, 4, 1)):
        model, X = _forest(C, trees, 60 + C, None, d=d, n=2000)
        arrays = _forest_arrays(model.estimators_)
        rows = _chunk_rows(d, 8 * C)
        base = _threshold_rows(X, arrays, rng)
        Xt = np.resize(base, (rows + 1000, d))
        l0 = _launches(eng)
        got = eng.forest_predict(Xt, *arrays)
        assert _launches(eng) - l0 == 2, ("chunks", C, _launches(eng) - l0)
        want = sr.forest_walk(Xt, *arrays)
        assert np.array_equal(got, want)
        assert np.array_equal(got, model.predict_proba(Xt))
    RAN.add(("forest", "chunks"))


# ---- (b) float tier -------------------------------------------------------------------------------------
D_FLOAT = [1, 17, 64, 300, 1000]
B_FLOAT = [3, 9, 65]


def _float_data(rng, n, d, B):
    X = (rng.standard_normal((n, d)) * rng.uniform(0.5, 2.0, d)).astype(np.float32)
    coef = (rng.standard_normal((B, d + 1)) / np.sqrt(d)).astype(np.float32)
    return X, coef


def _check_float_decision(X, coef, got, depth, label, discriminate):
    Z = sr.decision(X, coef)
    A = sr.decision_abs(X, coef)
    bound = sr.gamma(depth) * A
    err = np.abs(got.astype(np.float64) - Z)
    assert np.all(err <= bound), (label, (err / bound).max())
    if discriminate and X.shape[1] > 1:
        d = X.shape[1]
        for j in range(coef.shape[0]):
            terms = np.abs(X.astype(np.float64) * coef[j, :d].astype(np.float64)).mean(0)
            k = np.argsort(terms)[d // 2]
            wrong = Z[:, j] - X[:, k].astype(np.float64) * np.float64(coef[j, k])
            assert np.any(np.abs(got[:, j] - wrong) > bound[:, j]), (label, "bound cannot see one term", j)
    return Z, bound


@pytest.mark.parametrize("d", D_FLOAT)
def test_float_decision_and_predict(eng, d):
    rng = np.random.default_rng(3000 + d)
    n = 3000
    for B in B_FLOAT:
        X, coef = _float_data(rng, n, d, B)
        eng.stage_x(X)
        route = _decision_route(d, B)
        depth = sr.depth_predict(sr.round_up(d, 16)) if route == "predict" else sr.depth_fwd(d)
        _check_float_decision(X, coef, eng.linear_decision(coef), depth, "decision %s d=%d B=%d" % (route, d, B), True)
        got = eng.predict_linear(X, coef)
        _check_float_decision(X, coef, got, sr.depth_predict(sr.round_up(d, 4)), "predict d=%d B=%d" % (d, B), True)
        RAN.add(("float decision", route))


@pytest.mark.parametrize("d", [17, 300, 1000])
def test_float_accuracy_and_logloss(eng, d):
    """Accuracy counts equal the reference outside the rounding band of z; the binary log loss within its
    per-row bound (both on the CUDA cores)."""
    rng = np.random.default_rng(4000 + d)
    n, nf, B = 5001, 5, 65
    X, coef = _float_data(rng, n, d, B)
    coef[:, d] = 0.0
    coef[1, :d] *= 1e-3                                # many rows near z = 0
    ycls = rng.integers(0, 3, n).astype(np.int32)
    fold = _folds(rng, n, nf)
    _stage(eng, X, ycls, fold, nf)
    code = _codes(rng, nf, B)
    pos = rng.integers(0, 3, B).astype(np.int32)
    Z = sr.decision(X, coef)
    bound = sr.gamma(sr.depth_fwd(d)) * sr.decision_abs(X, coef)
    M = sr.select(code, fold, n)
    sure = np.abs(Z) > bound
    hit = (Z > 0) == (ycls[:, None] == pos[None, :])
    lo = (M & sure & hit).sum(0)
    band = (M & ~sure).sum(0)
    prev = eng.set_kernel(1)
    try:
        correct, count = eng.linear_score_batch(coef, code, pos)
        mean, count2 = eng.linear_logloss_batch(coef, code, pos)
    finally:
        eng.set_kernel(prev)
    assert np.array_equal(count, M.sum(0)) and np.array_equal(count2, M.sum(0))
    assert np.all(correct >= lo) and np.all(correct <= lo + band), (correct - lo, band)
    RAN.add(("float score", "simt"))
    z32 = Z.astype(np.float32)
    for j in range(B):
        m = M[:, j]
        yb = ycls[m] == pos[j]
        ref = sr.binary_logloss(z32[m, j], yb).sum()
        tol = sr.binary_logloss_bound(z32[m, j], yb, bound[m, j] + np.abs(Z[m, j] - z32[m, j])).sum() + 1e-12 * ref
        assert abs(mean[j] * count2[j] - ref) <= tol, (j, mean[j] * count2[j], ref, tol)
    RAN.add(("logloss", "binary"))


def test_exact_logloss(eng):
    """Integer data: z is exact, so the loss differs from the reference only by the rounding of p."""
    rng = np.random.default_rng(11)
    n, d, nf, B = 4097, 64, 40, 9
    X, e = _int_data(rng, n, d)
    ycls = rng.integers(0, 2, n).astype(np.int32)
    fold = _folds(rng, n, nf)
    _stage(eng, X, ycls, fold, nf)
    coef = _int_coef(rng, B, d, e + 5, b_range=3)        # z on a 1/32 grid, mostly inside (-20, 20)
    code = _codes(rng, nf, B)
    pos = rng.integers(0, 2, B).astype(np.int32)
    Z = sr.decision(X, coef)
    M = sr.select(code, fold, n)
    mean, count = eng.linear_logloss_batch(coef, code, pos)
    for j in range(B):
        m = M[:, j]
        yb = ycls[m] == pos[j]
        ref = sr.binary_logloss(Z[m, j].astype(np.float32), yb).sum()
        tol = sr.binary_logloss_bound(Z[m, j].astype(np.float32), yb, 0.0).sum() + 1e-12 * ref
        assert abs(mean[j] * count[j] - ref) <= tol, (j, mean[j] * count[j], ref, tol)
    RAN.add(("logloss", "exact"))


# ---- (c) public path ------------------------------------------------------------------------------------
def _quantised(est, rng, e):
    """Put a fitted linear model's coefficients on the exact grid: integers times 2^(-e_k - 3), z on a 1/8 grid."""
    est.coef_ = (rng.integers(-2, 3, est.coef_.shape) * np.exp2(-e - 3)).astype(est.coef_.dtype)
    est.intercept_ = rng.integers(-3, 4, est.intercept_.shape).astype(est.intercept_.dtype)


@pytest.mark.parametrize("kind", ["ovr10-d2000", "single-d20000"])
def test_public_predict_wide_rows(kind):
    """OneVsRest LogisticRegression over 10 classes at d = 2000 (4 + 4 + 2 cached models a pass) and one model at
    d = 20000 (uncached): scikit-learn's predict exactly (coefficients on the exact grid), predict_proba within
    float32 rounding."""
    from sklearn.linear_model import LogisticRegression
    from sklearn.multiclass import OneVsRestClassifier

    from skdist_b200.distribute.predict import batch_predict, get_prediction_udf
    rng = np.random.default_rng(12)
    d, K = (2000, 10) if kind.startswith("ovr") else (20000, 2)
    Xtr, e = _int_data(rng, 300, d)
    y = rng.integers(0, K, 300)
    y[:K] = np.arange(K)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if K > 2:
            model = OneVsRestClassifier(LogisticRegression(max_iter=5)).fit(Xtr, y)
            for est in model.estimators_:
                _quantised(est, rng, e)
        else:
            model = LogisticRegression(max_iter=5).fit(Xtr, y)
            _quantised(model, rng, e)
    X, _ = _int_data(rng, 700, d, e)
    assert np.array_equal(batch_predict(model, X), model.predict(X))
    cols = [X[:, k] for k in range(d)]
    assert np.array_equal(np.asarray(get_prediction_udf(model)(*cols)), model.predict(X))
    p = batch_predict(model, X, "predict_proba")
    np.testing.assert_allclose(p, model.predict_proba(X), rtol=2.0 ** -20, atol=2.0 ** -22)   # float32 rounding of p
    q = np.stack(get_prediction_udf(model, "predict_proba")(*cols).to_numpy())
    assert np.array_equal(p, q)
    ldx = sr.round_up(d, 4)
    RAN.update(("public", p_) for p_ in _predict_passes(ldx, K if K > 2 else 1))


def test_public_roc_auc_search_simt():
    """scoring="roc_auc" at d = 300: the fits and the decision values run on the CUDA cores."""
    from sklearn.linear_model import LogisticRegression
    from sklearn.model_selection import GridSearchCV

    from skdist.distribute.search import DistGridSearchCV
    from skdist_b200.datasets import make_g1_classification
    X, y = make_g1_classification(6000, 300, seed=34)
    grid = {"C": [0.001, 0.01, 0.1]}       # regularised enough that both solvers stop within 1e-5 of the optimum
    gs = DistGridSearchCV(LogisticRegression(), grid, None, cv=4, scoring="roc_auc").fit(X, y)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sk = GridSearchCV(LogisticRegression(), grid, cv=4, scoring="roc_auc").fit(X, y)
    np.testing.assert_allclose(gs.cv_results_["mean_test_score"], sk.cv_results_["mean_test_score"], rtol=0, atol=2e-5)
    assert gs.best_params_ == sk.best_params_
    RAN.add(("public", "roc_auc"))


def test_every_variant_ran():
    """Every planned (entry, kernel variant or route, regime) ran above."""
    want = {("decision", "predict"), ("decision", "simt"), ("float decision", "predict"), ("float decision", "simt")}
    want |= {("predict", (nb, cached)) for nb in (8, 4, 2, 1) for cached in (True, False)}
    want |= {("stream", s) for s in ("direct", "bounce", "pinned", "strided", "chunks", "output-bound")}
    want |= {("score", r) for r in ("auto", "forced")} | {("r2", r) for r in ("auto", "forced")}
    want |= {("auc", r) for r in ("ties", "B=1", "blocks", "beyond int32")}
    want |= {("forest", c) for c in (2, 8, 32, 0, "equality", "chunks")}
    want |= {("float score", "simt"), ("logloss", "binary"), ("logloss", "exact")}
    want |= {("public", (4, True)), ("public", (2, True)), ("public", (1, False)), ("public", "roc_auc")}
    assert RAN == want, (sorted(want - RAN, key=str), sorted(RAN - want, key=str))
