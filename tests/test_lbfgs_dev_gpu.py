"""The device L-BFGS-B driver (csrc/lbfgs_dev.cu on csrc/lbfgs_core.h) against the host build of the core and
scipy's L-BFGS-B, evaluation by evaluation, through skd_lbfgs_dev_*: the production optimiser kernels of the
binary (one warp per column, WarpPar) and multinomial (one CTA per candidate, CtaPar) fits fed with the partials
of tests/lbfgs_reference.py instead of an evaluation kernel.

Per round the device and the host core each evaluate at their own points.  Checked:
  (a) at every evaluation of every column up to the 60th: the integer state equal; x, f within 1e-10 relative
      to the host core, stp within 1e-9 and theta within 1e-8 over the first 30, within the looser TOL[True]
      from 30 to 60; and the final x of every run within FINAL_TOL.  The only differences are the order of the
      dot products and FMA contraction, whose rounding compounds over a run.  Where g'd at a trial point is
      zero up to rounding the two may take different sides of the line search's sign test; such a column is
      compared up to that point, and at most one column in 50 may end so;
  (b) evaluation count, nit, status and the final x against scipy on a few columns;
  (c) the plumbing, exactly: the slot list after every round equals a model of the dense or fold-grouped
      compaction, the slot / running counts and the round record equal the model, the exported fp32 rows are the
      new points, masked features stay 0, and finish returns fp32(x), min(nit, maxiter), f and the status.
Slots that hold no live column get NaN partials: a read of one would end its column with status 5."""
import numpy as np
import pytest

from skdist_b200 import _lib
from skdist_b200._lib import ptr
from tests import lbfgs_reference as lr

pytestmark = pytest.mark.gpu

RAN = set()
SEEN = set()
STALE = ("exact", "stale1", "stale4", "never")
N_CHECK = 60     # evaluations compared one by one (past them an ill-conditioned run's rounding drift compounds)
N_REAL = 30      # evaluations over which x, f, stp, theta are compared at the tight bound
# relative bounds on x, f, stp, theta against the host core: over the first N_REAL evaluations, and from there to
# N_CHECK, where the rounding of the device's dot-product order and FMA contraction has accumulated; LATE records
# the largest deviation seen past N_REAL and on the final points
# (largest seen on an H100 over this file between evaluations 30 and 60: x 1.1e-10, f 3.9e-10, stp 1.2e-9,
# theta 2.3e-8; the late bounds are about ten times those).  theta = y'y / s'y with s'y = (gd - gdold) stp
# cancels near convergence, and stp comes out of dcstep's interpolation, which divides differences of f and g.
TOL = {False: {"x": 1e-10, "f": 1e-10, "stp": 1e-9, "theta": 1e-8},
       True: {"x": 1e-9, "f": 4e-9, "stp": 1.2e-8, "theta": 3e-7}}
LATE = {"x": 0.0, "f": 0.0, "stp": 0.0, "theta": 0.0, "final x": 0.0}
FINAL_TOL = 5e-5   # final x of every run (largest seen: 4.7e-6, ill-conditioned runs of over 100 evaluations)
TIES = []          # (family, column, evaluation) where the device and the host core parted at a rounding tie
COMPARED = [0]     # columns compared with the host core


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _stage(eng, d):
    rng = np.random.default_rng(d)
    eng.stage_x(rng.standard_normal((96, d)).astype(np.float32))
    eng.stage_labels((rng.random(96) < 0.5).astype(np.int32))
    eng.stage_folds(None, 0)


def grouped_layout(col_fold):
    """the fold-grouped slot list: columns stable-sorted by fold, every fold segment padded to 128"""
    out = []
    for f in sorted(set(int(v) for v in col_fold)):
        seg = [(c, max(f, -1), 0, 0) for c in np.flatnonzero(col_fold == f)]
        seg += [(-1, max(f, -1), -1, 0)] * (-len(seg) % 128)
        out += seg
    return out


def _n_act_in(stale, hist, r, cap):
    if stale == "exact":
        return hist[-1]
    if stale == "stale1":
        return hist[-2] if len(hist) >= 2 else hist[0]
    if stale == "stale4":
        return hist[(r // 4) * 4]
    return cap


def run_device(eng, prob, maxiter, maxls, pgtol, grouped=False, use_reduce=False, col_fold=None, stale="exact"):
    """Drive skd_lbfgs_dev_* to the end, checking the plumbing after every round; per column the points it
    evaluated, its states after every evaluation, and the finish outputs."""
    lib = _lib.load()
    B, K, d, n, nz = prob.B, prob.K, prob.d, prob.n, prob.nz
    col_fold = np.full(B, -1, np.int32) if col_fold is None else np.asarray(col_fold, np.int32)
    dims = np.zeros(4, np.int32)
    gs = None if prob.gscale is None else ptr(np.ascontiguousarray(prob.gscale))
    fm = None if prob.fmask is None else ptr(np.ascontiguousarray(prob.fmask))
    h = lib.skd_lbfgs_dev_create(eng._h, B, K, d, int(prob.fit_intercept), int(grouped), ptr(col_fold), nz,
                                 int(use_reduce), maxiter, maxls, pgtol, lr.FTOL, ptr(prob.l2), ptr(prob.inv_n), gs,
                                 fm, ptr(dims))
    if not h:
        _lib.check(1, eng._h)
    n_var, cap, ldw, nrows = (int(v) for v in dims)
    assert n_var == n
    try:
        slots = grouped_layout(col_fold) if grouped else [(c, int(col_fold[c]), 0, 0) for c in range(B)]
        assert len(slots) == cap
        x = np.zeros((B, n))
        k = np.zeros(B, np.int64)
        running = np.ones(B, bool)
        hist = [cap]
        xs = [[] for _ in range(B)]
        sts = [[] for _ in range(B)]
        lp = np.zeros((B, nz))
        gsum = np.zeros((B * K, nz))
        gp = np.zeros((B * K, nz, d), np.float32)
        r = 0
        while running.any():
            n_in = _n_act_in(stale, hist, r, cap)
            cols = np.flatnonzero(running)
            rows = (cols[:, None] * K + np.arange(K)).ravel()
            lp[cols], gsum[rows], gp[rows] = prob.parts(x[cols], cols, k[cols])
            x_out = np.zeros((B, n))
            st = np.zeros(B, lr.STATE)
            slot_out = np.zeros((cap, 4), np.int32)
            counts = np.zeros(4, np.int32)
            rows_out = np.zeros(max(nrows, 1), np.float32)
            _lib.check(lib.skd_lbfgs_dev_step(h, n_in, ptr(lp), ptr(gsum), ptr(gp), ptr(x_out), ptr(st),
                                              ptr(slot_out), ptr(counts), ptr(rows_out)), eng._h)
            for c in cols:
                xs[c].append(x[c].copy())
                sts[c].append(st[c])
            k[cols] += 1
            assert (x_out[~running] == x[~running]).all()   # finished columns are not touched
            x = x_out
            running = st["status"] == lr.RUNNING
            # model of the compaction: running columns in their old order, per fold key when grouped
            kept = [s for s in slots[:hist[-1]] if s[0] >= 0 and running[s[0]]]
            if grouped:
                slots = []
                for f in range(-1, 128):
                    seg = [s for s in kept if s[1] == f]
                    slots += seg + [(-1, f, -1, 0)] * (-len(seg) % 128)
            else:
                slots = kept
            n_act = len(slots)
            assert [tuple(s) for s in slot_out[:n_act]] == slots, "slot list after round %d" % r
            n_run = int(running.sum())      # == n_act in the dense layout
            assert tuple(counts) == (n_act, n_run, n_act, n_run), (tuple(counts), n_act, n_run)
            hist.append(n_act)
            if nrows:     # exported fp32 rows of the dense layout and of the multinomial candidates
                W = rows_out[:nrows - B * K].reshape(B * K, ldw)
                bias = rows_out[nrows - B * K:]
                for s in range(n_act):
                    c = slots[s][0]
                    xk = x[c].reshape(K, d + 1).astype(np.float32)
                    for kk in range(K):
                        row = W[s * K + kk]
                        assert (row[:d] == xk[kk, :d]).all() and (row[d:] == 0).all(), "exported row %d" % s
                        assert bias[s * K + kk] == xk[kk, d]
            r += 1
        assert not (st["status"] == lr.NONFINITE).any() or prob.family.name == "non-finite"
        if prob.fmask is not None:
            masked = np.broadcast_to((prob.fmask == 0)[:, None, :], (B, K, d))
            for c in range(B):     # every iterate, not only the last
                pts = np.array(xs[c]).reshape(-1, K, d + 1)[:, :, :d]
                assert (pts[:, masked[c]] == 0).all()
            assert (x.reshape(B, K, d + 1)[:, :, :d][masked] == 0).all()
        if not prob.fit_intercept:
            assert (x.reshape(B, K, d + 1)[:, :, d] == 0).all()
        coef = np.zeros((B, n), np.float32)
        nit = np.zeros(B, np.int32)
        status = np.zeros(B, np.int32)
        loss = np.zeros(B)
        _lib.check(lib.skd_lbfgs_dev_finish(h, ptr(coef), ptr(nit), ptr(status), ptr(loss)), eng._h)
        assert (coef == x.astype(np.float32)).all()
        assert (nit == np.minimum(st["nit"], maxiter)).all()
        assert (status == st["status"]).all()
        assert (loss == st["f"]).all()
    finally:
        lib.skd_lbfgs_dev_free(h)
    for c in range(B):
        SEEN.update(lr.census(sts[c]))
    return xs, sts, x


def _tie(dev_st, host_st):
    """the device and the host core took different sides of the line search's sign test on g'd (dcsrch's stage
    switch f <= ftest and g'd >= 0) at a point where g'd is zero up to rounding: both sides are right"""
    return (dev_st["ls_stage"] != host_st["ls_stage"]
            and abs(host_st["gd"]) <= 1e-9 * abs(host_st["ginit"]) and abs(dev_st["gd"]) <= 1e-9 * abs(host_st["ginit"]))


def host_mismatches(prob, xs, sts, x_final, maxiter, maxls, pgtol, cols, m=lr.M, drop_pair=None, ints=True):
    """first disagreement of the device with the host core on every listed column ([] if none); ints=False
    compares the real values and the points only.  A column whose runs part at a rounding tie (_tie) is
    compared up to it."""
    bad = []
    for c in cols:
        ref = lr.run_core(prob, c, maxiter, maxls, pgtol, m=m, drop_pair=drop_pair)
        dx, ds = np.array(xs[c]), np.array(sts[c], lr.STATE)
        COMPARED[0] += 1
        for e in range(min(len(dx), len(ref["xs"]), N_CHECK)):
            hs = ref["states"][e]
            if ints and drop_pair is None and m == lr.M and _tie(ds[e], hs):
                TIES.append((prob.family.name, c, e))
                break
            late = e >= N_REAL
            for fld in lr.INT_FIELDS if ints and e < N_CHECK else ():
                if ds[e][fld] != hs[fld]:
                    bad.append((c, e, fld, int(ds[e][fld]), int(hs[fld])))
            for fld in lr.REAL_FIELDS:
                a, b = float(ds[e][fld]), float(hs[fld])
                dev = abs(a - b) / max(1.0, abs(b))
                if late:
                    LATE[fld] = max(LATE[fld], dev)
                if not dev <= TOL[late][fld]:
                    bad.append((c, e, fld, a, b))
            dev = np.abs(dx[e] - ref["xs"][e]).max() / (1.0 + np.abs(ref["xs"][e]).max())
            if late:
                LATE["x"] = max(LATE["x"], dev)
            if not dev <= TOL[late]["x"]:
                bad.append((c, e, "x", dev))
            if bad and bad[-1][0] == c:
                break
        else:
            if len(dx) != len(ref["xs"]):
                bad.append((c, "evaluations", len(dx), len(ref["xs"])))
                continue
            # the final point of every run, however long
            dev = np.abs(x_final[c] - ref["x"]).max() / (1.0 + np.abs(ref["x"]).max())
            LATE["final x"] = max(LATE["final x"], dev)
            if not dev <= FINAL_TOL:
                bad.append((c, "final x", dev))
    return bad


def check_run(eng, prob, maxiter=100, maxls=50, pgtol=1e-5, scipy_cols=2, host_cols=None, **kw):
    xs, sts, x = run_device(eng, prob, maxiter, maxls, pgtol, **kw)
    cols = range(prob.B) if host_cols is None else host_cols
    bad = host_mismatches(prob, xs, sts, x, maxiter, maxls, pgtol, cols)
    assert not bad, bad[:5]
    if prob.family.name != "non-finite":
        for c in list(cols)[:scipy_cols]:
            ref = lr.run_scipy(prob, c, maxiter, maxls, pgtol)
            last = sts[c][-1]
            # scipy does not call the function again at the point it has just evaluated; the driver asks again
            fresh = np.r_[True, (np.diff(np.array(xs[c]), axis=0) != 0).any(1)]
            assert fresh.sum() == len(ref["xs"])
            assert int(last["nit"]) == ref["nit"]
            assert lr.SCIPY_STATUS[int(last["status"])] == ref["status"]
            tol = 1e-8 if len(ref["xs"]) <= 40 or int(last["status"]) != lr.MAXITER else 1e-4
            if prob.family.name != "linear":     # scipy's z - x direction at |x| ~ 1e10: see the host test
                assert np.abs(x[c] - ref["x"]).max() <= tol * (1.0 + np.abs(ref["x"]).max())
    K = prob.K
    layout = "grouped" if kw.get("grouped") else "dense"
    path = "reduce" if kw.get("use_reduce") and prob.nz > 8 else "direct"
    RAN.add(("warp" if K == 1 else "cta", layout, path, kw.get("stale", "exact")))
    return xs, sts, x


@pytest.mark.parametrize("d", [1, 31, 32, 63, 255, 1000])
def test_binary_width(eng, d):
    """n = d + 1 around the warp stride of WarpPar and past the tensor-core width (dense layout)"""
    _stage(eng, d)
    for fam, nz in (("ill", 7), ("quadratic", 9), ("logistic", 1)):
        prob = lr.Problem(fam, d, 5, nz=nz, l2=1e-3 if fam == "logistic" else 0.0)
        check_run(eng, prob, maxiter=40)


def test_binary_intercept_off_mask_gscale(eng):
    d = 31
    _stage(eng, d)
    rng = np.random.default_rng(3)
    mask = (rng.random((6, d)) < 0.7).astype(np.uint8)
    gscale = 2.0 ** rng.integers(-4, 5, d).astype(float)
    for fi in (False, True):
        prob = lr.Problem("quadratic", d, 6, nz=8, fit_intercept=fi, fmask=mask, gscale=gscale)
        check_run(eng, prob, maxiter=60)


@pytest.mark.parametrize("nz,use_reduce", [(1, 0), (7, 0), (8, 0), (9, 0), (17, 0), (9, 1), (132, 1)])
def test_binary_partials(eng, nz, use_reduce):
    """the 8-wide partial loop and its tail, and lb_reduce_kernel for nz > 8: every chunk holds a share of the
    loss, intercept and gradient sums (lbfgs_reference.split), so a chunk left out or read twice shows"""
    d = 40
    _stage(eng, d)
    prob = lr.Problem("ill", d, 4, nz=nz, gscale=2.0 ** (np.arange(d) % 7 - 3.0))
    check_run(eng, prob, maxiter=30, use_reduce=bool(use_reduce))


@pytest.mark.parametrize("stale", STALE)
@pytest.mark.parametrize("B", [1, 5, 128, 129, 1024, 1025, 2500])
def test_binary_batch(eng, B, stale):
    """B around the 1024-thread compaction CTA (more than one pass from 1025 on)"""
    d = 3
    _stage(eng, d)
    prob = lr.Problem("wall", d, B, nz=2)
    check_run(eng, prob, maxiter=8, maxls=3, stale=stale, host_cols=range(0, B, max(1, B // 64)))


FOLDS = {
    "all -1": lambda: np.full(200, -1),
    "one fold": lambda: np.full(50, 3),
    "uneven": lambda: np.repeat([-1, 0, 2, 5], [7, 128, 129, 5]),
    "up to 127": lambda: np.arange(300) % 129 - 1,
}


@pytest.mark.parametrize("folds", list(FOLDS))
@pytest.mark.parametrize("use_reduce", [0, 1])
def test_grouped_layout(eng, folds, use_reduce):
    """the tensor-core fit's fold-grouped layout and lb_compact_grouped_kernel"""
    d = 24
    _stage(eng, d)
    cf = FOLDS[folds]().astype(np.int32)
    rng = np.random.default_rng(len(cf))
    cf = cf[rng.permutation(len(cf))]
    prob = lr.Problem("wall", d, len(cf), nz=12 if use_reduce else 5)
    stale = STALE[(len(cf) + use_reduce) % 4]
    check_run(eng, prob, maxiter=10, maxls=2, grouped=True, use_reduce=bool(use_reduce), col_fold=cf, stale=stale,
              host_cols=range(0, len(cf), 7))


@pytest.mark.parametrize("K,d", [(2, 63), (3, 42), (128, 16)])
def test_multinomial(eng, K, d):
    """K * (d + 1) around the 128 stride of CtaPar"""
    _stage(eng, d)
    rng = np.random.default_rng(K)
    mask = (rng.random((4, d)) < 0.8).astype(np.uint8)
    prob = lr.Problem("ill", d, 4, K=K, nz=3, fmask=mask)
    check_run(eng, prob, maxiter=25)
    prob = lr.Problem("logistic", d, 3, K=K, nz=9, l2=2e-3, inv_n=1 / 37.0, fit_intercept=K != 3)
    check_run(eng, prob, maxiter=25)


@pytest.mark.parametrize("stale", STALE)
def test_every_stale_mode(eng, stale):
    """every (policy, layout, gather path) with the host's slot count exact, one or four rounds stale, or never
    lowered"""
    d = 20
    _stage(eng, d)
    for grouped in (False, True):
        for use_reduce in (False, True):
            prob = lr.Problem("rosenbrock", d, 150, nz=10)
            check_run(eng, prob, maxiter=12, grouped=grouped, use_reduce=use_reduce, stale=stale,
                      col_fold=np.arange(150) % 3 - 1, host_cols=range(0, 150, 11))
    prob = lr.Problem("quadratic", d, 6, K=3, nz=4)
    check_run(eng, prob, maxiter=12, stale=stale)


@pytest.mark.parametrize("fam,maxls,maxiter,pgtol", [
    ("zero", 50, 100, 1e-4), ("quadratic", 50, 100, 1e-5), ("logistic", 50, 100, 1e-9), ("ill", 50, 100, 1e-9),
    ("linear", 50, 6, 1e-5), ("linear", 2, 6, 1e-5), ("wall", 1, 100, 1e-5), ("wall", 50, 100, 1e-5),
    ("nonfinite", 50, 100, 1e-9), ("rosenbrock", 3, 2, 1e-5), ("rosenbrock", 50, 1, 1e-5)])
def test_branches(eng, fam, maxls, maxiter, pgtol):
    """every exit path and every branch of the core, on the device"""
    d = 11
    _stage(eng, d)
    prob = lr.Problem(fam, d, 6, nz=3, l2=1e-3 if fam == "logistic" else 0.0)
    check_run(eng, prob, maxiter=maxiter, maxls=maxls, pgtol=pgtol)


def test_the_bound_bites(eng):
    """the comparison the device passes fails against a host core with memory 9 instead of 10, and against one
    that forgets a single (s, y) pair, on the real values and points alone as well as on the whole state"""
    d = 39
    _stage(eng, d)
    prob = lr.Problem("ill", d, 3, nz=2)
    xs, sts, x = run_device(eng, prob, 100, 50, 1e-9)
    assert not host_mismatches(prob, xs, sts, x, 100, 50, 1e-9, range(3))
    for broken in ({"m": 9}, {"drop_pair": 3}):
        assert host_mismatches(prob, xs, sts, x, 100, 50, 1e-9, range(3), **broken), broken
        bad = host_mismatches(prob, xs, sts, x, 100, 50, 1e-9, range(3), ints=False, **broken)
        assert any(isinstance(b[1], int) and b[1] < N_REAL for b in bad), (broken, bad)


def test_zz_every_variant_ran():
    want = {("warp", lay, path, s) for lay in ("dense", "grouped") for path in ("direct", "reduce") for s in STALE}
    want |= {("cta", "dense", "direct", s) for s in STALE}
    assert want <= RAN, sorted(want - RAN)
    branches = {"wrap", "skip", "restart", "abnormal", "maxiter", "ftol", "pgtol x0", "pgtol later", "nonfinite"}
    assert branches <= SEEN, sorted(branches - SEEN)
    print("largest relative deviation from the host core past evaluation %d: %s" % (N_REAL, LATE))
    print("rounding ties: %d of %d columns %s" % (len(TIES), COMPARED[0], TIES))
    assert len(TIES) <= COMPARED[0] // 50, TIES
    assert LATE["x"] > 0.0   # the runs above did go past N_REAL
