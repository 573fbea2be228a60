"""The host build of the L-BFGS-B core (csrc/lbfgs_core.h) against scipy's L-BFGS-B, evaluation by evaluation, on
every problem family of tests/lbfgs_reference.py -- smooth, ill-conditioned, gradient zero at x0, non-finite and
adversarial oracles that exhaust maxls, drop the memory, skip the pair update and end ABNORMAL -- at maxls 1, 2, 3
and 50 and maxiter 1, 2 and 100.  scipy and the core are given the same f, g: what the device forms from the
evaluation partials (lbfgs_reference.Problem.effective)."""
import numpy as np
import pytest

from tests import lbfgs_reference as lr

FAMILY_SHAPES = [("logistic", 12), ("quadratic", 20), ("ill", 40), ("rosenbrock", 12), ("zero", 6),
                 ("linear", 8), ("wall", 10)]
SEEN = set()


def _problem(family, n, col_count=3, **kw):
    kw.setdefault("l2", 1e-3 if family == "logistic" else 0.0)
    return lr.Problem(family, n - 1, col_count, nz=2, **kw)


def _compare(prob, col, maxiter, maxls, pgtol):
    ref = lr.run_scipy(prob, col, maxiter, maxls, pgtol)
    got = lr.run_core(prob, col, maxiter, maxls, pgtol)
    SEEN.update(lr.census(got["states"]))
    # scipy does not call the function again at the point it has just evaluated (a line search that has shrunk
    # its step to 0 requests the start point twice); the core counts every request
    xs = got["xs"]
    fresh = np.r_[True, (xs[1:] != xs[:-1]).any(1)]
    assert len(xs[fresh]) == len(ref["xs"]), (len(xs[fresh]), len(ref["xs"]))
    assert got["nfev"] == len(xs)
    assert fresh.sum() == ref["nfev"] == len(ref["xs"])
    assert got["nit"] == ref["nit"]
    assert lr.SCIPY_STATUS[got["status"]] == ref["status"], (got["status"], ref["status"])
    # scipy forms the direction as z - x: on the linear family x reaches 1e10 and that difference loses ~1e-6,
    # which later steps of up to 1e10 carry into the iterates; compare its first line search only
    upto = (got["states"]["iter"][fresh] == 0).sum() if prob.family.name == "linear" else len(ref["xs"])
    if len(ref["xs"]) <= 40:
        scale = 1.0 + np.abs(ref["xs"][:upto]).max()
        dev = np.abs(xs[fresh][:upto] - ref["xs"][:upto]).max() / scale
        assert dev <= 1e-9, dev
    # the two-loop recursion and scipy's compact representation round differently; on a long run that stops
    # unconverged (MAXITER on the ill-conditioned quadratic) the gap grows past 1e-8 by the last iterate
    tol = 1e-8 if len(ref["xs"]) <= 40 or got["status"] != lr.MAXITER else 1e-4
    if prob.family.name != "linear":
        assert np.abs(got["x"] - ref["x"]).max() <= tol * (1.0 + np.abs(ref["x"]).max())
    return got


@pytest.mark.parametrize("maxiter", [1, 2, 100])
@pytest.mark.parametrize("maxls", [1, 2, 3, 50])
@pytest.mark.parametrize("family,n", FAMILY_SHAPES)
def test_core_matches_scipy(family, n, maxls, maxiter):
    prob = _problem(family, n)
    pgtol = 1e-5 if family != "zero" else 1e-4
    for col in range(prob.B):
        _compare(prob, col, maxiter, maxls, pgtol)


@pytest.mark.parametrize("inv_n", [2.0 ** -3, 1.0 / 37.0])
def test_core_matches_scipy_rounding_tier(inv_n):
    """general l2 and inv_n on the smooth families: the effective f, g carry rounding, scipy and the core see the
    same values all the same"""
    for family, n in (("logistic", 9), ("quadratic", 17), ("rosenbrock", 6)):
        prob = _problem(family, n, l2=0.0137, inv_n=inv_n)
        for col in range(prob.B):
            _compare(prob, col, 100, 50, 1e-6)


def test_core_masked_and_intercept_off():
    """masked features and fit_intercept off: effective gradient 0 there, those variables stay exactly 0"""
    d = 11
    mask = np.ones((3, d), np.uint8)
    mask[:, [1, 4, 7]] = 0
    for fi in (True, False):
        prob = lr.Problem("quadratic", d, 3, nz=3, fit_intercept=fi, fmask=mask, gscale=2.0 ** np.arange(-3, d - 3))
        for col in range(3):
            got = _compare(prob, col, 100, 50, 1e-6)
            assert (got["xs"][:, [1, 4, 7]] == 0).all()
            if not fi:
                assert (got["xs"][:, d] == 0).all()


def test_core_nonfinite_stops_at_once():
    """f = inf or NaN: status 5 at that evaluation, nothing further requested"""
    prob = _problem("nonfinite", 15, col_count=6)
    for col in range(prob.B):
        got = lr.run_core(prob, col, 100, 50, 1e-8)
        SEEN.update(lr.census(got["states"]))
        assert got["status"] == lr.NONFINITE
        assert len(got["xs"]) == prob.family.k_bad[col] + 1
        assert got["nfev"] == len(got["xs"])


def test_nfev_counts_requested_evaluations_only():
    """a line search that runs out of maxls requests no further point: nfev is the number of evaluations"""
    for family, n in (("rosenbrock", 12), ("ill", 40), ("wall", 10), ("linear", 8)):
        prob = _problem(family, n)
        for maxls in (1, 2, 3):
            got = lr.run_core(prob, 0, 100, maxls, 1e-5)
            assert got["nfev"] == len(got["xs"]), (family, maxls, got["nfev"], len(got["xs"]))


def test_state_layout_matches_the_core():
    from skdist_b200 import _lib
    assert _lib.load().skd_lbfgs_state_bytes() == lr.STATE.itemsize
    core = lr.HostCore(7, 13, 5, 1e-3)
    s = core.state()
    assert (s["n"], s["m"], s["maxiter"], s["maxls"]) == (7, lr.M, 13, 5)
    assert (s["pgtol"], s["ftol_abs"], s["status"], s["ls_stage"]) == (1e-3, lr.FTOL, 0, 1)
    assert s["theta"] == 1.0
    core.close()


def test_zz_every_branch_ran():
    """the runs above went through every branch of the core"""
    want = {"wrap", "skip", "restart", "abnormal", "maxiter", "ftol", "pgtol x0", "pgtol later", "nonfinite"}
    assert want <= SEEN, sorted(want - SEEN)
