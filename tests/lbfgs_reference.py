"""float64 references for the L-BFGS-B optimiser (csrc/lbfgs_core.h, driven on the device by csrc/lbfgs_dev.cu):
problem families vectorised over columns, the splitter of a gradient into evaluation partials, and drivers for
scipy's L-BFGS-B and for the host build of the core that record every requested point and every state.

The device optimiser never sees f and g: it sees per-chunk partials (loss and intercept sums in float64, weight
gradient sums in fp32) and forms

  f = (sum_z loss_z) * inv_n + 0.5 * l2 * |w|^2,   g_k = (sum_z grad_zk) * gscale_k * inv_n + l2 * w_k

with the sums sequential in chunk order (gather_fg).  `Problem.parts` turns a family's f, g * n
into such partials -- every chunk holds a non-zero share of its value (`split`) -- and `Problem.effective` forms
the f, g the device forms from them, which is what scipy and the host core are given.  With l2 = 0, power-of-two inv_n
and gscale every device operation on them is exact (exact tier); otherwise FMA contraction and the order of
|w|^2 differ by rounding only (rounding tier).
"""
import ctypes

import numpy as np
from scipy import optimize

from skdist_b200 import _lib

EPS = np.finfo(np.float64).eps
FTOL = 64 * EPS          # what scikit-learn passes to scipy as ftol
M = 10                   # memory of every fit

# struct LbfgsScalars of csrc/lbfgs_core.h
_I, _D = np.int32, np.float64
STATE = np.dtype([("n", _I), ("m", _I), ("maxiter", _I), ("maxls", _I), ("pgtol", _D), ("ftol_abs", _D),
                  ("status", _I), ("started", _I), ("iter", _I), ("nit", _I), ("nfev", _I), ("col", _I),
                  ("head", _I), ("ifun", _I), ("iback", _I),
                  ("theta", _D), ("f", _D), ("fold", _D), ("gd", _D), ("gdold", _D), ("stp", _D), ("dnorm", _D),
                  ("dtd", _D), ("sbgnrm", _D), ("ls_brackt", _I), ("ls_stage", _I)]
                 + [(k, _D) for k in ("ginit", "gtest", "gx", "gy", "finit", "fx", "fy", "stx", "sty", "stmin",
                                      "stmax", "width", "width1")], align=True)
INT_FIELDS = ("status", "iter", "nit", "nfev", "col", "head", "ifun", "iback", "ls_brackt", "ls_stage")
REAL_FIELDS = ("f", "stp", "theta")

RUNNING, PGTOL, FTOL_CONV, MAXITER, ABNORMAL, NONFINITE = range(6)
SCIPY_STATUS = {PGTOL: 0, FTOL_CONV: 0, MAXITER: 1, ABNORMAL: 2}


# ---- problem families: f and g at the points x [cols, n] of the listed columns ---------------------------------
class Family:
    """f, g of every column at its point; k[cols] is the column's evaluation index (0 at x0)."""
    name = "?"

    def __init__(self, n, B, seed=0):
        self.n, self.B = n, B
        self.rng = np.random.default_rng(seed)

    def fg(self, X, cols, k):
        raise NotImplementedError


class Logistic(Family):
    """mean logistic loss of a fixed 48-row problem, labels and rows per column; bounded, smooth, ends in FTOL/PGTOL."""
    name = "logistic"

    def __init__(self, n, B, seed=0):
        super().__init__(n, B, seed)
        self.A = self.rng.standard_normal((48, n)) / np.sqrt(n)
        self.y = np.where(self.rng.random((B, 48)) < 0.5, -1.0, 1.0)

    def fg(self, X, cols, k):
        z = X @ self.A.T * self.y[cols]                           # [c, 48]
        f = np.logaddexp(0.0, -z).mean(1)
        r = -self.y[cols] / (1.0 + np.exp(z)) / 48.0
        return f, r @ self.A


class Quadratic(Family):
    """0.5 sum a_i (x_i - c_i)^2, a_i log-spaced up to `cond` (a random permutation per column)."""
    def __init__(self, n, B, seed=0, cond=10.0):
        super().__init__(n, B, seed)
        self.name = "quadratic(%g)" % cond
        a = np.logspace(0.0, np.log10(cond), n)
        self.a = np.stack([self.rng.permutation(a) for _ in range(min(B, 64))])
        self.c = self.rng.uniform(-1.0, 1.0, (min(B, 64), n))

    def fg(self, X, cols, k):
        a, c = self.a[cols % len(self.a)], self.c[cols % len(self.c)]
        r = X - c
        return 0.5 * (a * r * r).sum(1), a * r


class Rosenbrock(Family):
    """chained Rosenbrock from x0 = 0, scaled per column."""
    name = "rosenbrock"

    def __init__(self, n, B, seed=0):
        super().__init__(n, B, seed)
        self.s = self.rng.uniform(0.5, 2.0, B)

    def fg(self, X, cols, k):
        s = self.s[cols][:, None]
        a, b = X[:, :-1], X[:, 1:]
        t1, t2 = b - a * a, 1.0 - a
        f = (100.0 * t1 * t1 + t2 * t2).sum(1) * s[:, 0]
        g = np.zeros_like(X)
        g[:, :-1] += -400.0 * a * t1 - 2.0 * t2
        g[:, 1:] += 200.0 * t1
        return f, g * s


class ZeroGradient(Family):
    """constant f, g = 0 everywhere: PGTOL at x0 with nit = 0."""
    name = "zero gradient"

    def fg(self, X, cols, k):
        return np.full(len(cols), 3.0), np.zeros_like(X)


class NonFinite(Quadratic):
    """a quadratic whose f is inf or NaN at evaluation k_bad of the column (2 .. 6)."""
    def __init__(self, n, B, seed=0):
        super().__init__(n, B, seed, cond=100.0)
        self.name = "non-finite"
        self.k_bad = 2 + np.arange(B) % 5

    def fg(self, X, cols, k):
        f, g = super().fg(X, cols, k)
        bad = k >= self.k_bad[cols]
        f = np.where(bad, np.where(cols % 2 == 0, np.inf, np.nan), f)
        return f, g


class Linear(Family):
    """f = c.x with the constant gradient c: every line search extrapolates to stpmax (or runs out of maxls), and
    every pair has s'y = 0, so it is skipped; with a small maxls the first line search fails with no memory."""
    name = "linear"

    def __init__(self, n, B, seed=0):
        super().__init__(n, B, seed)
        self.c = self.rng.uniform(0.5, 1.5, (B, n)) * np.where(self.rng.random((B, n)) < 0.5, -1.0, 1.0)

    def fg(self, X, cols, k):
        c = self.c[cols]
        return (X * c).sum(1), c.copy()


class Wall(Quadratic):
    """a quadratic until evaluation k_wall of the column, then f reported above everything seen before with the
    true gradient: the line search under way runs out of maxls, the memory is dropped and the restart from
    steepest descent runs out too -> ABNORMAL."""
    def __init__(self, n, B, seed=0):
        super().__init__(n, B, seed, cond=30.0)
        self.name = "wall"
        self.k_wall = 5 + np.arange(B) % 4

    def fg(self, X, cols, k):
        f, g = super().fg(X, cols, k)
        a, c = self.a[cols % len(self.a)], self.c[cols % len(self.c)]
        top = 0.5 * (a * c * c).sum(1) + 1.0                        # f(x0) + 1
        return np.where(k >= self.k_wall[cols], top, f), g


FAMILIES = {"logistic": Logistic, "quadratic": lambda n, B, seed=0: Quadratic(n, B, seed, 10.0),
            "ill": lambda n, B, seed=0: Quadratic(n, B, seed, 1e4), "rosenbrock": Rosenbrock,
            "zero": ZeroGradient, "nonfinite": NonFinite, "linear": Linear, "wall": Wall}


# ---- the evaluation partials of a column and what the device makes of them -----------------------------------
def split(v, nz, dtype):
    """v into nz parts, none of them zero unless v is.  Parts 2 .. nz-1 (or 0 .. nz-2 in float64) take shares
    w_z / (w_z + ... + w_last + w_rest) of what is left to place, rounded to dtype, with w_z = 1 + (3 z mod 5), so that
    neighbouring parts differ by up to 5x and a lost, repeated or misplaced chunk changes the sum by a share of v,
    not by a rounding.  What is left goes to the last float64 part, or to fp32 parts 0 and 1 as hi = fp32(r),
    lo = fp32(r - hi): the chunk sum then stays within ~2^-48 |v| of v, a smooth function of the point, as the
    sums of a real evaluation are."""
    w = 1.0 + (3 * np.arange(nz)) % 5
    fp32 = np.dtype(dtype) == np.float32
    share = list(range(2, nz)) if fp32 else list(range(nz - 1))
    p = np.zeros(v.shape + (nz,), dtype)
    r = np.asarray(v, np.float64).copy()
    left = w[share].sum() + (w[0] if fp32 else w[nz - 1])      # the remainder's own share stays in r
    with np.errstate(invalid="ignore"):     # a non-finite f splits into non-finite parts
        for z in share:
            p[..., z] = (r * (w[z] / left)).astype(dtype)
            r = r - p[..., z].astype(np.float64)
            left -= w[z]
    if not fp32:
        p[..., nz - 1] = r
    else:
        p[..., 0] = r.astype(dtype)
        if nz > 1:
            p[..., 1] = (r - p[..., 0].astype(np.float64)).astype(dtype)
    return p


def chunk_sum(p):
    """sequential float64 sum over the last axis (chunk order), as gather_fg adds the partials."""
    acc = np.zeros(p.shape[:-1])
    for z in range(p.shape[-1]):
        acc = acc + p[..., z].astype(np.float64)
    return acc


class Problem:
    """B columns of K * (d + 1) variables (variable (k, j) at k * (d + 1) + j, j == d the intercept)."""

    def __init__(self, family, d, B, K=1, nz=1, fit_intercept=True, l2=None, inv_n=None, gscale=None, fmask=None,
                 seed=0):
        self.d, self.B, self.K, self.nz, self.fit_intercept = d, B, K, nz, bool(fit_intercept)
        self.dp = d + 1
        self.n = K * self.dp
        self.family = FAMILIES[family](self.n, B, seed) if isinstance(family, str) else family
        self.l2 = np.zeros(B) if l2 is None else np.broadcast_to(np.asarray(l2, float), (B,)).copy()
        self.inv_n = (np.full(B, 2.0 ** -6) if inv_n is None
                      else np.broadcast_to(np.asarray(inv_n, float), (B,)).copy())
        self.gscale = None if gscale is None else np.asarray(gscale, float)
        self.fmask = None if fmask is None else np.asarray(fmask, np.uint8)

    def parts(self, X, cols, k):
        """loss_parts [c, nz], gsum_parts [c * K, nz], grad_parts [c * K, nz, d] (fp32) at the points X [c, n]."""
        f, g = self.family.fg(X, cols, k)
        inv = self.inv_n[cols][:, None]
        G = (g / inv).reshape(len(cols), self.K, self.dp)
        gw = G[:, :, :self.d]
        if self.gscale is not None:
            gw = gw / self.gscale
        lp = split(f / self.inv_n[cols], self.nz, np.float64)
        gs = split(G[:, :, self.d].reshape(-1), self.nz, np.float64)
        gp = split(gw.reshape(-1, self.d), self.nz, np.float32).transpose(0, 2, 1).copy()
        return lp, gs, gp

    def effective(self, X, cols, lp, gs, gp):
        """f [c], g [c, n] that gather_fg forms from the partials."""
        c = len(cols)
        inv, l2 = self.inv_n[cols], self.l2[cols]
        acc = chunk_sum(gp.transpose(0, 2, 1)).reshape(c, self.K, self.d)
        if self.gscale is not None:
            acc = acc * self.gscale
        W = X.reshape(c, self.K, self.dp)
        g = np.empty((c, self.K, self.dp))
        g[:, :, :self.d] = acc * inv[:, None, None] + l2[:, None, None] * W[:, :, :self.d]
        if self.fmask is not None:
            g[:, :, :self.d] = np.where(self.fmask[cols][:, None, :] != 0, g[:, :, :self.d], 0.0)
        g[:, :, self.d] = chunk_sum(gs).reshape(c, self.K) * inv[:, None] if self.fit_intercept else 0.0
        wsq = (W[:, :, :self.d] ** 2).sum((1, 2))
        f = chunk_sum(lp) * inv + 0.5 * l2 * wsq
        return f, g.reshape(c, self.n)

    def fg(self, X, cols, k):
        X = np.atleast_2d(X)
        return self.effective(X, cols, *self.parts(X, cols, k))


# ---- drivers ---------------------------------------------------------------------------------------------
def run_scipy(prob, col, maxiter, maxls, pgtol, ftol=FTOL):
    """scipy's L-BFGS-B on column col from x0 = 0: every requested point, nit, nfev, status, x."""
    xs = []

    def fun(x):
        f, g = prob.fg(x[None, :], np.array([col]), np.array([len(xs)]))
        xs.append(x.copy())
        return f[0], g[0]

    res = optimize.minimize(fun, np.zeros(prob.n), jac=True, method="L-BFGS-B",
                            options={"maxiter": maxiter, "maxls": maxls, "gtol": pgtol, "ftol": ftol})
    return {"xs": np.array(xs), "nit": res.nit, "nfev": res.nfev, "status": res.status, "x": res.x}


class HostCore:
    """The host build of csrc/lbfgs_core.h on one column (skd_lbfgs_*)."""

    def __init__(self, n, maxiter, maxls, pgtol, ftol=FTOL, m=M):
        lib = _lib.load()
        assert lib.skd_lbfgs_state_bytes() == STATE.itemsize
        self.lib, self.n = lib, n
        self.h = lib.skd_lbfgs_create(n, m, maxiter, maxls, pgtol, ftol)
        self.x = np.ctypeslib.as_array(lib.skd_lbfgs_x(self.h), (n,))
        self.g = np.ctypeslib.as_array(lib.skd_lbfgs_g(self.h), (n,))

    def advance(self, f, g):
        self.g[:] = g
        self.lib.skd_lbfgs_advance(self.h, float(f))
        return self.state()

    def state(self):
        s = np.zeros(1, STATE)
        self.lib.skd_lbfgs_state(self.h, s.ctypes.data_as(ctypes.c_void_p))
        return s[0]

    def set_state(self, st):
        s = np.array([st], STATE)
        self.lib.skd_lbfgs_set_state(self.h, s.ctypes.data_as(ctypes.c_void_p))

    def close(self):
        if self.h:
            self.lib.skd_lbfgs_free(self.h)
            self.h = None

    def __del__(self):
        self.close()


def run_core(prob, col, maxiter, maxls, pgtol, ftol=FTOL, m=M, max_evals=100000, drop_pair=None):
    """The host core on column col: every requested point, the state after every evaluation, x.  drop_pair = j:
    a broken core that forgets the j-th stored (s, y) pair (1-based) right after storing it."""
    core = HostCore(prob.n, maxiter, maxls, pgtol, ftol, m)
    xs, states = [], []
    stored = 0
    while len(xs) < max_evals:
        x = core.x.copy()
        f, g = prob.fg(x[None, :], np.array([col]), np.array([len(xs)]))
        xs.append(x)
        before = core.state()
        st = core.advance(f[0], g[0])
        if st["iter"] > before["iter"] and st["col"] > before["col"]:
            stored += 1
            if stored == drop_pair:
                st = st.copy()
                st["col"] -= 1
                core.set_state(st)
        states.append(st)
        if st["status"] != RUNNING:
            break
    out = {"xs": np.array(xs), "states": np.array(states, STATE), "x": core.x.copy()}
    last = out["states"][-1]
    out.update(nit=int(last["nit"]), nfev=int(last["nfev"]), status=int(last["status"]))
    core.close()
    return out


def census(states):
    """Branches of the core that a sequence of per-evaluation states went through."""
    seen = set()
    s = np.asarray(states, STATE)
    if (s["head"] > 0).any():
        seen.add("wrap")
    for a, b in zip(s[:-1], s[1:]):
        if b["iter"] > a["iter"] and b["col"] == a["col"] and a["col"] < a["m"] and b["status"] == RUNNING:
            seen.add("skip")
        if a["col"] > 0 and b["col"] == 0:
            seen.add("restart")
    last = s[-1]
    st = int(last["status"])
    seen.add({PGTOL: "pgtol later" if last["nit"] > 0 else "pgtol x0", FTOL_CONV: "ftol", MAXITER: "maxiter",
              ABNORMAL: "abnormal", NONFINITE: "nonfinite"}.get(st, "running"))
    return seen
