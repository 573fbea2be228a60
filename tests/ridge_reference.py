"""Float64 statistics of batched Ridge fits, the normwise backward error of a computed solution, and a numpy
restatement of csrc/ridge.cu's arithmetic.  TEST INFRASTRUCTURE ONLY (tests/test_ridge_gpu.py,
tests/test_ridge_accumulation_host.py).

Backward error of w for  (A + alpha I) w = b  (Rigal-Gaches, infinity norm):

    eta = |(A + alpha I) w - b|_inf / (|A + alpha I|_inf |w|_inf + |b|_inf)

It is the smallest relative perturbation of A + alpha I and b for which w is exact, so it does not grow
with the condition number: an fp32 normal-equations solve (fp32 statistics, fp32 Cholesky) reaches a few
1e-8 on every problem, while a lost Gram tile or a cancelled target sum shows at 1e-5 and above.
"""
import numpy as np

CHUNK = 2048      # rows per fp32 partial sum (ridge.cu GR_CHUNK)
BLOCK = 16        # rows per fp32 block sum inside a chunk (ridge.cu GR_K)
ETA_BOUND = 1e-6
F32 = np.float32


class RidgeRef:
    """Training statistics of every "hold out fold h" fit from per-fold float64 block sums of the float32
    inputs.  The block sums are taken on data shifted by the float64 global means (an exact change of
    variables) so that the centring below cancels nothing; h = -1 holds out nothing."""

    def __init__(self, X, y, fold, n_folds, fit_intercept=True):
        X64, y64 = X.astype(np.float64), y.astype(np.float64)
        self.fit_intercept = fit_intercept
        self.gx = X64.mean(0) if fit_intercept else np.zeros(X.shape[1])
        self.gy = y64.mean() if fit_intercept else 0.0
        Xs, ys = X64 - self.gx, y64 - self.gy
        if fold is None:
            fold, n_folds = np.zeros(len(y), np.int64), 1
        self.fold = np.asarray(fold)
        self.n_folds = n_folds
        self.S, self.v, self.s, self.sy, self.cnt = [], [], [], [], []
        for f in range(n_folds):
            m = self.fold == f
            Xf, yf = Xs[m], ys[m]
            self.S.append(Xf.T @ Xf)
            self.v.append(Xf.T @ yf)
            self.s.append(Xf.sum(0))
            self.sy.append(yf.sum())
            self.cnt.append(m.sum())
        self._cache = {}

    def stats(self, h):
        """(A_h, b_h, xbar_h, ybar_h) in float64."""
        h = int(h)
        if h not in self._cache:
            keep = [f for f in range(self.n_folds) if f != h]
            A = sum(self.S[f] for f in keep)
            b = sum(self.v[f] for f in keep)
            ntr = sum(self.cnt[f] for f in keep)
            if self.fit_intercept and ntr > 0:
                s = sum(self.s[f] for f in keep)
                sy = sum(self.sy[f] for f in keep)
                A = A - np.outer(s, s) / ntr
                b = b - s * (sy / ntr)
                xbar, ybar = self.gx + s / ntr, self.gy + sy / ntr
            else:
                xbar, ybar = np.zeros(len(b)), 0.0
            self._cache[h] = (A, b, xbar, ybar)
        return self._cache[h]

    def solve(self, h, alphas):
        """w64[k] = (A_h + alphas[k] I)^-1 b_h from one eigendecomposition of A_h, and the intercepts."""
        A, b, xbar, ybar = self.stats(h)
        lam, Q = np.linalg.eigh(A)
        qb = Q.T @ b
        W = (qb[None, :] / (lam[None, :] + np.asarray(alphas, np.float64)[:, None])) @ Q.T
        return W, (ybar - W @ xbar) if self.fit_intercept else np.zeros(len(W))


def eta(A, b, alphas, W):
    """Normwise backward error of each row of W (one per alpha) for (A + alpha I) w = b."""
    W = np.atleast_2d(np.asarray(W, np.float64))
    alphas = np.asarray(alphas, np.float64).reshape(-1)
    R = W @ A + alphas[:, None] * W - b[None, :]
    diag = np.diag(A)
    rows = np.abs(A).sum(1)[None, :] - np.abs(diag)[None, :] + np.abs(diag[None, :] + alphas[:, None])
    normA = rows.max(1)
    return np.abs(R).max(1) / (normA * np.abs(W).max(1) + np.abs(b).max())


def _fma32(a, b, c):
    """fl32(a * b + c): the product of two float32 values is exact in float64, one rounding to float32
    (up to the rare double rounding through float64)."""
    return (a.astype(np.float64) * b + c).astype(F32)


def emulate_statistics(X, y, fold, n_folds, h, fit_intercept=True, shift_y=True, block=BLOCK):
    """The fp32 A_h, b_h, xbar_h and float64 ybar_h that ridge.cu hands its solve kernel.

    Global shift mu = fl32(mean x) (and yg = fl32(mean y) if shift_y); per chunk of <= 2048 rows of one
    fold: x - mu and y - yg in fp32; fp32 sums of the products and of x - mu, sequential inside each block of
    `block` rows and then over the block sums; float64 sums of y - yg; float64 across chunks and folds;
    centring in float64; A_h, b_h rounded to fp32."""
    n, d = X.shape
    if fold is None:
        fold, n_folds = np.zeros(n, np.int64), 1
    fold = np.asarray(fold)
    mu = X.astype(np.float64).mean(0).astype(F32) if fit_intercept else np.zeros(d, F32)
    yg = F32(y.astype(np.float64).mean()) if fit_intercept and shift_y else F32(0)
    S = np.zeros((n_folds, d, d))
    v = np.zeros((n_folds, d))
    s = np.zeros((n_folds, d))
    sy = np.zeros(n_folds)
    cnt = np.zeros(n_folds)
    for f in range(n_folds):
        rows = np.flatnonzero(fold == f)
        cnt[f] = len(rows)
        for c0 in range(0, len(rows), CHUNK):
            r = rows[c0:c0 + CHUNK]
            xc = (X[r] - mu).astype(F32)
            yc = (y[r] - yg).astype(F32)
            G = np.zeros((d, d), F32)
            av = np.zeros(d, F32)
            as_ = np.zeros(d, F32)
            for i0 in range(0, len(r), block):
                gb = np.zeros((d, d), F32)
                vb = np.zeros(d, F32)
                sb = np.zeros(d, F32)
                for i in range(i0, min(i0 + block, len(r))):
                    gb = _fma32(xc[i][:, None], xc[i][None, :], gb)
                    vb = _fma32(xc[i], yc[i], vb)
                    sb = (sb + xc[i]).astype(F32)
                G = (G + gb).astype(F32)
                av = (av + vb).astype(F32)
                as_ = (as_ + sb).astype(F32)
            S[f] += G
            v[f] += av
            s[f] += as_
            sy[f] += yc.astype(np.float64).sum()
    keep = [f for f in range(n_folds) if f != h]
    ntr = cnt[keep].sum()
    A, b = S[keep].sum(0), v[keep].sum(0)
    sr, syt = s[keep].sum(0), sy[keep].sum()
    if fit_intercept and ntr > 0:
        ybar = syt / ntr
        A = A - np.outer(sr, sr) / ntr
        b = b - sr * ybar
        xbar = (mu.astype(np.float64) + sr / ntr).astype(F32)
        ybar += float(yg)
    else:
        xbar, ybar = np.zeros(d, F32), 0.0
    return A.astype(F32), b.astype(F32), xbar, ybar


def cholesky_solve32(A32, b32, alpha):
    """ridge_solve_kernel: right-looking fp32 Cholesky of A + alpha I (lower triangle), then L z = b and
    L^T w = z; returns (w, ok) with ok False when a pivot is not positive."""
    d = len(b32)
    L = A32.astype(F32).copy()
    L[np.diag_indices(d)] = (L[np.diag_indices(d)] + F32(alpha)).astype(F32)
    ok = True
    for j in range(d):
        p = L[j, j]
        if not p > 0:
            ok, p = False, F32(1)
        L[j, j] = np.sqrt(p, dtype=F32)
        L[j + 1:, j] = (L[j + 1:, j] * (F32(1) / L[j, j])).astype(F32)
        col = L[j + 1:, j]
        L[j + 1:, j + 1:] = _fma32(-col[:, None], col[None, :], L[j + 1:, j + 1:])
    w = b32.astype(F32).copy()
    for j in range(d):
        w[j] = w[j] / L[j, j]
        w[j + 1:] = _fma32(-L[j + 1:, j], w[j], w[j + 1:])
    for j in range(d - 1, -1, -1):
        w[j] = w[j] / L[j, j]
        w[:j] = _fma32(-L[j, :j], w[j], w[:j])
    return w, ok
