"""float64 reference of the multinomial evaluation (csrc/logreg_multi.cu, gather_fg in csrc/lbfgs_dev.cu) and the
first-order error bound of its fp32 arithmetic, shared by the GPU tests and their host rehearsal.

With u = 2^-24 (one fp32 rounding), per training row i and class k of a candidate:

  forward     |dz_ik| <= u (sum_j |s_ijk| + |z_ik|)                     fp32 FMA over j = 0 .. d-1 in order, then
                         <= (d + 2) u (sum_j |x_ij w_kj| + |b_k|)       + b; s_ijk = sum_{l <= j} x_il w_kl exact
  pointwise   |dg_ik| <= p_ik (2 max_k' |dz_ik'| + 4 u) + u |g_ik|     softmax of perturbed z; exp, sum and quotient
                         (+ u |g_ik| with class weights)                rounded to fp32; p - [y = k]; times the weight
  backward    (rpc + 1) u sum_i |g_ik x_ij|                              fp32 FMA accumulation inside a row chunk

The per-chunk partials are added in float64, so the bound of a gradient component is the sum of these over the
training rows, divided by n_train (the sum of the weights when class weights are staged).  The loss of a row is
log(sum) + max - z_y in fp32: |dl_i| <= 2 max_k |dz_ik| + 3 u + u (|log(sum) + max| + 2 |l_i|).
"""
import numpy as np
from scipy.special import logsumexp, softmax

U = 2.0 ** -24
TINY = 2.0 ** -148     # fp32 exp results in the subnormal range carry an absolute, not relative, error
PASS_BUDGET = 6.0e9    # bytes of raw predictions and gradient partials per pass (candidates_per_pass)


def multi_chunks(n):
    """(chunks, rows per chunk) of logreg_multi.cu multi_chunks: at most 64 chunks, a multiple of 64 rows each."""
    want = max(1, min(64, (n + 63) // 64))
    r = (n + want - 1) // want
    r = (r + 63) // 64 * 64
    return (n + r - 1) // r, r


def candidates_per_pass(n, d, K, nz):
    ldx = (d + 15) // 16 * 16
    return max(1, int(PASS_BUDGET // (4.0 * K * (n + nz * ldx))))


def row_mask(n, fold, cf):
    """[n, B] training rows of every candidate (no folds staged, or col_fold < 0: every row)."""
    if fold is None:
        return np.ones((n, len(cf)), bool)
    return (fold[:, None] != cf[None, :]) | (cf[None, :] < 0)


def loss_grad(X, y, M, W, C, cw=None, fmask=None, fit_intercept=True, bounds=True, rpc=None):
    """float64 objective [B] and gradient [B, K, d + 1] of every candidate at the points W [B, K, d + 1].

    y: class ids [n]; M: [n, B] training rows; cw: [B, K] class weights or None (then n_train = rows);
    fmask: [B, d] feature masks or None.  The weights enter the products rounded to fp32, as scikit-learn casts
    them; the penalty is float64.  With bounds, also the error bound of every component ("bf", "bg") and the
    pieces needed to move the reference by one row ("G", "s").  rpc: rows per chunk (default multi_chunks)."""
    n, d = X.shape
    B, K = W.shape[0], W.shape[1]
    if rpc is None:
        rpc = multi_chunks(n)[1]
    X64 = X.astype(np.float64)
    Xa = np.abs(X64)
    W32 = W.astype(np.float32).astype(np.float64)
    onehot = np.zeros((n, K))
    onehot[np.arange(n), y] = 1.0
    out = dict(f=np.empty(B), g=np.zeros((B, K, d + 1)), pen=np.zeros((B, K, d + 1)), ntr=np.empty(B))
    if bounds:
        out.update(bf=np.empty(B), bg=np.zeros((B, K, d + 1)), G=[], s=[])
    for b in range(B):
        Wb = W32[b, :, :d]
        bias = W32[b, :, d] if fit_intercept else np.zeros(K)
        Z = X64 @ Wb.T + bias
        lse = logsumexp(Z, axis=1)
        P = softmax(Z, axis=1)
        G = P - onehot
        L = lse - Z[np.arange(n), y]
        s = M[:, b].astype(np.float64)
        if cw is not None:
            s = s * cw[b, y].astype(np.float64)
        ntr = s.sum()
        l2 = 1.0 / (C[b] * ntr)
        Gs = G * s[:, None]
        out["ntr"][b] = ntr
        out["f"][b] = (L * s).sum() / ntr + 0.5 * l2 * (W[b, :, :d] ** 2).sum()
        g = out["g"][b]
        g[:, :d] = (X64.T @ Gs).T / ntr + l2 * W[b, :, :d]
        g[:, d] = Gs.sum(0) / ntr if fit_intercept else 0.0
        out["pen"][b, :, :d] = l2 * W[b, :, :d]
        if fmask is not None:
            g[:, :d][:, fmask[b] == 0] = 0.0
            out["pen"][b, :, :d][:, fmask[b] == 0] = 0.0
        if not bounds:
            continue
        dz = U * (partial_sum_abs(X64, Wb) + np.abs(Z))
        dmax = dz.max(1)
        wu = 2.0 if cw is not None else 1.0
        eg = (P * (2.0 * dmax[:, None] + 4.0 * U) + wu * U * np.abs(G) + TINY) * s[:, None]
        sa = np.abs(s)
        bg = out["bg"][b]
        bg[:, :d] = ((Xa.T @ eg).T + (rpc + 1) * U * (Xa.T @ np.abs(Gs)).T) / ntr
        bg[:, d] = eg.sum(0) / ntr if fit_intercept else 0.0
        bg += 4.0 * 2.0 ** -53 * (np.abs(g) + np.abs(out["pen"][b]))     # float64 sums and products
        if fmask is not None:
            bg[:, :d][:, fmask[b] == 0] = 0.0
        el = 2.0 * dmax + 3.0 * U + U * (np.abs(lse) + (1.0 + wu) * np.abs(L))
        out["bf"][b] = (el * sa).sum() / ntr + 4.0 * 2.0 ** -53 * abs(out["f"][b])
        out["G"].append(G)
        out["s"].append(s)
    if bounds:
        out["fmask"] = fmask
    return out


def partial_sum_abs(X64, Wk, block=64):
    """[n, K] sum over j of |sum_{l <= j} x_il w_kl|: the magnitudes the FMA chain of fwd_kernel rounds."""
    n = X64.shape[0]
    out = np.empty((n, Wk.shape[0]))
    for r0 in range(0, n, block):
        prod = X64[r0:r0 + block, :, None] * Wk.T[None, :, :]          # [rows, d, K]
        out[r0:r0 + block] = np.abs(np.cumsum(prod, axis=1)).sum(1)
    return out


def ratio(err, bound):
    """error / bound; a zero bound allows no error."""
    return np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0), where=bound > 0)


def check_float(X, ref, f, g, label, fit_intercept=True):
    """Every component of (f, g) inside its bound; the largest ratio is printed.  The bound must also see one
    training row: a reference without one row of median |g| moves some component of every candidate past it."""
    assert np.all(np.isfinite(f)) and np.all(np.isfinite(g)), label
    rf = ratio(np.abs(f - ref["f"]), ref["bf"])
    rg = ratio(np.abs(g - ref["g"]), ref["bg"])
    print("%s: max error / bound  loss %.3f  gradient %.3f" % (label, rf.max(), rg.max()))
    b, k, j = np.unravel_index(np.argmax(rg), rg.shape)
    assert rg.max() <= 1.0, (label, "gradient", b, k, j, g[b, k, j], ref["g"][b, k, j], ref["bg"][b, k, j])
    assert rf.max() <= 1.0, (label, "loss", np.argmax(rf), rf.max())
    assert_bound_sees_one_row(X, ref, label, fit_intercept)
    return rf.max(), rg.max()


def assert_bound_sees_one_row(X, ref, label, fit_intercept=True):
    for b in range(ref["g"].shape[0]):
        s, G = ref["s"][b], ref["G"][b]
        rows = np.flatnonzero(s)
        mag = np.abs(G[rows]).sum(1)
        i = rows[np.argsort(mag)[len(rows) // 2]]
        ntr = ref["ntr"][b]
        data = ref["g"][b] - ref["pen"][b]
        xi = np.append(X[i].astype(np.float64), 1.0 if fit_intercept else 0.0)
        contrib = s[i] * np.outer(G[i], xi)
        if ref["fmask"] is not None:
            contrib[:, :-1][:, ref["fmask"][b] == 0] = 0.0
        moved = (data * ntr - contrib) / (ntr - s[i]) + ref["pen"][b]
        assert np.any(np.abs(moved - ref["g"][b]) > ref["bg"][b]), (label, "bound cannot see one row", b)


def emulate(X, y, M, W, C, cw=None, fit_intercept=True):
    """numpy restatement of the kernel's order in fp32: z by an fp32 dot product, softmax and p - [y = k] in
    fp32 as mn_pointwise_kernel, the weight gradient summed in fp32 within each row chunk of multi_chunks and
    in float64 across chunks, the loss per row in fp32 and summed in float64.  Returns (f, g)."""
    n, d = X.shape
    B, K = W.shape[0], W.shape[1]
    nz, rpc = multi_chunks(n)
    X32 = X.astype(np.float32)
    f = np.empty(B)
    g = np.zeros((B, K, d + 1))
    for b in range(B):
        Wb = W[b, :, :d].astype(np.float32)
        bias = W[b, :, d].astype(np.float32) if fit_intercept else np.zeros(K, np.float32)
        Z = np.zeros((n, K), np.float32)
        X64, W64 = X32.astype(np.float64), Wb.astype(np.float64)
        for j in range(d):         # one fused multiply-add per feature: exact product, one fp32 rounding
            Z = (Z.astype(np.float64) + X64[:, j:j + 1] * W64[None, :, j]).astype(np.float32)
        Z = (Z + bias[None, :]).astype(np.float32)
        mx = Z.max(1)
        e = np.exp(Z.astype(np.float64) - mx[:, None].astype(np.float64)).astype(np.float32)
        sum_f = e.astype(np.float64).sum(1).astype(np.float32)
        loss = (np.log(sum_f.astype(np.float64)) + mx.astype(np.float64)).astype(np.float32)
        loss = (loss - Z[np.arange(n), y]).astype(np.float32)
        p = (e / sum_f[:, None]).astype(np.float32)
        onehot = np.zeros((n, K), np.float32)
        onehot[np.arange(n), y] = 1.0
        G = (p - onehot).astype(np.float32)
        s = M[:, b].astype(np.float32)
        if cw is not None:
            s = (s * cw[b, y]).astype(np.float32)
        G = (G * s[:, None]).astype(np.float32)
        loss = (loss * s).astype(np.float32)
        ntr = s.astype(np.float64).sum()
        l2 = 1.0 / (C[b] * ntr)
        acc = np.zeros((K, d))
        for z in range(nz):
            r0, r1 = z * rpc, min(n, (z + 1) * rpc)
            # sequential fp32 accumulation over the rows of the chunk (cumsum adds in order, unlike sum)
            prod = (G[r0:r1, :, None] * X32[r0:r1, None, :]).astype(np.float32)
            acc += np.cumsum(prod, axis=0, dtype=np.float32)[-1]
        lsum = 0.0
        gsum = np.zeros(K)
        for z in range(nz):
            r0, r1 = z * rpc, min(n, (z + 1) * rpc)
            lsum += loss[r0:r1].astype(np.float64).sum()
            gsum += G[r0:r1].astype(np.float64).sum(0)
        f[b] = lsum / ntr + 0.5 * l2 * (W[b, :, :d] ** 2).sum()
        g[b, :, :d] = acc / ntr + l2 * W[b, :, :d]
        g[b, :, d] = gsum / ntr if fit_intercept else 0.0
    return f, g


def grad_at_zero(X, y, M, K, cw=None, fit_intercept=True):
    """Closed form at W = 0: p = 1/K, g = sum_train s_i (1/K - [y_i = k]) x_i / n_train, f = ln K.
    Exact in fp32 when K is a power of two and the data lie on power-of-two grids."""
    n, d = X.shape
    B = M.shape[1]
    X64 = X.astype(np.float64)
    g = np.zeros((B, K, d + 1))
    ntr = np.empty(B)
    for b in range(B):
        s = M[:, b].astype(np.float64)
        if cw is not None:
            s = s * cw[b, y].astype(np.float64)
        ntr[b] = s.sum()
        tot = s @ X64                                        # sum_train s_i x_i
        per = np.zeros((K, d))
        np.add.at(per, y, s[:, None] * X64)                  # sum over class k
        g[b, :, :d] = (tot[None, :] / K - per) / ntr[b]
        if fit_intercept:
            cnt = np.bincount(y, weights=s, minlength=K)
            g[b, :, d] = (ntr[b] / K - cnt) / ntr[b]
    return g, ntr
