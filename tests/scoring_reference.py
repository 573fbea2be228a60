"""float64 and integer references of the scoring and inference entries, shared by the GPU tests and their host
rehearsal.  Nothing here calls the engine.

  decision            z = X w + b in float64 (exact for the integer data of the exact tier)
  select              the rows a scoring code picks: f = fold f, -2 = every row, -3 - f = the rows outside fold f
  accuracy_counts     #{selected rows: (z > 0) == (y == pos)} and #selected, per column
  sse                 sum over the selected rows of (y - z)^2, per column
  auc_counts          2U, n_pos, n_neg of the Mann-Whitney statistic by sorting and counting tie groups
  binary_logloss      -log p of scikit-learn's float32 probabilities (expit, 1 - p1), clipped to float32 eps
  forest_walk         the soft vote of concatenated `Tree` arrays, compared as float64(x) <= threshold

Error bounds of the fp32 decision kernels (u = 2^-24, gamma_h = h u / (1 - h u)):

  fwd_kernel          one sequential FMA chain over k, then + b:        h = d + 1
  predict_kernel      per lane an FMA chain over its float4 quads (4 per quad, ceil(ldx / 128) quads), a
                      5-level shuffle tree, then + b:                   h = 4 ceil(ldx / 128) + 6

  |z32 - z64| <= gamma_h (sum_k |x_k w_k| + |b|).
"""
import numpy as np

U = 2.0 ** -24
EPS32 = float(np.finfo(np.float32).eps)


def round_up(v, m):
    return (v + m - 1) // m * m


def decision(X, coef):
    """[n, B] float64 decision values; coef [B, d + 1] (weights, intercept last) as the kernels read it (fp32)."""
    W = np.asarray(coef, np.float32).astype(np.float64)
    return np.asarray(X, np.float32).astype(np.float64) @ W[:, :-1].T + W[:, -1]


def decision_abs(X, coef):
    """[n, B] sum_k |x_k w_k| + |b|, the scale of the rounding error of z."""
    W = np.abs(np.asarray(coef, np.float32).astype(np.float64))
    return np.abs(np.asarray(X, np.float32).astype(np.float64)) @ W[:, :-1].T + W[:, -1]


def gamma(h):
    return h * U / (1.0 - h * U)


def depth_fwd(d):
    """Summation depth of fwd_kernel (logreg_simt.cu): a sequential FMA chain over k, then + b."""
    return d + 1


def depth_predict(ldx):
    """Summation depth of predict_kernel (predict.cu): lane-strided float4 FMA chains, 5 shuffle levels, + b."""
    return 4 * ((ldx + 127) // 128) + 6


def select(code, fold, n):
    """[n, B] rows chosen by every scoring code; fold None: no folds staged (row fold -1)."""
    code = np.asarray(code)
    f = np.full(n, -1) if fold is None else np.asarray(fold).astype(np.int64)
    return ((code[None, :] == -2)
            | ((code[None, :] >= 0) & (f[:, None] == code[None, :]))
            | ((code[None, :] <= -3) & (f[:, None] != (-3 - code)[None, :])))


def accuracy_counts(Z, ycls, pos, code, fold):
    """(correct, count) per column: prediction z > 0 (z == 0 predicts the negative class)."""
    M = select(code, fold, Z.shape[0])
    hit = (Z > 0) == (np.asarray(ycls)[:, None] == np.asarray(pos)[None, :])
    return (M & hit).sum(0).astype(np.int64), M.sum(0).astype(np.int64)


def sse(Z, yreal, code, fold):
    """(sum of squared residuals, count) per column over the selected rows."""
    M = select(code, fold, Z.shape[0])
    R = np.asarray(yreal, np.float32).astype(np.float64)[:, None] - Z
    return (np.where(M, R * R, 0.0)).sum(0), M.sum(0).astype(np.int64)


def auc_counts(z, positive):
    """(2U, n_pos, n_neg) as Python integers for scores z and a boolean positive mask: every positive row scores
    2 per negative row below it and 1 per negative row tied with it."""
    z = np.asarray(z, np.float64) + 0.0          # -0.0 and +0.0 are one value
    positive = np.asarray(positive, bool)
    vals, inv = np.unique(z, return_inverse=True)
    pos_g = np.bincount(inv, weights=positive, minlength=len(vals)).astype(np.int64)
    neg_g = np.bincount(inv, weights=~positive, minlength=len(vals)).astype(np.int64)
    neg_below = np.concatenate([[0], np.cumsum(neg_g)[:-1]])
    u2 = sum(2 * int(p) * int(nb) + int(p) * int(ng) for p, nb, ng in zip(pos_g, neg_below, neg_g) if p)
    return u2, int(positive.sum()), int((~positive).sum())


def auc_counts_batch(Z, ycls, pos, code, fold):
    """(2U, n_pos, n_neg) int64 arrays of every column on its selected rows."""
    M = select(code, fold, Z.shape[0])
    out = np.zeros((3, Z.shape[1]), np.int64)
    for j in range(Z.shape[1]):
        out[:, j] = auc_counts(Z[M[:, j], j], np.asarray(ycls)[M[:, j]] == pos[j])
    return out


def binary_proba32(z32):
    """p1 of scikit-learn's binary predict_proba on float32 decision values: expit in float32 arithmetic,
    1 / (1 + exp(-z)) with the exponential rounded once to float32."""
    z32 = np.asarray(z32, np.float32)
    e = np.exp(-z32.astype(np.float64)).astype(np.float32)
    with np.errstate(over="ignore"):
        return (np.float32(1.0) / (np.float32(1.0) + e)).astype(np.float32)


def binary_logloss(z32, positive):
    """Per row -log p_true with p0 = 1 - p1 in float32 and p clipped to [eps, 1 - eps] (float32 eps)."""
    p1 = binary_proba32(z32)
    p = np.where(positive, p1, np.float32(1.0) - p1).astype(np.float64)
    return -np.log(np.clip(p, EPS32, 1.0 - EPS32))


def binary_logloss_bound(z32, positive, dz):
    """Per-row bound on |loss_kernel - binary_logloss(z32)|: two float32 ulps of p1 (the rounding of the
    exponential), one of p_true (the rounding of 1 - p1) and the first-order effect of a decision error dz, all
    relative to the clipped p_true."""
    p1 = binary_proba32(z32).astype(np.float64)
    p = np.clip(np.where(positive, p1, 1.0 - p1), EPS32, 1.0 - EPS32)
    ulp = np.spacing(np.float32(p1)).astype(np.float64) * 2.0 + np.spacing(np.float32(p)).astype(np.float64)
    return (ulp + p1 * (1.0 - p1) * np.asarray(dz) * 1.01) / p


def forest_walk(X, off, left, right, feature, threshold, value):
    """[m, C] float64 mean over the trees of the leaf value each row reaches, trees added in order."""
    X = np.asarray(X, np.float32)
    m, C = X.shape[0], value.shape[1]
    acc = np.zeros((m, C))
    rows = np.arange(m)
    for t in range(len(off) - 1):
        base = off[t]
        k = np.zeros(m, np.int64)
        while True:
            live = left[base + k] != -1
            if not live.any():
                break
            r = rows[live]
            kk = base + k[live]
            go_left = X[r, feature[kk]].astype(np.float64) <= threshold[kk]
            k[live] = np.where(go_left, left[kk], right[kk])
        acc += value[base + k]
    return acc / (len(off) - 1)
