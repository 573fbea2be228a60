"""Float64 / integer restatement of the ranking scorers the rank kernel (csrc/auc.cu) serves -- never calls the
engine.  Per segment: 2U (twice the Mann-Whitney statistic, integer), n_pos, n_neg and the uninterpolated
average precision; then scikit-learn's averaging of roc_auc_ovr / roc_auc_ovo [_weighted] and
average_precision over the segments."""
import numpy as np

# a device probability lies within (K + 10) * 2^-23 of its value from numpy's (csrc/auc.cu, K = 1 for binary)
def proba_rel_tol(K):
    return (K + 10) * 2.0 ** -23


def f32_proba(Z):
    """float32 predict_proba of LogisticRegression from float32 decision values: expit for a 1-d Z, else
    sklearn.utils.extmath.softmax (what the scorer sees for float32 X)."""
    from scipy.special import expit
    from sklearn.utils.extmath import softmax
    Z = np.asarray(Z, dtype=np.float32)
    return expit(Z) if Z.ndim == 1 else softmax(Z.copy())


def segment_counts(s, pos):
    """(2U, n_pos, n_neg, ap) of one segment: scores s, positive flags pos."""
    s = np.asarray(s, dtype=np.float64)
    pos = np.asarray(pos, dtype=bool)
    neg = np.sort(s[~pos])
    P, N = int(pos.sum()), int((~pos).sum())
    sp = s[pos]
    below = np.searchsorted(neg, sp, side="left")
    tied = np.searchsorted(neg, sp, side="right") - below
    u2 = int(np.sum(2 * below.astype(np.int64) + tied))
    if P == 0:
        return u2, P, N, 0.0
    # tie groups in descending score: tp / fp = positives / negatives scoring >= the group
    vals, inv = np.unique(-s, return_inverse=True)
    pos_g = np.bincount(inv, weights=pos, minlength=len(vals)).astype(np.int64)
    neg_g = np.bincount(inv, weights=~pos, minlength=len(vals)).astype(np.int64)
    tp, fp = np.cumsum(pos_g), np.cumsum(neg_g)
    ap = float(np.sum(pos_g * (tp / (tp + fp))) / P)
    return u2, P, N, ap


def segments(S, y, K, pairs, pos=1):
    """[(scores, positive flags)] of one fit's segments in the kernel's order.  K == 1: S 1-d, positives
    y == pos; K > 2: S [n, K], one-vs-rest (class k) or ordered one-vs-one pairs (a, b) at
    a * (K - 1) + (b < a ? b : b - 1)."""
    y = np.asarray(y)
    if K == 1:
        return [(S, y == pos)]
    if not pairs:
        return [(S[:, k], y == k) for k in range(K)]
    out = []
    for a in range(K):
        for b in range(K):
            if b != a:
                m = (y == a) | (y == b)
                out.append((S[m, a], y[m] == a))
    return out


def rank_counts(S, y, K, pairs, pos=1):
    """{"u2", "n_pos", "n_neg", "ap"} arrays over one fit's segments."""
    c = [segment_counts(s, p) for s, p in segments(S, y, K, pairs, pos)]
    return {"u2": np.array([t[0] for t in c], np.int64), "n_pos": np.array([t[1] for t in c], np.int64),
            "n_neg": np.array([t[2] for t in c], np.int64), "ap": np.array([t[3] for t in c], np.float64)}


def u2_interval(s, pos, rel):
    """Smallest and largest 2U when every (positive, negative) pair whose scores lie within rel (relative to
    the larger magnitude) may rank either way."""
    s = np.asarray(s, dtype=np.float64)
    pos = np.asarray(pos, dtype=bool)
    neg = np.sort(s[~pos])
    lo = hi = 0
    for v in s[pos]:
        t = rel * np.maximum(abs(v), np.abs(neg))
        sure_below = np.sum(neg < v - t)
        close = np.sum(np.abs(neg - v) <= t)
        lo += 2 * sure_below
        hi += 2 * sure_below + 2 * close
    return lo, hi


def score(kind, average, y, S, K):
    """scikit-learn's value of a ranking scorer on one fit's rows, from rank_counts (None where scikit-learn
    raises: a class missing from y).  kind: roc_auc_ovr, roc_auc_ovo, average_precision; K == 1 binary."""
    if K == 1:
        r = rank_counts(S, y, 1, False)
        if kind == "average_precision":
            return r["ap"][0]
        return r["u2"][0] / (2.0 * r["n_pos"][0] * r["n_neg"][0]) if r["n_pos"][0] * r["n_neg"][0] else None
    counts = np.bincount(y, minlength=K)
    if np.any(counts == 0):
        return None
    r = rank_counts(S, y, K, kind == "roc_auc_ovo")
    auc = r["u2"] / (2.0 * r["n_pos"] * r["n_neg"])
    if kind == "average_precision":
        return float(np.mean(r["ap"]))
    if kind == "roc_auc_ovr":
        return float(np.average(auc, weights=counts if average == "weighted" else None))
    pair, prev = [], []
    for a in range(K):
        for b in range(a + 1, K):
            ab = auc[a * (K - 1) + b - 1]
            ba = auc[b * (K - 1) + a]
            pair.append((ab + ba) / 2.0)
            prev.append((counts[a] + counts[b]) / counts.sum())
    return float(np.average(pair, weights=prev if average == "weighted" else None))
