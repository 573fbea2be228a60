"""The work deal of the tensor-core logistic kernel (csrc/logreg_tc.cu, tc_eval_kernel) at many group counts.

Every CTA deals itself its share of the (group, chunk) units from the live slot count on the device, and a
consumer warpgroup whose 64 slots are all padding computes nothing.  Neither may change a result:

  * bit identity: a column fitted inside batches of 1 to 160 live groups of 128 slots (folds whose last
    group is one column, half empty, exactly half full, full, or one column into the next group; columns
    that converge at every round) gets the same coef, n_iter and loss bytes as fitted alone;
  * every unit exactly once: the exact tier of test_tc_eval_gpu (integer data on power-of-two grids) at the
    same group counts, through the loss/gradient entry at W = 0 and through the accuracy and squared-error
    counts.  A unit dealt twice or not at all moves a count or a gradient component far off its bound;
  * the trace (SKDIST_B200_TRACE=2) shows the deal at work: the live group count of every round, groups with
    a padding half, and CTA ranges that span two groups.
"""
import re

import numpy as np
import pytest

from tests.test_tc_eval_gpu import _exact_setup   # the exact tier's data: integers on power-of-two grids

pytestmark = pytest.mark.gpu

GROUP_COUNTS = [1, 2, 5, 7, 11, 12, 19, 20, 21, 67, 131, 132, 133, 160]
TAILS = [1, 63, 64, 65, 127, 128]      # columns in a fold's last group: 1 and 63 leave its second half padding
ROUND_RE = re.compile(r"round\s+(\d+) slots\s+(\d+) running\s+(\d+) groups\s+(\d+) half\s+(\d+) "
                      r"ctas\s+(\d+) cross\s+(\d+) eval")


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    e.set_kernel(2)
    yield e
    e.close()


def _fold_counts(groups, n_folds, minimum=()):
    """Columns per fold so that the fold-grouped layout has `groups` groups of 128 slots."""
    used = min(groups, n_folds)
    per = [groups // used + (1 if i < groups % used else 0) for i in range(used)]
    counts = [128 * (g - 1) + TAILS[(i + groups) % len(TAILS)] for i, g in enumerate(per)]
    for i, m in enumerate(minimum[:used]):
        if counts[i] < m:
            counts[i] = m
    return counts + [0] * (n_folds - used)


def _columns_of(counts):
    return np.concatenate([np.full(c, f, np.int32) for f, c in enumerate(counts)])


def _layout_groups(cf):
    return sum((np.count_nonzero(cf == f) + 127) // 128 for f in np.unique(cf))


# ---- every unit exactly once ----------------------------------------------------------------------------
@pytest.mark.parametrize("groups", GROUP_COUNTS)
def test_exact_gradient_at_zero_every_group_count(eng, groups):
    d = 17
    rng, X, e, ycls, fold, nf = _exact_setup(eng, (d, "M", "f40", 0), 900 + groups)
    cf = _columns_of(_fold_counts(groups, nf))
    assert _layout_groups(cf) == groups
    cf = cf[rng.permutation(len(cf))]
    B = len(cf)
    pos = (np.arange(B) % 3).astype(np.int32)
    f, g = eng.logreg_loss_grad(np.zeros((B, d + 1)), np.ones(B), cf, pos)
    Xs, Xa = X.astype(np.float64), np.abs(X.astype(np.float64))
    S = np.zeros((nf, 3, d)); A = np.zeros((nf, 3, d)); N = np.zeros((nf, 3))
    for k in range(nf):
        for c in range(3):
            m = (fold == k) & (ycls == c)
            S[k, c] = Xs[m].sum(0); A[k, c] = Xa[m].sum(0); N[k, c] = m.sum()
    St, At, Nt = S.sum(0) - S, A.sum(0) - A, N.sum(0) - N     # training rows per (held-out fold, class)
    ntr = Nt[cf].sum(1)
    want = (0.5 * St[cf].sum(1) - St[cf, pos]) / ntr[:, None]
    bound = 2.0 ** -20 * At[cf].sum(1) / ntr[:, None]
    err = np.abs(g[:, :d] - want)
    assert np.all(err <= bound), (groups, np.unravel_index(np.argmax(err / bound), err.shape))
    want_b = (0.5 * ntr - Nt[cf, pos]) / ntr
    assert np.all(np.abs(g[:, d] - want_b) <= 2.0 ** -20), groups
    assert np.all(np.isfinite(f))


@pytest.mark.parametrize("groups", GROUP_COUNTS)
def test_exact_score_and_r2_every_group_count(eng, groups):
    """Scoring lays the columns out densely: the last group holds 1 to 128 of them."""
    d = 40
    rng, X, e, ycls, fold, nf = _exact_setup(eng, (d, "M", "kfold", 0), 950 + groups)
    B = 128 * (groups - 1) + TAILS[groups % len(TAILS)]
    code = rng.integers(-2 - nf, nf, B).astype(np.int32)
    code[code == -1] = -2
    pos = (np.arange(B) % 3).astype(np.int32)
    coef = np.zeros((B, d + 1), np.float32)
    coef[:, :d] = rng.integers(-2, 3, (B, d)) * np.exp2(-e)
    coef[:, d] = rng.integers(-100, 101, B)
    yreal = rng.integers(-100, 101, X.shape[0]).astype(np.float32)
    eng.stage_targets(yreal)
    want_count, want_correct, want_sse = np.zeros(B, np.int64), np.zeros(B, np.int64), np.zeros(B)
    for j0 in range(0, B, 2048):     # float64 reference in column blocks (bounded host memory)
        j = slice(j0, min(B, j0 + 2048))
        c = code[j]
        Z = X.astype(np.float64) @ coef[j, :d].T.astype(np.float64) + coef[j, d].astype(np.float64)   # exact
        M = np.where(c[None, :] == -2, True,
                     np.where(c[None, :] >= 0, fold[:, None] == c[None, :], fold[:, None] != (-3 - c)[None, :]))
        want_count[j] = M.sum(0)
        want_correct[j] = (M & ((Z > 0) == (ycls[:, None] == pos[None, j]))).sum(0)
        R = yreal.astype(np.float64)[:, None] - Z
        want_sse[j] = (M * R * R).sum(0)
    correct, count = eng.linear_score_batch(coef, code, pos)
    assert np.array_equal(count, want_count), groups
    assert np.array_equal(correct, want_correct), groups
    sse, count = eng.linear_r2_batch(coef, code)
    assert np.array_equal(count, want_count), groups
    assert np.array_equal(sse, want_sse), groups


# ---- bit identity of fits ---------------------------------------------------------------------------------
N_FIT, D_FIT, FOLDS_FIT, MAX_ITER = 20000, 20, 5, 60
PROBES = [(0, 0.01), (0, 1.0), (0, 100.0), (1, 0.1), (1, 10.0)]   # (held-out fold, C)


@pytest.fixture(scope="module")
def fit_data(eng):
    rng = np.random.default_rng(77)
    X = rng.standard_normal((N_FIT, D_FIT)).astype(np.float32)
    y = (X @ rng.standard_normal(D_FIT) + rng.logistic(size=N_FIT) > 0).astype(np.int32)
    fold = (rng.permutation(N_FIT) % FOLDS_FIT).astype(np.int8)
    eng.stage_x(X); eng.stage_labels(y); eng.stage_folds(fold, FOLDS_FIT)
    alone = []
    for f, C in PROBES:
        r = eng.logreg_fit_batch(np.array([C]), np.array([f], np.int32), np.ones(1, np.int32), max_iter=MAX_ITER)
        alone.append({k: np.asarray(r[k])[0].copy() for k in ("coef", "n_iter", "loss")})
    return alone


def _batch(groups, seed):
    """Columns of a batch with `groups` live groups: the probes first, then columns whose C spreads over
    seven decades (so they converge at many different rounds, inside the host's round trips)."""
    counts = _fold_counts(groups, FOLDS_FIT, minimum=(3, 2))
    rng = np.random.default_rng(seed)
    cf, C, probe_at = [], [], {}
    for f, c in enumerate(counts):
        mine = [i for i, p in enumerate(PROBES) if p[0] == f][:c]
        for i in mine:
            probe_at[i] = len(cf)
            cf.append(f); C.append(PROBES[i][1])
        for _ in range(c - len(mine)):
            cf.append(f); C.append(10.0 ** rng.uniform(-4, 3))
    cf, C = np.array(cf, np.int32), np.array(C)
    perm = rng.permutation(len(cf))
    inv = np.argsort(perm)
    return cf[perm], C[perm], {i: int(inv[j]) for i, j in probe_at.items()}


@pytest.mark.parametrize("groups", GROUP_COUNTS)
def test_fit_bits_independent_of_group_count(eng, fit_data, groups):
    cf, C, probe_at = _batch(groups, 3000 + groups)
    assert _layout_groups(cf) == groups
    res = eng.logreg_fit_batch(C, cf, np.ones(len(cf), np.int32), max_iter=MAX_ITER)
    assert len(set(np.asarray(res["n_iter"]).tolist())) > 1
    for i, j in probe_at.items():
        for k in ("coef", "n_iter", "loss"):
            got = np.asarray(res[k])[j]
            assert np.asarray(got).tobytes() == fit_data[i][k].tobytes(), (groups, PROBES[i], k)


def test_trace_shows_the_deal(eng, fit_data, monkeypatch, capfd):
    """Round by round: the kernel counts the live groups itself, groups with a padding half occur, and
    some CTA ranges span two groups.  Round 0 runs on one CTA per SM."""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    cf, C, _ = _batch(20, 4020)
    monkeypatch.setenv("SKDIST_B200_TRACE", "2")
    eng.profile(1)
    capfd.readouterr()
    try:
        eng.logreg_fit_batch(C, cf, np.ones(len(cf), np.int32), max_iter=MAX_ITER)
    finally:
        err = capfd.readouterr().err
        eng.profile(0)
    rounds = [tuple(map(int, m.groups())) for m in ROUND_RE.finditer(err)]
    assert rounds, "no per-round deal lines in the trace"
    assert rounds[0][0] == 0 and rounds[0][3] == 20 and rounds[0][5] == sm, rounds[0]
    for r, slots, running, groups, half, ctas, cross in rounds:
        assert groups * 128 == slots, (r, slots, groups)      # the kernel's own live count
        assert half <= groups
    assert any(x[4] > 0 for x in rounds), "no group with a padding half"
    assert any(x[6] > 0 for x in rounds), "no CTA range spans two groups"
