"""Every variant of the SGD kernels against scikit-learn (run with -m gpu on an H100).

Hinge-loss SGD promises coefficients, intercepts, n_iter_ and t_ bit-identical to SGDClassifier on both device
paths: the warp-per-column `sgd_epoch_spec_kernel` (csrc/sgd.cu) and the tensor-core path (csrc/sgd_tc.cu:
`sgd_export_kernel`, `sgd_gemm_kernel`, `sgd_scan_kernel`).  Each kernel has one instantiation per DPL =
weights per lane = 1, 2, 4, 8, 16, 32 (d <= 32 DPL).  The tests fit through `Engine.sgd_fit_batch` and compare
every column with `SGDClassifier(**same params).fit(X, y == k)` on the same float32 X; a column with no positive
row (which scikit-learn refuses to fit) is compared with `oracle.sgd_oracle.fit_binary_sgd`, itself bit-identical
to scikit-learn (tests/test_multiclass_host.py).

`SKDIST_B200_SGD_KERNEL` picks the path and `SKDIST_B200_TRACE=2` makes the fit print one line per epoch
("sgd epoch" or "sgd-tc epoch", with the active column count) and, on the tensor-core path, the screening
counters; every test asserts from those lines that the intended path ran.  Batches wider than 128 columns repeat
classes in `col_pos`: each duplicate must equal scikit-learn's one fit of its class.

log_loss goes through CUDA's exp / log / log1p instead of glibc's, so it is compared within scikit-learn's own
sensitivity: how far its fit moves when the last mantissa bit of 0.1 % of the inputs flips.  With a small
constant or invscaling step that envelope is about 1e-7, so the comparison is tight.
"""
import re
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import SGDClassifier

from oracle import sgd_oracle
from skdist_b200.datasets import make_multiclass

pytestmark = pytest.mark.gpu

BLOCK = 2048            # samples per block of the tensor-core path (ST_T)
KERNELS = ("spec", "log_loss", "scan", "export")
RAN = set()             # (kernel, DPL) run by the tests of this module
REACHED = set()         # tensor-core conditions reached: "ring_wrap", "kgroups>1", "active_crosses_128"

EPOCH_RE = re.compile(r"\[skd trace\] (sgd|sgd-tc) epoch +(\d+) active +(\d+) ")
COUNT_RE = re.compile(r"screened by the tensor-core margins (\d+), exact dot products (\d+), violators (\d+), "
                      r"violator-log overflows (\d+)")


def _dpl(d):
    p = 1
    while 32 * p < d:
        p *= 2
    return p


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _device_fit(eng, monkeypatch, capfd, path, X, y, col_pos, params):
    """sgd_fit_batch on the chosen path; returns its result and what the trace says ran."""
    monkeypatch.setenv("SKDIST_B200_SGD_KERNEL", path)
    monkeypatch.setenv("SKDIST_B200_TRACE", "2")
    capfd.readouterr()
    eng.stage_x(X)
    eng.stage_labels(np.asarray(y, np.int32))
    eng.stage_folds(None, 0)
    res = eng.sgd_fit_batch(SGDClassifier(**params), np.asarray(col_pos, np.int32))
    err = capfd.readouterr().err
    epochs = [(m.group(1), int(m.group(2)), int(m.group(3))) for m in EPOCH_RE.finditer(err)]
    assert epochs, "no SGD epoch trace lines"
    want = "sgd" if path == "simt" else "sgd-tc"
    assert {e[0] for e in epochs} == {want}, "expected the %s path, the trace shows %s" % (path, {e[0] for e in epochs})
    assert len(epochs) == int(res["n_iter"].max())
    d = X.shape[1]
    info = {"active": [e[2] for e in epochs]}
    if path == "simt":
        RAN.add(("spec" if params.get("loss", "hinge") == "hinge" else "log_loss", _dpl(d)))
    else:
        RAN.add(("scan", _dpl(d)))
        RAN.add(("export", _dpl(d)))
        if (d + 63) // 64 > 4:
            REACHED.add("ring_wrap")
        groups = [(a + 127) // 128 for a in info["active"]]
        if max(groups) > 1:
            REACHED.add("kgroups>1")
        if len(set(groups)) > 1:
            REACHED.add("active_crosses_128")
        m = COUNT_RE.search(err)
        assert m, "no screening counter line"
        info.update(zip(("screened", "exact", "violators", "overflows"), map(int, m.groups())))
    return res, info


def _sk_params(params):
    p = dict(random_state=0)
    p.update(params)
    return p


def _reference(X, y, classes, params):
    """{class: (coef float32[d], intercept, n_iter, t)} from scikit-learn (or the oracle without a positive row)."""
    out = {}
    for k in classes:
        yk = (y == k).astype(int)
        if 0 < yk.sum() < len(yk):
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                m = SGDClassifier(**params).fit(X, yk)
            assert m.coef_.dtype == np.float32
            out[k] = (m.coef_[0], float(m.intercept_[0]), int(m.n_iter_), float(m.t_))
        else:
            p = {"loss": "hinge", "alpha": 1e-4, "fit_intercept": True, "max_iter": 1000, "tol": 1e-3,
                 "shuffle": True, "random_state": 0, "n_iter_no_change": 5}
            assert set(params) <= set(p) | {"learning_rate"} and params.get("learning_rate", "optimal") == "optimal"
            p.update(params)
            p["tol"] = -np.inf if p["tol"] is None else p["tol"]
            w, b, it, t = sgd_oracle.fit_binary_sgd(X, np.where(yk == 1, 1, -1), **p)
            out[k] = (w, float(b), int(it), float(t))
    return out


def _ulps(a, b):
    a = np.atleast_1d(np.asarray(a))
    b = np.atleast_1d(np.asarray(b))
    it = np.int64 if a.dtype == np.float64 else np.int32
    return int(np.abs(a.view(it).astype(np.int64) - b.view(it).astype(np.int64)).max())


def _assert_bit_identical(res, col_pos, ref, label):
    for j, k in enumerate(col_pos):
        w, b, it, t = ref[int(k)]
        where = "%s column %d (class %d)" % (label, j, k)
        assert int(res["status"][j]) != 5, where + ": non-finite weights"
        assert int(res["n_iter"][j]) == it, "%s: n_iter %d, scikit-learn %d" % (where, res["n_iter"][j], it)
        assert float(res["t"][j]) == t, "%s: t %r, scikit-learn %r" % (where, res["t"][j], t)
        got = res["coef32"][j]
        assert np.array_equal(got, w), "%s: %d coefficients differ, by up to %d ulp" % (
            where, int((got != w).sum()), _ulps(got, w))
        assert float(res["intercept"][j]) == b, "%s: intercept %r vs %r (%d ulp)" % (
            where, float(res["intercept"][j]), b, _ulps(np.float64(res["intercept"][j]), np.float64(b)))


def _col_pos(B, k):
    return np.tile(np.arange(k), (B + k - 1) // k)[:B].astype(np.int32)


# --------------------------------------------------------------------------------------------------------------
# (a) hinge shape matrix, both paths
# --------------------------------------------------------------------------------------------------------------
# d, n, B, k: every DPL; kchunks = ceil(d / 64) both <= 4 and > 4 (the TMA ring of 4 stages wraps); B = 1, 128, 129
# and >= 257; n < 2048, = 2048, a multiple of 2048 and ragged last blocks (of 1 sample too)
SHAPES = [
    (1, 1500, 3, 3),
    (20, 2500, 1, 3),
    (32, 6145, 129, 5),
    (33, 2048, 7, 7),
    (65, 2049, 300, 5),
    (129, 8192, 128, 4),
    (256, 4097, 129, 5),
    (257, 6145, 7, 7),
    (512, 4096, 300, 5),
    (513, 2049, 3, 3),
    (1024, 6145, 129, 5),
]
_CACHE = {}


def _shape_case(d, n, B, k):
    key = ("shape", d, n, B, k)
    if key not in _CACHE:
        X, y = make_multiclass(n, d, k, seed=d + n)
        col_pos = _col_pos(B, k)
        _CACHE[key] = (X, y, col_pos, _reference(X, y, sorted(set(col_pos.tolist())), _sk_params({})))
    return _CACHE[key]


@pytest.mark.parametrize("path", ["simt", "tc"])
@pytest.mark.parametrize("d,n,B,k", SHAPES, ids=["d%d-n%d-B%d" % s[:3] for s in SHAPES])
def test_hinge_shapes_bit_identical(eng, monkeypatch, capfd, path, d, n, B, k):
    X, y, col_pos, ref = _shape_case(d, n, B, k)
    res, info = _device_fit(eng, monkeypatch, capfd, path, X, y, col_pos, _sk_params({}))
    _assert_bit_identical(res, col_pos, ref, "%s d=%d n=%d B=%d" % (path, d, n, B))


# --------------------------------------------------------------------------------------------------------------
# (b) hinge edges: hyper-parameters and data, one small-d and one d > 256 shape, both paths
# --------------------------------------------------------------------------------------------------------------
EDGE_SHAPES = {"small": (3000, 24, 4), "wide": (4500, 300, 3)}
EDGES = {
    "no_intercept": {"fit_intercept": False},
    "no_shuffle": {"shuffle": False},
    "constant": {"learning_rate": "constant", "eta0": 0.01},
    "reset_every_sample": {"learning_rate": "constant", "eta0": 1.0, "alpha": 1.0},
    "invscaling": {"learning_rate": "invscaling", "eta0": 0.01},
    "alpha_100": {"alpha": 100.0},
    "alpha_1e-7": {"alpha": 1e-7},
    "tol_none_max_iter_3": {"tol": None, "max_iter": 3},
    "n_iter_no_change_1": {"n_iter_no_change": 1},
    "n_iter_no_change_10": {"n_iter_no_change": 10},
    "random_labels": {},
    "data_edges": {},
    "one_or_no_positive": {},
}
RESET_EDGES = ("reset_every_sample", "alpha_100")
EDGE_N = {"alpha_100": 12000}      # the second reset of alpha = 100 comes near sample 31 624 of the fit, in epoch 2


def _edge_data(edge, n, d, k, seed):
    X, y = make_multiclass(n, d, k, seed=seed)
    classes = list(range(k))
    if edge == "random_labels":                 # violators stay frequent in every epoch
        y = np.random.default_rng(seed).integers(0, k, n)
    elif edge == "data_edges":
        X *= np.logspace(-3, 3, d, dtype=np.float32)[np.random.default_rng(seed).permutation(d)]
        X[:, d // 2] = 0.0                      # an all-zero feature
        X[7] = 0.0                              # an all-zero row
        big = np.abs(X).max()
        for r in (11, 12, 13):                  # rows at about 2^-20 of max |X| (inside the screening precondition)
            X[r] *= np.float32(2.0 ** -20 * big / np.linalg.norm(X[r].astype(np.float64)))
        X[100:140] = X[300:340]                 # duplicated rows
        y[100:140] = y[300:340]
    elif edge == "one_or_no_positive":
        y[5] = k                                # class k has one positive row, class k + 1 none
        classes = list(range(k + 2))
    return np.ascontiguousarray(X, np.float32), y, np.array(classes, np.int32)


def _edge_case(edge, shape):
    key = ("edge", edge, shape)
    if key not in _CACHE:
        n, d, k = EDGE_SHAPES[shape]
        n = EDGE_N.get(edge, n)
        X, y, col_pos = _edge_data(edge, n, d, k, seed=d + len(edge))
        params = _sk_params(EDGES[edge])
        _CACHE[key] = (X, y, col_pos, params, _reference(X, y, col_pos.tolist(), params))
    return _CACHE[key]


def _schedule_cfac(params, n, epochs):
    """The per-sample factor max(0, 1 - eta * alpha) as float, for `epochs` epochs of n samples."""
    alpha = params.get("alpha", 1e-4)
    t = 1.0 + np.arange(epochs * n, dtype=np.float64)
    lr = params.get("learning_rate", "optimal")
    if lr == "optimal":
        typw = np.sqrt(1.0 / np.sqrt(alpha))
        eta = 1.0 / (alpha * (1.0 / (typw * alpha) + t - 1.0))     # hinge: optimal_init = 1 / (typw * alpha)
    elif lr == "constant":
        eta = np.full_like(t, params["eta0"])
    else:
        eta = params["eta0"] / t ** params.get("power_t", 0.5)
    return np.maximum(0.0, 1.0 - eta * alpha).astype(np.float32).astype(np.float64)


def _reset_samples(params, n, epochs):
    """Sample indices (within their epoch) where wscale *= c_t falls below 1e-6 and reset_wscale fires."""
    ws, out = 1.0, []
    for i, c in enumerate(_schedule_cfac(params, n, epochs)):
        ws *= c
        if ws < 1e-6:
            out.append(i % n)
            ws = 1.0
    return np.array(out, np.int64)


@pytest.mark.parametrize("path", ["simt", "tc"])
@pytest.mark.parametrize("shape", sorted(EDGE_SHAPES))
@pytest.mark.parametrize("edge", list(EDGES))
def test_hinge_edges_bit_identical(eng, monkeypatch, capfd, edge, shape, path):
    X, y, col_pos, params, ref = _edge_case(edge, shape)
    n = X.shape[0]
    if edge in RESET_EDGES:                     # the replay of the lazy scale puts a reset strictly inside a block
        epochs = max(r[2] for r in ref.values())
        resets = _reset_samples(params, n, epochs)
        assert np.any(resets % BLOCK != 0), "no reset_wscale inside a block: %s" % resets[:10]
    if edge == "one_or_no_positive":
        assert (y == col_pos[-2]).sum() == 1 and (y == col_pos[-1]).sum() == 0
    res, info = _device_fit(eng, monkeypatch, capfd, path, X, y, col_pos, params)
    _assert_bit_identical(res, col_pos, ref, "%s %s %s" % (path, edge, shape))
    if path == "tc" and edge == "random_labels":
        # the violator log (96 updates per column and block) overflows in more scans than epoch 0 has
        blocks = (n + BLOCK - 1) // BLOCK
        assert info["overflows"] > blocks * len(col_pos), info


# --------------------------------------------------------------------------------------------------------------
# (c) log_loss on the warp kernel, every DPL: within scikit-learn's own sensitivity
# --------------------------------------------------------------------------------------------------------------
LOG_D = (20, 40, 100, 200, 400, 800)
LOG_SCHEDULES = {"constant": {"learning_rate": "constant", "eta0": 1e-3},
                 "invscaling": {"learning_rate": "invscaling", "eta0": 0.01}}


@pytest.mark.parametrize("schedule", sorted(LOG_SCHEDULES))
@pytest.mark.parametrize("d", LOG_D)
def test_log_loss_every_dpl_within_envelope(eng, monkeypatch, capfd, d, schedule):
    n, k = 3000, 5
    X, y = make_multiclass(n, d, k, seed=12 + d)
    params = _sk_params(dict(LOG_SCHEDULES[schedule], loss="log_loss", shuffle=False))
    Xp = X.copy()
    Xp.view(np.int32)[np.random.RandomState(0).rand(*X.shape) < 1e-3] ^= 1
    ref, ref_p = _reference(X, y, range(k), params), _reference(Xp, y, range(k), params)
    envelope = max(np.abs(ref_p[c][0] - ref[c][0]).max() / np.abs(ref[c][0]).max() for c in range(k))
    assert envelope <= 1e-5, envelope           # the tier bites: the reference is stable under this schedule
    col_pos = np.arange(k, dtype=np.int32)
    res, _ = _device_fit(eng, monkeypatch, capfd, "simt", X, y, col_pos, params)
    for c in range(k):
        w, b, it, _ = ref[c]
        scale = np.abs(w).max()
        assert int(res["n_iter"][c]) == it, (c, res["n_iter"][c], it)
        err = np.abs(res["coef32"][c] - w).max()
        assert err <= 3 * envelope * scale, (c, err / scale, envelope)
        assert abs(res["intercept"][c] - b) <= 3 * envelope * max(abs(b), scale), (c, res["intercept"][c], b, envelope)


# --------------------------------------------------------------------------------------------------------------
# overflow and max_iter through the one-vs-rest wrapper, as scikit-learn reports them
# --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["simt", "tc"])
def test_ovr_overflow_raises_like_sklearn(monkeypatch, path):
    from sklearn.multiclass import OneVsRestClassifier
    from skdist.distribute.multiclass import DistOneVsRestClassifier
    monkeypatch.setenv("SKDIST_B200_SGD_KERNEL", path)
    X, y = make_multiclass(1500, 20, 4, seed=3)
    X = X * np.float32(1e18)
    mk = lambda: SGDClassifier(learning_rate="constant", eta0=1e20, random_state=0)
    with pytest.raises(ValueError) as ref:
        OneVsRestClassifier(mk()).fit(X, y)
    with pytest.raises(ValueError) as ours:
        DistOneVsRestClassifier(mk(), None).fit(X, y)
    assert "under-/overflow occurred at epoch" in str(ref.value)
    assert str(ours.value) == str(ref.value)


@pytest.mark.parametrize("path", ["simt", "tc"])
def test_ovr_max_iter_warns_like_sklearn(monkeypatch, path):
    from sklearn.multiclass import OneVsRestClassifier
    from skdist.distribute.multiclass import DistOneVsRestClassifier
    monkeypatch.setenv("SKDIST_B200_SGD_KERNEL", path)
    X, y = make_multiclass(2500, 20, 3, seed=4)
    mk = lambda: SGDClassifier(max_iter=2, random_state=0)
    with pytest.warns(ConvergenceWarning, match="Maximum number of iteration reached before convergence"):
        ref = OneVsRestClassifier(mk()).fit(X, y)
    with pytest.warns(ConvergenceWarning, match="Maximum number of iteration reached before convergence"):
        ours = DistOneVsRestClassifier(mk(), None).fit(X, y)
    for a, b in zip(ours.estimators_, ref.estimators_):
        assert a.n_iter_ == b.n_iter_ == 2
        np.testing.assert_array_equal(a.coef_, b.coef_)


# --------------------------------------------------------------------------------------------------------------
# (d) bookkeeping
# --------------------------------------------------------------------------------------------------------------
def test_every_variant_ran():
    """All 24 instantiations (spec, log_loss, scan, export x DPL 1..32) ran in the tests above, the TMA ring of
    sgd_gemm_kernel wrapped, a batch had more than one 128-column group and an active count crossed 128."""
    want = {(kern, p) for kern in KERNELS for p in (1, 2, 4, 8, 16, 32)}
    assert RAN == want, sorted(want - RAN)
    assert REACHED == {"ring_wrap", "kgroups>1", "active_crosses_128"}, REACHED
