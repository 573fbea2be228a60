"""Forest classifiers with class_weight, host side (no GPU): the weights staged for the device, the fit
pipeline on an engine double that builds the restated reference trees, the refusals, and the float32
screening bound of the weighted throughput builder restated in numpy."""
from fractions import Fraction

import numpy as np
import pytest
from sklearn.utils import check_random_state
from sklearn.utils.class_weight import compute_class_weight, compute_sample_weight

from skdist_b200.distribute.ensemble import MAX_RAND_SEED, _tree_inputs
from tests.forest_class_weight_restate import WeightedForestEngine, restated_forest, tree_class_weights


@pytest.fixture
def weighted_engine():
    from skdist_b200 import engine
    engine.set_engine_factory(WeightedForestEngine)
    yield
    engine.set_engine_factory(None)


def _data(n=400, d=6, k=3, seed=2):
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 12, size=(n, d)).astype(np.float32)
    s = X[:, 0] + 0.5 * X[:, 1] + rng.standard_normal(n) * 2
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, k + 1)[1:-1]))
    return X, y


def _seed_map(rs, n_trees, n):
    from skdist_b200.engine import get_engine
    states = check_random_state(rs).randint(MAX_RAND_SEED, size=n_trees)
    eng = get_engine()
    eng.seed_of_rand_r = {int(_tree_inputs(s, n, False)[1]): int(s) for s in states}
    return eng


def _same_trees(ests, trees):
    assert len(ests) == len(trees)
    for a, b in zip(ests, trees):
        np.testing.assert_array_equal(a.tree_.children_left, b.tree_.children_left)
        np.testing.assert_array_equal(a.tree_.threshold, b.tree_.threshold)
        np.testing.assert_array_equal(a.tree_.n_node_samples, b.tree_.n_node_samples)
        np.testing.assert_array_equal(a.tree_.weighted_n_node_samples, b.tree_.weighted_n_node_samples)
        np.testing.assert_array_equal(a.tree_.value, b.tree_.value)


@pytest.mark.parametrize("cw,bootstrap", [({0: 2.0, 1: 0.0}, True), ({0: 0.5, 2: 3.0}, False), ("balanced", True),
                                          ("balanced", False), ("balanced_subsample", True),
                                          ("balanced_subsample", False)])
def test_staged_weights_are_scikit_learns(weighted_engine, cw, bootstrap):
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = _data()
    y = y + 3                                              # original labels 3, 4, 5: dict keys are labels
    cwl = {k + 3: v for k, v in cw.items()} if isinstance(cw, dict) else cw
    eng = _seed_map(4, 5, len(y))
    DistRandomForestClassifier(n_estimators=5, random_state=4, bootstrap=bootstrap, class_weight=cwl,
                               min_weight_fraction_leaf=0.01).fit(X, y)
    (st,) = eng.staged                                     # one chunk: one staging call
    assert st[0] == 3 and st[3] == 0.01
    if cw == "balanced_subsample" and bootstrap:
        assert st[2] and st[1] is None
    else:
        want = compute_class_weight("balanced" if cw == "balanced_subsample" else cwl, classes=np.unique(y), y=y)
        assert not st[2]
        np.testing.assert_array_equal(st[1], want)
        # compute_sample_weight of the reference's expanded_class_weight, class by class
        np.testing.assert_array_equal(st[1][y - 3], compute_sample_weight(
            "balanced" if cw == "balanced_subsample" else cwl, y))


def test_subsample_weights_of_a_tree_are_compute_sample_weights():
    """The per-tree balanced_subsample weights n / (K_present N_k) that the builders form from the bootstrap
    class counts: compute_sample_weight("balanced", y, indices=...) bit for bit, absent classes 0."""
    rng = np.random.default_rng(0)
    y = np.r_[np.zeros(300, int), np.ones(40, int), np.full(3, 2)]
    for s in rng.integers(0, MAX_RAND_SEED, size=30):
        counts, _ = _tree_inputs(int(s), len(y), True)
        nk = np.bincount(y, weights=counts.astype(np.float64), minlength=3)
        mine = np.where(nk > 0, counts.sum() / (np.count_nonzero(nk) * np.where(nk > 0, nk, 1.0)), 0.0)
        np.testing.assert_array_equal(mine, tree_class_weights("balanced_subsample", y, 3, int(s), True))


def test_unweighted_fit_stages_nothing(weighted_engine):
    from skdist.distribute.ensemble import DistExtraTreesClassifier
    X, y = _data()
    eng = _seed_map(1, 3, len(y))
    DistExtraTreesClassifier(n_estimators=3, random_state=1).fit(X, y)
    assert eng.staged == []


@pytest.mark.parametrize("kind", ["rf", "et"])
@pytest.mark.parametrize("cw", [{0: 2.0, 1: 0.0, 2: 0.5}, "balanced", "balanced_subsample"])
def test_fit_pipeline_equals_the_restatement(weighted_engine, monkeypatch, kind, cw):
    """Several chunks (each stages again), trees wrapped into scikit-learn trees: the forest equals the
    restated reference tree for tree; with balanced_subsample it also equals scikit-learn's own forest."""
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier
    monkeypatch.setenv("SKDIST_B200_FOREST_CHUNK", "3")
    X, y = _data(k=3)
    n_trees, rs = 7, 11
    eng = _seed_map(rs, n_trees, len(y))
    Dist, Sk = (DistRandomForestClassifier, RandomForestClassifier) if kind == "rf" else \
        (DistExtraTreesClassifier, ExtraTreesClassifier)
    bootstrap = kind == "rf"
    kw = dict(n_estimators=n_trees, random_state=rs, class_weight=cw, max_depth=6, min_samples_leaf=2)
    ours = Dist(**kw).fit(X, y)
    assert len(eng.staged) == 3
    trees = restated_forest(X, y, n_trees, rs, cw, bootstrap, splitter=0 if kind == "rf" else 1,
                            max_features="sqrt", max_depth=6, min_samples_leaf=2)
    _same_trees(ours.estimators_, trees)
    if cw == "balanced_subsample" or not bootstrap:      # scikit-learn 1.9 agrees in these cases
        _same_trees(ours.estimators_, Sk(**kw).fit(X, y).estimators_)


def test_warm_start_with_class_weight(weighted_engine):
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = _data()
    _seed_map(9, 7, len(y))
    warm = DistRandomForestClassifier(n_estimators=3, random_state=9, warm_start=True, class_weight="balanced").fit(X, y)
    warm.set_params(n_estimators=7)
    warm.fit(X, y)
    cold = DistRandomForestClassifier(n_estimators=7, random_state=9, class_weight="balanced").fit(X, y)
    _same_trees(warm.estimators_, cold.estimators_)


@pytest.mark.parametrize("cw", ["subsample", [{0: 1.0, 1: 2.0}], "unknown"])
def test_unsupported_class_weights_raise(weighted_engine, cw):
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = _data(k=2)
    with pytest.raises(NotImplementedError, match="class_weight"):
        DistRandomForestClassifier(n_estimators=2, random_state=0, class_weight=cw).fit(X, y)


def test_sample_weight_still_raises(weighted_engine):
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = _data(k=2)
    with pytest.raises(NotImplementedError):
        DistRandomForestClassifier(n_estimators=2, class_weight="balanced").fit(X, y, sample_weight=np.ones(len(y)))


# ---- the weighted float32 rank of csrc/forest_fast.cu (ff_rank<CM, true>) ----------------------------------

def _rank32_weighted(sl, st, cw):
    """ff_rank<CM, true>: weights scaled by the power of two that brings the largest into [1/2, 1), rounded to
    float32; a_c = cw_c * l_c and b_c = cw_c * r_c rounded to float32; w_l, w_r their float32 sums; fused
    multiply-adds; two divisions (__fdividef: within 2 ulp, added by the caller).  Returns the rank in the
    units of the unscaled weights (the device compares it with bars scaled by the same factor)."""
    _, e = np.frexp(cw.max())
    scale = np.ldexp(1.0, -int(e))
    cwf = (cw * scale).astype(np.float32)
    wl = wr = sql = sqr = np.float32(0)
    for c in range(len(st)):
        a = np.float32(cwf[c] * np.float32(sl[c]))
        b = np.float32(cwf[c] * np.float32(st[c] - sl[c]))
        wl = np.float32(wl + a)
        wr = np.float32(wr + b)
        sql = np.float32(np.float64(a) * np.float64(a) + np.float64(sql))
        sqr = np.float32(np.float64(b) * np.float64(b) + np.float64(sqr))
    r32 = np.float32(sql / wl) + np.float32(sqr / wr)
    return float(r32) / scale, (float(sql / wl) + float(sqr / wr)) / scale


@pytest.mark.parametrize("C", [2, 3, 4])
def test_weighted_float32_rank_is_within_its_bar(C):
    """|rank32 - exact| <= 2^-18 * w_node for weighted sums (bar FF_BAR_W = 2^-17 * w_node: a candidate more
    than the bar below the best cannot win in float64 either), on weights spread over the 2^40 the host
    allows the fast builder, "balanced"-like weights and node sums up to 2^32."""
    rng = np.random.default_rng(10 + C)
    worst = 0.0
    for trial in range(3000):
        scale = 10 ** rng.integers(0, 9)
        st = rng.integers(1, 10 * scale, size=C).astype(np.int64)
        if st.sum() >= 2 ** 32:
            st = (st * (2 ** 32 - 1) // st.sum()).clip(1)
        sl = np.array([rng.integers(0, s + 1) for s in st], dtype=np.int64)
        if sl.sum() == 0 or sl.sum() == st.sum():
            continue
        if trial % 3 == 0:
            cw = st.sum() / (C * st.astype(np.float64))          # "balanced"-like
        else:
            cw = 2.0 ** rng.uniform(-40, 0, size=C) * 10.0 ** rng.uniform(-3, 3)
        r32, mag = _rank32_weighted(sl, st, cw)
        fc = [Fraction(float(x)) for x in cw]
        a = [fc[c] * int(sl[c]) for c in range(C)]
        b = [fc[c] * int(st[c] - sl[c]) for c in range(C)]
        wl, wr = sum(a), sum(b)
        wn = wl + wr
        exact = sum(x * x for x in a) / wl + sum(x * x for x in b) / wr
        err = abs(float(Fraction(r32) - exact)) + 2.0 ** -22 * mag
        worst = max(worst, err / float(wn))
        # the weighted proxy_impurity_improvement is rank - w_node exactly
        proxy = -wr * (1 - sum(x * x for x in b) / wr ** 2) - wl * (1 - sum(x * x for x in a) / wl ** 2)
        assert proxy == exact - wn
    assert worst <= 2.0 ** -18, worst


# ---- the restatement against the unmodified reference (tests/golden/make_forest_class_weight_pins.py) -------

def test_restatement_reproduces_the_reference_trees():
    """The reference's own `_build_trees` with dict (a weight of 0 among them), "balanced" and (without
    bootstrap) "balanced_subsample" weights, RandomForest and ExtraTrees, bootstrap on and off, recorded as
    pins: the restatement every parity test here and on the device compares with builds the same trees bit
    for bit -- including dict and "balanced" with bootstrap, where scikit-learn's own forests differ."""
    from tests.golden.make_forest_class_weight_pins import CASES, N_TREES, OUT, PARAMS, RANDOM_STATE
    pins = np.load(OUT)
    X, y = pins["X"], pins["y"]
    for name, splitter, cw, bootstrap in CASES:
        trees = restated_forest(X, y, N_TREES, RANDOM_STATE, cw, bootstrap, splitter, **PARAMS)
        for t, tree in enumerate(trees):
            tr = tree.tree_
            for field in ("children_left", "children_right", "feature", "threshold", "impurity",
                          "n_node_samples", "weighted_n_node_samples"):
                np.testing.assert_array_equal(getattr(tr, field), pins["%s_%d_%s" % (name, t, field)],
                                              err_msg="%s tree %d %s" % (name, t, field))
            np.testing.assert_array_equal(tr.value[:, 0, :], pins["%s_%d_value" % (name, t)])
