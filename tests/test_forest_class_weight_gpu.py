"""Forest classifiers with class_weight on the device, both tree builders, against the restated reference
task (tests/forest_class_weight_restate.py): bit for bit when every weighted sum is exact (integer or dyadic
weights), and otherwise node statistics to rounding with every differing split inside the rounding envelope
of DESIGN.md §4."""
from fractions import Fraction

import numpy as np
import pytest

from tests.forest_class_weight_restate import restated_forest, restated_tree, tree_class_weights

pytestmark = pytest.mark.gpu

BUILDERS = ["default", "general"]


@pytest.fixture
def builder(request, monkeypatch):
    if request.param == "general":
        monkeypatch.setenv("SKDIST_B200_FOREST_KERNEL", "general")
    return request.param


def lattice(n, d, k, seed, levels=24, counts=None):
    rng = np.random.default_rng(seed)
    Z = rng.standard_normal((n, d))
    X = np.clip(np.floor((Z + 3.0) / 6.0 * levels), 0, levels - 1).astype(np.float32)
    s = Z[:, 0] + 0.5 * Z[:, 1] * Z[:, 2] - 0.7 * Z[:, 3] + 0.8 * rng.standard_normal(n)
    order = np.argsort(s, kind="stable")
    y = np.empty(n, np.int64)
    if counts is None:
        counts = [n // k + (1 if j < n % k else 0) for j in range(k)]
    y[order] = np.repeat(np.arange(k), counts)
    return X, y


def same_trees(ests, trees, wscale=1.0):
    assert len(ests) == len(trees)
    for a, b in zip(ests, trees):
        x, z = a.tree_, b.tree_
        assert x.node_count == z.node_count and x.max_depth == z.max_depth
        np.testing.assert_array_equal(x.children_left, z.children_left)
        np.testing.assert_array_equal(x.children_right, z.children_right)
        np.testing.assert_array_equal(x.feature, z.feature)
        np.testing.assert_array_equal(x.threshold, z.threshold)
        np.testing.assert_array_equal(x.n_node_samples, z.n_node_samples)
        np.testing.assert_array_equal(x.weighted_n_node_samples, z.weighted_n_node_samples * wscale)
        np.testing.assert_array_equal(x.impurity, z.impurity)
        np.testing.assert_array_equal(x.value, z.value)


def _classes(kind):
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier
    return (DistRandomForestClassifier, 0) if kind == "rf" else (DistExtraTreesClassifier, 1)


DYADIC = {2: {0: 0.5, 1: 2.0}, 3: {0: 4.0, 1: 0.0, 2: 0.5}, 4: {0: 2.0, 1: 0.25, 2: 1.0, 3: 3.0},
          8: {0: 2.0, 1: 0.5, 2: 0.0, 3: 4.0, 5: 0.125, 6: 3.0, 7: 1.5}}
VARIANTS = [dict(), dict(bootstrap=False, max_depth=7), dict(min_samples_leaf=3, max_features=5),
            dict(min_weight_fraction_leaf=0.02), dict(min_impurity_decrease=0.002)]


@pytest.mark.parametrize("builder", BUILDERS, indirect=True)
@pytest.mark.parametrize("kind", ["rf", "et"])
@pytest.mark.parametrize("k", [2, 3, 4, 8])
def test_dyadic_weights_bit_identical(builder, kind, k):
    """Dict weights (a 0 among them) and "balanced" weights that the class counts n/8, n/8, n/4, n/2 make
    dyadic: every weighted sum is exact, so the trees equal the restated reference bit for bit."""
    from skdist.distribute.predict import batch_predict
    Dist, splitter = _classes(kind)
    X, y = lattice(4096, 12, k, seed=k)
    for i, v in enumerate(VARIANTS):
        bootstrap = v.get("bootstrap", kind == "rf")
        kw = dict(n_estimators=3, random_state=i + 3, **v)
        ours = Dist(class_weight=DYADIC[k], **kw).fit(X, y)
        params = {p: v[p] for p in v if p != "bootstrap"}
        params.setdefault("max_features", "sqrt")
        want = restated_forest(X, y, 3, i + 3, DYADIC[k], bootstrap, splitter, **params)
        same_trees(ours.estimators_, want)
    np.testing.assert_array_equal(batch_predict(ours, X[:500], "predict_proba"), ours.predict_proba(X[:500]))
    np.testing.assert_array_equal(batch_predict(ours, X[:500], "predict"), ours.predict(X[:500]))
    if k == 4:
        Xb, yb = lattice(4096, 12, 4, seed=9, counts=[512, 512, 1024, 2048])
        for bs in (True, False):
            ours = Dist(n_estimators=3, random_state=1, bootstrap=bs, class_weight="balanced").fit(Xb, yb)
            same_trees(ours.estimators_, restated_forest(Xb, yb, 3, 1, "balanced", bs, splitter, max_features="sqrt"))


@pytest.mark.parametrize("builder", BUILDERS, indirect=True)
@pytest.mark.parametrize("kind", ["rf", "et"])
def test_unit_weights_and_power_of_two_scaling(builder, kind):
    """{k: 1.0} gives the bytes of class_weight=None; scaling every weight by 2^k keeps structure, values and
    impurities and scales weighted_n_node_samples exactly."""
    Dist, _ = _classes(kind)
    X, y = lattice(5000, 10, 3, seed=4)
    a = Dist(n_estimators=4, random_state=2).fit(X, y)
    b = Dist(n_estimators=4, random_state=2, class_weight={0: 1.0, 1: 1.0, 2: 1.0}).fit(X, y)
    same_trees(b.estimators_, a.estimators_)
    cw = {0: 0.3, 1: 1.7, 2: 0.9}
    for e in (-3, 5):
        base = Dist(n_estimators=3, random_state=6, class_weight=cw, min_weight_fraction_leaf=0.01).fit(X, y)
        scaled = Dist(n_estimators=3, random_state=6, class_weight={c: w * 2.0 ** e for c, w in cw.items()},
                      min_weight_fraction_leaf=0.01).fit(X, y)
        same_trees(scaled.estimators_, base.estimators_, wscale=2.0 ** e)


def _node_rows(tree, X, rows):
    """rows of `rows` reaching each node of `tree`, as a dict node -> index array."""
    out = {0: rows}
    for node in range(tree.node_count):
        if node not in out or tree.children_left[node] < 0:
            continue
        r = out[node]
        go = X[r, tree.feature[node]].astype(np.float64) <= tree.threshold[node]
        out[tree.children_left[node]] = r[go]
        out[tree.children_right[node]] = r[~go]
    return out


def envelope(n_node, C, w_node):
    """DESIGN.md §4: each computation's Gini proxy is within E = (11 kappa + C + 8) 2^-53 w_node of the exact
    one, kappa = 2 n_node + C + 2, provided both children weigh at least 4 kappa 2^-53 w_node; two splits
    chosen differently by the two computations have exact proxies within 2 E.  Returns (2 E, kappa 2^-53
    w_node)."""
    kappa = 2 * n_node + C + 2
    return 2 * (11 * kappa + C + 8) * 2.0 ** -53 * w_node, kappa * 2.0 ** -53 * w_node


def _exact_rank(X, y, counts, cw, rows, f, thr):
    """sum_l^2 / w_l + sum_r^2 / w_r of a split with the exact weights counts_i * cw[y_i] (rationals), and the
    smaller child weight."""
    fc = [Fraction(float(w)) for w in cw]
    left = X[rows, f].astype(np.float64) <= thr
    tot = []
    for side in (rows[left], rows[~left]):
        s = [Fraction(0)] * len(cw)
        for c in range(len(cw)):
            s[c] = fc[c] * int(counts[side][y[side] == c].sum())
        tot.append(s)
    (a, b) = tot
    return sum(x * x for x in a) / sum(a) + sum(x * x for x in b) / sum(b), float(min(sum(a), sum(b)))


def check_to_rounding(dev_tree, ref_tree, X, y, counts, cw, rtol=1e-11):
    """Walk both trees in lockstep, in build order (depth first, left child first).  Where they agree,
    n_node_samples match and weighted_n_node_samples, value and impurity agree within rtol.  At the first
    node where they split differently, both splits' exact proxies, on the node's rows, lie within the envelope
    of DESIGN.md §4 (`envelope`), or the node is pure and one of them split it on impurity rounding noise.
    The walk stops there: every later node draws its features from a random stream that the differing
    subtree has already advanced differently.  Returns 1 if the trees diverge."""
    a, b = dev_tree.tree_, ref_tree.tree_
    keep = np.flatnonzero((counts > 0) & (np.asarray(cw)[y] > 0))
    rows = _node_rows(a, X, keep)
    diverged = 0
    stack = [(0, 0)]
    while stack and not diverged:
        i, j = stack.pop()
        assert a.n_node_samples[i] == b.n_node_samples[j]
        np.testing.assert_allclose(a.weighted_n_node_samples[i], b.weighted_n_node_samples[j], rtol=rtol)
        np.testing.assert_allclose(a.value[i], b.value[j], rtol=rtol, atol=1e-300)
        np.testing.assert_allclose(a.impurity[i], b.impurity[j], rtol=1e-9, atol=1e-12)
        la, lb = a.children_left[i], b.children_left[j]
        if la < 0 and lb < 0:
            continue
        if la < 0 or lb < 0:
            # a pure node: its impurity is 0 in exact arithmetic, but sum_right = sum_total - sum_left and
            # w_right = w_node - w_left round differently in the two computations, and the rounding noise
            # can land on either side of EPSILON (one of them then splits the pure node)
            assert len(np.unique(y[rows[i]])) == 1, "one tree splits an impure node the other leaves as a leaf"
            diverged = 1
            continue
        if a.feature[i] == b.feature[j] and a.threshold[i] == b.threshold[j]:
            stack += [(a.children_right[i], b.children_right[j]), (la, lb)]
            continue
        diverged += 1
        r = rows[i]
        pa, wmin_a = _exact_rank(X, y, counts, cw, r, a.feature[i], a.threshold[i])
        pb, wmin_b = _exact_rank(X, y, counts, cw, r, b.feature[j], b.threshold[j])
        env, kappa_w = envelope(len(r), len(cw), a.weighted_n_node_samples[i])
        assert min(wmin_a, wmin_b) >= 4 * kappa_w, "the envelope's condition on the children's weights fails"
        assert abs(float(pa - pb)) <= env, (float(pa - pb), env)
    return diverged


@pytest.mark.parametrize("builder", BUILDERS, indirect=True)
@pytest.mark.parametrize("kind,k", [("rf", 2), ("rf", 3), ("rf", 4), ("rf", 8), ("et", 3)])
@pytest.mark.parametrize("cw", ["balanced", "balanced_subsample"])
def test_non_dyadic_weights_agree_to_rounding(builder, kind, k, cw):
    from skdist.distribute.ensemble import MAX_RAND_SEED, _tree_inputs
    from sklearn.utils import check_random_state
    from sklearn.utils.class_weight import compute_sample_weight
    Dist, splitter = _classes(kind)
    X, y = lattice(3001, 10, k, seed=11 + k, counts=None)
    y[:7] = k - 1                                                  # uneven class counts: non-dyadic weights
    bootstrap = kind == "rf"
    ours = Dist(n_estimators=4, random_state=3, class_weight=cw, max_depth=10).fit(X, y)
    states = check_random_state(3).randint(MAX_RAND_SEED, size=4)
    for t, s in zip(ours.estimators_, states):
        counts, _ = _tree_inputs(s, len(y), bootstrap)
        ref, w = restated_tree(X, y, k, s, cw, bootstrap, splitter, max_features="sqrt", max_depth=10)
        check_to_rounding(t, ref, X, y, counts.astype(np.int64), w)
        if cw == "balanced_subsample" and bootstrap:                 # the root value: scikit-learn's weights
            idx = check_random_state(s).randint(0, len(y), len(y))
            sw = compute_sample_weight("balanced", y, indices=idx) * counts
            root = np.bincount(y, weights=sw, minlength=k)
            np.testing.assert_allclose(t.tree_.value[0, 0], root / root.sum(), rtol=1e-13)
            np.testing.assert_allclose(t.tree_.weighted_n_node_samples[0], root.sum(), rtol=1e-13)
        # a restatement with one weight off by 1 % is told apart
        bad, wb = restated_tree(X, y, k, s, cw, bootstrap, splitter, cw_scale={0: 1.01}, max_features="sqrt",
                                max_depth=10)
        with pytest.raises(AssertionError):
            check_to_rounding(t, bad, X, y, counts.astype(np.int64), w)


@pytest.mark.parametrize("builder", BUILDERS, indirect=True)
def test_agrees_with_scikit_learns_own_forests(builder):
    """"balanced_subsample", and any weights without bootstrap: scikit-learn 1.9's forests fit the same trees."""
    from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier
    X, y = lattice(4096, 12, 4, seed=2, counts=[512, 512, 1024, 2048])
    kw = dict(n_estimators=4, random_state=8, class_weight="balanced_subsample")
    ours = DistRandomForestClassifier(**kw).fit(X, y)
    ref = RandomForestClassifier(**kw).fit(X, y)
    n_div = 0
    for t, r in zip(ours.estimators_, ref.estimators_):
        from skdist_b200.distribute.ensemble import _tree_inputs
        counts, _ = _tree_inputs(r.random_state, len(y), True)
        n_div += check_to_rounding(t, r, X, y, counts.astype(np.int64),
                                   tree_class_weights("balanced_subsample", y, 4, r.random_state, True))
    if n_div == 0:
        np.testing.assert_allclose(ours.predict_proba(X[:300]), ref.predict_proba(X[:300]), rtol=0, atol=1e-12)
    kw = dict(n_estimators=3, random_state=5, class_weight={0: 0.5, 1: 2.0, 2: 1.0, 3: 4.0})
    same_trees(DistExtraTreesClassifier(**kw).fit(X, y).estimators_, ExtraTreesClassifier(**kw).fit(X, y).estimators_)
    same_trees(DistRandomForestClassifier(bootstrap=False, **kw).fit(X, y).estimators_,
               RandomForestClassifier(bootstrap=False, **kw).fit(X, y).estimators_)


@pytest.mark.parametrize("k", [2, 3, 4])
@pytest.mark.parametrize("cw", ["balanced", "balanced_subsample", {0: 0.3, 1: 1.7, 2: 0.9, 3: 2.2}])
def test_builders_agree_bit_for_bit_with_non_dyadic_weights(monkeypatch, k, cw):
    """The throughput builder (float32 screening, compact records expanded on the host) and the general
    builder evaluate the same float64 expressions: with non-dyadic weights too they build the same trees and
    report the same node statistics, right children's impurities included."""
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = lattice(6001, 16, k, seed=30 + k)
    y[:11] = k - 1
    cwk = {c: w for c, w in cw.items() if c < k} if isinstance(cw, dict) else cw
    kw = dict(n_estimators=6, random_state=12, class_weight=cwk, min_weight_fraction_leaf=0.001)
    fast = DistRandomForestClassifier(**kw).fit(X, y)
    monkeypatch.setenv("SKDIST_B200_FOREST_KERNEL", "general")
    general = DistRandomForestClassifier(**kw).fit(X, y)
    same_trees(fast.estimators_, general.estimators_)
