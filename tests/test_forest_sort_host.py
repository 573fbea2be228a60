"""scikit-learn's best splitter over raw float32 values restated in numpy, the contract the general tree builder's
sort-based mode (csrc/forest.cu, FO_SORT) implements: sort the node's values, call the feature constant when
max <= min + 1e-7 in float32, put a candidate after position p - 1 when v[p] > v[p-1] + 1e-7 in float32 (runs
chained by smaller gaps stay whole), skip candidates that break min_samples_leaf, keep the first strictly
larger proxy, threshold v[p-1]/2 + v[p]/2 in float64, and send (double)x <= threshold left.  The restated trees
are checked against DecisionTreeClassifier / DecisionTreeRegressor on adversarial columns.  Then the
SKDIST_B200_FOREST_SORT switch on an engine double.  No GPU."""
import numpy as np
import pytest
from sklearn.tree import DecisionTreeClassifier, DecisionTreeRegressor

from skdist_b200.distribute.ensemble import _tree_inputs
from tests.fake_engine import FakeEngine
from tests.test_forest_continuous_host import EPSILON, FEATURE_THRESHOLD, _Stats, adversarial, is_constant, rand_r


def best_split(v, rows, st, min_samples_leaf):
    """node_split_best for one feature (rules 1-6): (proxy, threshold, left mask) or None."""
    order = np.argsort(v, kind="stable")          # any order of equal values gives the same candidates
    vs = v[order]
    w = len(rows)
    onehot = st.k and np.eye(st.k)[st.y[rows[order]]]
    cum = np.cumsum(onehot, axis=0) if st.k else None
    best, best_proxy = None, -np.inf
    for p in range(1, w):
        if not vs[p] > vs[p - 1] + FEATURE_THRESHOLD:      # float32: the same run
            continue
        if p < min_samples_leaf or w - p < min_samples_leaf:
            continue
        if st.k:                                           # integer counts: exact in any order
            sl = cum[p - 1]
            sr = cum[-1] - sl
        else:
            sl, sr = st.of(rows[order[:p]]), st.of(rows[order[p:]])
        proxy = st.proxy(sl, sr)
        if proxy > best_proxy:
            thr = float(vs[p - 1]) / 2.0 + float(vs[p]) / 2.0
            if thr == float(vs[p]) or np.isinf(thr):
                thr = float(vs[p - 1])
            best_proxy, best = proxy, (thr, sl, sr)
    if best is None:
        return None
    thr, sl, sr = best
    left = v.astype(np.float64) <= thr                     # rule 7: the partition by value gives the left side
    np.testing.assert_array_equal(st.of(rows[left]), sl)
    return best_proxy, thr, left, sl, sr


def restated_tree(X, y, n_classes, seed, max_features, max_depth=None, min_samples_split=2, min_samples_leaf=1):
    """DepthFirstTreeBuilder + node_split_best over raw values; n_classes = 0: squared error."""
    n, d = X.shape
    st = _Stats(y, n_classes)
    _, rs = _tree_inputs(seed, n, False)
    state = np.array([rs], np.uint64)
    max_depth = np.iinfo(np.int32).max if max_depth is None else max_depth
    features, constant = list(range(d)), [0] * d
    nodes = []
    stack = [(np.arange(n), 0, -1, False, np.inf, 0)]
    first = True
    while stack:
        rows, depth, parent, is_left, impurity, n_known = stack.pop()
        s = st.of(rows)
        w = len(rows)
        is_leaf = depth >= max_depth or w < min_samples_split or w < 2 * min_samples_leaf
        if first:
            impurity, first = st.impurity(s), False
        is_leaf = is_leaf or impurity <= EPSILON
        best = None
        n_total = n_known
        if not is_leaf:
            f_i, n_visited, n_found, n_drawn, best_proxy = d, 0, 0, 0, -np.inf
            while f_i > n_total and (n_visited < max_features or n_visited <= n_found + n_drawn):
                n_visited += 1
                f_j = n_drawn + rand_r(state) % (f_i - n_found - n_drawn)
                if f_j < n_known:
                    features[n_drawn], features[f_j] = features[f_j], features[n_drawn]
                    n_drawn += 1
                    continue
                f_j += n_found
                f = features[f_j]
                v = X[rows, f]
                if is_constant(v.min(), v.max()):
                    features[f_j], features[n_total] = features[n_total], f
                    n_found += 1
                    n_total += 1
                    continue
                f_i -= 1
                features[f_i], features[f_j] = features[f_j], features[f_i]
                r = best_split(v, rows, st, min_samples_leaf)
                if r is not None and r[0] > best_proxy:          # across features in draw order, strict '>'
                    best_proxy, best = r[0], (f,) + r[1:]
            features[:n_known] = constant[:n_known]
            constant[n_known:n_total] = features[n_known:n_total]
            if best is not None:
                f, thr, left, sl, sr = best
                il, ir = st.impurity(sl), st.impurity(sr)
                wl, wr = sl[0] if not n_classes else sl.sum(), sr[0] if not n_classes else sr.sum()
                improvement = (w / n) * (impurity - wr / w * ir - wl / w * il)
                is_leaf = improvement + EPSILON < 0.0
        node = len(nodes)
        if parent >= 0:
            nodes[parent]["left" if is_left else "right"] = node
        nodes.append(dict(left=-1, right=-1, feature=-2, threshold=-2.0, n=w, impurity=impurity, value=st.value(s)))
        if not is_leaf and best is not None:
            f, thr, left, sl, sr = best
            nodes[node].update(feature=f, threshold=thr)
            stack.append((rows[~left], depth + 1, node, False, st.impurity(sr), n_total))
            stack.append((rows[left], depth + 1, node, True, st.impurity(sl), n_total))
    return {k: np.array([nd[k] for nd in nodes]) for k in nodes[0]}


def check_against_sklearn(X, y, n_classes, seed, **params):
    cls = DecisionTreeClassifier if n_classes else DecisionTreeRegressor
    t = cls(random_state=int(seed), **params).fit(X, y).tree_
    mf = params.get("max_features")
    mf_i = {None: X.shape[1], "sqrt": max(1, int(np.sqrt(X.shape[1])))}.get(mf, mf)
    got = restated_tree(X, y, n_classes, seed, mf_i, **{k: v for k, v in params.items() if k != "max_features"})
    np.testing.assert_array_equal(got["left"], t.children_left)
    np.testing.assert_array_equal(got["right"], t.children_right)
    np.testing.assert_array_equal(got["feature"], t.feature)
    np.testing.assert_array_equal(got["threshold"], t.threshold)
    np.testing.assert_array_equal(got["n"], t.n_node_samples)
    np.testing.assert_array_equal(got["impurity"], t.impurity)
    np.testing.assert_array_equal(got["value"], t.value[:, 0, :])


def extra_columns(n, seed):
    """Runs chained by gaps <= 1e-7 spanning more than 1e-7, adjacent float32 values near 1e6, signed zeros."""
    rng = np.random.default_rng(seed)
    ulp = np.float32(2.0 ** -24)                                   # float32 spacing in [0.5, 1): 6e-8
    chain = np.where(rng.random(n) < 0.5, np.float32(0.5), np.float32(0.75)) + rng.integers(0, 12, n) * ulp
    big = np.float32(1e6) + rng.integers(0, 40, n).astype(np.float32) * np.float32(0.0625)
    zeros = rng.choice(np.array([-0.0, 0.0, 1.0, -1.0], np.float32), n)
    return np.stack([chain.astype(np.float32), big.astype(np.float32), zeros], axis=1)


def test_run_rule_chains_small_gaps():
    """Three values 6e-8 apart: two float32 gaps below 1e-7, one run although it spans 1.2e-7."""
    a = np.float32(0.5)
    v = np.array([a, a + np.float32(2.0 ** -24), a + np.float32(2.0 ** -23)], np.float32)
    assert float(v[2]) - float(v[0]) > 1e-7
    assert not any(v[p] > v[p - 1] + FEATURE_THRESHOLD for p in (1, 2))
    st = _Stats(np.array([0, 1, 1]), 2)
    assert best_split(v, np.arange(3), st, 1) is None


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_classifier_matches_scikit_learn(seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((300, 6)).astype(np.float32)
    y = (X[:, 0] + X[:, 1] * X[:, 2] + 0.3 * rng.standard_normal(300) > 0).astype(np.int64) + (X[:, 3] > 1)
    check_against_sklearn(X, y, 3, 100 + seed, max_features="sqrt")
    check_against_sklearn(X, y, 3, 200 + seed, max_features="sqrt", max_depth=4, min_samples_leaf=5)
    check_against_sklearn(X, y, 3, 300 + seed, min_samples_split=10)


def test_adversarial_columns_match_scikit_learn():
    X = np.concatenate([adversarial(400, 5), extra_columns(400, 6)], axis=1)
    rng = np.random.default_rng(6)
    s = X[:, 2] + X[:, 3] * 0.3 + (X[:, 4] - 1e6) / 50 + X[:, 6] + (X[:, 7] > 0.6) + (X[:, 9] > 0.5)
    y = ((s + rng.standard_normal(400)) > 0).astype(np.int64)
    for seed in (7, 8, 9):
        check_against_sklearn(X, y, 2, seed, max_features="sqrt")
        check_against_sklearn(X, y, 2, seed, max_depth=4)
        check_against_sklearn(X, y.astype(np.float64) * 3 + (X[:, 8] > 1e6 + 1.2), 0, seed, max_features=1)


# ---------------------------------------------------------------- the switch

class SortEngine(FakeEngine):
    """The engine double, with the library's splitter 2 (best splitter, sorts features that have no bin
    codes) and its refusal of splitter 0 on a feature with more than 256 distinct values."""

    def __init__(self, device=0):
        super().__init__(device)
        self.splitters = []

    def forest_fit(self, sample_counts, rand_states, n_classes, max_features, max_depth, min_samples_split,
                   min_samples_leaf, min_weight_leaf, min_impurity_decrease, splitter=0, y_regression=None):
        self.splitters.append(splitter)
        distinct = [len(np.unique(self.X[:, f])) for f in range(self.d)]
        if splitter == 0 and max(distinct) > 256:
            f = int(np.argmax(np.array(distinct) > 256))
            raise NotImplementedError("forest: feature %d has %d distinct values; the histogram splitter needs "
                                      "<= 256 (continuous features need the sort-based splitter, not built yet)"
                                      % (f, distinct[f]))
        return super().forest_fit(sample_counts, rand_states, n_classes, max_features, max_depth, min_samples_split,
                                  min_samples_leaf, min_weight_leaf, min_impurity_decrease,
                                  0 if splitter == 2 else splitter, y_regression)


@pytest.fixture
def sort_engine(monkeypatch):
    from skdist_b200 import engine
    monkeypatch.delenv("SKDIST_B200_FOREST_SORT", raising=False)
    monkeypatch.delenv("SKDIST_B200_FOREST_MAX_BINS", raising=False)
    engine.set_engine_factory(SortEngine)
    yield engine.get_engine()
    engine.set_engine_factory(None)


def continuous(n=600, d=5, seed=3):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    return X, (X[:, 0] + 0.5 * X[:, 1] > 0).astype(int)


def seeds(eng, n, n_trees, random_state):
    from sklearn.utils import check_random_state
    from skdist_b200.distribute.ensemble import MAX_RAND_SEED
    states = check_random_state(random_state).randint(MAX_RAND_SEED, size=n_trees)
    eng.seed_of_rand_r = {int(_tree_inputs(s, n, False)[1]): int(s) for s in states}


def test_switch_selects_splitter_2_for_random_forests_only(sort_engine, monkeypatch):
    from sklearn.ensemble import RandomForestClassifier
    from skdist.distribute.ensemble import (DistExtraTreesClassifier, DistExtraTreesRegressor,
                                            DistRandomForestClassifier, DistRandomForestRegressor)
    X, y = continuous()
    seeds(sort_engine, len(y), 3, 4)
    monkeypatch.setenv("SKDIST_B200_FOREST_SORT", "1")
    ours = DistRandomForestClassifier(n_estimators=3, random_state=4).fit(X, y)
    ref = RandomForestClassifier(n_estimators=3, random_state=4).fit(X, y)
    for a, b in zip(ours.estimators_, ref.estimators_):
        np.testing.assert_array_equal(a.tree_.threshold, b.tree_.threshold)
    DistRandomForestRegressor(n_estimators=3, random_state=4).fit(X, y.astype(float))
    assert sort_engine.splitters == [2, 2]
    sort_engine.splitters.clear()
    DistExtraTreesClassifier(n_estimators=3, random_state=4).fit(X, y)
    DistExtraTreesRegressor(n_estimators=3, random_state=4).fit(X, y.astype(float))
    assert sort_engine.splitters == [1, 1]


def test_switch_unset_refuses_with_both_switches_named(sort_engine):
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = continuous()
    seeds(sort_engine, len(y), 2, 0)
    with pytest.raises(NotImplementedError, match="SKDIST_B200_FOREST_MAX_BINS") as e:
        DistRandomForestClassifier(n_estimators=2, random_state=0).fit(X, y)
    assert "SKDIST_B200_FOREST_SORT=1" in str(e.value) and "SKDIST_B200_FOREST_MAX_BINS=256" in str(e.value)
    assert sort_engine.splitters == [0]


@pytest.mark.parametrize("value", ["0", "2", "yes", ""])
def test_switch_bad_value_raises(sort_engine, monkeypatch, value):
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier
    X, y = continuous()
    monkeypatch.setenv("SKDIST_B200_FOREST_SORT", value)
    for cls in (DistRandomForestClassifier, DistExtraTreesClassifier):
        with pytest.raises(ValueError, match="SKDIST_B200_FOREST_SORT must be unset or 1"):
            cls(n_estimators=2, random_state=0).fit(X, y)
    assert sort_engine.splitters == []


def test_both_switches_raise(sort_engine, monkeypatch):
    from skdist.distribute.ensemble import DistRandomForestClassifier, DistRandomForestRegressor
    X, y = continuous()
    monkeypatch.setenv("SKDIST_B200_FOREST_SORT", "1")
    monkeypatch.setenv("SKDIST_B200_FOREST_MAX_BINS", "256")
    with pytest.raises(ValueError, match="different trees"):
        DistRandomForestClassifier(n_estimators=2, random_state=0).fit(X, y)
    with pytest.raises(ValueError, match="different trees"):
        DistRandomForestRegressor(n_estimators=2, random_state=0).fit(X, y.astype(float))
    assert sort_engine.splitters == []
