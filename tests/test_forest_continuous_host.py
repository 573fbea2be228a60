"""scikit-learn's random splitter over raw float32 values restated in numpy, the arithmetic the general tree
builder's random branch (csrc/forest.cu) performs: min and max of the node's values, the constant test in
float32, one threshold rand_uniform(min, max) in float64 that falls back to min when it lands on max, and
(double)x <= threshold to the left.  The restated trees are checked against ExtraTreeClassifier /
ExtraTreeRegressor on small continuous inputs, adversarial columns included.  No GPU."""
import numpy as np
import pytest
from sklearn.tree import ExtraTreeClassifier, ExtraTreeRegressor

from skdist_b200.distribute.ensemble import RAND_R_MAX, _tree_inputs

FEATURE_THRESHOLD = np.float32(1e-7)
EPSILON = np.finfo(np.float64).eps


def rand_r(state):
    """SK/utils/_random.pxd our_rand_r on a one-element uint32 state."""
    s = int(state[0]) or 1
    s ^= (s << 13) & 0xFFFFFFFF
    s ^= s >> 17
    s ^= (s << 5) & 0xFFFFFFFF
    state[0] = s
    return s % (RAND_R_MAX + 1)


def is_constant(lo, hi):
    """max <= min + FEATURE_THRESHOLD, evaluated in float32."""
    return bool(np.float32(hi) <= np.float32(lo) + FEATURE_THRESHOLD)


def draw_threshold(lo, hi, r):
    """rand_uniform(min, max) (SK/tree/_utils.pyx) in float64; min when it lands on max."""
    lo, hi = float(lo), float(hi)
    thr = (hi - lo) * float(r) / float(RAND_R_MAX) + lo
    return lo if thr == hi else thr


def goes_left(values, thr):
    return values.astype(np.float64) <= thr


class _Stats:
    """Node statistics: class counts (Gini) or (w, sum y, sum y^2) (squared error), unit weights."""

    def __init__(self, y, n_classes):
        self.y, self.k = y, n_classes

    def of(self, rows):
        if self.k:
            return np.bincount(self.y[rows], minlength=self.k).astype(np.float64)
        y = self.y[rows]
        return np.array([float(len(rows)), float(np.sum(y)), float(np.sum(y * y))])

    def impurity(self, s):
        if self.k:
            w = s.sum()
            return 1.0 - float(np.sum(s * s)) / (w * w)
        m = s[1] / s[0]
        return s[2] / s[0] - m * m

    def proxy(self, sl, sr):
        if self.k:
            return -sr.sum() * self.impurity(sr) - sl.sum() * self.impurity(sl)
        return sl[1] * sl[1] / sl[0] + sr[1] * sr[1] / sr[0]

    def value(self, s):
        return s / s.sum() if self.k else np.array([s[1] / s[0]])


def restated_extra_tree(X, y, n_classes, seed, max_features, max_depth=None, min_samples_split=2,
                        min_samples_leaf=1):
    """DepthFirstTreeBuilder + node_split_random over raw values (SK/tree/_tree.pyx, _splitter.pyx);
    n_classes = 0: squared error.  Returns the node arrays."""
    n, d = X.shape
    st = _Stats(y, n_classes)
    _, rs = _tree_inputs(seed, n, False)
    state = np.array([rs], np.uint64)
    max_depth = np.iinfo(np.int32).max if max_depth is None else max_depth
    features, constant = list(range(d)), [0] * d
    nodes = []
    rows0 = np.arange(n)
    stack = [(rows0, 0, -1, False, np.inf, 0)]
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
                lo, hi = v.min(), v.max()
                if is_constant(lo, hi):
                    features[f_j], features[n_total] = features[n_total], f
                    n_found += 1
                    n_total += 1
                    continue
                f_i -= 1
                features[f_i], features[f_j] = features[f_j], features[f_i]
                thr = draw_threshold(lo, hi, rand_r(state))
                left = goes_left(v, thr)
                n_left = int(left.sum())
                if n_left < min_samples_leaf or w - n_left < min_samples_leaf:
                    continue
                sl, sr = st.of(rows[left]), st.of(rows[~left])
                proxy = st.proxy(sl, sr)
                if proxy > best_proxy:
                    best_proxy, best = proxy, (f, thr, left, sl, sr)
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
    cls = ExtraTreeClassifier if n_classes else ExtraTreeRegressor
    t = cls(random_state=int(seed), **params).fit(X, y).tree_
    mf = params.get("max_features", "sqrt" if n_classes else None)
    mf_i = {None: X.shape[1], "sqrt": max(1, int(np.sqrt(X.shape[1])))}.get(mf, mf)
    got = restated_extra_tree(X, y, n_classes, seed, mf_i, **{k: v for k, v in params.items() if k != "max_features"})
    np.testing.assert_array_equal(got["left"], t.children_left)
    np.testing.assert_array_equal(got["right"], t.children_right)
    np.testing.assert_array_equal(got["feature"], t.feature)
    np.testing.assert_array_equal(got["threshold"], t.threshold)
    np.testing.assert_array_equal(got["n"], t.n_node_samples)
    np.testing.assert_array_equal(got["impurity"], t.impurity)
    np.testing.assert_array_equal(got["value"], t.value[:, 0, :])


def adversarial(n, seed):
    rng = np.random.default_rng(seed)
    one = np.float32(1.0)
    return np.stack([np.full(n, 3.5, np.float32),
                     np.where(rng.random(n) < 0.5, one, np.nextafter(one, np.float32(2))).astype(np.float32),
                     np.where(rng.random(n) < 0.3, -1.0, 2.0).astype(np.float32),
                     np.round(rng.standard_normal(n) * 2).astype(np.float32),
                     (1e6 + rng.standard_normal(n) * 50).astype(np.float32),
                     rng.integers(0, 7, n).astype(np.float32),
                     rng.standard_normal(n).astype(np.float32)], axis=1)


def test_constant_test_is_float32():
    one = np.float32(1.0)
    ulp = np.nextafter(one, np.float32(2))
    assert is_constant(one, ulp)                      # one float32 ulp (1.19e-7) apart: constant in float32 ...
    assert not float(ulp) <= float(one) + 1e-7        # ... but not in float64
    assert not is_constant(one, np.nextafter(ulp, np.float32(2)))
    assert is_constant(2.5, 2.5)


def test_threshold_is_float64_and_falls_back_to_min():
    lo, hi = np.float32(-1.25), np.float32(3.0)
    assert draw_threshold(lo, hi, 0) == -1.25
    assert draw_threshold(lo, hi, RAND_R_MAX) == -1.25            # lands on max: min
    t = draw_threshold(lo, hi, 123456789)
    assert t == (3.0 + 1.25) * 123456789.0 / RAND_R_MAX - 1.25 and t != float(np.float32(t))
    v = np.array([lo, np.float32(t), np.nextafter(np.float32(t), np.float32(9)), hi], np.float32)
    left = goes_left(v, t)                                          # (double)x <= thr
    assert left[0] and not left[3] and left[2] == (float(v[2]) <= t) and left[1] == (float(v[1]) <= t)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_classifier_matches_scikit_learn(seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((300, 6)).astype(np.float32)
    y = (X[:, 0] + X[:, 1] * X[:, 2] + 0.3 * rng.standard_normal(300) > 0).astype(np.int64) + (X[:, 3] > 1)
    check_against_sklearn(X, y, 3, 100 + seed)
    check_against_sklearn(X, y, 3, 200 + seed, max_depth=4, min_samples_leaf=5)
    check_against_sklearn(X, y, 3, 300 + seed, max_features=None, min_samples_split=10)


@pytest.mark.parametrize("seed", [0, 1])
def test_regressor_matches_scikit_learn(seed):
    rng = np.random.default_rng(10 + seed)
    X = rng.standard_normal((250, 5)).astype(np.float32)
    y = np.round(3 * X[:, 0] + X[:, 1] ** 2 + rng.standard_normal(250))      # integers: exact sums
    check_against_sklearn(X, y, 0, 400 + seed)
    check_against_sklearn(X, y, 0, 500 + seed, max_features=1, max_depth=6)


def test_adversarial_columns_match_scikit_learn():
    X = adversarial(400, 5)
    rng = np.random.default_rng(6)
    y = ((X[:, 2] + X[:, 3] * 0.3 + (X[:, 4] - 1e6) / 50 + X[:, 6] + rng.standard_normal(400)) > 0).astype(np.int64)
    for seed in (7, 8, 9):
        check_against_sklearn(X, y, 2, seed)
        check_against_sklearn(X, y, 2, seed, max_features=None)
        check_against_sklearn(X, y.astype(np.float64), 0, seed, max_features=1)
