"""criterion="entropy" of the forest classifiers, without a GPU.

scikit-learn's entropy restated in numpy (SK/tree/_criterion.pyx Entropy, impurity in bits with
log(x) = ln(x) / ln(2.0) of SK/tree/_utils.pyx, zero classes skipped, the base proxy -w_r * imp_r - w_l * imp_l)
over both splitters on raw float32 values, bootstrap multiplicities as integer sample weights.  The restated
trees must equal DecisionTreeClassifier / ExtraTreeClassifier and the trees of RandomForestClassifier /
ExtraTreesClassifier bit for bit, impurity included.  The general tree builder (csrc/forest.cu, ENT
instantiations) makes the same choices with CUDA's log; the tie-sensitivity guard re-runs the restatement with
a log that is one ulp off on a few percent of its inputs, on every dataset of tests/test_forest_entropy_gpu.py,
and asserts the same structure, so a device mismatch there points at a bug and not at the last bit of log.
Then the criterion plumbing of the estimators on an engine double."""
import math

import numpy as np
import pytest
from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier
from sklearn.tree import DecisionTreeClassifier, ExtraTreeClassifier

from skdist_b200.distribute.ensemble import _tree_inputs
from tests.fake_engine import FakeEngine
from tests.test_forest_continuous_host import (EPSILON, FEATURE_THRESHOLD, adversarial, draw_threshold, goes_left,
                                               is_constant, rand_r)
from tests.test_forest_sort_host import extra_columns, seeds

LN2 = math.log(2.0)
_glibc_log = np.vectorize(math.log, otypes=[np.float64])    # the libm log scikit-learn calls (not numpy's SIMD log)


def perturbed_log(fraction=0.03):
    """math.log moved by one ulp (up or down) on about `fraction` of its inputs, chosen by a hash of the bits."""
    cut = int(fraction * 2 ** 16)

    def one(x):
        v = math.log(x)
        h = (np.float64(x).view(np.uint64).item() * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
        if (h >> 48) < cut:
            v = math.nextafter(v, math.inf if (h >> 47) & 1 else -math.inf)
        return v
    return np.vectorize(one, otypes=[np.float64])


def entropy(S, W, log):
    """Entropy in bits of every row of class sums S [m, k] with weights W [m], scikit-learn's operation order."""
    S = np.atleast_2d(S)
    W = np.atleast_1d(np.asarray(W, np.float64))
    e = np.zeros(len(W))
    for c in range(S.shape[1]):
        s = S[:, c]
        pos = s > 0
        p = np.where(pos, s / np.where(W > 0, W, 1.0), 1.0)
        t = p * (log(p) / LN2)
        e = np.where(pos, e - t, e)
    return e


def restated_entropy_tree(X, y, k, seed, max_features, splitter="best", bootstrap=False, max_depth=None,
                          min_samples_split=2, min_samples_leaf=1, min_impurity_decrease=0.0, log=_glibc_log):
    """DepthFirstTreeBuilder with node_split_best / node_split_random over raw values and the Entropy
    criterion; the bootstrap multiplicities of `seed` are the sample weights.  Returns the node arrays."""
    n, d = X.shape
    counts, rs = _tree_inputs(seed, n, bootstrap)
    cnt = counts.astype(np.float64)
    state = np.array([rs], np.uint64)
    max_depth = np.iinfo(np.int32).max if max_depth is None else max_depth
    of = lambda rows: np.bincount(y[rows], weights=cnt[rows], minlength=k)   # noqa: E731
    rows0 = np.flatnonzero(counts)                  # rows of weight 0 leave the tree (Splitter.init)
    w_total = cnt.sum()
    features, constant = list(range(d)), [0] * d
    nodes = []
    stack = [(rows0, 0, -1, False, np.inf, 0)]
    first = True
    while stack:
        rows, depth, parent, is_left, impurity, n_known = stack.pop()
        s = of(rows)
        w, m = s.sum(), len(rows)
        is_leaf = depth >= max_depth or m < min_samples_split or m < 2 * min_samples_leaf
        if first:
            impurity, first = entropy(s, w, log)[0], False
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
                if splitter == "random":
                    thr = draw_threshold(lo, hi, rand_r(state))
                    left = goes_left(v, thr)
                    n_left = int(left.sum())
                    if n_left < min_samples_leaf or m - n_left < min_samples_leaf:
                        continue
                    SL = of(rows[left])[None, :]
                    cand = [(thr, left)]
                else:
                    order = np.argsort(v, kind="stable")
                    vs = v[order]
                    M = np.zeros((m, k))
                    M[np.arange(m), y[rows[order]]] = cnt[rows[order]]
                    cum = np.cumsum(M, axis=0)                     # integer sums: exact in any order
                    p = np.arange(1, m)
                    ok = (vs[1:] > vs[:-1] + FEATURE_THRESHOLD) & (p >= min_samples_leaf) & (m - p >= min_samples_leaf)
                    p = p[ok]
                    if not len(p):
                        continue
                    SL = cum[p - 1]
                    cand = p
                SR = s[None, :] - SL
                wl = SL.sum(axis=1)
                wr = w - wl
                il, ir = entropy(SL, wl, log), entropy(SR, wr, log)
                proxy = (-wr) * ir - wl * il
                j = int(np.argmax(proxy))                          # the first of equal maxima: strict '>'
                if proxy[j] > best_proxy:
                    if splitter == "random":
                        thr, left = cand[0]
                    else:
                        q = cand[j]
                        thr = float(vs[q - 1]) / 2.0 + float(vs[q]) / 2.0
                        if thr == float(vs[q]) or np.isinf(thr):
                            thr = float(vs[q - 1])
                        left = goes_left(v, thr)
                    best_proxy, best = proxy[j], (f, thr, left, il[j], ir[j], wl[j], wr[j])
            features[:n_known] = constant[:n_known]
            constant[n_known:n_total] = features[n_known:n_total]
            if best is not None:
                f, thr, left, il, ir, wl, wr = best
                improvement = (w / w_total) * (impurity - wr / w * ir - wl / w * il)
                is_leaf = improvement + EPSILON < min_impurity_decrease
        node = len(nodes)
        if parent >= 0:
            nodes[parent]["left" if is_left else "right"] = node
        nodes.append(dict(left=-1, right=-1, feature=-2, threshold=-2.0, n=m, wn=w, impurity=impurity, value=s / w))
        if not is_leaf and best is not None:
            f, thr, left, il, ir, wl, wr = best
            nodes[node].update(feature=f, threshold=thr)
            stack.append((rows[~left], depth + 1, node, False, ir, n_total))
            stack.append((rows[left], depth + 1, node, True, il, n_total))
    return {key: np.array([nd[key] for nd in nodes]) for key in nodes[0]}


def assert_tree_equal(got, t, structure_only=False):
    np.testing.assert_array_equal(got["left"], t.children_left)
    np.testing.assert_array_equal(got["right"], t.children_right)
    np.testing.assert_array_equal(got["feature"], t.feature)
    np.testing.assert_array_equal(got["threshold"], t.threshold)
    np.testing.assert_array_equal(got["n"], t.n_node_samples)
    if structure_only:
        return
    np.testing.assert_array_equal(got["wn"], t.weighted_n_node_samples)
    np.testing.assert_array_equal(got["impurity"], t.impurity)
    np.testing.assert_array_equal(got["value"], t.value[:, 0, :])


def _mf(mf, d):
    if isinstance(mf, float):
        return max(1, int(mf * d))
    return {None: d, "sqrt": max(1, int(np.sqrt(d)))}.get(mf, mf)


def check_single_tree(X, y, k, seed, splitter="best", criterion="entropy", **params):
    cls = ExtraTreeClassifier if splitter == "random" else DecisionTreeClassifier
    mf = params.pop("max_features", "sqrt")
    t = cls(criterion=criterion, random_state=int(seed), max_features=mf, **params).fit(X, y).tree_
    got = restated_entropy_tree(X, y, k, seed, _mf(mf, X.shape[1]), splitter, False, **params)
    assert_tree_equal(got, t)


def check_forest(X, y, k, forest_cls, n_trees, random_state, log=_glibc_log, structure_only=False, **params):
    """Every tree of scikit-learn's forest against the restatement with `log`."""
    f = forest_cls(n_estimators=n_trees, criterion="entropy", random_state=random_state, **params).fit(X, y)
    splitter = "random" if forest_cls is ExtraTreesClassifier else "best"
    p = dict(params)
    bootstrap = p.pop("bootstrap", forest_cls is RandomForestClassifier)
    mf = _mf(p.pop("max_features", "sqrt"), X.shape[1])
    for est in f.estimators_:
        got = restated_entropy_tree(X, y, k, est.random_state, mf, splitter, bootstrap, log=log, **p)
        assert_tree_equal(got, est.tree_, structure_only)


# ------------------------------------------------------------------------- datasets

def lattice(n, d, k, seed):
    """Features on a lattice of <= 16 values (the histogram splitter), k classes."""
    rng = np.random.default_rng(seed)
    X = rng.integers(0, 16, (n, d)).astype(np.float32)
    s = X[:, 0] + 0.7 * X[:, 1] - 0.4 * X[:, 2] + rng.normal(0, 3, n)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, k + 1)[1:-1])).astype(np.int64)
    return X, y


def gaussian(n, d, k, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    s = X[:, 0] + X[:, 1] * X[:, 2] + 0.5 * rng.standard_normal(n)
    y = np.digitize(s, np.quantile(s, np.linspace(0, 1, k + 1)[1:-1])).astype(np.int64)
    return X, y


# The datasets of tests/test_forest_entropy_gpu.py: (name, builder, forest class, n_trees, random_state, params)
GPU_CASES = [
    ("lattice3", lambda: lattice(2000, 12, 3, 0), RandomForestClassifier, 4, 0, {}),
    ("lattice3_nobs", lambda: lattice(2000, 12, 3, 1), RandomForestClassifier, 3, 1,
     dict(bootstrap=False, max_features=0.5, max_depth=7, min_samples_leaf=3)),
    ("lattice3_decrease", lambda: lattice(2000, 12, 3, 2), RandomForestClassifier, 3, 2,
     dict(min_impurity_decrease=0.002)),
    ("gauss_sort", lambda: gaussian(9000, 6, 3, 3), RandomForestClassifier, 2, 3, {}),
    ("gauss_extra", lambda: gaussian(3000, 8, 4, 4), ExtraTreesClassifier, 4, 4, {}),
    ("gauss_extra_bs", lambda: gaussian(3000, 8, 2, 5), ExtraTreesClassifier, 3, 5,
     dict(bootstrap=True, max_depth=9, min_samples_leaf=2)),
] + [("lattice_k%d" % k, (lambda k=k: lattice(1500, 10, k, 10 + k)), RandomForestClassifier, 2, 10 + k, {})
     for k in (2, 4, 5, 8, 9, 16)]


# ------------------------------------------------------------------------- restatement vs scikit-learn

def test_log_base_is_the_hosts():
    assert LN2 == 0.6931471805599453
    assert entropy(np.array([[1.0, 1.0]]), 2.0, _glibc_log)[0] == 1.0


@pytest.mark.parametrize("k", [2, 3, 5])
@pytest.mark.parametrize("splitter", ["best", "random"])
def test_single_trees_match_scikit_learn(k, splitter):
    for seed, (X, y) in enumerate([lattice(400, 6, k, k), gaussian(400, 6, k, k + 1)]):
        check_single_tree(X, y, k, 100 + seed, splitter)
        check_single_tree(X, y, k, 200 + seed, splitter, max_depth=4, min_samples_leaf=5)
        check_single_tree(X, y, k, 300 + seed, splitter, max_features=None, min_impurity_decrease=0.01)
        check_single_tree(X, y, k, 400 + seed, splitter, criterion="log_loss", min_samples_split=9)


@pytest.mark.parametrize("splitter", ["best", "random"])
def test_adversarial_columns_match_scikit_learn(splitter):
    X = np.concatenate([adversarial(400, 5), extra_columns(400, 6)], axis=1)
    rng = np.random.default_rng(6)
    s = X[:, 2] + X[:, 3] * 0.3 + (X[:, 4] - 1e6) / 50 + X[:, 6] + (X[:, 7] > 0.6) + (X[:, 9] > 0.5)
    y = np.digitize(s + rng.standard_normal(400), [-1.0, 1.0]).astype(np.int64)
    for seed in (7, 8, 9):
        check_single_tree(X, y, 3, seed, splitter)
        check_single_tree(X, y, 3, seed, splitter, max_depth=4, max_features=None)


@pytest.mark.parametrize("forest_cls", [RandomForestClassifier, ExtraTreesClassifier])
def test_forest_trees_match_scikit_learn(forest_cls):
    """Bootstrap multiplicities as sample weights: the forests' own trees."""
    X, y = gaussian(500, 7, 3, 11)
    check_forest(X, y, 3, forest_cls, 3, 12)
    check_forest(X, y, 3, forest_cls, 2, 13, bootstrap=True, max_depth=5, min_impurity_decrease=0.005)


@pytest.mark.parametrize("case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_gpu_datasets_are_not_tie_sensitive(case):
    """Each dataset of the GPU test, restated with a log one ulp off on ~3 % of its inputs: the same trees,
    structure and thresholds.  (The restatement with the host's log is checked against scikit-learn too.)"""
    name, make, forest_cls, n_trees, rs, params = case
    X, y = make()
    k = int(y.max()) + 1
    n_check = 1 if len(y) > 5000 else n_trees      # the large sorted case: its first tree (the slow restatement)
    check_forest(X, y, k, forest_cls, n_check, rs, log=perturbed_log(), structure_only=True, **params)


def test_perturbed_log_differs():
    x = np.linspace(0.01, 0.99, 2000)
    d = perturbed_log()(x) != _glibc_log(x)
    assert 0.005 < d.mean() < 0.1


# ------------------------------------------------------------------------- plumbing on an engine double

class CriterionEngine(FakeEngine):
    """The engine double with the library's one-shot criterion: stage_forest_criterion sets it for the next
    forest_fit, which clears it; the trees are scikit-learn's under that criterion."""

    def __init__(self, device=0):
        super().__init__(device)
        self.staged = 0
        self.log = []

    def stage_forest_criterion(self, criterion):
        assert criterion in (0, 1)
        self.log.append(("stage", criterion))
        self.staged = criterion

    def forest_fit(self, sample_counts, rand_states, n_classes, max_features, max_depth, min_samples_split,
                   min_samples_leaf, min_weight_leaf, min_impurity_decrease, splitter=0, y_regression=None):
        crit, self.staged = self.staged, 0
        if crit and y_regression is not None:
            raise RuntimeError("forest: criterion entropy is staged but this is a regression fit")
        self.log.append(("fit", len(rand_states), crit))
        out = super().forest_fit(sample_counts, rand_states, n_classes, max_features, max_depth, min_samples_split,
                                 min_samples_leaf, min_weight_leaf, min_impurity_decrease, splitter, y_regression)
        return out


@pytest.fixture
def crit_engine(monkeypatch):
    from skdist_b200 import engine
    for v in ("SKDIST_B200_FOREST_SORT", "SKDIST_B200_FOREST_MAX_BINS", "SKDIST_B200_FOREST_CHUNK"):
        monkeypatch.delenv(v, raising=False)
    engine.set_engine_factory(CriterionEngine)
    yield engine.get_engine()
    engine.set_engine_factory(None)


def small(n=60, seed=0):
    X, y = lattice(n, 5, 3, seed)
    return X, y


@pytest.mark.parametrize("criterion", ["entropy", "log_loss"])
@pytest.mark.parametrize("cls_name", ["DistRandomForestClassifier", "DistExtraTreesClassifier"])
def test_entropy_stages_criterion_before_every_chunk(crit_engine, monkeypatch, criterion, cls_name):
    import skdist.distribute.ensemble as ens
    X, y = small()
    seeds(crit_engine, len(y), 5, 3)
    monkeypatch.setenv("SKDIST_B200_FOREST_CHUNK", "2")
    f = getattr(ens, cls_name)(n_estimators=5, criterion=criterion, random_state=3).fit(X, y)
    assert crit_engine.log == [("stage", 1), ("fit", 2, 1), ("stage", 1), ("fit", 2, 1), ("stage", 1), ("fit", 1, 1)]
    assert [e.criterion for e in f.estimators_] == [criterion] * 5
    assert f.criterion == criterion


@pytest.mark.parametrize("cls_name", ["DistRandomForestClassifier", "DistExtraTreesClassifier"])
def test_gini_never_stages(crit_engine, cls_name):
    import skdist.distribute.ensemble as ens
    X, y = small()
    seeds(crit_engine, len(y), 3, 4)
    f = getattr(ens, cls_name)(n_estimators=3, random_state=4).fit(X, y)
    assert [e for e in crit_engine.log if e[0] == "stage"] == []
    assert all(e.criterion == "gini" for e in f.estimators_)


def test_chunk_sizes(crit_engine):
    """Gini keeps the throughput builder's chunk (1036 trees); entropy takes the general builder's (296)."""
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = small(40, 5)
    seeds(crit_engine, len(y), 300, 6)
    DistRandomForestClassifier(n_estimators=300, max_depth=2, random_state=6).fit(X, y)
    assert [e[1] for e in crit_engine.log if e[0] == "fit"] == [300]
    crit_engine.log.clear()
    DistRandomForestClassifier(n_estimators=300, max_depth=2, criterion="entropy", random_state=6).fit(X, y)
    assert [e[1] for e in crit_engine.log if e[0] == "fit"] == [296, 4]


@pytest.mark.parametrize("criterion", ["entropy", "log_loss", "gini"])
def test_regressors_refuse_classification_criteria(crit_engine, criterion):
    from skdist.distribute.ensemble import DistExtraTreesRegressor, DistRandomForestRegressor
    X, y = small()
    for cls in (DistRandomForestRegressor, DistExtraTreesRegressor):
        with pytest.raises(NotImplementedError, match="criterion"):
            cls(n_estimators=2, criterion=criterion, random_state=0).fit(X, y.astype(float))
    assert crit_engine.log == []


@pytest.mark.parametrize("criterion", ["Entropy", "hellinger", "squared_error", None, ["entropy"]])
def test_other_strings_raise(crit_engine, criterion):
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier
    X, y = small()
    for cls in (DistRandomForestClassifier, DistExtraTreesClassifier):
        with pytest.raises(NotImplementedError, match="criterion"):
            cls(n_estimators=2, criterion=criterion, random_state=0).fit(X, y)
    assert crit_engine.log == []


def test_trees_on_the_double_are_scikit_learns(crit_engine):
    """The estimators carry the user's criterion into their trees' parameters."""
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = small()
    seeds(crit_engine, len(y), 2, 8)
    f = DistRandomForestClassifier(n_estimators=2, criterion="log_loss", random_state=8).fit(X, y)
    assert [e.get_params()["criterion"] for e in f.estimators_] == ["log_loss", "log_loss"]
