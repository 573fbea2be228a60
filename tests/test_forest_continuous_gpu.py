"""ExtraTrees forests and RandomTreesEmbedding on continuous float32 features: when a feature has more than
256 distinct values the random splitter of the general builder reads raw values (min / max pass, drawn
threshold, left-side pass), and the trees are scikit-learn's bit for bit wherever the node sums are exact."""
import numpy as np
import pytest

from tests.forest_class_weight_restate import restated_forest

pytestmark = pytest.mark.gpu

FIELDS = ("children_left", "children_right", "feature", "threshold", "n_node_samples", "weighted_n_node_samples",
          "impurity", "value")


def same_trees(ours, ref):
    assert len(ours) == len(ref)
    for a, b in zip(ours, ref):
        assert a.tree_.node_count == b.tree_.node_count and a.tree_.max_depth == b.tree_.max_depth
        for f in FIELDS:
            np.testing.assert_array_equal(getattr(a.tree_, f), getattr(b.tree_, f), err_msg=f)


def normal(n, d, k, seed):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    s = X[:, 0] + 0.5 * X[:, 1] * X[:, 2] - 0.7 * X[:, 3 % d] + 0.8 * rng.standard_normal(n)
    y = np.digitize(s, np.quantile(s, np.arange(1, k) / k))
    return X, y


def adversarial(n, seed):
    """A constant column, a column one float32 ulp wide (constant for the 1e-7 test), a two-valued column,
    heavy ties, magnitudes around 1e6, lattice columns next to continuous ones."""
    rng = np.random.default_rng(seed)
    base = np.float32(1.0)
    cols = [np.full(n, 3.5, np.float32),
            np.where(rng.random(n) < 0.5, base, np.nextafter(base, np.float32(2))).astype(np.float32),
            np.where(rng.random(n) < 0.3, -1.0, 2.0).astype(np.float32),
            np.round(rng.standard_normal(n) * 2).astype(np.float32),
            (1e6 + rng.standard_normal(n) * 50).astype(np.float32),
            rng.integers(0, 7, n).astype(np.float32),
            rng.standard_normal(n).astype(np.float32),
            rng.uniform(-1e-3, 1e-3, n).astype(np.float32)]
    X = np.stack(cols, axis=1)
    s = X[:, 2] + X[:, 3] * 0.3 + (X[:, 4] - 1e6) / 50 + X[:, 6] + 0.5 * rng.standard_normal(n)
    return X, (s > np.median(s)).astype(int) + (s > np.quantile(s, 0.9))


@pytest.mark.parametrize("n,d,k", [(3000, 16, 2), (20000, 64, 2), (5000, 10, 5)])
def test_extra_trees_classifier_bit_for_bit(n, d, k):
    from sklearn.ensemble import ExtraTreesClassifier
    from skdist.distribute.ensemble import DistExtraTreesClassifier
    X, y = normal(n, d, k, seed=n + k)
    variants = [dict(), dict(max_depth=6), dict(min_samples_leaf=5, min_samples_split=12),
                dict(max_features=0.5), dict(bootstrap=True)]
    for i, v in enumerate(variants):
        kw = dict(n_estimators=3, random_state=i, **v)
        ours = DistExtraTreesClassifier(**kw).fit(X, y)
        ref = ExtraTreesClassifier(**kw).fit(X, y)
        same_trees(ours.estimators_, ref.estimators_)
        np.testing.assert_array_equal(ours.predict_proba(X[:2000]), ref.predict_proba(X[:2000]))


def test_class_weight_on_continuous_features():
    """Dyadic dict weights and "balanced" weights that the class counts make dyadic: every weighted sum is
    exact, so the trees are the restated reference's bit for bit."""
    from sklearn.ensemble import ExtraTreesClassifier
    from skdist.distribute.ensemble import DistExtraTreesClassifier
    X, y = normal(4096, 12, 4, seed=3)
    cw = {0: 0.5, 1: 2.0, 2: 1.0, 3: 4.0}
    for bootstrap in (False, True):
        ours = DistExtraTreesClassifier(n_estimators=3, random_state=4, class_weight=cw, bootstrap=bootstrap).fit(X, y)
        same_trees(ours.estimators_, restated_forest(X, y, 3, 4, cw, bootstrap, 1, max_features="sqrt"))
    ours = DistExtraTreesClassifier(n_estimators=3, random_state=5, class_weight="balanced").fit(X, y)
    same_trees(ours.estimators_, ExtraTreesClassifier(n_estimators=3, random_state=5, class_weight="balanced").fit(X, y).estimators_)
    # balanced_subsample with bootstrap: non-dyadic weights from each tree's bootstrap class counts, so node
    # statistics to rounding and any differing split within the rounding envelope (DESIGN.md §4)
    from sklearn.utils import check_random_state
    from skdist.distribute.ensemble import MAX_RAND_SEED, _tree_inputs
    from tests.forest_class_weight_restate import restated_tree
    from tests.test_forest_class_weight_gpu import check_to_rounding
    yb = np.repeat([0, 1, 2, 3], [512, 512, 1024, 2048])
    ours = DistExtraTreesClassifier(n_estimators=3, random_state=6, bootstrap=True, max_depth=10,
                                    class_weight="balanced_subsample").fit(X, yb)
    for t, s in zip(ours.estimators_, check_random_state(6).randint(MAX_RAND_SEED, size=3)):
        counts, _ = _tree_inputs(s, len(yb), True)
        ref, w = restated_tree(X, yb, 4, s, "balanced_subsample", True, 1, max_features="sqrt", max_depth=10)
        check_to_rounding(t, ref, X, yb, counts.astype(np.int64), w)


def test_extra_trees_regressor():
    from sklearn.ensemble import ExtraTreesRegressor
    from skdist.distribute.ensemble import DistExtraTreesRegressor
    X, _ = normal(6000, 12, 2, seed=8)
    rng = np.random.default_rng(9)
    y_int = np.round(X[:, 0] * 3 + X[:, 1] ** 2 + rng.standard_normal(len(X)))
    for kw in (dict(), dict(max_depth=8, min_samples_leaf=3), dict(bootstrap=True, max_features=0.5)):
        ours = DistExtraTreesRegressor(n_estimators=3, random_state=1, **kw).fit(X, y_int)
        same_trees(ours.estimators_, ExtraTreesRegressor(n_estimators=3, random_state=1, **kw).fit(X, y_int).estimators_)
    # real-valued y: the float64 node sums are formed in another order than scikit-learn's (a child's total is
    # its parent's minus its sibling's), so where two drawn splits of a small node score within rounding of each
    # other the trees can choose differently.  Walk both trees in lockstep: every node they share agrees to
    # rounding, a node where the splits differ is small, and the walk does not descend below it.
    y = X[:, 0] * 3.1 + np.sin(X[:, 1]) + 0.1 * rng.standard_normal(len(X))
    ours = DistExtraTreesRegressor(n_estimators=3, random_state=2, max_depth=8).fit(X, y)
    ref = ExtraTreesRegressor(n_estimators=3, random_state=2, max_depth=8).fit(X, y)
    for a, b in zip(ours.estimators_, ref.estimators_):
        x, z = a.tree_, b.tree_
        stack, shared = [(0, 0)], 0
        while stack:
            i, j = stack.pop()
            shared += 1
            assert x.n_node_samples[i] == z.n_node_samples[j]
            # absolute 1e-10: a nearly pure node's impurity is a difference of the derived sums (~1e4 at the root)
            np.testing.assert_allclose(x.value[i], z.value[j], rtol=1e-12, atol=1e-10)
            np.testing.assert_allclose(x.impurity[i], z.impurity[j], rtol=1e-12, atol=1e-10)
            if (x.children_left[i] < 0) != (z.children_left[j] < 0) or (x.children_left[i] >= 0 and (
                    x.feature[i] != z.feature[j] or x.threshold[i] != z.threshold[j])):
                assert x.n_node_samples[i] <= 16, (i, x.n_node_samples[i])
                continue
            if x.children_left[i] >= 0:
                stack += [(x.children_right[i], z.children_right[j]), (x.children_left[i], z.children_left[j])]
        assert shared >= 0.9 * z.node_count
    again = DistExtraTreesRegressor(n_estimators=3, random_state=2, max_depth=8).fit(X, y)
    same_trees(again.estimators_, ours.estimators_)


@pytest.mark.parametrize("max_depth", [5, 30])
def test_random_trees_embedding(max_depth):
    from sklearn.ensemble import RandomTreesEmbedding
    from skdist.distribute.ensemble import DistRandomTreesEmbedding
    X, _ = normal(5000, 10, 2, seed=12)
    ours = DistRandomTreesEmbedding(n_estimators=8, max_depth=max_depth, random_state=3)
    ref = RandomTreesEmbedding(n_estimators=8, max_depth=max_depth, random_state=3)
    got, want = ours.fit_transform(X), ref.fit_transform(X)
    assert got.shape == want.shape and (got != want).nnz == 0
    X2, _ = normal(700, 10, 2, seed=13)
    assert (ours.transform(X2) != ref.transform(X2)).nnz == 0


def test_adversarial_columns():
    from sklearn.ensemble import ExtraTreesClassifier, ExtraTreesRegressor
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistExtraTreesRegressor
    X, y = adversarial(6000, seed=21)
    for kw in (dict(), dict(max_features=None), dict(max_features=1, max_depth=20)):
        ours = DistExtraTreesClassifier(n_estimators=4, random_state=7, **kw).fit(X, y)
        same_trees(ours.estimators_, ExtraTreesClassifier(n_estimators=4, random_state=7, **kw).fit(X, y).estimators_)
    ours = DistExtraTreesRegressor(n_estimators=3, random_state=8).fit(X, y.astype(float))
    same_trees(ours.estimators_, ExtraTreesRegressor(n_estimators=3, random_state=8).fit(X, y.astype(float)).estimators_)


def test_warm_start_equals_cold_fit():
    from skdist.distribute.ensemble import DistExtraTreesClassifier
    X, y = normal(4000, 12, 3, seed=30)
    warm = DistExtraTreesClassifier(n_estimators=3, random_state=2, warm_start=True).fit(X, y)
    warm.set_params(n_estimators=6)
    warm.fit(X, y)
    cold = DistExtraTreesClassifier(n_estimators=6, random_state=2).fit(X, y)
    same_trees(warm.estimators_, cold.estimators_)


def test_batch_predict_and_udf():
    from sklearn.ensemble import ExtraTreesClassifier
    from skdist.distribute.ensemble import DistExtraTreesClassifier
    from skdist.distribute.predict import batch_predict, get_prediction_udf
    X, y = normal(6000, 16, 3, seed=40)
    ours = DistExtraTreesClassifier(n_estimators=5, random_state=1).fit(X, y)
    ref = ExtraTreesClassifier(n_estimators=5, random_state=1).fit(X, y)
    Xt, _ = normal(3000, 16, 3, seed=41)
    want = ref.predict_proba(Xt)
    np.testing.assert_array_equal(batch_predict(ours, Xt, "predict_proba"), want)
    import pandas as pd
    out = get_prediction_udf(ours, method="predict_proba")(*[pd.Series(Xt[:500, j]) for j in range(16)])
    np.testing.assert_array_equal(np.vstack(out.values), want[:500])


def test_best_splitter_still_refuses_continuous_features():
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier
    X, y = normal(3000, 8, 2, seed=50)
    DistExtraTreesClassifier(n_estimators=2, random_state=0).fit(X, y)      # raw values staged alongside the codes
    with pytest.raises(NotImplementedError, match="SKDIST_B200_FOREST_MAX_BINS"):
        DistRandomForestClassifier(n_estimators=2, random_state=0).fit(X, y)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_values_raise(bad):
    from skdist.distribute.ensemble import DistExtraTreesClassifier
    from skdist_b200.engine import get_engine
    X, y = normal(3000, 8, 2, seed=60)
    X[1234, 5] = bad
    with pytest.raises(ValueError, match="NaN or infinity"):
        DistExtraTreesClassifier(n_estimators=2, random_state=0).fit(X, y)
    X[1234, 5] = 0.25                                                       # the device is still usable
    DistExtraTreesClassifier(n_estimators=2, random_state=0).fit(X, y)
    get_engine()
