"""RandomForest forests on continuous float32 features with SKDIST_B200_FOREST_SORT=1: the best splitter sorts
the node's raw values of every drawn feature that has more than 256 distinct values (a CTA radix sort in shared
memory up to 4096 samples, an LSD radix sort in global scratch above), and the trees are scikit-learn's bit for
bit wherever the node sums are exact."""
import numpy as np
import pytest

from tests.forest_class_weight_restate import restated_forest
from tests.test_forest_continuous_gpu import adversarial, normal, same_trees

pytestmark = pytest.mark.gpu

S = 4096   # the largest node sorted in shared memory (csrc/forest.cu FO_SORT_S)


@pytest.fixture(autouse=True)
def sort_switch(monkeypatch):
    monkeypatch.setenv("SKDIST_B200_FOREST_SORT", "1")
    monkeypatch.delenv("SKDIST_B200_FOREST_MAX_BINS", raising=False)


def fit_both(X, y, **kw):
    from sklearn.ensemble import RandomForestClassifier
    from skdist.distribute.ensemble import DistRandomForestClassifier
    ours = DistRandomForestClassifier(**kw).fit(X, y)
    ref = RandomForestClassifier(**kw).fit(X, y)
    same_trees(ours.estimators_, ref.estimators_)
    return ours, ref


VARIANTS = [dict(), dict(max_depth=6), dict(min_samples_leaf=5, min_samples_split=12), dict(max_features=None),
            dict(max_features=0.5), dict(max_features=1), dict(bootstrap=False),
            dict(min_weight_fraction_leaf=0.01), dict(min_impurity_decrease=1e-3)]


@pytest.mark.parametrize("n,d,k", [(3000, 16, 2), (20000, 64, 2)])
def test_classifier_bit_for_bit(n, d, k):
    """3000 x 16: every node sorts in shared memory; 20000 x 64: the root and the first levels in global scratch."""
    X, y = normal(n, d, k, seed=n + k)
    for i, v in enumerate(VARIANTS):
        ours, ref = fit_both(X, y, n_estimators=3, random_state=i, **v)
        np.testing.assert_array_equal(ours.predict_proba(X[:2000]), ref.predict_proba(X[:2000]))


def test_classifier_large_nodes():
    """200000 rows: several levels of every tree go through the global radix sort."""
    X, y = normal(200000, 16, 2, seed=7)
    for v in (dict(), dict(max_depth=6, bootstrap=False)):
        fit_both(X, y, n_estimators=2, random_state=3, **v)


@pytest.mark.parametrize("k", [3, 5, 9, 16])
def test_class_counts(k):
    """Every class-count instantiation of the builder (4, 8, 16 classes)."""
    X, y = normal(6000, 10, k, seed=100 + k)
    fit_both(X, y, n_estimators=3, random_state=k)
    fit_both(X, y, n_estimators=2, random_state=k + 1, max_depth=5, bootstrap=False)


@pytest.mark.parametrize("n", [S - 1, S, S + 1, S + 2])
def test_regime_boundary(n):
    """The root holds every row (no bootstrap): n <= S sorts in shared memory, n > S in global scratch."""
    X, y = normal(n, 6, 3, seed=n)
    fit_both(X, y, n_estimators=2, random_state=1, bootstrap=False, max_depth=2)
    fit_both(X, y, n_estimators=2, random_state=2, bootstrap=False, max_features=None)


def extra_columns(n, seed):
    """Runs chained by gaps <= 1e-7 whose span exceeds 1e-7 (adjacent float32 values near 0.5 are 6e-8
    apart), adjacent float32 values near 1e6 (0.0625 apart) that are all valid split points, signed zeros."""
    rng = np.random.default_rng(seed)
    ulp = np.float32(2.0 ** -24)
    chain = np.where(rng.random(n) < 0.5, np.float32(0.5), np.float32(0.75)) + rng.integers(0, 12, n) * ulp
    chain = np.where(rng.random(n) < 0.2, rng.standard_normal(n), chain)
    big = np.float32(1e6) + rng.integers(0, 40, n).astype(np.float32) * np.float32(0.0625)
    zeros = rng.choice(np.array([-0.0, 0.0, 1.0, -1.0], np.float32), n, p=[0.35, 0.35, 0.15, 0.15])
    return np.stack([chain.astype(np.float32), big.astype(np.float32), zeros], axis=1)


def test_adversarial_columns():
    from sklearn.ensemble import RandomForestRegressor
    from skdist.distribute.ensemble import DistRandomForestRegressor
    for n in (3000, 12000):          # shared memory only, and the global sort near the root
        X, y = adversarial(n, seed=21)
        E = extra_columns(n, seed=22)
        X = np.ascontiguousarray(np.concatenate([X, E], axis=1))
        y = y + (E[:, 0] > 0.6) + (E[:, 1] > 1e6 + 1.2) * 2 + (E[:, 2] > 0.5)
        for kw in (dict(), dict(max_features=None), dict(max_features=1, max_depth=20), dict(bootstrap=False)):
            fit_both(X, y, n_estimators=3, random_state=7, **kw)
        ours = DistRandomForestRegressor(n_estimators=3, random_state=8).fit(X, y.astype(float))
        same_trees(ours.estimators_, RandomForestRegressor(n_estimators=3, random_state=8).fit(X, y.astype(float)).estimators_)


def test_class_weight():
    """Dyadic dict weights and "balanced" weights that the class counts make dyadic are exact: the restated
    reference's trees bit for bit.  balanced_subsample with bootstrap: to rounding (DESIGN.md §4)."""
    from sklearn.utils import check_random_state
    from skdist.distribute.ensemble import MAX_RAND_SEED, DistRandomForestClassifier, _tree_inputs
    from tests.forest_class_weight_restate import restated_tree
    from tests.test_forest_class_weight_gpu import check_to_rounding
    X, y = normal(8192, 12, 4, seed=3)
    cw = {0: 0.5, 1: 2.0, 2: 1.0, 3: 4.0}
    for bootstrap in (False, True):
        ours = DistRandomForestClassifier(n_estimators=3, random_state=4, class_weight=cw, bootstrap=bootstrap).fit(X, y)
        same_trees(ours.estimators_, restated_forest(X, y, 3, 4, cw, bootstrap, 0, max_features="sqrt"))
        ours = DistRandomForestClassifier(n_estimators=3, random_state=5, class_weight="balanced", bootstrap=bootstrap).fit(X, y)
        same_trees(ours.estimators_, restated_forest(X, y, 3, 5, "balanced", bootstrap, 0, max_features="sqrt"))
    yb = np.repeat([0, 1, 2, 3], [1024, 1024, 2048, 4096])
    ours = DistRandomForestClassifier(n_estimators=3, random_state=6, bootstrap=True, max_depth=10,
                                      class_weight="balanced_subsample").fit(X, yb)
    for t, s in zip(ours.estimators_, check_random_state(6).randint(MAX_RAND_SEED, size=3)):
        counts, _ = _tree_inputs(s, len(yb), True)
        ref, w = restated_tree(X, yb, 4, s, "balanced_subsample", True, 0, max_features="sqrt", max_depth=10)
        check_to_rounding(t, ref, X, yb, counts.astype(np.int64), w)


def test_regressor():
    from sklearn.ensemble import RandomForestRegressor
    from skdist.distribute.ensemble import DistRandomForestRegressor
    X, _ = normal(6000, 12, 2, seed=8)
    rng = np.random.default_rng(9)
    y_int = np.round(X[:, 0] * 3 + X[:, 1] ** 2 + rng.standard_normal(len(X)))
    for kw in (dict(), dict(max_depth=8, min_samples_leaf=3), dict(bootstrap=False, max_features=0.5)):
        ours = DistRandomForestRegressor(n_estimators=3, random_state=1, **kw).fit(X, y_int)
        same_trees(ours.estimators_, RandomForestRegressor(n_estimators=3, random_state=1, **kw).fit(X, y_int).estimators_)
    # real-valued y: the float64 prefix sums are formed in another order than scikit-learn's, so where two
    # candidates of a small node score within rounding of each other the trees can choose differently.  Walk
    # both trees in lockstep: shared nodes agree to rounding, a node where the splits differ is small.
    y = X[:, 0] * 3.1 + np.sin(X[:, 1]) + 0.1 * rng.standard_normal(len(X))
    ours = DistRandomForestRegressor(n_estimators=3, random_state=2, max_depth=8).fit(X, y)
    ref = RandomForestRegressor(n_estimators=3, random_state=2, max_depth=8).fit(X, y)
    for a, b in zip(ours.estimators_, ref.estimators_):
        x, z = a.tree_, b.tree_
        stack, shared = [(0, 0)], 0
        while stack:
            i, j = stack.pop()
            shared += 1
            assert x.n_node_samples[i] == z.n_node_samples[j]
            np.testing.assert_allclose(x.value[i], z.value[j], rtol=1e-12, atol=1e-10)
            np.testing.assert_allclose(x.impurity[i], z.impurity[j], rtol=1e-12, atol=1e-10)
            if (x.children_left[i] < 0) != (z.children_left[j] < 0) or (x.children_left[i] >= 0 and (
                    x.feature[i] != z.feature[j] or x.threshold[i] != z.threshold[j])):
                assert x.n_node_samples[i] <= 16, (i, x.n_node_samples[i])
                continue
            if x.children_left[i] >= 0:
                stack += [(x.children_right[i], z.children_right[j]), (x.children_left[i], z.children_left[j])]
        assert shared >= 0.9 * z.node_count
    again = DistRandomForestRegressor(n_estimators=3, random_state=2, max_depth=8).fit(X, y)
    same_trees(again.estimators_, ours.estimators_)


def test_node_capacity_retry(monkeypatch):
    """Trees that outgrow a small node array are rebuilt with the full one: the same trees."""
    monkeypatch.setenv("SKDIST_B200_FOREST_NODECAP", "64")
    X, y = normal(5000, 12, 3, seed=31)
    fit_both(X, y, n_estimators=4, random_state=3)


def test_warm_start_equals_cold_fit():
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = normal(4000, 12, 3, seed=30)
    warm = DistRandomForestClassifier(n_estimators=3, random_state=2, warm_start=True).fit(X, y)
    warm.set_params(n_estimators=6)
    warm.fit(X, y)
    cold = DistRandomForestClassifier(n_estimators=6, random_state=2).fit(X, y)
    same_trees(warm.estimators_, cold.estimators_)


def test_batch_predict_and_udf():
    from skdist.distribute.predict import batch_predict, get_prediction_udf
    X, y = normal(6000, 16, 3, seed=40)
    ours, ref = fit_both(X, y, n_estimators=5, random_state=1)
    Xt, _ = normal(3000, 16, 3, seed=41)
    want = ref.predict_proba(Xt)
    np.testing.assert_array_equal(batch_predict(ours, Xt, "predict_proba"), want)
    import pandas as pd
    out = get_prediction_udf(ours, method="predict_proba")(*[pd.Series(Xt[:500, j]) for j in range(16)])
    np.testing.assert_array_equal(np.vstack(out.values), want[:500])


def test_lattice_data_unchanged(monkeypatch):
    """Every feature with <= 256 distinct values: the switch changes nothing (the histogram builders run)."""
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = normal(8000, 12, 3, seed=50)
    Xq = np.round(X * 8).astype(np.float32)
    on, _ = fit_both(Xq, y, n_estimators=4, random_state=5)
    monkeypatch.delenv("SKDIST_B200_FOREST_SORT")
    off = DistRandomForestClassifier(n_estimators=4, random_state=5).fit(Xq, y)
    same_trees(on.estimators_, off.estimators_)
