"""criterion="entropy" / "log_loss" of DistRandomForestClassifier and DistExtraTreesClassifier on the device (the
general tree builder's ENT instantiations, histogram, sort and raw modes) against scikit-learn's own forests:
every tree array-equal, impurity included (formed on the host with the host's log).  Every dataset here is
checked in tests/test_forest_entropy_host.py against a log one ulp off on a few percent of its inputs, so a
mismatch is not a last-bit difference of CUDA's log: the failure message prints the competing proxies."""
import math

import numpy as np
import pytest
from sklearn.ensemble import ExtraTreesClassifier, RandomForestClassifier

from tests.test_forest_entropy_host import GPU_CASES, gaussian, lattice

pytestmark = pytest.mark.gpu

FIELDS = ("children_left", "children_right", "feature", "threshold", "n_node_samples", "weighted_n_node_samples",
          "value", "impurity")


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for v in ("SKDIST_B200_FOREST_SORT", "SKDIST_B200_FOREST_MAX_BINS", "SKDIST_B200_FOREST_NODECAP",
              "SKDIST_B200_FOREST_KERNEL", "SKDIST_B200_FOREST_CHUNK"):
        monkeypatch.delenv(v, raising=False)


def _entropy(s):
    w = float(np.sum(s))
    e = 0.0
    for v in s:
        if v > 0:
            p = v / w
            e -= p * (math.log(p) / math.log(2.0))
    return e, w


def _proxy(X, y, k, sw, rows, f, thr):
    left = X[rows, f].astype(np.float64) <= thr
    (il, wl), (ir, wr) = (_entropy(np.bincount(y[r], weights=sw[r], minlength=k)) for r in (rows[left], rows[~left]))
    return -wr * ir - wl * il


def _first_difference(a, b, X, y, k, sw):
    """Walk both trees in build order to the first node that differs; describe it with both splits' proxies."""
    rows = {0: np.flatnonzero(sw > 0)}
    stack = [(0, 0)]
    while stack:
        i, j = stack.pop()
        r = rows[i]
        same = a.feature[i] == b.feature[j] and a.threshold[i] == b.threshold[j] and \
            (a.children_left[i] < 0) == (b.children_left[j] < 0)
        if not same:
            msg = "node %d (%d rows): device (f %d, thr %r), scikit-learn (f %d, thr %r)" % (
                i, len(r), a.feature[i], a.threshold[i], b.feature[j], b.threshold[j])
            if a.children_left[i] >= 0 and b.children_left[j] >= 0:
                msg += "; proxies %r vs %r" % (_proxy(X, y, k, sw, r, a.feature[i], a.threshold[i]),
                                               _proxy(X, y, k, sw, r, b.feature[j], b.threshold[j]))
            return msg
        for f in ("n_node_samples", "weighted_n_node_samples", "impurity"):
            if getattr(a, f)[i] != getattr(b, f)[j]:
                return "node %d: %s %r vs %r" % (i, f, getattr(a, f)[i], getattr(b, f)[j])
        if a.children_left[i] >= 0:
            go = X[r, a.feature[i]].astype(np.float64) <= a.threshold[i]
            rows[a.children_left[i]], rows[a.children_right[i]] = r[go], r[~go]
            stack += [(a.children_right[i], b.children_right[j]), (a.children_left[i], b.children_left[j])]
    return "no structural difference"


def same_trees(ours, ref, X, y, bootstrap):
    from skdist_b200.distribute.ensemble import _tree_inputs
    assert len(ours.estimators_) == len(ref.estimators_)
    k = len(ref.classes_)
    for a, b in zip(ours.estimators_, ref.estimators_):
        assert a.criterion == b.criterion
        ta, tb = a.tree_, b.tree_
        ok = ta.node_count == tb.node_count and all(np.array_equal(getattr(ta, f), getattr(tb, f)) for f in FIELDS)
        if not ok:
            counts, _ = _tree_inputs(b.random_state, len(y), bootstrap)
            pytest.fail("tree of seed %d differs: %s" % (b.random_state, _first_difference(
                ta, tb, X, np.searchsorted(ref.classes_, y), k, counts.astype(np.float64))))


def fit_both(X, y, forest="rf", criterion="entropy", **kw):
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier
    Dist, Ref = ((DistRandomForestClassifier, RandomForestClassifier) if forest == "rf" else
                 (DistExtraTreesClassifier, ExtraTreesClassifier))
    ours = Dist(criterion=criterion, **kw).fit(X, y)
    ref = Ref(criterion=criterion, **kw).fit(X, y)
    same_trees(ours, ref, X, y, kw.get("bootstrap", forest == "rf"))
    return ours, ref


@pytest.mark.parametrize("case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_trees_equal_scikit_learns(case, monkeypatch):
    """Histogram mode (lattice), sort mode (continuous, root nodes above 4096 samples, deeper ones below),
    raw random splitter (ExtraTrees, continuous), every class-count instantiation up to 16 classes."""
    name, make, forest_cls, n_trees, rs, params = case
    X, y = make()
    if name == "gauss_sort":
        monkeypatch.setenv("SKDIST_B200_FOREST_SORT", "1")
    fit_both(X, y, "rf" if forest_cls is RandomForestClassifier else "et", n_estimators=n_trees, random_state=rs,
             **params)


def test_log_loss_alias():
    X, y = lattice(2000, 12, 3, 0)
    fit_both(X, y, criterion="log_loss", n_estimators=2, random_state=5)
    fit_both(X, y, "et", criterion="log_loss", n_estimators=2, random_state=5)


def test_warm_start_equals_cold_fit():
    from skdist.distribute.ensemble import DistRandomForestClassifier
    X, y = lattice(2000, 12, 3, 0)
    warm = DistRandomForestClassifier(n_estimators=2, criterion="entropy", random_state=2, warm_start=True).fit(X, y)
    warm.set_params(n_estimators=4)
    warm.fit(X, y)
    ref = RandomForestClassifier(n_estimators=4, criterion="entropy", random_state=2).fit(X, y)
    same_trees(warm, ref, X, y, True)


def test_node_capacity_retry(monkeypatch):
    monkeypatch.setenv("SKDIST_B200_FOREST_NODECAP", "64")
    X, y = lattice(2000, 12, 3, 0)
    fit_both(X, y, n_estimators=4, random_state=0)


def test_dyadic_class_weight():
    """Dict weights that are powers of two keep every sum exact.  Without bootstrap scikit-learn's forests fit
    the trees the reference's per-tree sample weights give."""
    X, y = lattice(2000, 12, 3, 0)
    cw = {0: 0.5, 1: 2.0, 2: 1.0}
    fit_both(X, y, n_estimators=3, random_state=0, class_weight=cw, bootstrap=False)
    fit_both(X, y, "et", n_estimators=3, random_state=0, class_weight=cw)


def _lockstep_to_rounding(a, b, X, y, k, sw):
    """Where both trees agree, node statistics agree to rounding; at the first node where they split
    differently both splits' proxies, formed in float64 on the node's rows, lie within a relative 1e-9 of each
    other (a near-tie that rounding of the non-dyadic weighted sums decides).  Returns 1 on divergence."""
    rows = {0: np.flatnonzero(sw > 0)}
    stack = [(0, 0)]
    while stack:
        i, j = stack.pop()
        r = rows[i]
        assert a.n_node_samples[i] == b.n_node_samples[j]
        np.testing.assert_allclose(a.weighted_n_node_samples[i], b.weighted_n_node_samples[j], rtol=1e-11)
        np.testing.assert_allclose(a.value[i], b.value[j], rtol=1e-11, atol=1e-300)
        np.testing.assert_allclose(a.impurity[i], b.impurity[j], rtol=1e-9, atol=1e-12)
        la, lb = a.children_left[i], b.children_left[j]
        if la < 0 and lb < 0:
            continue
        if la < 0 or lb < 0:
            assert len(np.unique(y[r])) == 1, "one tree splits an impure node the other leaves as a leaf"
            return 1
        if a.feature[i] == b.feature[j] and a.threshold[i] == b.threshold[j]:
            go = X[r, a.feature[i]].astype(np.float64) <= a.threshold[i]
            rows[la], rows[a.children_right[i]] = r[go], r[~go]
            stack += [(a.children_right[i], b.children_right[j]), (la, lb)]
            continue
        pa = _proxy(X, y, k, sw, r, a.feature[i], a.threshold[i])
        pb = _proxy(X, y, k, sw, r, b.feature[j], b.threshold[j])
        assert abs(pa - pb) <= 1e-9 * a.weighted_n_node_samples[i], (pa, pb)
        return 1
    return 0


@pytest.mark.parametrize("cw,bootstrap", [("balanced", False), ("balanced_subsample", True)])
@pytest.mark.parametrize("forest", ["rf", "et"])
def test_non_dyadic_class_weight_to_rounding(cw, bootstrap, forest):
    """"balanced" without bootstrap and "balanced_subsample" with it: scikit-learn's forests use the same
    weights; the sums are not exact, so trees agree to rounding (DESIGN.md §4)."""
    from sklearn.utils import check_random_state
    from sklearn.utils.class_weight import compute_sample_weight
    from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomForestClassifier, _tree_inputs
    X, y = lattice(3001, 10, 3, 21)
    y[:7] = 2
    Dist, Ref = ((DistRandomForestClassifier, RandomForestClassifier) if forest == "rf" else
                 (DistExtraTreesClassifier, ExtraTreesClassifier))
    kw = dict(n_estimators=3, random_state=3, criterion="entropy", class_weight=cw, bootstrap=bootstrap, max_depth=10)
    ours, ref = Dist(**kw).fit(X, y), Ref(**kw).fit(X, y)
    for a, b in zip(ours.estimators_, ref.estimators_):
        counts, _ = _tree_inputs(b.random_state, len(y), bootstrap)
        if bootstrap:
            idx = check_random_state(b.random_state).randint(0, len(y), len(y))
            sw = compute_sample_weight("balanced", y, indices=idx) * counts
        else:
            sw = compute_sample_weight("balanced", y)
        _lockstep_to_rounding(a.tree_, b.tree_, X, y, 3, sw)


def test_predict_proba_udf():
    import pandas as pd
    from skdist.distribute.predict import get_prediction_udf
    X, y = gaussian(3000, 8, 4, 4)
    ours, ref = fit_both(X, y, "et", n_estimators=4, random_state=4)
    Xt, _ = gaussian(500, 8, 4, 40)
    out = get_prediction_udf(ours, method="predict_proba")(*[pd.Series(Xt[:, j]) for j in range(8)])
    np.testing.assert_array_equal(np.vstack(out.values), ref.predict_proba(Xt))


def test_gini_after_entropy_is_gini():
    """The staged criterion is one-shot: a Gini fit straight after an entropy fit builds Gini trees, also after
    a fit that failed with entropy staged."""
    from skdist.distribute.ensemble import DistRandomForestClassifier
    from skdist_b200.engine import get_engine
    X, y = lattice(2000, 12, 3, 0)
    fit_both(X, y, n_estimators=2, random_state=1)
    eng = get_engine()
    eng.stage_forest_criterion(1)
    with pytest.raises(Exception, match="regression"):
        eng.forest_fit(None, np.array([1], np.uint32), 1, 3, 5, 2, 1, 0.0, 0.0, 0, y.astype(np.float64))
    ours = DistRandomForestClassifier(n_estimators=2, random_state=1).fit(X, y)
    ref = RandomForestClassifier(n_estimators=2, random_state=1).fit(X, y)
    same_trees(ours, ref, X, y, True)
    with pytest.raises(Exception, match="criterion must be"):
        eng.stage_forest_criterion(2)
