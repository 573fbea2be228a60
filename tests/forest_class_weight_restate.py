"""Restatement of the reference's per-tree task `_build_trees` (ref ensemble.py:68-109) with class weights,
and an engine double that builds its trees with it.  No GPU: both are scikit-learn on the host.

Tree t of a forest with seed s: counts = bootstrap multiplicities of s (`_tree_inputs`, or 1 without
bootstrap), w_i = counts_i * cw[y_i] in float64, then DecisionTreeClassifier / ExtraTreeClassifier
(random_state=s).fit(X, y, sample_weight=w).  cw is compute_class_weight(dict or "balanced", classes, y) on
all of y, or -- "balanced_subsample" with bootstrap -- compute_sample_weight("balanced", y, indices=bootstrap
indices), which gives absent classes 0."""
import numpy as np
from sklearn.tree import DecisionTreeClassifier, ExtraTreeClassifier
from sklearn.utils import check_random_state
from sklearn.utils.class_weight import compute_class_weight, compute_sample_weight

from skdist_b200.distribute.ensemble import MAX_RAND_SEED, _tree_inputs
from tests.fake_engine import FakeEngine


def tree_class_weights(class_weight, y_enc, n_classes, state, bootstrap):
    """[n_classes] float64 weights of one tree (y_enc: labels 0 .. n_classes - 1)."""
    classes = np.arange(n_classes)
    if isinstance(class_weight, str) and class_weight == "balanced_subsample":
        if not bootstrap:
            return compute_class_weight("balanced", classes=classes, y=y_enc)
        indices = check_random_state(state).randint(0, len(y_enc), len(y_enc))      # ref :51-55
        sw = compute_sample_weight("balanced", y_enc, indices=indices)
        w = np.zeros(n_classes)
        for k in classes:
            rows = np.flatnonzero(y_enc == k)
            w[k] = sw[rows[0]] if len(rows) else 0.0
        return w
    return compute_class_weight(class_weight, classes=classes, y=y_enc)


def restated_tree(X, y_enc, n_classes, state, class_weight, bootstrap, splitter=0, cw_scale=None, **params):
    """The reference's tree for seed `state`.  cw_scale: {class: factor} applied to the weights (tests that
    the parity checks reject a wrong weight)."""
    counts, _ = _tree_inputs(state, len(y_enc), bootstrap)
    cw = tree_class_weights(class_weight, y_enc, n_classes, state, bootstrap)
    for k, f in (cw_scale or {}).items():
        cw[k] *= f
    w = counts.astype(np.float64) * cw[y_enc]
    cls = ExtraTreeClassifier if splitter else DecisionTreeClassifier
    return cls(random_state=int(state), **params).fit(X, y_enc, sample_weight=w), cw


def restated_forest(X, y, n_estimators, random_state, class_weight, bootstrap, splitter=0, **params):
    """Every tree of a forest (seeds drawn as ref ensemble.py:278)."""
    classes, y_enc = np.unique(y, return_inverse=True)
    if isinstance(class_weight, dict):                 # keys are the original labels
        class_weight = {int(np.flatnonzero(classes == k)[0]): v for k, v in class_weight.items()}
    states = check_random_state(random_state).randint(MAX_RAND_SEED, size=n_estimators)
    return [restated_tree(X, y_enc, len(classes), s, class_weight, bootstrap, splitter, **params)[0] for s in states]


class WeightedForestEngine(FakeEngine):
    """FakeEngine whose forest_fit honours staged forest class weights the way the library does: one-shot,
    the staged fraction replaces min_weight_leaf, balanced_subsample forms each tree's weights from the
    bootstrap class counts it is handed.  Every staging call is recorded in `staged`."""

    def __init__(self, device=0):
        super().__init__(device)
        self.staged = []
        self._cw = None

    def stage_forest_class_weights(self, n_classes, w=None, balanced_subsample=False, min_weight_fraction_leaf=0.0):
        entry = None
        if n_classes:
            entry = (int(n_classes), None if balanced_subsample else np.array(w, np.float64),
                     bool(balanced_subsample), float(min_weight_fraction_leaf))
        self.staged.append(entry)
        self._cw = entry

    def forest_fit(self, sample_counts, rand_states, n_classes, max_features, max_depth, min_samples_split,
                   min_samples_leaf, min_weight_leaf, min_impurity_decrease, splitter=0, y_regression=None):
        cw, self._cw = self._cw, None
        if cw is None:
            return super().forest_fit(sample_counts, rand_states, n_classes, max_features, max_depth,
                                      min_samples_split, min_samples_leaf, min_weight_leaf, min_impurity_decrease,
                                      splitter, y_regression)
        assert y_regression is None and cw[0] == n_classes
        self.calls.append(("forest_fit", len(rand_states)))
        self.last_forest_seconds = 0.0
        out = []
        for t, r in enumerate(rand_states):
            seed = self.seed_of_rand_r[int(r)]
            counts = np.ones(self.n) if sample_counts is None else sample_counts[t].astype(np.float64)
            if cw[2]:
                nk = np.bincount(self.y, weights=counts, minlength=n_classes)
                w_cls = np.where(nk > 0, counts.sum() / (np.count_nonzero(nk) * np.where(nk > 0, nk, 1.0)), 0.0)
            else:
                w_cls = cw[1]
            sw = counts * w_cls[self.y]
            cls = ExtraTreeClassifier if splitter else DecisionTreeClassifier
            est = cls(max_features=max_features, max_depth=None if max_depth >= 2 ** 31 - 1 else max_depth,
                      min_samples_split=min_samples_split, min_samples_leaf=min_samples_leaf,
                      min_weight_fraction_leaf=cw[3], min_impurity_decrease=min_impurity_decrease,
                      random_state=seed)
            est.fit(self.X, self.y, sample_weight=sw)
            tr = est.tree_
            out.append({"left": tr.children_left.astype(np.int32), "right": tr.children_right.astype(np.int32),
                        "feature": tr.feature.astype(np.int32), "threshold": tr.threshold.copy(),
                        "impurity": tr.impurity.copy(), "n_node_samples": tr.n_node_samples.astype(np.int32),
                        "weighted_n_node_samples": tr.weighted_n_node_samples.copy(),
                        "missing_go_to_left": np.zeros(tr.node_count, np.uint8),
                        "value": tr.value[:, 0, :].copy(), "max_depth": tr.max_depth})
        return out
