"""Generate tests/golden/forest_class_weight_pins.npz: trees of the UNMODIFIED reference's per-tree task
`_build_trees` (ref ensemble.py:68-109, imported through oracle/refshim.py) for forest classifiers with
class weights, so that tests/test_forest_class_weight_host.py can show, without the reference tree, that the
restatement in tests/forest_class_weight_restate.py builds the same trees.

    SKDIST_REFERENCE_ROOT=<sk-dist checkout> python tests/golden/make_forest_class_weight_pins.py

What the reference's `fit` does before the fan-out (ref ensemble.py:224-238) is replayed here:
`_validate_y_class_weight` (scikit-learn's ForestClassifier method, which the reference class inherits)
turns y into class indices and class_weight into per-row weights, and those are `_build_trees`'
sample_weight.  The reference's constructor and `fit` do not run on scikit-learn 1.9 (the constructor passes
`min_impurity_split`, `fit` calls `_validate_y_class_weight(y)` without the now required sample_weight), so
the instance is made with object.__new__ and the method is called with sample_weight=None, which is what the
one-argument call meant.

"balanced_subsample" is not pinned: with bootstrap the reference calls
`compute_sample_weight("balanced", y, indices)` with `indices` positional, and scikit-learn 1.9 makes that
argument keyword-only, so the unmodified task raises a TypeError.  (Without bootstrap scikit-learn maps
"balanced_subsample" to "balanced", which is pinned.)
"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "forest_class_weight_pins.npz")

# (name, splitter, class_weight, bootstrap); classes are labelled 3, 4, 5 so that dict keys are labels
CASES = [
    ("rf_dict_zero_boot", 0, {3: 2.0, 4: 0.0, 5: 0.5}, True),
    ("rf_dict_boot", 0, {3: 0.3, 5: 1.7}, True),
    ("rf_balanced_boot", 0, "balanced", True),
    ("rf_balanced_noboot", 0, "balanced", False),
    ("rf_dict_noboot", 0, {3: 1.5, 4: 0.25, 5: 3.0}, False),
    ("et_dict_zero_noboot", 1, {3: 0.0, 4: 1.0, 5: 4.0}, False),
    ("et_balanced_boot", 1, "balanced", True),
    ("rf_balanced_subsample_noboot", 0, "balanced_subsample", False),
]
N_TREES, RANDOM_STATE = 3, 7
PARAMS = dict(max_features="sqrt", max_depth=8, min_samples_leaf=2)


def data():
    """A small lattice with three uneven classes (labels 3, 4, 5)."""
    rng = np.random.default_rng(21)
    X = rng.integers(0, 10, size=(600, 6)).astype(np.float32)
    s = X[:, 0] + 0.6 * X[:, 1] - 0.3 * X[:, 2] + rng.standard_normal(600) * 2.0
    y = np.digitize(s, np.quantile(s, [0.15, 0.55])) + 3
    return X, y


def main():
    from sklearn.tree import DecisionTreeClassifier, ExtraTreeClassifier
    warnings.simplefilter("ignore")
    _, _, ref_ens = refshim.load()
    X, y = data()
    out = {"X": X, "y": y}
    for name, splitter, cw, bootstrap in CASES:
        est = object.__new__(ref_ens.DistRandomForestClassifier)
        est.class_weight, est.bootstrap, est.warm_start, est.n_outputs_ = cw, bootstrap, False, 1   # ref :226
        y_idx, expanded = est._validate_y_class_weight(y.reshape(-1, 1), None)      # ref :229
        y_idx = np.ascontiguousarray(y_idx, dtype=np.float64)                          # ref :231-232
        states = np.random.RandomState(RANDOM_STATE).randint(ref_ens.MAX_RAND_SEED, size=N_TREES)   # ref :278
        base = (ExtraTreeClassifier if splitter else DecisionTreeClassifier)(**PARAMS)
        for t, s in enumerate(states):
            tree = ref_ens._build_trees(base, (), {}, X, y_idx, expanded, s, N_TREES,
                                        class_weight=cw, bootstrap=bootstrap).tree_
            for field in ("children_left", "children_right", "feature", "threshold", "impurity",
                          "n_node_samples", "weighted_n_node_samples"):
                out["%s_%d_%s" % (name, t, field)] = np.asarray(getattr(tree, field))
            out["%s_%d_value" % (name, t)] = tree.value[:, 0, :].copy()
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
