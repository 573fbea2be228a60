"""Generate tests/golden/reference_pins.npz and tests/golden/reference_surface.json: what the tests that
pin this package against the UNMODIFIED reference (sk-dist, imported under oracle/refshim.py) compare with,
stored so that those tests run without the reference tree.

    SKDIST_REFERENCE_ROOT=<sk-dist checkout> python tests/golden/make_reference_pins.py
"""
import inspect
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refshim, search_oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
SURFACE = {
    "search": ["DistGridSearchCV", "DistRandomizedSearchCV", "DistMultiModelSearch"],
    "multiclass": ["DistOneVsRestClassifier", "DistOneVsOneClassifier"],
    "ensemble": ["DistRandomForestClassifier", "DistRandomForestRegressor", "DistExtraTreesClassifier",
                 "DistExtraTreesRegressor", "DistRandomTreesEmbedding"],
    "eliminate": ["DistFeatureEliminator"],
}
NEGATIVES = [(300, "ratio"), (0.2, "ratio"), (2, "multiplier"), (1.5, "multiplier"), (10 ** 6, "ratio")]
ELIMINATE = [(2, 3, None), (3, 4, 3)]          # (step, cv folds, min_features_to_select; None = d // 2)


def MULTI_MODELS():
    from sklearn.linear_model import LogisticRegression
    return [("a", LogisticRegression(), {"C": [0.01, 0.1, 1.0, 10.0]}),
            ("b", LogisticRegression(fit_intercept=False), {"C": [0.5, 5.0], "tol": [1e-4, 1e-3]})]


def params(cls):
    out = []
    for k, v in inspect.signature(cls.__init__).parameters.items():
        if k != "self":
            out.append([k, v.kind == v.VAR_KEYWORD, None if v.default is inspect._empty else repr(v.default)])
    return out


def eliminate_sets(X, y, base, step, min_keep):
    """Feature sets as the reference's eliminator builds them (ref eliminate.py:131-154)."""
    from sklearn.base import clone
    d = X.shape[1]
    coefs = clone(base).fit(X, y).coef_
    ranks = np.ravel(np.argsort((coefs ** 2).sum(axis=0)))[: d - min_keep]
    sets, k = [np.array([])], 0
    while k < d - min_keep:
        k += step
        sets.append(ranks[:k])
    return sets


def main():
    from sklearn.linear_model import LogisticRegression, SGDClassifier
    from sklearn.metrics import check_scoring
    from sklearn.model_selection import ParameterGrid, StratifiedKFold
    from sklearn.tree import DecisionTreeClassifier
    from skdist_b200.datasets import make_g1_classification, make_multiclass
    from tests.golden.make_golden import reference_task
    from tests.test_eliminate_host import _data
    from tests.test_forest_host import MAX_RAND_SEED, lattice
    warnings.simplefilter("ignore")
    ref_search, ref_mc, ref_ens = refshim.load()
    ref_elim = refshim.load_module("skdist.distribute.eliminate")
    mods = {"search": ref_search, "multiclass": ref_mc, "ensemble": ref_ens, "eliminate": ref_elim}
    surface = {name: {"params": params(getattr(mods[m], name)),
                      "public": sorted(n for n in dir(getattr(mods[m], name)) if not n.startswith("_"))}
               for m, names in SURFACE.items() for name in names}
    with open(os.path.join(HERE, "reference_surface.json"), "w") as f:
        json.dump(surface, f, indent=1, sort_keys=True)

    out = {}
    # reference _fit_and_score on a small search (tests/test_oracle.py)
    X, y = make_g1_classification(1500, 8, seed=5)
    a = search_oracle.search_cv(LogisticRegression(), list(ParameterGrid({"C": [0.1, 10.0]})), X, y, cv=3,
                                task_fn=reference_task(ref_search))
    out["task_mean_test_score"] = np.asarray(a["cv_results_"]["mean_test_score"], np.float64)
    out["task_best_C"] = np.float64(a["best_params_"]["C"])
    # reference DistOneVsRestClassifier(SGDClassifier), sc=None (tests/test_multiclass_host.py)
    X, y = make_multiclass(500, 6, 4, seed=8)
    r = ref_mc.DistOneVsRestClassifier(SGDClassifier(random_state=0)).fit(X, y)
    out["ovr_sgd_coef"] = np.stack([e.coef_.ravel() for e in r.estimators_])
    # reference _negatives_mask rows
    rng = np.random.default_rng(0)
    n = 5000
    Xn = np.arange(n, dtype=np.float64)[:, None]
    yn = (rng.random(n) < 0.07).astype(int)
    for i, (mn, method) in enumerate(NEGATIVES):
        for rs in (0, 7):
            Xr, _ = ref_mc._negatives_mask(Xn, yn, max_negatives=mn, random_state=rs, method=method)
            out["negatives_rows_%d_%d" % (i, rs)] = np.sort(Xr[:, 0].astype(np.int64))
    # reference eliminator task function (tests/test_eliminate_host.py)
    X, y = _data()
    for i, (step, n_cv, min_keep) in enumerate(ELIMINATE):
        base = LogisticRegression(C=0.3)
        sets = eliminate_sets(X, y, base, step, X.shape[1] // 2 if min_keep is None else min_keep)
        scorer = check_scoring(base, scoring=None)
        out["eliminate_scores_%d" % i] = np.array(
            [np.mean([ref_elim._fit_and_score_one(idx, base, X, y, scorer, tr, te, False, {})
                      for tr, te in StratifiedKFold(n_cv).split(X, y)]) for idx in sets])
    # reference _build_trees (tests/test_forest_host.py)
    X, y = lattice(1500, 8, 3)
    states = np.random.RandomState(5).randint(MAX_RAND_SEED, size=3)
    for i, s in enumerate(states):
        tr = ref_ens._build_trees(DecisionTreeClassifier(max_features="sqrt"), (), {}, X,
                                  y.astype(np.float64)[:, None], None, s, 3, bootstrap=True)
        out["trees_threshold_%d" % i] = tr.tree_.threshold
        out["trees_children_left_%d" % i] = tr.tree_.children_left.astype(np.int64)
    X, y = lattice(300, 4, 6)
    out["oof"] = ref_ens.get_oof(LogisticRegression(), X, y, n_splits=3)[1]
    # reference DistMultiModelSearch task functions, Spark semantics (tests/test_search_host.py)
    import copy
    from itertools import product
    X, y = make_g1_classification(400, 5, seed=6)
    models = MULTI_MODELS()
    folds = list(StratifiedKFold(4).split(X, y))
    param_sets = ref_search._raw_sampler(models, n=3, random_state=11)
    scores = [ref_search._fit_one_fold((f, copy.deepcopy(ps)), models, X, y, None, {})
              for f, ps in product(folds, param_sets)]
    results = ref_search._get_results(scores)
    out["multi_model_params"] = np.array(json.dumps(list(results["param_set"])))
    out["multi_model_index"] = np.asarray(results["model_index"], np.int64)
    out["multi_model_score"] = np.asarray(results["score"].values, np.float64)
    np.savez_compressed(os.path.join(HERE, "reference_pins.npz"), **out)


if __name__ == "__main__":
    main()
