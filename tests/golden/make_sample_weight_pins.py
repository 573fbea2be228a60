"""Generate tests/golden/sample_weight_pins.npz: the scores of the UNMODIFIED reference's `_fit_and_score`
(sk-dist, imported under oracle/refshim.py) with fit_params={"sample_weight": w}, so that
tests/test_sample_weight_host.py pins tests/weighted_search_oracle.py against it without the reference tree.

    SKDIST_REFERENCE_ROOT=<sk-dist checkout> python tests/golden/make_sample_weight_pins.py
"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402
from tests import weighted_search_oracle as wso  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def reference_task(ref_search, fit_params):
    def task(estimator, X, y, scorer, train, test, params):
        # the call DistBaseSearchCV.fit makes (ref search.py:391-406), with the search's fit_params
        return ref_search._fit_and_score(
            estimator, X, y, {"score": scorer}, train, test, 0, params, fit_params=fit_params,
            return_train_score=False, return_n_test_samples=True, return_times=True,
            return_parameters=False, error_score="raise")
    return task


def main():
    from sklearn.linear_model import LogisticRegression
    warnings.simplefilter("ignore")
    ref_search, _, _ = refshim.load()
    out = {}
    for n_classes in (2, 4):
        X, y, w, cands, cv = wso.sample_weight_case(n_classes)
        fp = {"sample_weight": w}
        a = wso.search_cv(LogisticRegression(), cands, X, y, cv=cv, fit_params=fp, refit=False,
                          task_fn=reference_task(ref_search, fp))
        res = a["cv_results_"]
        for i in range(a["n_splits_"]):
            out["k%d_split%d_test_score" % (n_classes, i)] = np.asarray(res["split%d_test_score" % i], np.float64)
        out["k%d_mean_test_score" % n_classes] = np.asarray(res["mean_test_score"], np.float64)
        out["k%d_best_index" % n_classes] = np.int64(a["best_index_"])
    np.savez_compressed(os.path.join(HERE, "sample_weight_pins.npz"), **out)


if __name__ == "__main__":
    main()
