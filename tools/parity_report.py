"""Predictions that differ from the reference (`flips` per held-out fold) on every logistic fixture,
for the fp32 CUDA-core kernels and for the tensor-core kernel separately, next to the reference's own
run-to-run envelope stored with the fixture.  One JSON line per (fixture, kernel); DESIGN.md section 4
quotes them.   python tools/parity_report.py"""
import json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from skdist_b200.engine import get_engine
from tests.test_gpu_parity import GOLD, _case, _fold_ids
eng = get_engine()
for name in ["search_logreg_g1_4000x16", "search_logreg_g1_20000x64", "search_logreg_g1_200000x256"]:
    g = np.load(os.path.join(GOLD, name + ".npz"))
    X, y, cv = _case(name)
    fold = _fold_ids(y, cv)
    eng.stage_x(X); eng.stage_labels(y); eng.stage_folds(fold, cv)
    Cs = g["C"]; C = np.repeat(Cs, cv); cf = np.tile(np.arange(cv, dtype=np.int32), len(Cs))
    gold = np.stack([g["split%d_test_score" % i] for i in range(cv)], 1).ravel()
    nf = g["noise_flips"].ravel(); nc = g["noise_coef"].ravel(); gi = g["n_iter"].ravel()
    gc = g["coef"].reshape(len(C), -1)
    stable = (nf == 0) & (nc < 1e-4) & (gi < 100)
    for kernel, kname in ((1, "simt-fp32"), (2, "tensor-core")):
        eng.set_kernel(kernel)
        res = eng.logreg_fit_batch(C, cf, np.ones(len(C), np.int32))
        correct, count = eng.linear_score_batch(res["coef"], cf, np.ones(len(C), np.int32))
        eng.set_kernel(0)
        flips = np.abs(correct - np.rint(gold * count))
        rel = np.abs(res["coef"] - gc).max(1) / np.abs(gc).max(1)
        mean = np.average((correct / count).reshape(len(Cs), cv), axis=1, weights=count[:cv])
        print(json.dumps({"fixture": name, "kernel": kname, "test_rows_per_fold": int(count[0]), "columns": len(C),
                          "flips_max": int(flips.max()), "flips_mean": float(flips.mean()),
                          "reference_envelope_flips_max": int(nf.max()), "reference_envelope_flips_mean": float(nf.mean()),
                          "excess_over_envelope_max": int(np.max(flips - nf)), "columns_above_envelope": int(np.sum(flips > nf)),
                          "stable_columns": int(stable.sum()), "flips_on_stable": int(flips[stable].sum()),
                          "coef_rel_on_stable_max": float(rel[stable].max()) if stable.any() else None,
                          "n_iter_diff_on_stable_max": int(np.abs(res["n_iter"][stable] - gi[stable]).max()) if stable.any() else None,
                          "max_abs_d_mean_test_score": float(np.abs(mean - g["mean_test_score"]).max()),
                          "best_index_device": int(mean.argmax()), "best_index_reference": int(g["best_index"])}))
