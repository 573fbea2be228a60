"""Ranking scorers on the device: scoring time of roc_auc_ovr[_weighted], roc_auc_ovo[_weighted] and
average_precision next to the fit time, for BASELINE config 1 (digits, 4 C x 3 folds, 10 classes) and a
200k x 128, 10-class, 32 C x 5 fold search; scikit-learn's CPU scorer time on a sample of the fitted
(candidate, fold) estimators; the card's name and power limit.  One JSON line."""
import argparse, json, os, subprocess, sys, time, warnings
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
warnings.simplefilter("ignore")

p = argparse.ArgumentParser()
p.add_argument("--n", type=int, default=200_000)
p.add_argument("--d", type=int, default=128)
p.add_argument("--classes", type=int, default=10)
p.add_argument("--cands", type=int, default=32)
p.add_argument("--folds", type=int, default=5)
p.add_argument("--cpu-sample", type=int, default=2)
a = p.parse_args()

from sklearn.datasets import load_digits
from sklearn.linear_model import LogisticRegression
from sklearn.metrics import get_scorer
from sklearn.model_selection import StratifiedKFold
from skdist_b200 import engine as E
from skdist_b200.datasets import make_multiclass
from skdist_b200.distribute.folds import _fold_ids
from skdist_b200.distribute.logreg_family import _MultinomialFamily

SCORERS = ["roc_auc_ovr", "roc_auc_ovr_weighted", "roc_auc_ovo", "roc_auc_ovo_weighted", "average_precision"]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the card name still comes from torch below
        return "nvidia-smi unavailable: %s" % e


def case(X, y, Cs, n_splits):
    X = np.ascontiguousarray(X, dtype=np.float32)
    eng = E.get_engine()
    splits = list(StratifiedKFold(n_splits).split(X, y))
    fold = _fold_ids(splits, len(y))
    K = len(np.unique(y))
    fam = _MultinomialFamily(LogisticRegression(), [{"C": c} for c in Cs], X, y,
                             {s: get_scorer(s) for s in SCORERS})
    fam.stage(eng, X, fold, n_splits)
    C = np.repeat(np.asarray(Cs, dtype=np.float64), n_splits)
    f = np.tile(np.arange(n_splits, dtype=np.int32), len(Cs))
    t0 = time.perf_counter()
    res = eng.logreg_multinomial_fit_batch(C, f, K)
    fit_s = time.perf_counter() - t0
    out = {"fits": len(C), "fit_seconds": fit_s, "score_seconds": {}}
    for s in SCORERS:
        one = _MultinomialFamily(LogisticRegression(), [{}], X, y, {s: get_scorer(s)})
        one.score_columns(eng, res["coef"], f)                 # warm-up (scratch pool, cub temp sizes)
        t0 = time.perf_counter()
        v = one.score_columns(eng, res["coef"], f)[s]
        out["score_seconds"][s] = time.perf_counter() - t0
        out.setdefault("mean_score", {})[s] = float(np.nanmean(v))
    cpu = {}
    for s in SCORERS:
        t = 0.0
        for i in range(min(a.cpu_sample, len(C))):
            est = fam.make_estimator({"C": C[i]}, res["coef"][i], res["n_iter"][i], np.float32, X.shape[1])
            te = splits[f[i]][1]
            t0 = time.perf_counter()
            get_scorer(s)(est, X[te], y[te])
            t += time.perf_counter() - t0
        cpu[s] = t / max(1, min(a.cpu_sample, len(C)))
    out["sklearn_cpu_seconds_per_fit"] = cpu
    return out


line = {"card": card()}
try:
    import torch
    line["device"] = torch.cuda.get_device_name(0)
except Exception:
    pass
dg = load_digits()
line["config1_digits"] = case(dg.data, dg.target, [0.01, 0.1, 1.0, 10.0], 3)
X, y = make_multiclass(a.n, a.d, a.classes, seed=0)
line["synthetic_%dx%d_k%d" % (a.n, a.d, a.classes)] = case(X, y, list(np.logspace(-3, 2, a.cands)), a.folds)
print(json.dumps(line))
