"""DistGridSearchCV(SGDClassifier) over alpha: (candidate, fold) fits per second on the device with X resident,
next to scikit-learn's GridSearchCV(n_jobs=-1) on a row subsample of the same grid.

Workloads: binary hinge and log_loss on make_g1_classification 500k x 256 (32 alphas x 5 folds), and 10-class
hinge on make_multiclass 200k x 64 (16 alphas x 3 folds).  The device time is the search family's fit + score
of every (candidate, fold) column after X, labels and folds are staged (one skd_sgd_fit_groups launch per
workload); the end-to-end DistGridSearchCV.fit time (staging, scoring, refit) is printed beside it.  The card
name and power limit are printed in the same run.  One JSON line per stage of each workload.  With alpha down
to 1e-7 the slowest columns of the full-size workloads run hundreds of epochs; --scale shrinks every row count."""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
p = argparse.ArgumentParser()
p.add_argument("--scale", type=float, default=1.0, help="multiplies every row count")
p.add_argument("--cpu-rows", type=int, default=20000, help="rows of the scikit-learn subsample")
p.add_argument("--skip-cpu", action="store_true")
p.add_argument("--skip-e2e", action="store_true", help="device launch only")
p.add_argument("--only", default="", help="comma-separated workloads to run: hinge, log_loss, multiclass")
a = p.parse_args()

from sklearn.linear_model import SGDClassifier
from sklearn.model_selection import GridSearchCV, check_cv

from skdist.distribute.search import DistGridSearchCV
from skdist_b200.datasets import make_g1_classification, make_multiclass
from skdist_b200.distribute.folds import _cv_fold_ids
from skdist_b200.distribute.search import _pick_family
from skdist_b200.distribute.utils import _check_multimetric_scoring
from skdist_b200.engine import get_engine


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        return "unknown (%s)" % e


def device(est, grid, X, y, cv):
    """(fits/s with X resident, seconds of the fit + score launch, epochs of the slowest column)."""
    eng = get_engine()
    cands = [{"alpha": float(v)} for v in grid["alpha"]]
    scorers, _ = _check_multimetric_scoring(est, scoring=None)
    splitter = check_cv(cv, y, classifier=True)
    fold, k = _cv_fold_ids(splitter, X, y, None, len(y))
    fam = _pick_family(est, cands, X, y, scorers)
    fam.stage(eng, X, fold, k)
    cols = np.arange(len(cands) * k)
    fam.run_columns(eng, cols[:k], k, False)         # warm-up: one candidate's folds
    t0 = time.perf_counter()
    out = fam.run_columns(eng, cols, k, False)
    dt = time.perf_counter() - t0
    return len(cols) / dt, dt, int(out["n_iter"].max())


def run(name, est, X, y, n_alpha, cv):
    """One JSON line per stage, printed as soon as it is measured: the device launch, the end-to-end search,
    scikit-learn on the subsample."""
    grid = {"alpha": np.logspace(-7, -2, n_alpha)}
    base = {"workload": name, "rows": len(y), "d": X.shape[1], "alphas": n_alpha, "folds": cv, "gpu": gpu}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        fits_s, dt, epochs = device(est, grid, X, y, cv)
        print(json.dumps(dict(base, stage="device, X resident", fits_per_s=fits_s, seconds=dt, max_epochs=epochs)),
              flush=True)
        if a.skip_e2e:
            return
        t0 = time.perf_counter()
        DistGridSearchCV(est, grid, cv=cv).fit(X, y)
        print(json.dumps(dict(base, stage="DistGridSearchCV.fit end to end", seconds=time.perf_counter() - t0)),
              flush=True)
        if not a.skip_cpu:
            m = min(a.cpu_rows, len(y))
            sub = np.random.RandomState(0).choice(len(y), m, replace=False)
            t0 = time.perf_counter()
            GridSearchCV(est, grid, cv=cv, n_jobs=-1).fit(X[sub], y[sub])
            cdt = time.perf_counter() - t0
            print(json.dumps(dict(base, stage="scikit-learn GridSearchCV(n_jobs=-1), row subsample", rows=m,
                                  fits_per_s=n_alpha * cv / cdt, seconds=cdt, cores=os.cpu_count())), flush=True)


get_engine()          # CUDA context / library load: process start-up, not part of a search
gpu = card()
only = set(a.only.split(",")) if a.only else {"hinge", "log_loss", "multiclass"}
X, y = make_g1_classification(int(500_000 * a.scale), 256, seed=0)
if "hinge" in only:
    run("binary hinge", SGDClassifier(random_state=0), X, y, 32, 5)
if "log_loss" in only:
    run("binary log_loss", SGDClassifier(loss="log_loss", random_state=0), X, y, 32, 5)
if "multiclass" in only:
    X, y = make_multiclass(int(200_000 * a.scale), 64, 10, seed=0)
    run("10-class hinge", SGDClassifier(random_state=0), X, y, 16, 3)
