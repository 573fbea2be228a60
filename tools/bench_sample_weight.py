#!/usr/bin/env python
"""A LogisticRegression grid search at a user-sized shape (200k x 64 fp32, binary, 16 C values x 5 folds) in
four variants, alternated and repeated in one process: unweighted, class_weight="balanced", integer sample
weights 0..3 and log-normal sample weights.  Prints the wall time of each DistGridSearchCV.fit (fits, scoring
and refit; X staged by every fit as a user's call stages it) with the card's name and power limit.

Then the cost of the per-row load in the weighted epilogue alone: one batched fit of 512 C values x 5 folds on
the same data with class weights {0: 1, 1: 3}, without and with all-ones sample weights (the same objective, so
the same iterations; only the row-weight load differs), alternated, device seconds of each (`gpu_seconds`).

    python tools/bench_sample_weight.py [--n N] [--d D] [--candidates K] [--reps R]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=200_000)
    p.add_argument("--d", type=int, default=64)
    p.add_argument("--candidates", type=int, default=16)
    p.add_argument("--folds", type=int, default=5)
    p.add_argument("--reps", type=int, default=3)
    a = p.parse_args()
    from sklearn.linear_model import LogisticRegression
    from skdist.distribute.search import DistGridSearchCV
    from skdist_b200.datasets import make_g1_classification
    X, y = make_g1_classification(a.n, a.d, seed=0)
    rng = np.random.default_rng(0)
    variants = {
        "none": ({}, {}),
        "balanced": ({"class_weight": "balanced"}, {}),
        "int_0_3": ({}, {"sample_weight": rng.integers(0, 4, a.n).astype(np.float64)}),
        "lognormal": ({}, {"sample_weight": np.exp(rng.normal(0.0, 1.0, a.n))}),
    }
    grid = {"C": list(np.logspace(-3, 3, a.candidates))}

    def run(name):
        kw, fp = variants[name]
        gs = DistGridSearchCV(LogisticRegression(**kw), grid, None, cv=a.folds)
        t0 = time.time()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gs.fit(X, y, **fp)
        return time.time() - t0, float(gs.best_score_)

    for k in variants:      # warm-up of every variant
        run(k)
    secs = {k: [] for k in variants}
    best = {}
    for _ in range(a.reps):
        for k in variants:
            s, best[k] = run(k)
            secs[k].append(s)
    # the weighted epilogue with and without its per-row load, at the engine level
    from skdist_b200.distribute.logreg_family import _ClassWeights
    from skdist_b200.engine import get_engine
    eng = get_engine()
    yc = np.asarray(y).astype(np.int32)
    fold = (np.arange(a.n) % a.folds).astype(np.int8)
    eng.stage_x(np.asarray(X, np.float32))
    eng.stage_labels(yc)
    eng.stage_folds(fold, a.folds)
    C = np.repeat(np.logspace(-4, 4, 512), a.folds)
    cf = np.tile(np.arange(a.folds, dtype=np.int32), 512)
    pos = np.ones(len(C), np.int32)
    cw = _ClassWeights(np.array([0, 1]), yc)
    cw.set_folds(fold)
    cols = [cw.column({0: 1, 1: 3}, f) for f in cf]
    W, sw = np.stack([c[0] for c in cols]), np.array([c[1] for c in cols])
    ones = np.ones(a.n, np.float32)

    def fit(rows):
        eng.stage_class_weights(W, sw)
        if rows:
            eng.stage_sample_weights(ones)
        r = eng.logreg_fit_batch(C, cf, pos)
        return r["gpu_seconds"], int(r["n_evals"].sum())

    fit(False), fit(True)
    epi = {"class_weight": [], "class_weight+ones": []}
    evals = {}
    for _ in range(a.reps):
        for k in epi:
            t, evals[k] = fit(k != "class_weight")
            epi[k].append(t)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"shape": [a.n, a.d], "fits": a.candidates * a.folds, "card": card,
                      "search_seconds": {k: [round(v, 3) for v in s] for k, s in secs.items()},
                      "median_seconds": {k: round(float(np.median(s)), 3) for k, s in secs.items()},
                      "best_score": best,
                      "epilogue_fit_columns": len(C),
                      "epilogue_gpu_seconds": {k: [round(v, 4) for v in s] for k, s in epi.items()},
                      "epilogue_column_evaluations": evals}))


if __name__ == "__main__":
    main()
