#!/usr/bin/env python
"""Weighted against unweighted fits at the headline shape: 1M x 256 fp32, 512 C values x 5 folds, binary
LogisticRegression with class_weight={0: 1, 1: 3} and with class_weight=None, alternated in one process.
Prints candidate-fits/s of each (the batched lbfgs solve, X / labels / folds already on the device) with
the card's name and power limit.

    python tools/bench_class_weight.py [--n N] [--d D] [--candidates K] [--reps R]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--n", type=int, default=1_000_000)
    p.add_argument("--d", type=int, default=256)
    p.add_argument("--candidates", type=int, default=512)
    p.add_argument("--folds", type=int, default=5)
    p.add_argument("--reps", type=int, default=3)
    a = p.parse_args()
    from skdist_b200.datasets import make_g1_classification
    from skdist_b200.distribute.logreg_family import _ClassWeights
    from skdist_b200.engine import Engine
    X, y = make_g1_classification(a.n, a.d, seed=0)
    y = np.asarray(y).astype(np.int32)
    fold = (np.arange(a.n) % a.folds).astype(np.int8)
    eng = Engine(0)
    eng.stage_x(X)
    eng.stage_labels(y)
    eng.stage_folds(fold, a.folds)
    C = np.repeat(np.logspace(-4, 4, a.candidates), a.folds)
    cf = np.tile(np.arange(a.folds, dtype=np.int32), a.candidates)
    pos = np.ones(len(C), np.int32)
    cw = _ClassWeights(np.array([0, 1]), y)
    cw.set_folds(fold)
    cols = [cw.column({0: 1, 1: 3}, f) for f in cf]
    W, sw = np.stack([c[0] for c in cols]), np.array([c[1] for c in cols])

    def run(weighted):
        if weighted:
            eng.stage_class_weights(W, sw)
        t0 = time.time()
        res = eng.logreg_fit_batch(C, cf, pos)
        dt = time.time() - t0
        return len(C) / dt, int(res["n_evals"].sum()) / dt

    run(False), run(True)       # warm-up of both variants
    rates = {"none": [], "class_weight": []}
    evals = {"none": [], "class_weight": []}     # the two objectives take different numbers of evaluations
    for _ in range(a.reps):
        for k in rates:
            r, e = run(k == "class_weight")
            rates[k].append(r)
            evals[k].append(e)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"shape": [a.n, a.d], "columns": len(C), "card": card,
                      "fits_per_s": {k: [round(v, 1) for v in r] for k, r in rates.items()},
                      "column_evaluations_per_s": {k: [round(v) for v in r] for k, r in evals.items()}}))


if __name__ == "__main__":
    main()
