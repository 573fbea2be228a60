"""DistRandomForestClassifier on continuous float32 features with SKDIST_B200_FOREST_SORT=1 (the sort-based best
splitter), on the config-4 generator of bench_configs.py: 2M x 64 standard-normal draws, binary target.  In the
same process it also times the same data with SKDIST_B200_FOREST_MAX_BINS=256 (the histogram approximation),
the config-4 lattice (floor to 256 levels) with and without the switch (the same histogram builders run, so
the two should agree within spread), and a smaller point; a CPU scikit-learn fit of the first tree of the
smaller point is the bit-identity check.  One JSON line per run: device seconds (`last_forest_seconds` summed
over the fit), builder-kernel seconds, end-to-end seconds, nodes per tree.  Set SKDIST_B200_LIBPATH to time
another build."""
import argparse, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
p = argparse.ArgumentParser()
p.add_argument("--n", type=int, default=2_000_000)
p.add_argument("--small-n", type=int, default=200_000)
p.add_argument("--d", type=int, default=64)
p.add_argument("--trees", type=int, default=32)
p.add_argument("--cpu-sample", type=int, default=1, help="trees of the smaller point fitted by scikit-learn (0: none)")
p.add_argument("--reps", type=int, default=1)
a = p.parse_args()

from sklearn.ensemble import RandomForestClassifier
from skdist.distribute.ensemble import DistRandomForestClassifier
from skdist_b200.engine import get_engine


def data(kind, n):
    rng = np.random.default_rng(0)
    Z = rng.standard_normal((n, a.d))
    s = Z[:, 0] + 0.5 * Z[:, 1] * Z[:, 2] - 0.7 * Z[:, 3] + 0.8 * rng.standard_normal(n)
    if kind == "lattice":
        X = np.clip(np.floor((Z + 4.0) / 8.0 * 256), 0, 255).astype(np.float32)
    else:
        X = Z.astype(np.float32)
    return X, (s > 0).astype(np.int64)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        return "unknown (%s)" % e


def run(kind, n, mode, X, y):
    os.environ.pop("SKDIST_B200_FOREST_SORT", None)
    os.environ.pop("SKDIST_B200_FOREST_MAX_BINS", None)
    if mode == "sort":
        os.environ["SKDIST_B200_FOREST_SORT"] = "1"
    elif mode == "max_bins=256":
        os.environ["SKDIST_B200_FOREST_MAX_BINS"] = "256"
    for rep in range(a.reps):
        t0 = time.perf_counter()
        est = DistRandomForestClassifier(n_estimators=a.trees, random_state=0).fit(X, y)
        dt = time.perf_counter() - t0
        line = {"estimator": "randomforest", "mode": mode, "data": "%s %dx%d fp32" % (kind, n, a.d), "trees": a.trees,
                "rep": rep, "seconds_e2e": dt, "device_seconds": est.device_seconds_,
                "builder_kernel_seconds": est.kernel_seconds_, "trees_per_s_device": a.trees / est.device_seconds_,
                "nodes_mean": float(np.mean([e.tree_.node_count for e in est.estimators_])),
                "lib": os.environ.get("SKDIST_B200_LIBPATH", "in-tree"), "gpu": gpu}
        print(json.dumps(line), flush=True)
    return est


get_engine()          # CUDA context / library load: process start-up, not part of a fit
gpu = card()
X, y = data("continuous", a.n)
run("continuous", a.n, "sort", X, y)
run("continuous", a.n, "max_bins=256", X, y)
X, y = data("lattice", a.n)
run("lattice", a.n, "sort", X, y)
run("lattice", a.n, "unset", X, y)
X, y = data("continuous", a.small_n)
est = run("continuous", a.small_n, "sort", X, y)
if a.cpu_sample:
    t0 = time.perf_counter()
    ref = RandomForestClassifier(n_estimators=a.cpu_sample, random_state=0).fit(X, y)
    dtc = time.perf_counter() - t0
    # the first tree seeds of a forest do not depend on n_estimators
    same = all(np.array_equal(r.tree_.threshold, o.tree_.threshold) and
               np.array_equal(r.tree_.children_left, o.tree_.children_left) and
               np.array_equal(r.tree_.value, o.tree_.value)
               for r, o in zip(ref.estimators_, est.estimators_))
    print(json.dumps({"cpu_sample": {"data": "continuous %dx%d fp32" % (a.small_n, a.d), "trees": a.cpu_sample,
                                     "seconds": dtc, "bit_identical_to_gpu": same}, "gpu": gpu}), flush=True)
os.environ.pop("SKDIST_B200_FOREST_SORT", None)
