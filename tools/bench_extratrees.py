"""DistExtraTreesClassifier and DistRandomTreesEmbedding on the config-4 generator of bench_configs.py: the
lattice (floor to 256 levels) and the same draws without the floor (continuous float32).  One JSON line per
(estimator, data): device seconds (`last_forest_seconds` summed over the fit), end-to-end seconds, and a CPU
scikit-learn fit of the first trees as a parity check.  Set SKDIST_B200_LIBPATH to time another build."""
import argparse, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
p = argparse.ArgumentParser()
p.add_argument("--n", type=int, default=2_000_000)
p.add_argument("--d", type=int, default=64)
p.add_argument("--trees", type=int, default=32)
p.add_argument("--embedding-trees", type=int, default=100)
p.add_argument("--cpu-sample", type=int, default=1, help="trees fitted by scikit-learn for the parity check (0: none)")
p.add_argument("--data", choices=["both", "continuous", "lattice"], default="both")
p.add_argument("--reps", type=int, default=1)
a = p.parse_args()

from sklearn.ensemble import ExtraTreesClassifier, RandomTreesEmbedding
from skdist.distribute.ensemble import DistExtraTreesClassifier, DistRandomTreesEmbedding
from skdist_b200.engine import get_engine


def data(kind):
    rng = np.random.default_rng(0)
    Z = rng.standard_normal((a.n, a.d))
    s = Z[:, 0] + 0.5 * Z[:, 1] * Z[:, 2] - 0.7 * Z[:, 3] + 0.8 * rng.standard_normal(a.n)
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


get_engine()          # CUDA context / library load: process start-up, not part of a fit
gpu = card()
kinds = ["continuous", "lattice"] if a.data == "both" else [a.data]
for kind in kinds:
    X, y = data(kind)
    for name in ("extratrees", "embedding"):
        for rep in range(a.reps):
            t0 = time.perf_counter()
            if name == "extratrees":
                est = DistExtraTreesClassifier(n_estimators=a.trees, random_state=0).fit(X, y)
            else:
                est = DistRandomTreesEmbedding(n_estimators=a.embedding_trees, random_state=0).fit(X)
            dt = time.perf_counter() - t0
            nt = a.trees if name == "extratrees" else a.embedding_trees
            line = {"estimator": name, "data": "%s %dx%d fp32" % (kind, a.n, a.d), "trees": nt, "rep": rep,
                    "seconds_e2e": dt, "device_seconds": est.device_seconds_, "builder_kernel_seconds": est.kernel_seconds_, "trees_per_s_device": nt / est.device_seconds_,
                    "nodes_mean": float(np.mean([e.tree_.node_count for e in est.estimators_])),
                    "lib": os.environ.get("SKDIST_B200_LIBPATH", "in-tree"), "gpu": gpu}
            if a.cpu_sample and rep == 0:
                t0 = time.perf_counter()
                if name == "extratrees":
                    ref = ExtraTreesClassifier(n_estimators=a.cpu_sample, random_state=0).fit(X, y)
                else:
                    ref = RandomTreesEmbedding(n_estimators=a.cpu_sample, random_state=0).fit(X)
                dtc = time.perf_counter() - t0
                # the first tree seeds of a forest do not depend on n_estimators
                same = all(np.array_equal(r.tree_.threshold, o.tree_.threshold) and
                           np.array_equal(r.tree_.children_left, o.tree_.children_left)
                           for r, o in zip(ref.estimators_, est.estimators_))
                line["cpu_sample"] = {"trees": a.cpu_sample, "seconds": dtc, "trees_per_s": a.cpu_sample / dtc,
                                      "bit_identical_to_gpu": same}
            print(json.dumps(line), flush=True)
