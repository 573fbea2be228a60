"""DistRandomForestClassifier with criterion="entropy" against Gini on the same forest: a config-4-like lattice
(2M x 64 features floored to 256 levels, 3 classes) timed under three settings -- Gini on the default
(throughput) builder, Gini with SKDIST_B200_FOREST_KERNEL=general, and entropy (always the general builder) --
then one continuous case with SKDIST_B200_FOREST_SORT=1, Gini and entropy.  The card name and power limit are
printed in the same run.  One JSON line per fit: device seconds (`last_forest_seconds` summed over the fit),
builder-kernel seconds, end-to-end seconds, nodes per tree."""
import argparse, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
p = argparse.ArgumentParser()
p.add_argument("--n", type=int, default=2_000_000)
p.add_argument("--d", type=int, default=64)
p.add_argument("--trees", type=int, default=64)
p.add_argument("--sort-n", type=int, default=500_000)
p.add_argument("--sort-trees", type=int, default=8)
a = p.parse_args()

from skdist.distribute.ensemble import DistRandomForestClassifier
from skdist_b200.engine import get_engine


def data(kind, n):
    rng = np.random.default_rng(0)
    Z = rng.standard_normal((n, a.d))
    s = Z[:, 0] + 0.5 * Z[:, 1] * Z[:, 2] - 0.7 * Z[:, 3] + 0.8 * rng.standard_normal(n)
    X = np.clip(np.floor((Z + 4.0) / 8.0 * 256), 0, 255).astype(np.float32) if kind == "lattice" else Z.astype(np.float32)
    return X, np.digitize(s, np.quantile(s, [1 / 3, 2 / 3])).astype(np.int64)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        return "unknown (%s)" % e


def run(kind, X, y, criterion, trees, env):
    for v in ("SKDIST_B200_FOREST_SORT", "SKDIST_B200_FOREST_KERNEL"):
        os.environ.pop(v, None)
    os.environ.update(env)
    t0 = time.perf_counter()
    est = DistRandomForestClassifier(n_estimators=trees, criterion=criterion, random_state=0).fit(X, y)
    dt = time.perf_counter() - t0
    print(json.dumps({"criterion": criterion, "env": env, "data": "%s %dx%d fp32, 3 classes" % (kind, len(y), a.d),
                      "trees": trees, "seconds_e2e": dt, "device_seconds": est.device_seconds_,
                      "builder_kernel_seconds": est.kernel_seconds_,
                      "nodes_mean": float(np.mean([e.tree_.node_count for e in est.estimators_])), "gpu": gpu}),
          flush=True)


get_engine()          # CUDA context / library load: process start-up, not part of a fit
gpu = card()
X, y = data("lattice", a.n)
run("lattice", X, y, "gini", a.trees, {})
run("lattice", X, y, "gini", a.trees, {"SKDIST_B200_FOREST_KERNEL": "general"})
run("lattice", X, y, "entropy", a.trees, {})
X, y = data("continuous", a.sort_n)
run("continuous", X, y, "gini", a.sort_trees, {"SKDIST_B200_FOREST_SORT": "1"})
run("continuous", X, y, "entropy", a.sort_trees, {"SKDIST_B200_FOREST_SORT": "1"})
for v in ("SKDIST_B200_FOREST_SORT", "SKDIST_B200_FOREST_KERNEL"):
    os.environ.pop(v, None)
