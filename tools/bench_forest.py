"""Config 4 of BASELINE.json: DistRandomForestClassifier on synthetic lattice-valued n x d fp32;
prints one JSON line (trees/s) with a sampled CPU baseline (sklearn tree fit = the reference's
per-tree task) and checks the first tree against it bit for bit."""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
p = argparse.ArgumentParser()
p.add_argument("--n", type=int, default=2_000_000)
p.add_argument("--d", type=int, default=64)
p.add_argument("--trees", type=int, default=64)
p.add_argument("--cpu-sample", type=int, default=1)
p.add_argument("--cpu-jobs", type=int, default=0, help="0 = one sklearn tree per sampled core (cpu-sample trees, n_jobs=cpu-sample)")
p.add_argument("--class-weight", choices=["none", "balanced", "balanced_subsample"], default="none",
               help="class_weight of the forest (weighted instantiations of the builders)")
a = p.parse_args()
cw = None if a.class_weight == "none" else a.class_weight
from sklearn.ensemble import RandomForestClassifier
from skdist.distribute.ensemble import DistRandomForestClassifier
from skdist_b200.engine import get_engine
from tests.test_forest_gpu import lattice_data
X, y = lattice_data(a.n, a.d, seed=0)
get_engine()          # CUDA context / library load: one-time process start-up, not part of a fit
t0 = time.perf_counter()
rf = DistRandomForestClassifier(n_estimators=a.trees, random_state=0, class_weight=cw).fit(X, y)
dt = time.perf_counter() - t0
eng = get_engine()
nodes = np.array([e.tree_.node_count for e in rf.estimators_])
internal = [e.tree_.n_node_samples[e.tree_.children_left != -1].sum() for e in rf.estimators_]
mf = max(1, int(np.sqrt(a.d)))
alg_bytes = 8.0 * (mf + 1) * float(np.sum(internal))
line = {"workload": "DistRandomForestClassifier(n_estimators=%d, random_state=0, class_weight=%r) on lattice %dx%d fp32"
        % (a.trees, cw, a.n, a.d),
        "trees_per_s_e2e": a.trees / dt, "seconds": dt, "device_seconds": rf.device_seconds_,
        "nodes_mean": float(nodes.mean()), "depth_max": int(max(e.tree_.max_depth for e in rf.estimators_)),
        "builder_kernel_seconds": rf.kernel_seconds_,
        "algorithmic_bytes": alg_bytes, "algorithmic_GBps_device": alg_bytes / rf.device_seconds_ / 1e9,
        "algorithmic_GBps_builder_kernel": alg_bytes / max(rf.kernel_seconds_, 1e-9) / 1e9,
        "kernel": os.environ.get("SKDIST_B200_FOREST_KERNEL", "auto")}
if a.cpu_sample and cw != "balanced":     # scikit-learn 1.9 draws a "balanced" forest's bootstrap differently
    t0 = time.time()
    nj = a.cpu_jobs or a.cpu_sample
    ref = RandomForestClassifier(n_estimators=a.cpu_sample, random_state=0, n_jobs=nj, class_weight=cw).fit(X, y)
    dtc = time.time() - t0
    same = all(np.array_equal(r.tree_.threshold, o.tree_.threshold) and np.array_equal(r.tree_.children_left, o.tree_.children_left)
               for r, o in zip(ref.estimators_, rf.estimators_))
    line["cpu_baseline"] = {"value": a.cpu_sample / dtc, "unit": "trees/s", "cores": nj, "kind": "port", "host_cores": os.cpu_count(),
                            "sample": "%d tree(s) in %.1f s, %d at a time (one tree per core, as the reference's tasks)" % (a.cpu_sample, dtc, nj),
                            "bit_identical_to_gpu": bool(same)}
print(json.dumps(line))
