"""bench.py --config {3,4,5}: the other BASELINE.json configurations, same JSON schema as the headline.

  3  DistOneVsRestClassifier(SGDClassifier) 1000 classes on synthetic 500k x 512   label-fits/s
  4  DistRandomForestClassifier(n_estimators=1024) on synthetic 2M x 64 (lattice)     trees/s
  5  DistRandomizedSearchCV(Ridge) n_iter=2048 x 5 folds on synthetic 1M x 256        fits/s
     (+ skdist.predict batched inference on 10M rows, reported under config.predict)

`value`: whole-job throughput of the engine call with X, y (and folds) already staged in HBM, device
time from CUDA events on the library's stream, max over ranks.  `e2e`: the public estimator's
`fit` on HOST numpy arrays (staging, fits, results back, sklearn objects built), wall clock, max over
ranks.  `roofline`: SURVEY.md section 8(d)'s algorithmic bytes / flops of the whole call over its
device time.  `cpu_baseline` and
`--impl reference`: scikit-learn's own estimator (what every reference task runs) fanned out over the
host cores with joblib, one bounded wave.
"""
import json
import os
import time
import warnings

import numpy as np

UNITS = {3: ("label-fits/sec DistOneVsRestClassifier(SGDClassifier) K=1000 500kx512", "label-fits/s"),
         4: ("trees/sec DistRandomForestClassifier(n_estimators=1024) 2Mx64", "trees/s"),
         5: ("candidate-fits/sec (params x folds) DistRandomizedSearchCV(Ridge) 1Mx256", "fits/s")}


def sizes(a):
    if a.config == 3:
        return dict(n=a.n or 500_000, d=a.d or 512, k=a.candidates if a.candidates != 512 else 1000)
    if a.config == 4:
        return dict(n=a.n or 2_000_000, d=a.d or 64, trees=a.candidates if a.candidates != 512 else 1024)
    return dict(n=a.n or 1_000_000, d=a.d or 256, n_iter=a.candidates if a.candidates != 512 else 2048, folds=a.folds,
                predict_rows=10_000_000)


def workload_name(a, z):
    if a.config == 3:
        return "DistOneVsRestClassifier(SGDClassifier(random_state=0)) K=%d, synthetic %dx%d fp32" % (z["k"], z["n"], z["d"])
    if a.config == 4:
        return "DistRandomForestClassifier(n_estimators=%d, random_state=0), synthetic lattice %dx%d fp32" % (
            z["trees"], z["n"], z["d"])
    return "DistRandomizedSearchCV(Ridge, alpha~loguniform(1e-3,1e3)) n_iter=%d x %d folds, synthetic G1 %dx%d fp32" % (
        z["n_iter"], z["folds"], z["n"], z["d"])


def make_data(a, z):
    from skdist_b200 import datasets
    if a.config == 3:
        return datasets.make_multiclass(z["n"], z["d"], z["k"], seed=0)
    if a.config == 4:
        rng = np.random.default_rng(0)
        Z = rng.standard_normal((z["n"], z["d"]))
        X = np.clip(np.floor((Z + 4.0) / 8.0 * 256), 0, 255).astype(np.float32)
        s = Z[:, 0] + 0.5 * Z[:, 1] * Z[:, 2] - 0.7 * Z[:, 3] + 0.8 * rng.standard_normal(z["n"])
        return X, (s > 0).astype(np.int64)
    return datasets.make_g1_regression(z["n"], z["d"], seed=0)


# ---------------------------------------------------------------------------------------------
# CPU legs (scikit-learn's own estimators = what each reference task runs)
# ---------------------------------------------------------------------------------------------
def cpu_leg(a, z, X, y, n_units):
    """Run a bounded sample of the workload's units on the host cores.  Returns
    (units/s, seconds, description, cores used, per-unit results for the parity check)."""
    from joblib import Parallel, delayed, parallel_config
    cores = os.cpu_count() or 1
    warnings.simplefilter("ignore")
    if a.config == 3:
        from sklearn.linear_model import SGDClassifier
        ks = list(range(min(n_units, z["k"])))
        nj = min(len(ks), cores)

        def one(k):   # ref multiclass.py:109-152 `_fit_binary` on column k of the label matrix
            m = SGDClassifier(random_state=0).fit(X, (y == k).astype(int))
            return m.coef_[0].copy(), float(m.intercept_[0]), int(m.n_iter_)
        t0 = time.time()
        with parallel_config(backend="loky", n_jobs=nj, inner_max_num_threads=1):
            out = Parallel()(delayed(one)(k) for k in ks)
        dt = time.time() - t0
        return len(ks) / dt, dt, "%d label columns, %d at a time (SGD is single-threaded per column)" % (len(ks), nj), nj, out
    if a.config == 4:
        from sklearn.ensemble import RandomForestClassifier
        nt = min(n_units, z["trees"])
        nj = min(nt, cores)
        t0 = time.time()
        ref = RandomForestClassifier(n_estimators=nt, random_state=0, n_jobs=nj).fit(X, y)
        dt = time.time() - t0
        return nt / dt, dt, "%d trees, %d at a time (one tree per core, as the reference's tasks)" % (nt, nj), nj, ref.estimators_
    from sklearn.linear_model import Ridge
    from sklearn.model_selection import KFold, ParameterSampler
    from scipy.stats import loguniform
    cands = list(ParameterSampler({"alpha": loguniform(1e-3, 1e3)}, n_iter=z["n_iter"], random_state=0))
    splits = list(KFold(z["folds"]).split(X))
    idx = np.unique(np.linspace(0, len(cands) - 1, max(1, n_units // z["folds"])).round().astype(int))
    tasks = [(int(ci), f) for ci in idx for f in range(z["folds"])]
    nj = max(1, min(len(tasks), 32, cores))
    inner = max(1, cores // nj)

    def one(ci, f):   # ref search.py:180-288 `_fit_and_score`
        tr, te = splits[f]
        m = Ridge(**cands[ci]).fit(X[tr], y[tr])
        return float(m.score(X[te], y[te]))
    t0 = time.time()
    with parallel_config(backend="loky", n_jobs=nj, inner_max_num_threads=inner):
        out = Parallel()(delayed(one)(ci, f) for ci, f in tasks)
    dt = time.time() - t0
    return len(tasks) / dt, dt, "%d (alpha, fold) fits, joblib n_jobs=%d x %d BLAS threads" % (len(tasks), nj, inner), cores, (tasks, out)


def run_reference(a):
    if int(os.environ.get("RANK", 0)) != 0:
        return
    z = sizes(a)
    X, y = make_data(a, z)
    cores = os.cpu_count() or 1
    n_units = max(a.cpu_sample, min(64, cores))
    v, dt, desc, used, _ = cpu_leg(a, z, X, y, n_units)
    metric, unit = UNITS[a.config]
    line = {"impl": "reference", "metric": metric, "value": v, "unit": unit, "n_gpus": a.gpus, "steps": a.steps,
            "warmup": a.warmup, "ms_per_step": 1e3 * dt / max(1, a.steps), "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": {3: "f32", 4: "u8", 5: "f32"}[a.config], "data": "synthetic",
            "config": {"workload": workload_name(a, z), "inputs": "exceed L2"},
            "cpu_baseline": {"value": v, "unit": unit, "cores": used, "host_cores": cores, "kind": "port",
                             "sample": desc + "; all steps run as one wave"},
            "e2e": {"value": v, "unit": unit, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}, "gpu_launches": 0}
    print(json.dumps(line))


# ---------------------------------------------------------------------------------------------
# device arms
# ---------------------------------------------------------------------------------------------
def run(a, ClockSampler, peaks, dump_outputs):
    import torch
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", 1))
    rank = int(os.environ.get("RANK", 0))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from skdist_b200 import parallel
    from skdist_b200.engine import get_engine
    warnings.simplefilter("ignore")
    z = sizes(a)
    X, y = make_data(a, z)
    eng = get_engine()
    metric, unit = UNITS[a.config]

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    extra = {}
    # ---- resident arm: one step = the engine call over this rank's share of the units
    if a.config == 3:
        from sklearn.linear_model import SGDClassifier
        eng.stage_x(X)
        eng.stage_labels(y.astype(np.int32))
        eng.stage_folds(None, 0)
        mine = parallel.shard_indices(z["k"], rank, world).astype(np.int32)
        n_units = z["k"]
        res_box = {}

        def step():
            res_box["r"] = eng.sgd_fit_batch(SGDClassifier(random_state=0), mine)
    elif a.config == 4:
        from skdist_b200.bootstrap import bootstrap_counts
        from sklearn.utils import check_random_state
        eng.stage_x(X)
        eng.stage_labels(y.astype(np.int32))
        eng.stage_folds(None, 0)
        states = list(check_random_state(0).randint(np.iinfo(np.int32).max, size=z["trees"]))
        mine = parallel.shard_indices(z["trees"], rank, world)
        counts, rs = bootstrap_counts([states[i] for i in mine], z["n"], bootstrap=True,
                                      n_threads=max(1, min(64, (os.cpu_count() or 8) // world)))
        n_units = z["trees"]
        res_box = {}
        mf = max(1, int(np.sqrt(z["d"])))

        def step():
            res_box["r"] = eng.forest_fit(counts, rs, 2, mf, np.iinfo(np.int32).max, 2, 1, 0.0, 0.0)
    else:
        from scipy.stats import loguniform
        from sklearn.model_selection import ParameterSampler
        cands = list(ParameterSampler({"alpha": loguniform(1e-3, 1e3)}, n_iter=z["n_iter"], random_state=0))
        fold = np.repeat(np.arange(z["folds"], dtype=np.int8),
                         np.full(z["folds"], z["n"] // z["folds"]) + (np.arange(z["folds"]) < z["n"] % z["folds"]))
        eng.stage_x(X)
        eng.stage_targets(y)
        eng.stage_folds(fold, z["folds"])
        n_units = z["n_iter"] * z["folds"]
        cols = parallel.shard_indices(n_units, rank, world)
        alpha = np.array([cands[c // z["folds"]]["alpha"] for c in cols])
        f_cols = (cols % z["folds"]).astype(np.int32)
        res_box = {}

        def step():
            r = eng.ridge_fit_batch(alpha, f_cols)
            res_box["r"] = r
            res_box["score"] = eng.linear_r2_batch(r["coef"], f_cols)

    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    for _ in range(a.warmup):
        step()
    barrier()
    sampler.begin()
    c0 = eng.counters()
    eng.timer_start()
    for _ in range(a.steps):
        step()
    dev_s = eng.timer_stop()
    barrier()
    sampler.end()
    c1 = eng.counters()
    clocks = sampler.stop() if rank == 0 else None
    if a.dump_outputs and rank == 0:
        dump_outputs(a.dump_outputs, res_box)
    tt = torch.tensor([dev_s], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    t_steps = float(tt.item())
    value = n_units * a.steps / t_steps

    # ---- end-to-end arm: the public estimator on host arrays
    e2e_times, h2d, d2h, est = [], 0, 0, None
    reps = 1 if a.config == 4 else 2
    for i in range(1 + reps):
        barrier()
        cc0 = eng.counters()
        t0 = time.perf_counter()
        if a.config == 3:
            from sklearn.linear_model import SGDClassifier
            from skdist.distribute.multiclass import DistOneVsRestClassifier
            est = DistOneVsRestClassifier(SGDClassifier(random_state=0), None).fit(X, y)
        elif a.config == 4:
            from skdist.distribute.ensemble import DistRandomForestClassifier
            est = None          # a fitted config-4 forest is 38 GB of node records: release it before the next fit
            est = DistRandomForestClassifier(n_estimators=z["trees"], random_state=0).fit(X, y)
        else:
            from scipy.stats import loguniform
            from sklearn.linear_model import Ridge
            from skdist.distribute.search import DistRandomizedSearchCV
            est = DistRandomizedSearchCV(Ridge(), {"alpha": loguniform(1e-3, 1e3)}, None, n_iter=z["n_iter"],
                                         cv=z["folds"], random_state=0, refit=False).fit(X, y)
        barrier()
        e2e_times.append(time.perf_counter() - t0)
        cc1 = eng.counters()
        h2d, d2h = cc1["h2d_bytes"] - cc0["h2d_bytes"], cc1["d2h_bytes"] - cc0["d2h_bytes"]
    te = torch.tensor(e2e_times[1:], dtype=torch.float64, device="cuda")
    if world > 1:
        dist.all_reduce(te, op=dist.ReduceOp.MAX)
    e2e_all = sorted(float(v) for v in te.tolist())
    e2e_s = e2e_all[len(e2e_all) // 2]

    if a.config == 5 and rank == 0 and world == 1:     # batched inference tail of config 5 (ref predict.py:74-179)
        from skdist.distribute.predict import batch_predict
        from sklearn.linear_model import Ridge
        from skdist_b200 import datasets
        m = Ridge(alpha=1.0)
        r = res_box["r"]
        m.coef_ = r["coef"][0, :z["d"]].astype(np.float32)
        m.intercept_ = np.float32(r["coef"][0, z["d"]])
        m.n_features_in_ = z["d"]
        rows = 0
        chunk = 1_000_000
        Xn, _ = datasets.make_g1_regression(chunk, z["d"], seed=1)
        batch_predict(m, Xn[:1000])
        t0 = time.perf_counter()
        for _ in range(z["predict_rows"] // chunk):
            batch_predict(m, Xn)
            rows += chunk
        dtp = time.perf_counter() - t0
        extra["predict"] = {"rows": rows, "rows_per_s_from_host_arrays": rows / dtp,
                            "algorithmic_GBps": rows * (4.0 * z["d"] + 4.0) / dtp / 1e9,
                            "note": "skdist.predict batch path on host rows (1M-row chunks of the seed-1 generator, reused), H2D inside"}

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    pk = peaks()
    # ---- roofline: SURVEY.md section 8(d) algorithmic work of the whole call / its device time
    if a.config == 3:
        r = res_box["r"]
        epochs = float(np.sum(r["n_iter"])) * (z["k"] / max(1, len(mine)))     # this rank's columns scaled to the job
        flops = 4.0 * z["n"] * z["d"] * epochs
        achieved = flops * a.steps / t_steps / 1e12
        roof = {"bound": "tensor", "achieved": achieved, "peak": pk["bf16_sustained"], "unit": "TFLOP/s",
                "frac": achieved / pk["bf16_sustained"], "traffic": None,
                "algorithmic_flops": "4 * n * d per label column per epoch x the epochs every column ran",
                "kernel": "whole sgd_fit_batch call (screening products on the tensor cores + ordered scan)"}
        extra["epochs_min_mean_max"] = [int(np.min(r["n_iter"])), float(np.mean(r["n_iter"])), int(np.max(r["n_iter"]))]
    elif a.config == 4:
        trees = res_box["r"]
        internal = sum(float(t["n_node_samples"][t["left"] != -1].sum()) for t in trees) * (z["trees"] / max(1, len(trees)))
        mf = max(1, int(np.sqrt(z["d"])))
        nbytes = 8.0 * (mf + 1) * internal
        achieved = nbytes * a.steps / t_steps / 1e9
        roof = {"bound": "hbm", "achieved": achieved, "peak": pk["hbm"], "unit": "GB/s", "frac": achieved / pk["hbm"],
                "traffic": None,
                "algorithmic_bytes": "8 * (max_features + 1) * sum over internal nodes of n_node_samples (SURVEY 8d)",
                "kernel": "whole forest_fit call (builder kernel + copies of bootstrap counts in, node arrays out)"}
        extra["nodes_mean"] = float(np.mean([len(t["left"]) for t in trees]))
    else:
        nbytes = 4.0 * z["n"] * z["d"]
        achieved = nbytes * a.steps / t_steps / 1e9
        roof = {"bound": "hbm", "achieved": achieved, "peak": pk["hbm"], "unit": "GB/s", "frac": achieved / pk["hbm"],
                "traffic": None, "algorithmic_bytes": "4 * n * d (one read of X; the Gram flops 2 n d^2 are second order)",
                "kernel": "whole ridge_fit_batch + linear_r2_batch call"}
    line = {"metric": metric, "value": value, "unit": unit, "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
            "ms_per_step": 1e3 * t_steps / a.steps, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": {3: "f32", 4: "u8", 5: "f32"}[a.config], "data": "synthetic",
            "config": dict({"workload": workload_name(a, z), "inputs": "exceed L2 (X is %.2f GB)" % (X.nbytes / 1e9),
                            "parallelism": "units dealt round-robin over %d rank(s), X replicated" % world}, **extra),
            "e2e": {"value": n_units / e2e_s, "unit": unit, "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
                    "seconds": e2e_s, "seconds_all": e2e_all},
            "gpu_launches": int(c1["launches"] - c0["launches"]), "clocks": clocks, "roofline": roof}
    if world == 1 and a.cpu_sample > 0:
        cores = os.cpu_count() or 1
        v, dt, desc, used, out = cpu_leg(a, z, X, y, max(a.cpu_sample if a.cpu_sample != 40 else 0, min(64, cores)))
        line["cpu_baseline"] = {"value": v, "unit": unit, "cores": used, "host_cores": cores, "kind": "port",
                                "sample": "%s in %.1f s" % (desc, dt)}
        # parity of the sampled units against the device results of the same units
        if a.config == 3:
            same = all(np.array_equal(c, est.estimators_[k].coef_[0]) and b == float(est.estimators_[k].intercept_[0])
                       and it == int(est.estimators_[k].n_iter_) for k, (c, b, it) in enumerate(out))
            line["parity"] = {"n_compared": len(out), "bit_identical_coef_intercept_n_iter": bool(same),
                              "checker": "sklearn SGDClassifier.fit on label column k (ref multiclass.py:109-152)"}
        elif a.config == 4:
            same = all(np.array_equal(r.tree_.threshold, o.tree_.threshold) and np.array_equal(r.tree_.children_left, o.tree_.children_left)
                       and np.array_equal(r.tree_.value, o.tree_.value) for r, o in zip(out, est.estimators_))
            line["parity"] = {"n_compared": len(out), "bit_identical_trees": bool(same),
                              "checker": "sklearn RandomForestClassifier(random_state=0) trees (ref ensemble.py:68-109)"}
        else:
            tasks, sc = out
            dev = np.array([est.cv_results_["split%d_test_score" % f][ci] for ci, f in tasks])
            line["parity"] = {"n_compared": len(tasks), "max_rel_dscore_split": float(np.max(np.abs(dev - np.array(sc)) / np.abs(sc))),
                              "checker": "sklearn Ridge fit + r2 on the same (alpha, fold) (ref search.py:180-288)"}
    print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()
