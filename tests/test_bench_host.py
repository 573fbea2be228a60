"""bench.py's checker pieces on the CPU: the task sample of the CPU leg and the `parity` block that compares its
scores with cv_results_ at the same (candidate, fold) -- on an engine double whose fits are scikit-learn's, so the
block must report no difference."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def test_cpu_tasks_are_whole_candidates_spread_over_the_grid():
    import bench
    tasks = bench.cpu_tasks(512, 5, 40)
    assert len(tasks) == 40
    cands = sorted({c for c, _ in tasks})
    assert cands[0] == 0 and cands[-1] == 511 and len(cands) == 8
    assert all(sorted(f for c, f in tasks if c == ci) == list(range(5)) for ci in cands)
    assert len(bench.cpu_tasks(512, 5, 3)) == 3


def test_parity_block_against_the_cpu_leg(fake_engine):
    import bench
    from sklearn.linear_model import LogisticRegression
    from skdist.distribute.search import DistGridSearchCV
    from skdist_b200.datasets import make_g1_classification
    X, y = make_g1_classification(3000, 12, seed=2)
    Cs = np.logspace(-3, 2, 6)
    fold = bench.fold_ids(y, 3)
    gs = DistGridSearchCV(LogisticRegression(), {"C": list(Cs)}, None, cv=3).fit(X, y)
    tasks = bench.cpu_tasks(len(Cs), 3, 9)
    fps, dt, scores, n_jobs, inner = bench.cpu_fits_per_sec(X, y, fold, Cs, tasks, n_jobs=1)
    assert fps > 0 and len(scores) == len(tasks) == 9
    blk = bench.parity_block(gs.cv_results_, tasks, scores, fold, Cs, 3)
    assert blk["n_compared"] == 9 and blk["max_flips_per_fold"] == 0 and blk["max_abs_dscore"] < 1e-12
    assert blk["best_C_equal_on_subgrid"] and blk["best_C_tied"]
    assert blk["test_rows_per_fold"] == 1000
    # a device result that differs by 3 test rows in one fold is reported as such
    bad = {k: np.array(v, dtype=float).copy() if k.startswith(("split", "mean_test")) else v for k, v in gs.cv_results_.items()}
    ci, f = tasks[4]
    bad["split%d_test_score" % f][ci] -= 3 / 1000
    assert bench.parity_block(bad, tasks, scores, fold, Cs, 3)["max_flips_per_fold"] == 3


def test_dump_outputs_writes_float_arrays_within_the_limit(tmp_path, monkeypatch):
    import bench
    res = {"fit": {"coef": np.arange(12, dtype=np.float32).reshape(4, 3), "n_iter": np.array([3, 4, 5, 6], np.int32)},
           "correct": np.array([1, 2, 3, 4], np.int64)}
    bench.dump_outputs(str(tmp_path / "a"), res)
    coef = np.load(tmp_path / "a" / "fit_coef.npy")
    assert coef.dtype == np.float32 and np.array_equal(coef, res["fit"]["coef"])
    assert np.load(tmp_path / "a" / "fit_n_iter.npy").dtype == np.float64
    assert np.array_equal(np.load(tmp_path / "a" / "correct.npy"), [1, 2, 3, 4])
    # over the limit: every file counted; arrays of the same length share one seeded row sample
    monkeypatch.setattr(bench, "DUMP_LIMIT", 8192)
    big = {"x": np.arange(4000, dtype=np.float64).reshape(1000, 4), "y": np.arange(1000, dtype=np.float32),
           "z": np.arange(300, dtype=np.int32), "s": 3.5}
    for d in ("b", "c"):
        bench.dump_outputs(str(tmp_path / d), big)
        assert sum(f.stat().st_size for f in (tmp_path / d).iterdir()) <= 8192
    rows = np.load(tmp_path / "b" / "sample_rows_1000.npy").astype(int)
    assert 0 < len(rows) < 1000 and not (tmp_path / "b" / "x_rows.npy").exists()
    np.testing.assert_array_equal(np.load(tmp_path / "b" / "x.npy"), big["x"][rows])
    np.testing.assert_array_equal(np.load(tmp_path / "b" / "y.npy"), big["y"][rows])
    zrows = np.load(tmp_path / "b" / "sample_rows_300.npy").astype(int)
    np.testing.assert_array_equal(np.load(tmp_path / "b" / "z.npy"), big["z"][zrows])
    assert float(np.load(tmp_path / "b" / "s.npy")) == 3.5
    for f in (tmp_path / "b").iterdir():
        np.testing.assert_array_equal(np.load(f), np.load(tmp_path / "c" / f.name))
