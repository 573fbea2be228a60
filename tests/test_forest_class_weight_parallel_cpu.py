"""Forest classifiers with class_weight over two gloo ranks (CPU, engine double): every rank stages the same
dict / "balanced" weights, "balanced_subsample" is formed per tree from the tree's own bootstrap, and the
trees of the other rank arrive through the all-gather -- so both ranks end with the single-process forest."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [{0: 2.0, 1: 0.0, 2: 0.7}, "balanced", "balanced_subsample"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _data():
    rng = np.random.default_rng(12)
    X = rng.integers(0, 10, size=(500, 6)).astype(np.float32)
    s = X[:, 0] + 0.5 * X[:, 1] + rng.standard_normal(500) * 2
    y = np.digitize(s, np.quantile(s, [0.2, 0.6]))
    return X, y


def _forests():
    """{case: per-tree arrays} of DistRandomForestClassifier(n_estimators=7) fits on the engine double."""
    from sklearn.utils import check_random_state
    from skdist.distribute.ensemble import DistRandomForestClassifier
    from skdist_b200 import engine
    from skdist_b200.distribute.ensemble import MAX_RAND_SEED, _tree_inputs
    from tests.forest_class_weight_restate import WeightedForestEngine
    engine.set_engine_factory(WeightedForestEngine)
    try:
        X, y = _data()
        seeds = check_random_state(4).randint(MAX_RAND_SEED, size=7)
        engine.get_engine().seed_of_rand_r = {int(_tree_inputs(s, len(y), False)[1]): int(s) for s in seeds}
        out = {}
        for i, cw in enumerate(CASES):
            rf = DistRandomForestClassifier(n_estimators=7, random_state=4, class_weight=cw).fit(X, y)
            assert len(rf.estimators_) == 7
            for t, e in enumerate(rf.estimators_):
                for f in ("threshold", "children_right", "weighted_n_node_samples", "impurity"):
                    out["%d_%d_%s" % (i, t, f)] = getattr(e.tree_, f)
                out["%d_%d_value" % (i, t)] = e.tree_.value
            out["%d_proba" % i] = rf.predict_proba(X)
        return out
    finally:
        engine.set_engine_factory(None)


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank), SKDIST_B200_FOREST_GATHER="all")
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    np.savez(os.path.join(out_dir, "cw%d.npz" % rank), **_forests())
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_weighted_forests_equal_one_rank(tmp_path):
    import torch.multiprocessing as mp
    port = _free_port()
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(tmp_path / "cw0.npz"), np.load(tmp_path / "cw1.npz")
    single = _forests()
    assert set(r0.files) == set(single) == set(r1.files)
    for k in single:
        np.testing.assert_array_equal(r0[k], single[k], err_msg=k)
        np.testing.assert_array_equal(r1[k], single[k], err_msg=k)
