"""SGDClassifier search over two gloo ranks on the CPU engine double: each rank forms order groups from the
(candidate, fold) columns it is dealt, and every rank ends with the single-process cv_results_."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRID = {"alpha": [1e-5, 1e-4, 1e-3, 1e-2, 1e-1]}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _search(X, y, Xm, ym):
    from sklearn.linear_model import SGDClassifier
    from skdist.distribute.search import DistGridSearchCV
    gs = DistGridSearchCV(SGDClassifier(random_state=0), GRID, cv=3, return_train_score=True).fit(X, y)
    gm = DistGridSearchCV(SGDClassifier(random_state=1, max_iter=20, tol=None), GRID, cv=3,
                          scoring="f1_macro").fit(Xm, ym)
    return gs, gm


def _data():
    from skdist_b200.datasets import make_g1_classification, make_multiclass
    X, y = make_g1_classification(900, 8, seed=9)
    Xm, ym = make_multiclass(600, 6, 4, seed=5)
    return X, y, Xm, ym


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import warnings
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from skdist_b200 import engine
    from tests.sgd_fake_engine import SGDFakeEngine
    engine.set_engine_factory(SGDFakeEngine)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gs, gm = _search(*_data())
    cols = sum(c[1] for c in engine.get_engine().calls if c[0] == "sgd_fit_groups")
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **{k: np.asarray(v) for k, v in gs.cv_results_.items()
                                                             if k.startswith(("split", "mean_test", "rank"))},
             multi=gm.cv_results_["mean_test_score"], coef=gs.best_estimator_.coef_, mcoef=gm.best_estimator_.coef_,
             cols=cols)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_two_rank_sgd_search_matches_single_process(tmp_path):
    import warnings
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1 = np.load(tmp_path / "rank0.npz"), np.load(tmp_path / "rank1.npz")
    from skdist_b200 import engine
    from tests.sgd_fake_engine import SGDFakeEngine
    engine.set_engine_factory(SGDFakeEngine)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            gs, gm = _search(*_data())
    finally:
        engine.set_engine_factory(None)
    for k in r0.files:
        if k in gs.cv_results_:
            np.testing.assert_array_equal(r0[k], r1[k], err_msg=k)
            np.testing.assert_array_equal(r0[k], gs.cv_results_[k], err_msg=k)
    np.testing.assert_array_equal(r0["multi"], gm.cv_results_["mean_test_score"])
    np.testing.assert_array_equal(r1["multi"], gm.cv_results_["mean_test_score"])
    np.testing.assert_array_equal(r0["coef"], gs.best_estimator_.coef_)
    np.testing.assert_array_equal(r1["mcoef"], gm.best_estimator_.coef_)
    # the 15 binary and 15 x 4 multiclass columns were split between the ranks (plus one refit each)
    assert int(r0["cols"]) + int(r1["cols"]) == 15 + 15 * 4 + 2 * (1 + 4)
    assert int(r0["cols"]) < 15 + 15 * 4 + 5
