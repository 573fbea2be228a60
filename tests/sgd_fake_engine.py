"""FakeEngine plus the order-group SGD call -- TEST DOUBLE, CPU only.

`sgd_fit_groups` fits every column with scikit-learn's own exact-order SGD loop (`_plain_sgd32`, the
Cython routine SGDClassifier.fit runs) on X[rows of its group], in the group's row order, with the column's
alpha and the group's seed -- what one (candidate, fold, class) fit of scikit-learn's search computes.
Every call is recorded in `calls` as ("sgd_fit_groups", B, G)."""
import re

import numpy as np

from tests.fake_engine import FakeEngine


def plain_sgd(X, y_pos, params, alpha, seed):
    """(coef float32 [d], intercept, n_iter, t_, status) of one binary fit of scikit-learn's _plain_sgd32 on
    the rows of X in the given order; status 5 where scikit-learn raises its overflow error (n_iter = that
    epoch), 3 when all max_iter epochs ran, else 1."""
    from sklearn.linear_model import SGDClassifier
    from sklearn.linear_model._base import make_dataset
    from sklearn.linear_model._sgd_fast import _plain_sgd32
    est = SGDClassifier(**{k: v for k, v in params.items() if k != "alpha"}, alpha=alpha)
    loss_fn = est._get_loss_function(est.loss)
    X = np.ascontiguousarray(X, dtype=np.float32)
    y = np.where(y_pos, 1.0, 0.0 if est.loss == "log_loss" else -1.0).astype(np.float32)
    dataset, decay = make_dataset(X, y, np.ones(len(y), np.float32), random_state=np.random.RandomState(0))
    tol = -np.inf if est.tol is None else float(est.tol)
    try:
        coef, b, _, _, n_iter = _plain_sgd32(
            np.zeros(X.shape[1], np.float32), 0.0, None, 0.0, loss_fn, est._get_penalty_type("l2"), float(alpha),
            0.0, dataset, np.zeros(len(y), np.uint8), False, None, int(est.n_iter_no_change), int(est.max_iter),
            tol, int(est.fit_intercept), 0, int(est.shuffle), int(seed), 1.0, 1.0,
            est._get_learning_rate_type(est.learning_rate), float(est.eta0), float(est.power_t), 0, 1.0, decay, 0)
    except ValueError as e:
        m = re.search(r"epoch #(\d+)", str(e))
        return np.full(X.shape[1], np.nan, np.float32), np.nan, int(m.group(1)), np.nan, 5
    status = 3 if n_iter == est.max_iter else 1
    return coef, float(b), int(n_iter), 1.0 + n_iter * len(y), status


class SGDFakeEngine(FakeEngine):
    def sgd_fit_groups(self, params, col_pos, col_group, col_alpha, group_rows, group_seeds):
        B = len(col_pos)
        self.calls.append(("sgd_fit_groups", B, len(group_rows)))
        for a in col_alpha:
            assert a > 0
        out = {"coef32": np.zeros((B, self.d), np.float32), "intercept": np.zeros(B), "n_iter": np.zeros(B, np.int32),
               "t": np.zeros(B), "status": np.zeros(B, np.int32)}
        for j in range(B):
            rows = np.asarray(group_rows[col_group[j]])
            w, b, it, t, st = plain_sgd(self.X[rows], self.y[rows] == col_pos[j], params, float(col_alpha[j]),
                                        int(group_seeds[col_group[j]]))
            out["coef32"][j], out["intercept"][j], out["n_iter"][j], out["t"][j], out["status"][j] = w, b, it, t, st
        out["coef"] = np.concatenate([out["coef32"].astype(np.float64), out["intercept"][:, None]], axis=1)
        out["gpu_seconds"] = 0.0
        return out
