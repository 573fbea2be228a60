"""(candidate x fold) columns of dense Ridge regression on the device.

Replaces, for `DistGridSearchCV/DistRandomizedSearchCV(Ridge(), ...)`, the per-task
`Ridge.fit` + r2 scoring that the reference fans out (ref search.py:180-288): one pass over X
gives every fold's Gram block; each (alpha, fold) is then a 256x256 Cholesky solve
(csrc/ridge.cu) and one r2 epilogue pass scores all columns (csrc/logreg_tc.cu TC_R2)."""
import time
from collections import defaultdict

import numpy as np

from .. import parallel
from .base import _clone, _merged_params
from .folds import _train_codes

_RIDGE_SEARCHABLE = {"alpha", "fit_intercept"}
# each column's packed Cholesky factor lives in one CTA's shared memory (csrc/ridge.cu RIDGE_MAX_D)
_RIDGE_MAX_FEATURES = 338


def _resolve(estimator, params):
    est = _clone(estimator)
    if params:
        est.set_params(**params)
    return est


def _check_ridge(est):
    p = est if isinstance(est, dict) else est.get_params(deep=False)
    bad = []
    if p.get("solver", "auto") not in ("auto", "cholesky"):
        bad.append("solver=%r (only 'auto'/'cholesky')" % p["solver"])
    if p.get("positive", False):
        bad.append("positive=True")
    if np.ndim(p.get("alpha", 1.0)) != 0:
        bad.append("per-target alpha")
    if bad:
        raise NotImplementedError("Ridge configuration without a device path: " + ", ".join(bad))
    return p


class _RidgeFamily:
    name = "ridge"

    def __init__(self, estimator, candidate_params, X, y, scorers):
        self.estimator = estimator
        for p in candidate_params:
            extra = set(p) - _RIDGE_SEARCHABLE
            if extra:
                raise NotImplementedError(
                    "searching Ridge over %s has no device path (searchable: %s)"
                    % (sorted(extra), sorted(_RIDGE_SEARCHABLE)))
        self.cands = [_check_ridge(q) for q in _merged_params(estimator, candidate_params)]
        if np.ndim(y) != 1:
            raise NotImplementedError("multi-target Ridge has no device path")
        if X.shape[1] > _RIDGE_MAX_FEATURES:
            raise NotImplementedError("Ridge with %d features has no device path (supported: n_features <= %d)"
                                      % (X.shape[1], _RIDGE_MAX_FEATURES))
        self.y = np.asarray(y, dtype=np.float32)
        # scorers that are functions of the per-column (sum of squared residuals, row count):
        # r2 (also estimator.score), neg_mean_squared_error, neg_root_mean_squared_error
        self.metrics = {}
        for name, scorer in scorers.items():
            kind = None
            if type(scorer).__name__ == "_PassthroughScorer":
                kind = "r2"
            else:
                f = getattr(getattr(scorer, "_score_func", None), "__name__", "")
                sign, kw = getattr(scorer, "_sign", 1), dict(getattr(scorer, "_kwargs", {}) or {})
                if f == "r2_score" and sign == 1 and not kw:
                    kind = "r2"
                elif f == "mean_squared_error" and sign == -1 and not kw:
                    kind = "neg_mse"
                elif f == "root_mean_squared_error" and sign == -1 and not kw:
                    kind = "neg_rmse"
            if kind is None:
                raise NotImplementedError(
                    "scorer %r has no device path for regressors (supported: r2, neg_mean_squared_error, "
                    "neg_root_mean_squared_error)" % (scorer,))
            self.metrics[name] = kind

    @staticmethod
    def _metric(kind, sse, count, sst):
        if kind == "r2":
            return 1.0 - sse / sst
        mse = sse / np.maximum(count, 1)
        return -mse if kind == "neg_mse" else -np.sqrt(mse)

    def stage(self, eng, X, fold, n_splits, x_staged=False):
        if not x_staged:
            parallel.stage_x_replicated(eng, X)
        eng.stage_targets(self.y)
        eng.stage_folds(fold, n_splits)
        if getattr(self, "fold", None) is not fold:
            self.prepare(fold, n_splits)

    def prepare(self, fold, n_splits):
        """Total sums of squares of the test / train part of every fold (denominators of r2); host-only,
        so the search runs it while X is still on its way to the device."""
        self.fold = fold
        y64 = self.y.astype(np.float64)
        self.sst_test = np.zeros(n_splits)
        self.sst_train = np.zeros(n_splits)
        for k in range(n_splits):
            t = y64[fold == k]
            self.sst_test[k] = np.sum((t - t.mean()) ** 2)
            t = y64[fold != k]
            self.sst_train[k] = np.sum((t - t.mean()) ** 2)

    def run_columns(self, eng, cols, n_splits, return_train_score):
        cols = np.asarray(cols, dtype=np.int64)
        out = {
            "n_test": np.zeros(len(cols), dtype=np.int64),
            "fit_time": np.zeros(len(cols)), "score_time": np.zeros(len(cols)),
            "n_iter": np.zeros(len(cols), dtype=np.int32), "status": np.zeros(len(cols), dtype=np.int32),
        }
        for name in self.metrics:
            out["test_%s" % name] = np.zeros(len(cols))
            if return_train_score:
                out["train_%s" % name] = np.zeros(len(cols))
        cand = cols // n_splits
        fold = (cols % n_splits).astype(np.int32)
        groups = defaultdict(list)
        for i, c in enumerate(cand):
            groups[bool(self.cands[c]["fit_intercept"])].append(i)
        for fi, idx in groups.items():
            idx = np.asarray(idx)
            alpha = np.array([self.cands[c]["alpha"] for c in cand[idx]], dtype=np.float64)
            t0 = time.time()
            res = eng.ridge_fit_batch(alpha, fold[idx], fit_intercept=fi)
            t1 = time.time()
            sse, count = eng.linear_r2_batch(res["coef"], fold[idx])
            t2 = time.time()
            for name, kind in self.metrics.items():
                score = self._metric(kind, sse, count, self.sst_test[fold[idx]])
                score[res["status"] != 1] = np.nan
                out["test_%s" % name][idx] = score
            out["n_test"][idx] = count
            out["fit_time"][idx] = (t1 - t0) / len(idx)
            out["score_time"][idx] = (t2 - t1) / len(idx)
            out["status"][idx] = res["status"]
            if return_train_score:
                sse2, n2 = eng.linear_r2_batch(res["coef"], _train_codes(fold[idx]))
                for name, kind in self.metrics.items():
                    out["train_%s" % name][idx] = self._metric(kind, sse2, n2, self.sst_train[fold[idx]])
        return out

    def refit(self, eng, params, X_dtype, n_features):
        p = _check_ridge(_resolve(self.estimator, params))
        res = eng.ridge_fit_batch(np.array([p["alpha"]]), np.array([-1], dtype=np.int32),
                                  fit_intercept=p["fit_intercept"])
        return self.make_estimator(params, res["coef"][0], X_dtype, n_features)

    def make_estimator(self, params, coef_row, X_dtype, n_features):
        """A genuine fitted sklearn Ridge (attributes as SK/linear_model/_ridge.py:1016-1020 leaves
        them) so inherited predict/score work."""
        est = _resolve(self.estimator, params)
        dt = np.float64 if X_dtype == np.float64 else np.float32
        est.coef_ = coef_row[:n_features].astype(dt)
        est.intercept_ = dt(coef_row[n_features]) if est.fit_intercept else 0.0
        est.n_iter_ = None
        est.solver_ = "cholesky"
        est.n_features_in_ = n_features
        return est

    def fold_proba(self, eng, params, fold, n_splits):
        """preds_ (ref search.py:551-560): regressors have no predict_proba -> predict."""
        p = _check_ridge(_resolve(self.estimator, params))
        f = np.arange(n_splits, dtype=np.int32)
        res = eng.ridge_fit_batch(np.full(n_splits, p["alpha"]), f, fit_intercept=p["fit_intercept"])
        dec = eng.linear_decision(res["coef"])
        return np.vstack([dec[fold == k, k][:, None] for k in range(n_splits)])
