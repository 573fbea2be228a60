"""(candidate x fold) columns of dense Ridge regression on the device.

Replaces, for `DistGridSearchCV/DistRandomizedSearchCV(Ridge(), ...)`, the per-task
`Ridge.fit` + r2 scoring that the reference fans out (ref search.py:180-288): one pass over X
gives every fold's Gram block; each (alpha, fold) is then a 256x256 Cholesky solve
(csrc/ridge.cu) and one r2 epilogue pass scores all columns (csrc/logreg_tc.cu TC_R2)."""
import numpy as np

from .. import parallel
from .base import _merged_params
from .family import _Family, _resolve

# each column's packed Cholesky factor lives in one CTA's shared memory (csrc/ridge.cu RIDGE_MAX_D)
_RIDGE_MAX_FEATURES = 338


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


class _RidgeFamily(_Family):
    name = "ridge"
    searchable = frozenset({"alpha", "fit_intercept"})

    def __init__(self, estimator, candidate_params, X, y, scorers):
        self.estimator = estimator
        self._check_searchable(candidate_params)
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
        if self.fold is not fold:
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

    @staticmethod
    def _launch_key(p):
        return bool(p["fit_intercept"])

    def _launch(self, eng, cands, folds):
        alpha = np.array([p["alpha"] for p in cands], dtype=np.float64)
        res = eng.ridge_fit_batch(alpha, folds, fit_intercept=self._launch_key(cands[0]))
        return res["coef"], 0, res["status"], res["status"] != 1, np.zeros(len(cands), dtype=bool)

    def score_columns(self, eng, coef, codes):
        """({scorer name: per-column value}, rows per column) on the rows the scoring codes select; r2 takes the
        total sum of squares of those rows."""
        sse, count = eng.linear_r2_batch(coef, codes)
        sst = np.where(codes >= 0, self.sst_test[np.maximum(codes, 0)], self.sst_train[np.maximum(-3 - codes, 0)])
        return {name: self._metric(kind, sse, count, sst) for name, kind in self.metrics.items()}, count

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
