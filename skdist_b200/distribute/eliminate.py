"""Distributed feature elimination on H100 GPUs.

Counterpart of /root/reference/skdist/distribute/eliminate.py (`DistFeatureEliminator`, :47-284).
The reference ranks the features by the squared coefficients of one fit on all features, builds
nested sets of features to remove (`step` at a time) and fans one task per (feature set, fold)
out over Spark; every task copies X without the removed columns (`_drop_col`, :22-26) and fits
(`_fit_and_score_one`, :29-38).

Here a (feature set, fold) pair is one column of the batched logistic solve with a per-column
FEATURE MASK next to the per-row fold mask: a masked feature's gradient entry is forced to zero,
so its weight stays exactly 0 and the L-BFGS iterates are those of the fit on the remaining
columns (csrc/lbfgs_dev.cu gather_fg).  No column-dropped copies of X are made; scoring uses the
zero-padded coefficient rows on the full X.

Base estimator with a device path: ``LogisticRegression(solver="lbfgs")`` (binary or multiclass target) with
scoring=None / "accuracy" / "roc_auc".  Anything else raises NotImplementedError (no CPU fallback).
"""
import numpy as np
from sklearn.utils.metaestimators import available_if
from sklearn.base import BaseEstimator, ClassifierMixin, is_classifier
from sklearn.linear_model import LogisticRegression
from sklearn.model_selection import check_cv
from sklearn.utils import check_X_y
from sklearn.utils.validation import check_is_fitted

from .. import parallel
from ..engine import get_engine
from .base import _clone, _parse_partitions, _ScParamMixin
from .folds import _fold_ids
from .logreg_family import _check_logreg, _ClassWeights, _count_metric
from .utils import _check_multimetric_scoring

__all__ = ["DistFeatureEliminator"]


class DistFeatureEliminator(_ScParamMixin, ClassifierMixin, BaseEstimator):
    """Cross-validated backward feature elimination with all (feature set, fold) fits batched
    on the device.  Constructor mirrors ref eliminate.py:77-100 (``sc`` 2nd positional)."""

    def __init__(self, estimator, sc=None, partitions="auto", min_features_to_select=None, step=1, cv=5,
                 scoring=None, verbose=False, n_jobs=None, pre_dispatch=None, mask=True):
        self.estimator = estimator
        self.sc = sc
        self.partitions = partitions
        self.min_features_to_select = min_features_to_select
        self.step = step
        self.cv = cv
        self.scoring = scoring
        self.verbose = verbose
        self.n_jobs = n_jobs
        self.pre_dispatch = pre_dispatch
        self.mask = mask

    def fit(self, X, y=None, groups=None, **fit_params):
        """ref eliminate.py:102-237"""
        if fit_params:
            raise NotImplementedError("fit_params are not supported on the device path")
        X, y = check_X_y(X, y, "csr", ensure_min_features=2)
        if hasattr(X, "tocsr"):
            raise NotImplementedError("sparse X has no device path")
        if type(self.estimator) is not LogisticRegression:
            raise NotImplementedError(
                "%s has no device path in DistFeatureEliminator; supported: LogisticRegression(solver='lbfgs')."
                "  (No CPU fallback by design.)" % type(self.estimator).__name__)
        p = _check_logreg(_clone(self.estimator), class_weight=True)
        scorers, _ = _check_multimetric_scoring(self.estimator, scoring=self.scoring)
        metric = _count_metric(scorers["score"])
        if metric is None or metric[0] not in ("accuracy", "roc_auc"):
            raise NotImplementedError("scoring=None / 'accuracy' / 'roc_auc' are scored on the device")
        classes = np.unique(y)
        n_classes = len(classes)
        if n_classes < 2:
            raise ValueError("the target has a single class")
        multi = n_classes > 2          # LogisticRegression(lbfgs) is multinomial there (SK/linear_model/_logistic.py:523-547)
        if multi and metric[0] == "roc_auc":
            raise NotImplementedError("roc_auc on a multiclass target has no device path")
        cv = check_cv(self.cv, y, classifier=is_classifier(self.estimator))
        n_samples, n_features = X.shape
        min_features_to_select = n_features // 2 if self.min_features_to_select is None \
            else self.min_features_to_select                               # ref :120-123
        step = int(max(1, self.step * n_features)) if 0.0 < self.step < 1.0 else int(self.step)   # ref :124-127
        if step <= 0:
            raise ValueError("Step must be >0")

        rank, world, _ = parallel.dist_info()
        eng = get_engine()
        ycls = np.searchsorted(classes, y).astype(np.int32)
        cv_splits = list(cv.split(X, y, groups))
        n_splits = len(cv_splits)
        fold = _fold_ids(cv_splits, n_samples)
        parallel.stage_x_replicated(eng, X)
        eng.stage_labels(ycls)
        eng.stage_folds(fold, n_splits)
        kw = dict(fit_intercept=p["fit_intercept"], tol=p["tol"], max_iter=p["max_iter"])
        one = np.ones(1, np.int32)
        weights = _ClassWeights(classes, ycls)
        weights.set_folds(fold, [np.asarray(train) for train, _ in cv_splits])

        def fit(C, folds):
            weights.stage(eng, [p["class_weight"]] * len(C), folds)
            if multi:
                return eng.logreg_multinomial_fit_batch(C, folds, n_classes, **kw)
            return eng.logreg_fit_batch(C, folds, np.ones(len(C), np.int32), **kw)

        # initial fit on every feature -> ranking by squared coefficient, summed over the class rows of a
        # multiclass model (ref :141-156)
        res0 = fit(np.array([p["C"]]), np.array([-1], np.int32))
        coefs = res0["coef"][0][..., :n_features].astype(np.float64)
        ranks = np.argsort((coefs ** 2).sum(axis=0) if multi else coefs ** 2)
        ranks = np.ravel(ranks)[: (n_features - min_features_to_select)]
        this_step = 0
        features_to_remove = [np.array([], dtype=np.int64)]
        while this_step < (n_features - min_features_to_select):               # ref :150-154
            this_step += step
            features_to_remove.append(ranks[:this_step])

        # (feature set, fold) columns, set-major like product(features_to_remove, cv_splits) (ref :156)
        n_sets = len(features_to_remove)
        n_cols = n_sets * n_splits
        _parse_partitions(self.partitions, n_cols)
        mine = parallel.shard_indices(n_cols, rank, world)
        masks = np.ones((len(mine), n_features), dtype=np.uint8)
        for i, col in enumerate(mine):
            masks[i, features_to_remove[col // n_splits]] = 0
        f_cols = (np.asarray(mine) % n_splits).astype(np.int32)
        pos = np.ones(len(mine), np.int32)
        if len(mine):
            eng.stage_column_masks(masks)
            res = fit(np.full(len(mine), p["C"]), f_cols)
            if multi:
                correct, count = eng.multinomial_score_batch(res["coef"], f_cols)
                loc = correct / np.maximum(count, 1)
            elif metric[0] == "roc_auc":       # the reference's examples/eliminate/basic_usage.py scorer
                loc, _ = eng.linear_auc_batch(res["coef"], f_cols, pos)
            else:
                correct, count = eng.linear_score_batch(res["coef"], f_cols, pos)
                loc = correct / np.maximum(count, 1)
        else:
            loc = np.zeros(0)
        scores = np.asarray(parallel.all_gather_columns(loc, n_cols, rank, world), dtype=np.float64)
        self.scores_ = [float(np.mean(s)) for s in scores.reshape(n_sets, n_splits)]   # ref :214-217
        best_set_ = int(np.argmax(self.scores_))
        self.best_score_ = self.scores_[best_set_]
        if len(features_to_remove[best_set_]) > 0:                                      # ref :220-225
            self.best_features_ = np.delete(range(n_features), features_to_remove[best_set_])
        else:
            self.best_features_ = range(n_features)

        # final fit on the best feature set (ref :226-227): the full-data column with that mask
        m = np.zeros((1, n_features), np.uint8)
        m[0, np.asarray(self.best_features_, dtype=np.int64)] = 1
        eng.stage_column_masks(m)
        resb = fit(np.array([p["C"]]), np.array([-1], np.int32))
        keep = np.asarray(self.best_features_, dtype=np.int64)
        est = _clone(self.estimator)
        dt = np.float64 if X.dtype == np.float64 else np.float32
        rows = np.atleast_2d(resb["coef"][0])                 # (1, d+1) binary, (K, d+1) multiclass
        est.coef_ = rows[:, :n_features][:, keep].astype(dt)
        est.intercept_ = (rows[:, n_features].astype(dt) if est.fit_intercept
                          else np.zeros(rows.shape[0], dtype=dt))
        est.classes_ = classes
        est.n_iter_ = np.array([int(resb["n_iter"][0])], dtype=np.int32)
        est.n_features_in_ = len(keep)
        self.best_estimator_ = est
        self.n_features_ = len(self.best_features_)
        self.__dict__.pop("sc", None)
        return self

    # ---- prediction surface (ref eliminate.py:239-284) --------------------------------------
    def _apply_mask(self, X):
        self._check_is_fitted()
        return np.asarray(X)[:, self.best_features_] if self.mask else X

    def _check_is_fitted(self):
        check_is_fitted(self, "best_estimator_")

    def predict(self, X):
        return self.best_estimator_.predict(self._apply_mask(X))

    def predict_proba(self, X):
        return self.best_estimator_.predict_proba(self._apply_mask(X))

    def predict_log_proba(self, X):
        return self.best_estimator_.predict_log_proba(self._apply_mask(X))

    def decision_function(self, X):
        return self.best_estimator_.decision_function(self._apply_mask(X))

    # ref eliminate.py:271-275: present only when the estimator has it (if_delegate_has_method)
    @available_if(lambda self: hasattr(getattr(self, "best_estimator_", None), "transform"))
    def transform(self, X):
        return self.best_estimator_.transform(self._apply_mask(X))

    def score(self, X, y):
        return self.best_estimator_.score(self._apply_mask(X), y)

    @property
    def classes_(self):
        self._check_is_fitted()
        return self.best_estimator_.classes_
