"""Distributed hyper-parameter search meta-estimators on H100 GPUs.

Drop-in for /root/reference/skdist/distribute/search.py (class names, constructor
signatures incl. positional order, fitted attributes).  The reference fans
``_fit_and_score`` (search.py:180-288) out over Spark executors, one task per
(candidate, fold) (search.py:378-437); here every (candidate, fold) pair is one *column*
of a batched solve on the GPU(s):

  reference                                    this module
  ---------                                    -----------
  cv.split -> (train_idx, test_idx) per task   one int8 fold id per row      (_fold_ids)
  _safe_split copies X[train], X[test]         none: rows are masked by fold id in-kernel
  estimator.fit per task                       Engine.logreg_fit_batch / ridge_cv (all columns)
  scorer(estimator, X_test, y_test)            Engine.linear_score_batch (accuracy counts) / r2
  sc.parallelize(...).map(...).collect()       round-robin column shards over ranks + all_gather
  cv_results_ assembly, best_*, refit          same arithmetic as search.py:461-550 (host)

Base estimators with a device path: ``LogisticRegression`` (binary y, penalty l2, solver
lbfgs), ``Ridge`` (dense, single target) and ``SGDClassifier`` (hinge / log_loss, penalty l2,
searched over alpha; sgd_family.py).  Anything else raises NotImplementedError: by
design there is no CPU fallback (the reference's joblib branch, search.py:388-409, is what
the CPU baseline in bench.py times).
"""
import numbers
import time
from collections import defaultdict
from functools import partial

import numpy as np
from sklearn.utils.metaestimators import available_if
from numpy.ma import MaskedArray
from scipy.stats import rankdata
from sklearn.base import BaseEstimator, is_classifier
from sklearn.linear_model import LogisticRegression, Ridge, SGDClassifier
from sklearn.model_selection import (GridSearchCV, ParameterGrid, ParameterSampler,
                                     RandomizedSearchCV, check_cv)
from sklearn.utils.validation import indexable

from .. import parallel
from ..engine import get_engine
from .base import _parse_partitions, _ScParamMixin
from .utils import _check_multimetric_scoring
from .validation import _check_estimator, _check_n_iter, _validate_models

__all__ = ["DistGridSearchCV", "DistRandomizedSearchCV", "DistMultiModelSearch"]


from .folds import _cv_fold_groups, _cv_fold_ids, _encode_target
from .family import _check_engine_entries
from .logreg_family import _fit_sample_weight, _LogRegFamily, _MultinomialFamily


# ----------------------------------------------------------------------------------------
# estimator families with a device path (family.py; logreg_family.py, sgd_family.py, ridge_family.py)
# ----------------------------------------------------------------------------------------
def _pick_family(estimator, candidate_params, X, y, scorers, enc=None):
    if type(estimator) is LogisticRegression:
        n_classes = len(enc.classes) if enc is not None and enc.y is y else len(np.unique(y))
        if n_classes > 2:
            return _MultinomialFamily(estimator, candidate_params, X, y, scorers, enc)
        return _LogRegFamily(estimator, candidate_params, X, y, scorers, enc)
    if type(estimator) is Ridge:
        from .ridge_family import _RidgeFamily
        return _RidgeFamily(estimator, candidate_params, X, y, scorers)
    if type(estimator) is SGDClassifier:
        from .sgd_family import _SGDFamily
        return _SGDFamily(estimator, candidate_params, X, y, scorers, enc)
    raise NotImplementedError(
        "%s has no device path; supported base estimators: LogisticRegression(solver='lbfgs'), "
        "Ridge, SGDClassifier.  (No CPU fallback by design.)" % type(estimator).__name__)


# ----------------------------------------------------------------------------------------
# the meta-estimators
# ----------------------------------------------------------------------------------------
class DistBaseSearchCV(_ScParamMixin):
    """Same role as the reference's DistBaseSearchCV (search.py:291-581)."""

    def fit(self, X, y=None, groups=None, **fit_params):
        """Run fit with all sets of parameters (ref search.py:315-571).

        fit_params: `sample_weight` of a LogisticRegression base (any other key raises the TypeError of
        LogisticRegression.fit; other bases raise NotImplementedError).  As in the reference, each
        (candidate, fold) fit takes the weights of its training rows (ref search.py:208-211) and the refit
        takes all of them (:548); the scores stay unweighted (:264)."""
        _check_estimator(self, verbose=self.verbose)
        estimator = self.estimator
        cv = check_cv(self.cv, y, classifier=is_classifier(estimator))
        scorers, self.multimetric_ = _check_multimetric_scoring(self.estimator, scoring=self.scoring)
        if self.multimetric_:                                   # ref search.py:340-358
            if self.refit is not False and (not isinstance(self.refit, str) or self.refit not in scorers):
                raise ValueError(
                    "For multi-metric scoring, the parameter refit must be set to a scorer key to refit an "
                    "estimator with the best parameter setting on the whole data and make the best_* "
                    "attributes available for that metric. If this is not needed, refit should be set to "
                    "False explicitly. %r was passed." % self.refit)
            refit_metric = self.refit
        else:
            refit_metric = "score"

        X, y, groups = indexable(X, y, groups)
        n_splits = cv.get_n_splits(X, y, groups)

        X_arr = np.asarray(X)
        if X_arr.ndim != 2:
            raise ValueError("X must be a 2-d array")
        y_arr = np.asarray(y)
        n_samples, n_features = X_arr.shape
        sample_weight = _fit_sample_weight(estimator, fit_params, n_samples)
        # the host-to-device copy of X (the C-ABI call releases the GIL) runs while the host draws the
        # candidates (ParameterSampler: one scipy rvs call per candidate), computes the cv splits and
        # validates the candidates
        eng = get_engine()
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=1) as pool:
            staged = pool.submit(parallel.stage_x_replicated, eng, X_arr)
            time.sleep(0)       # hand the GIL to the worker so that the copy starts before the host work below
            try:
                candidate_params = list(self._get_param_iterator())
                n_candidates = len(candidate_params)
                if self.verbose > 0:
                    print("Fitting {0} folds for each of {1} candidates, totalling {2} fits".format(
                        n_splits, n_candidates, n_candidates * n_splits))
                _parse_partitions(self.partitions, n_candidates * n_splits)
                enc = _encode_target(y_arr) if is_classifier(estimator) else None   # one hash pass over y for both
                train_orders = []       # train index arrays of the splits, when the splitter gave them
                layouts, n_splits = _cv_fold_groups(cv, X, y_arr, groups, n_samples, enc, train_orders)
                fold = layouts[0][0]
                family = _pick_family(estimator, candidate_params, X_arr, y_arr, scorers, enc)
                _check_engine_entries(family, eng)
                if sample_weight is not None:
                    family.set_sample_weight(sample_weight)
                if self.refit and self.preds and not hasattr(family, "fold_proba"):
                    raise NotImplementedError("preds=True has no device path for %s" % type(estimator).__name__)
                family.prepare(fold, layouts[0][1])     # host-only statistics of the folds (no engine calls)
            finally:
                staged.result()

        rank, world, _ = parallel.dist_info()
        metric_names = list(family.metrics)
        keys = ["n_test", "fit_time", "score_time"] + ["test_%s" % m for m in metric_names]
        if self.return_train_score:
            keys += ["train_%s" % m for m in metric_names]
        # task order: candidate-major, fold-minor (ref search.py:378-383), column = cand * n_splits + split.
        # A cross-validator whose test sets overlap (ShuffleSplit, RepeatedKFold ...) comes as several
        # fold-id layouts of disjoint test sets; the fold ids (n bytes) are re-staged per layout, X once.
        n_cols = n_candidates * n_splits
        full = np.zeros((n_cols, len(keys)))
        for li, (fold_l, nf_l, idx_l) in enumerate(layouts):
            if li > 0:
                family.prepare(fold_l, nf_l)
            family.stage(eng, X_arr, fold_l, nf_l, x_staged=True)
            # training rows of every local fold, in the splitter's order
            family.set_train_rows([train_orders[s] if train_orders else None for s in idx_l])
            k_l = len(idx_l)
            # local columns cand * nf_l + f, f < k_l (the extra fold id of a layout is never held out).
            # Ranks are dealt blocks of 128 consecutive candidates of ONE fold (fold-major order).
            cols_l = (np.arange(n_candidates)[None, :] * nf_l + np.arange(k_l)[:, None]).ravel()
            col_cost = family.column_cost(nf_l)[cols_l] if world > 1 else None
            pick = parallel.shard_blocks(len(cols_l), rank, world, cost=col_cost)
            loc = family.run_columns(eng, cols_l[pick], nf_l, bool(self.return_train_score))
            # one collective per layout for all per-column results (counts are exact in float64)
            stacked = np.stack([np.asarray(loc[k], dtype=np.float64) for k in keys], axis=1)
            gathered = parallel.all_gather_blocks(stacked, len(cols_l), rank, world, cost=col_cost)
            cand_l, f_l = cols_l // nf_l, cols_l % nf_l
            full[cand_l * n_splits + np.asarray(idx_l)[f_l]] = gathered
        res = {k: full[:, i] for i, k in enumerate(keys)}
        res["n_test"] = np.rint(res["n_test"]).astype(np.int64)
        if len(layouts) > 1 and self.refit and self.preds:
            raise NotImplementedError("preds=True needs a cross-validator whose test sets partition the rows")

        error_score = self.error_score
        for m in metric_names:
            bad = ~np.isfinite(res["test_%s" % m])
            if np.any(bad):
                # ref search.py:226-259 semantics for a failed fit
                if isinstance(error_score, numbers.Number):
                    res["test_%s" % m][bad] = error_score
                else:
                    raise ValueError("a fit produced a non-finite score and error_score=%r" % (error_score,))

        results = {}

        def _store(key_name, array, weights=None, splits=False, rank=False):
            """ref search.py:463-484"""
            array = np.array(array, dtype=np.float64).reshape(n_candidates, n_splits)
            if splits:
                for split_i in range(n_splits):
                    results["split%d_%s" % (split_i, key_name)] = array[:, split_i]
            array_means = np.average(array, axis=1, weights=weights)
            results["mean_%s" % key_name] = array_means
            array_stds = np.sqrt(np.average((array - array_means[:, np.newaxis]) ** 2, axis=1,
                                            weights=weights))
            results["std_%s" % key_name] = array_stds
            if rank:
                results["rank_%s" % key_name] = np.asarray(rankdata(-array_means, method="min"),
                                                           dtype=np.int32)

        _store("fit_time", res["fit_time"])
        _store("score_time", res["score_time"])
        param_results = defaultdict(partial(MaskedArray, np.empty(n_candidates,), mask=True, dtype=object))
        for cand_i, params in enumerate(candidate_params):
            for name, value in params.items():
                param_results["param_%s" % name][cand_i] = value
        results.update(param_results)
        results["params"] = candidate_params

        # ref search.py:510-519: weights = test-fold sizes when `iid` is truthy ("warn" default)
        test_sample_counts = np.array(res["n_test"][:n_splits], dtype=int)
        for m in metric_names:                                  # ref search.py:512-533
            _store("test_%s" % m, res["test_%s" % m], splits=True, rank=True,
                   weights=test_sample_counts if self.iid else None)
            if self.return_train_score:
                _store("train_%s" % m, res["train_%s" % m], splits=True)

        # ref search.py:535-541: best_* only when a refit metric is defined
        if self.refit or not self.multimetric_:
            self.best_index_ = results["rank_test_%s" % refit_metric].argmin()
            self.best_params_ = candidate_params[self.best_index_]
            self.best_score_ = results["mean_test_%s" % refit_metric][self.best_index_]

        if self.refit:
            # ref search.py:543-550 (one more full-data fit, here on the device)
            t0 = time.time()
            self.best_estimator_ = family.refit(eng, self.best_params_, X_arr.dtype, n_features)
            self.refit_time_ = time.time() - t0
            if self.preds:
                self.preds_ = family.fold_proba(eng, self.best_params_, fold, n_splits)

        self.scorer_ = scorers if self.multimetric_ else scorers["score"]   # ref search.py:563
        self.cv_results_ = results
        self.n_splits_ = n_splits

        # ref search.py:568-570
        self.__dict__.pop("sc", None)
        if hasattr(self.estimator, "sc"):
            del self.estimator.sc
        return self

    def get_preds(self):
        """Get CV predictions (ref search.py:573-576)."""
        if hasattr(self, "preds_"):
            return self.preds_

    def drop_preds(self):
        """Remove preds_ attribute (ref search.py:578-581)."""
        if hasattr(self, "preds_"):
            del self.preds_


class DistGridSearchCV(DistBaseSearchCV, GridSearchCV):
    """Same as sklearn `GridSearchCV` but with the fits batched on H100 GPUs.
    Constructor mirrors ref search.py:608-641 (``sc`` is the 3rd positional argument)."""

    def __init__(self, estimator, param_grid, sc=None, partitions="auto", preds=False,
                 scoring=None, n_jobs=None, iid="warn", refit=True, cv=5, verbose=0,
                 pre_dispatch="2*n_jobs", error_score="raise-deprecating",
                 return_train_score=False):
        self.estimator = estimator
        self.param_grid = param_grid
        self.sc = sc
        self.partitions = partitions
        self.preds = preds
        self.scoring = scoring
        self.n_jobs = n_jobs
        self.iid = iid
        self.refit = refit
        self.cv = cv
        self.verbose = verbose
        self.pre_dispatch = pre_dispatch
        self.error_score = error_score
        self.return_train_score = return_train_score

    def _get_param_iterator(self):
        """ref search.py:643-645"""
        return ParameterGrid(self.param_grid)


class DistRandomizedSearchCV(DistBaseSearchCV, RandomizedSearchCV):
    """Same as sklearn `RandomizedSearchCV` but with the fits batched on H100 GPUs.
    Constructor mirrors ref search.py:671-708."""

    def __init__(self, estimator, param_distributions, sc=None, partitions="auto", preds=False,
                 n_iter=10, scoring=None, n_jobs=None, iid="warn", refit=True, cv=5, verbose=0,
                 pre_dispatch="2*n_jobs", random_state=None, error_score="raise-deprecating",
                 return_train_score=False):
        self.estimator = estimator
        self.param_distributions = param_distributions
        self.sc = sc
        self.partitions = partitions
        self.preds = preds
        self.n_iter = n_iter
        self.scoring = scoring
        self.n_jobs = n_jobs
        self.iid = iid
        self.refit = refit
        self.cv = cv
        self.verbose = verbose
        self.pre_dispatch = pre_dispatch
        self.random_state = random_state
        self.error_score = error_score
        self.return_train_score = return_train_score

    def _get_param_iterator(self):
        """ref search.py:710-714"""
        return ParameterSampler(self.param_distributions, self.n_iter, random_state=self.random_state)


# ----------------------------------------------------------------------------------------
# multi-model randomized search (ref search.py:60-177, 717-908)
# ----------------------------------------------------------------------------------------
def _raw_sampler(models, n, random_state=None):
    """`n` sampled parameter sets per model, every model sampled with the same random_state
    (ref search.py:60-90)."""
    param_sets = []
    for index, (_, _, dist) in enumerate(models):
        sampler = list(ParameterSampler(dist, n_iter=_check_n_iter(n, dist), random_state=random_state))
        for sample_index, params in enumerate(sampler):
            param_sets.append({"model_index": index, "params_index": sample_index, "param_set": params})
    return param_sets


class DistMultiModelSearch(_ScParamMixin, BaseEstimator):
    """Randomized search over several (name, estimator, param_set) models at once; the
    (model, sampled params, fold) fits of every model run as columns of that model's batched
    device solve.  Constructor and fitted attributes mirror ref search.py:717-908."""

    def __init__(self, models, sc=None, partitions="auto", n=5, cv=5, scoring=None, random_state=None,
                 verbose=0, refit=True, n_jobs=None, pre_dispatch="2*n_jobs"):
        self.models = models
        self.sc = sc
        self.partitions = partitions
        self.n = n
        self.cv = cv
        self.scoring = scoring
        self.random_state = random_state
        self.verbose = verbose
        self.refit = refit
        self.n_jobs = n_jobs
        self.pre_dispatch = pre_dispatch

    def fit(self, X, y=None, groups=None, **fit_params):
        """ref search.py:800-866"""
        if fit_params:
            raise NotImplementedError("fit_params are not supported on the device path")
        _check_estimator(self, verbose=self.verbose)
        models = _validate_models(self.models, self)
        cv = check_cv(self.cv, y, classifier=is_classifier(models[0][1]))
        X, y, groups = indexable(X, y, groups)
        X_arr, y_arr = np.asarray(X), np.asarray(y)
        n_samples, n_features = X_arr.shape
        fold, n_splits = _cv_fold_ids(cv, X, y, groups, n_samples)
        param_sets = _raw_sampler(models, self.n, random_state=self.random_state)
        _parse_partitions(self.partitions, len(param_sets) * n_splits)

        rank, world, _ = parallel.dist_info()
        eng = get_engine()
        scores = np.zeros(len(param_sets))
        families = {}
        for index, (_, estimator, _) in enumerate(models):
            rows = [i for i, ps in enumerate(param_sets) if ps["model_index"] == index]
            cands = [param_sets[i]["param_set"] for i in rows]
            scorers, _ = _check_multimetric_scoring(estimator, scoring=self.scoring)
            family = _pick_family(estimator, cands, X_arr, y_arr, scorers)
            _check_engine_entries(family, eng)
            families[index] = family
            family.stage(eng, X_arr, fold, n_splits)
            n_cols = len(cands) * n_splits
            deal_order = (np.arange(len(cands))[None, :] * n_splits + np.arange(n_splits)[:, None]).ravel()
            my_cols = parallel.shard_blocks(n_cols, rank, world, deal_order)
            loc = family.run_columns(eng, my_cols, n_splits, False)
            test = parallel.all_gather_blocks(loc["test_score"], n_cols, rank, world, deal_order)
            # plain mean over folds (ref search.py:166-176: groupby(...).agg({"score": "mean"}))
            scores[rows] = np.asarray(test, dtype=np.float64).reshape(len(cands), n_splits).mean(axis=1)
        if self.verbose:
            for index, (name, _, _) in enumerate(models):
                best = max(scores[i] for i, ps in enumerate(param_sets) if ps["model_index"] == index)
                print("model %d (%s): best score %.6f" % (index, name, best))

        best_index = int(np.argmax(scores))                              # ref :838
        self.best_model_index_ = param_sets[best_index]["model_index"]
        self.best_model_name_ = models[self.best_model_index_][0]
        self.best_params_ = param_sets[best_index]["param_set"]
        self.best_score_ = scores[best_index]
        self.worst_score_ = scores[best_index]                           # sic (ref :843)
        self.cv_results_ = {                                             # ref :844-859
            "model_index": [ps["model_index"] for ps in param_sets],
            "model_name": [models[ps["model_index"]][0] for ps in param_sets],
            "params": [ps["param_set"] for ps in param_sets],
            "rank_test_score": list(np.asarray(rankdata(-scores), dtype=np.int32)),
            "mean_test_score": list(scores),
        }
        if self.refit:                                                   # ref :861-864
            family = families[self.best_model_index_]
            family.stage(eng, X_arr, fold, n_splits)
            self.best_estimator_ = family.refit(eng, self.best_params_, X_arr.dtype, n_features)
        self.__dict__.pop("sc", None)
        return self

    def _check_is_fitted(self):
        """ref search.py:868-880"""
        from sklearn.exceptions import NotFittedError
        if not self.refit:
            raise NotFittedError(
                "This %s instance was initialized with refit=False. The method is available only after "
                "refitting on the best parameters. You can refit an estimator manually using the "
                "``best_params_`` attribute" % (type(self).__name__))
        from sklearn.utils.validation import check_is_fitted
        check_is_fitted(self, "best_estimator_")

    def _delegate(self, name, X):
        self._check_is_fitted()
        if not hasattr(self.best_estimator_, name):
            raise AttributeError("%s has no %s" % (type(self.best_estimator_).__name__, name))
        return getattr(self.best_estimator_, name)(X)

    def predict(self, X):
        return self._delegate("predict", X)

    def predict_proba(self, X):
        return self._delegate("predict_proba", X)

    def predict_log_proba(self, X):
        return self._delegate("predict_log_proba", X)

    def decision_function(self, X):
        return self._delegate("decision_function", X)

    # ref search.py:895-903: present only when the (best) estimator has them (if_delegate_has_method)
    @available_if(lambda self: hasattr(getattr(self, "best_estimator_", None), "transform"))
    def transform(self, X):
        return self._delegate("transform", X)

    @available_if(lambda self: hasattr(getattr(self, "best_estimator_", None), "inverse_transform"))
    def inverse_transform(self, Xt):
        return self._delegate("inverse_transform", Xt)

    @property
    def classes_(self):
        self._check_is_fitted()
        return self.best_estimator_.classes_
