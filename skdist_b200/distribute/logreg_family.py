"""LogisticRegression families of the search (family.py): what one (candidate, fold) task of the reference
(`_fit_and_score`, ref search.py:180-288) computes, for all tasks of a search at once.

  _LogRegFamily        binary target: columns of the batched lbfgs solve (csrc/logreg_tc.cu,
                       logreg_simt.cu, lbfgs_dev.cu)
  _MultinomialFamily   more than two classes: multinomial problems (csrc/logreg_multi.cu)"""
import warnings

import numpy as np

from .base import _merged_params
from .family import _count_metric, _Family, _resolve, SUPPORTED_CLASSIFIER_SCORERS
# the scoring helpers these families were written with, importable from here as before
from .family import _metric_from_confusion, _RANK_SCORE, _rank_average  # noqa: F401
from .folds import _classes_and_ids, _train_rows


def _check_logreg(est, class_weight=False):
    """Raise unless `est` is a configuration the batched lbfgs kernel path reproduces
    (SK/linear_model/_logistic.py:1355-1593).  class_weight=True: the caller passes the class weights
    to the engine."""
    p = est if isinstance(est, dict) else est.get_params(deep=False)
    bad = []
    if p.get("solver", "lbfgs") != "lbfgs":
        bad.append("solver=%r (only 'lbfgs')" % p["solver"])
    pen = p.get("penalty", "deprecated")
    if pen not in ("l2", "deprecated"):
        bad.append("penalty=%r (only 'l2')" % (pen,))
    if p.get("l1_ratio", 0.0) not in (None, 0, 0.0):
        bad.append("l1_ratio=%r" % (p["l1_ratio"],))
    if not class_weight and p.get("class_weight", None) is not None:
        bad.append("class_weight")
    if p.get("dual", False):
        bad.append("dual=True")
    if p.get("warm_start", False):
        bad.append("warm_start=True")
    if bad:
        raise NotImplementedError(
            "LogisticRegression configuration without a device path: " + ", ".join(bad))
    return p


def _fit_sample_weight(estimator, fit_params, n_samples):
    """The float32 `sample_weight` a fit of `estimator` takes from `fit_params`, checked as LogisticRegression.fit
    checks it (SK/utils/validation.py _check_sample_weight: length, finite values), or None.  Every other
    key raises the TypeError that LogisticRegression.fit raises for it.  The device restriction: weights
    must be >= 0 (ValueError).  Only LogisticRegression has a weighted device path: fit_params for any other
    estimator raise NotImplementedError."""
    if not fit_params:
        return None
    from sklearn.linear_model import LogisticRegression
    if type(estimator) is not LogisticRegression:
        raise NotImplementedError("fit_params %s of %s are not supported on the device path (sample_weight: "
                                  "LogisticRegression only)" % (sorted(fit_params), type(estimator).__name__))
    for key in fit_params:
        if key != "sample_weight":
            raise TypeError("LogisticRegression.fit() got an unexpected keyword argument %r" % key)
    sw = fit_params["sample_weight"]
    if sw is None:
        return None
    from sklearn.utils.validation import _check_sample_weight
    sw = _check_sample_weight(sw, np.empty((n_samples, 0), dtype=np.float32), dtype=np.float32, copy=True)
    if np.any(sw < 0):
        raise ValueError("sample_weight must be >= 0 on the device path (negative weights make the logistic "
                         "objective non-convex)")
    return sw


class _ClassWeights:
    """Per-column class weights of LogisticRegression(class_weight=...) fits, as
    SK/linear_model/_logistic.py:409-474 forms them: compute_class_weight on the labels of the fit's own
    training rows (classes = the labels present there; with sample weights, "balanced" counts them), cast to
    float32, and sw_sum = the float32 sum of the per-row weights (sample weight times class weight, a float32
    product) in the order of those rows.  Weights depend on (class_weight, held-out fold) only."""

    def __init__(self, classes, y_class):
        self.classes, self.y_class = classes, y_class
        self.fold, self.train_rows, self.cache = None, None, {}
        self.sample_weight = None

    def set_sample_weight(self, sample_weight):
        """float32 sample weight of every row (None: none); each fit takes those of its training rows."""
        self.sample_weight, self.cache = sample_weight, {}

    def set_folds(self, fold, train_rows=None):
        """fold ids of the staged layout; train_rows[f] = training rows of local fold f in the splitter's
        order (None: the rows outside fold f in ascending order, as every partition splitter gives them)."""
        self.fold, self.train_rows, self.cache = np.asarray(fold), train_rows, {}

    def column(self, class_weight, f):
        """(float32 weight of every class id, sw_sum) of a fit on the training rows of fold f (-1: all rows)."""
        key = (repr(class_weight), int(f))
        if key not in self.cache:
            rows = _train_rows(self.fold, self.train_rows, f)
            sw = None if self.sample_weight is None else self.sample_weight[rows]
            self.cache[key] = _fit_class_weights(class_weight, self.y_class[rows], self.classes, sw)
        return self.cache[key]

    def stage(self, eng, class_weights, folds):
        """Stage the weights of columns (class_weight, held-out fold) for the next fit, and the sample weights
        when there are any; nothing when no column is weighted (the unweighted kernels then run)."""
        if self.sample_weight is None and all(cw is None for cw in class_weights):
            return
        _stage_columns(eng, [self.column(cw, f) for cw, f in zip(class_weights, folds)], self.sample_weight)


def _fit_class_weights(class_weight, ids, classes, sw=None):
    """(float32 weight of every class id, sw_sum) of ONE fit whose training rows, in the fit's order, carry
    the class ids `ids` (labels classes[ids]) and the float32 sample weights `sw` (None: none): what
    SK/linear_model/_logistic.py:409-474 forms from class_weight and sample_weight (classes = the labels
    present in the fit, compute_class_weight with the fit's sample weights, weights cast to float32, sw_sum =
    the float32 sum of the per-row weights sw * class_weight_[y]).  Errors of compute_class_weight propagate;
    sample weights that sum to 0 over the fit's rows raise ValueError."""
    from sklearn.utils.class_weight import compute_class_weight
    w = np.ones(len(classes), dtype=np.float32)
    if class_weight is None:
        if sw is None:
            return w, float(len(ids))
        rw = sw
    else:
        present = np.unique(ids)
        w[:] = 0.0      # a class without training rows carries no weight
        w[present] = compute_class_weight(class_weight, classes=classes[present], y=classes[ids],
                                          sample_weight=sw).astype(np.float32)
        rw = w[ids] if sw is None else sw * w[ids]
    sw_sum = float(np.sum(rw))
    if sw is not None and not sw_sum > 0:
        raise ValueError("the sample weights of a fit's training rows sum to %r: a fit needs a positive sum" % sw_sum)
    return w, sw_sum


def _stage_columns(eng, cols, sample_weight=None):
    """Stage [(weights, sw_sum)] of the columns of the next fit, and the float32 sample weights of every staged
    row when not None.  If a staging call fails, both are cleared: staged inputs are one-shot, and class weights
    without the sample weights they were summed over must not reach a later fit."""
    try:
        eng.stage_class_weights(np.stack([c[0] for c in cols]), np.array([c[1] for c in cols]))
        if sample_weight is not None:
            eng.stage_sample_weights(sample_weight)
    except Exception:
        eng.stage_class_weights(None, None)
        if sample_weight is not None:
            eng.stage_sample_weights(None)
        raise




class _LogRegFamily(_Family):
    """(candidate x fold) columns of binary L2 logistic regression."""

    name = "logreg"
    searchable = frozenset({"C", "tol", "max_iter", "fit_intercept", "class_weight"})

    def __init__(self, estimator, candidate_params, X, y, scorers, enc=None):
        self.estimator = estimator
        self.cands = [_check_logreg(q, class_weight=True) for q in _merged_params(estimator, candidate_params)]
        self._check_searchable(candidate_params)
        self.classes_, self.y_class = _classes_and_ids(y, enc)
        self.n_classes = len(self.classes_)
        self._set_metrics(scorers)
        self.weights = _ClassWeights(self.classes_, self.y_class)

    def _set_metrics(self, scorers):
        if self.n_classes != 2:
            raise NotImplementedError(
                "this family is binary (got %d classes)" % self.n_classes)
        metrics = {}
        for name, scorer in scorers.items():
            metrics[name] = _count_metric(scorer)
            if metrics[name] is None:
                raise NotImplementedError(
                    "scorer %r has no device path for classifiers (supported: %s)"
                    % (scorer, SUPPORTED_CLASSIFIER_SCORERS))
        self._set_binary_metrics(metrics)

    def stage(self, eng, X, fold, n_splits, x_staged=False):
        super().stage(eng, X, fold, n_splits, x_staged)
        self.weights.set_folds(self.fold)

    def set_sample_weight(self, sample_weight):
        """float32 sample weight of every row (None: none), indexed by each fit's training rows as the
        reference indexes fit_params (ref search.py:208-211); the refit takes all of them."""
        self.weights.set_sample_weight(sample_weight)

    def set_train_rows(self, train_rows):
        """Training rows of every fold of the staged layout in the splitter's order (None entries: the
        rows outside the fold, ascending): the order sw_sum of a weighted column is summed in."""
        super().set_train_rows(train_rows)
        self.weights.set_folds(self.fold, train_rows)

    def column_cost(self, n_splits):
        """Expected relative duration of every (candidate, fold) column, for the multi-GPU block deal."""
        from ..parallel import logreg_column_cost
        return np.repeat(logreg_column_cost([p["C"] for p in self.cands]), n_splits)

    @staticmethod
    def _launch_key(p):
        return bool(p["fit_intercept"]), float(p["tol"]), int(p["max_iter"])

    def fit_columns(self, eng, cands, folds):
        """The engine result of one batched fit: column i fits candidate cands[i] (parameter dict; all share
        the launch key) on the training rows of fold folds[i] (-1: all rows), with its class and sample
        weights staged first."""
        self.weights.stage(eng, [p["class_weight"] for p in cands], folds)
        C = np.array([p["C"] for p in cands], dtype=np.float64)
        fi, tol, mi = self._launch_key(cands[0])
        if self.n_classes > 2:
            return eng.logreg_multinomial_fit_batch(C, folds, self.n_classes, fit_intercept=fi, tol=tol,
                                                    max_iter=mi)
        return eng.logreg_fit_batch(C, folds, np.ones(len(C), dtype=np.int32), fit_intercept=fi, tol=tol,
                                    max_iter=mi)

    def _launch(self, eng, cands, folds):
        # a column whose objective went non-finite (status 5) has no usable coefficients; max_iter /
        # line-search stops only warn, as scikit-learn does (SK/linear_model/_logistic.py:599)
        res = self.fit_columns(eng, cands, folds)
        status = res["status"]
        n_slow = int(np.sum((status == 3) | (status == 4)))
        if n_slow:
            from sklearn.exceptions import ConvergenceWarning
            warnings.warn("lbfgs failed to converge within max_iter=%d for %d of %d (candidate, fold) fits"
                          % (self._launch_key(cands[0])[2], n_slow, len(cands)), ConvergenceWarning)
        return res["coef"], res["n_iter"], status, status == 5, status == 5

    def score_columns(self, eng, coef, codes):
        """({scorer name: per-column value}, rows per column) of fitted coefficients on the rows the scoring
        codes select."""
        return self._binary_scores(eng, coef, codes)

    def refit(self, eng, params, X_dtype, n_features):
        p = _check_logreg(_resolve(self.estimator, params), class_weight=True)
        res = self.fit_columns(eng, [p], np.array([-1], dtype=np.int32))
        return self.make_estimator(params, res["coef"][0], res["n_iter"][0], X_dtype, n_features)

    def make_estimator(self, params, coef_rows, n_iter, X_dtype, n_features):
        """A genuine fitted sklearn LogisticRegression (attributes as set by
        SK/linear_model/_logistic.py:1561-1593) so inherited predict* work: coef_ (1 or K, d), intercept_
        (1 or K,), n_iter_ (1,).  coef_rows: [d + 1] (binary) or [K, d + 1], intercept last."""
        est = _resolve(self.estimator, params)
        dt = np.float64 if X_dtype == np.float64 else np.float32
        rows = np.atleast_2d(coef_rows)
        est.coef_ = rows[:, :n_features].astype(dt)
        if est.fit_intercept:
            est.intercept_ = rows[:, n_features].astype(dt)
        else:
            est.intercept_ = np.zeros(len(rows), dtype=dt)
        est.classes_ = self.classes_
        est.n_iter_ = np.array([n_iter], dtype=np.int32)
        est.n_features_in_ = n_features
        return est

    def _fold_fits(self, eng, params, n_splits):
        """Coefficients of the best params refitted on the training rows of every fold (preds_ support, ref
        search.py:551-560)."""
        p = _check_logreg(_resolve(self.estimator, params), class_weight=True)
        return self.fit_columns(eng, [p] * n_splits, np.arange(n_splits, dtype=np.int32))["coef"]

    def fold_proba(self, eng, params, fold, n_splits):
        """preds_: predict_proba of every held-out row under its fold's refit, stacked in fold order."""
        dec = eng.linear_decision(self._fold_fits(eng, params, n_splits))
        preds = []
        for k in range(n_splits):
            z = dec[fold == k, k].astype(np.float64)
            p1 = 1.0 / (1.0 + np.exp(-z))
            preds.append(np.column_stack([1.0 - p1, p1]))
        return np.vstack(preds)


class _MultinomialFamily(_LogRegFamily):
    """(candidate x fold) problems of multinomial L2 logistic regression: what LogisticRegression(lbfgs)
    fits when the target has more than two classes (SK/linear_model/_logistic.py:523-547).  One
    device optimiser problem per (candidate, fold) with n_classes x (d + 1) variables."""

    name = "logreg_multinomial"

    def _set_metrics(self, scorers):
        self.metrics = {}
        for name, scorer in scorers.items():
            m = _count_metric(scorer)
            if m is None or m[1] == "binary" or m[0] == "roc_auc":    # scikit-learn itself rejects these on a multiclass target
                raise NotImplementedError(
                    "scorer %r has no device path for a multiclass target (supported: accuracy, "
                    "balanced_accuracy, precision / recall / f1 with average micro, macro or weighted, "
                    "roc_auc_ovr, roc_auc_ovr_weighted, roc_auc_ovo, roc_auc_ovo_weighted, average_precision, "
                    "neg_log_loss)" % (scorer,))
            self.metrics[name] = m

    def _launch(self, eng, cands, folds):
        res = self.fit_columns(eng, cands, folds)
        keep = np.zeros(len(cands), dtype=bool)
        return res["coef"], res["n_iter"], res["status"], keep, keep

    def score_columns(self, eng, coef, codes):
        return self._multiclass_scores(eng, coef, codes)

    def fold_proba(self, eng, params, fold, n_splits):
        from sklearn.utils.extmath import softmax
        coef = self._fold_fits(eng, params, n_splits)
        K = self.n_classes
        dec = eng.linear_decision(coef.reshape(n_splits * K, -1))
        return np.vstack([softmax(dec[fold == k, k * K:(k + 1) * K].astype(np.float64)) for k in range(n_splits)])
