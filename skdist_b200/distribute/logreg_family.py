"""LogisticRegression families of the search: what one (candidate, fold) task of the reference
(`_fit_and_score`, ref search.py:180-288) computes, for all tasks of a search at once.

  _LogRegFamily        binary target: columns of the batched lbfgs solve (csrc/logreg_tc.cu,
                       logreg_simt.cu, lbfgs_dev.cu)
  _MultinomialFamily   more than two classes: multinomial problems (csrc/logreg_multi.cu)

Scorers are functions of device-side counts / sums: confusion counts (accuracy, balanced accuracy,
precision / recall / f1 with any averaging), ranked counts per segment (csrc/auc.cu: roc_auc on the decision
values, roc_auc_ovr / roc_auc_ovo [_weighted] on float32 predict_proba, average_precision on the decision
values) and a sum of -log p (neg_log_loss)."""
import time
from collections import defaultdict

import numpy as np

from .. import parallel
from .base import _clone, _merged_params
from .folds import _classes_and_ids, _train_codes

_LOGREG_SEARCHABLE = {"C", "tol", "max_iter", "fit_intercept", "class_weight"}


def _resolve(estimator, params):
    est = _clone(estimator)
    if params:
        est.set_params(**params)
    return est


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


_COUNT_METRICS = {"accuracy_score": "accuracy", "f1_score": "f1", "precision_score": "precision",
                  "recall_score": "recall", "balanced_accuracy_score": "balanced_accuracy"}


def _count_metric(scorer):
    """(kind, average) of the count-based metric a scikit-learn scorer computes on predict(), or None.
    average is None for accuracy / balanced accuracy, else "binary" / "micro" / "macro" / "weighted".
    All of them are functions of the confusion counts the scoring kernels deliver."""
    if type(scorer).__name__ == "_PassthroughScorer":       # estimator.score == accuracy (ref utils.py:75-143)
        return "accuracy", None
    f = getattr(scorer, "_score_func", None)
    kind = _COUNT_METRICS.get(getattr(f, "__name__", ""))
    kwargs = dict(getattr(scorer, "_kwargs", {}) or {})
    if getattr(f, "__name__", "") == "log_loss" and not kwargs and getattr(scorer, "_sign", 1) == -1:
        # scoring="neg_log_loss": -log_loss(y, predict_proba(X)) -- summed on the device (csrc/logreg_multi.cu)
        return "neg_log_loss", None
    if getattr(f, "__name__", "") == "roc_auc_score" and not kwargs and getattr(scorer, "_sign", 1) == 1:
        # scoring="roc_auc": roc_auc_score(y, decision_function(X)) -- exact pair counts on the device (csrc/auc.cu)
        return "roc_auc", None
    rank = _ranking_metric(getattr(f, "__name__", ""), dict(kwargs), getattr(scorer, "_response_method", None),
                           getattr(scorer, "_sign", 1))
    if rank is not None:
        return rank
    if kind is None or getattr(scorer, "_sign", 1) != 1:
        return None
    if kind in ("accuracy", "balanced_accuracy"):
        return None if kwargs else (kind, None)
    average = kwargs.pop("average", "binary")
    pos_label = kwargs.pop("pos_label", 1)      # the named averaged scorers ("f1_weighted", ...) carry pos_label=None
    if kwargs or average not in ("binary", "micro", "macro", "weighted"):
        return None
    if pos_label != 1 and not (average != "binary" and pos_label is None):
        return None
    return kind, average


# ranking scorers -> the score the device ranks: "proba" = float32 predict_proba, "decision" = decision_function
_RANK_SCORE = {"roc_auc_ovr": "proba", "roc_auc_ovo": "proba", "average_precision": "decision"}
SUPPORTED_CLASSIFIER_SCORERS = (
    "accuracy, balanced_accuracy, precision / recall / f1 with average binary (binary target), micro, macro or "
    "weighted, roc_auc (binary target), roc_auc_ovr, roc_auc_ovr_weighted, roc_auc_ovo, roc_auc_ovo_weighted, "
    "average_precision, neg_log_loss")


def _ranking_metric(func_name, kwargs, response_method, sign):
    """(kind, average) of a ranking scorer the rank kernel serves, or None:
      roc_auc_score(multi_class="ovr" | "ovo", average="macro" | "weighted") on predict_proba
          -> ("roc_auc_ovr" | "roc_auc_ovo", average)
      average_precision_score() on decision_function first -> ("average_precision", None)"""
    if sign != 1:
        return None
    rm = tuple(response_method) if isinstance(response_method, (list, tuple)) else (response_method,)
    if func_name == "roc_auc_score" and rm == ("predict_proba",):
        multi_class = kwargs.pop("multi_class", "raise")
        average = kwargs.pop("average", "macro")
        if kwargs or multi_class not in ("ovr", "ovo") or average not in ("macro", "weighted"):
            return None
        return "roc_auc_" + multi_class, average
    if func_name == "average_precision_score" and not kwargs and rm and rm[0] == "decision_function":
        return "average_precision", None
    return None


def _is_rank(metric):
    """True for the (kind, average) of a ranking scorer served by the rank kernel."""
    return isinstance(metric, tuple) and metric[0] in _RANK_SCORE


def _rank_entries(metrics):
    """Engine entries the scorers in `metrics` call beyond the fit and count kernels."""
    return ("linear_rank_batch",) if any(_is_rank(k) for k in metrics.values()) else ()


def _check_engine_entries(family, eng):
    """Raise NotImplementedError before any fit when the engine lacks an entry the family's scorers call: a
    scorer whose kernel the engine does not provide has no device path (and no CPU fallback)."""
    missing = [e for e in getattr(family, "engine_entries", ()) if not hasattr(eng, e)]
    if missing:
        raise NotImplementedError(
            "scorers %s need %s, which %s does not provide: no device path on this engine"
            % (sorted(family.metrics), ", ".join(missing), type(eng).__name__))


def _label_one(classes):
    """Class id of the label 1 (the pos_label of the average_precision scorer), or None when no class is 1."""
    hits = [i for i, c in enumerate(classes) if not isinstance(c, (str, bytes)) and c == 1]
    return hits[0] if hits else None


def _auc(r):
    """ROC-AUC per segment from {2U, n_pos, n_neg}: NaN where a class is missing."""
    den = 2.0 * r["n_pos"].astype(np.float64) * r["n_neg"].astype(np.float64)
    return np.divide(r["u2"].astype(np.float64), den, out=np.full(den.shape, np.nan), where=den > 0)


def _rank_average(kind, average, r, K):
    """Per-column score of a ranking scorer from the per-segment counts r ([B, S] arrays), averaged as
    SK/metrics/_ranking.py averages them.  K == 1: binary columns, one segment each.  K > 2: a column whose
    rows miss a class gets NaN (scikit-learn raises "Number of classes in y_true not equal to the number of
    columns in 'y_score'", and y_true / y_score shapes differ for average_precision)."""
    if K == 1:
        return r["ap"][:, 0] if kind == "average_precision" else _auc(r)[:, 0]
    if kind == "roc_auc_ovo":
        # segment a * (K - 1) + (b < a ? b : b - 1): positives y == a, negatives y == b
        n_cls = r["n_pos"][:, ::K - 1]                                   # rows of class a (segment (a, *))
        auc = _auc(r)
        a, b = np.triu_indices(K, 1)
        ab = a * (K - 1) + b - 1
        ba = b * (K - 1) + a
        pair = (auc[:, ab] + auc[:, ba]) / 2.0
        if average == "macro":
            val = pair.mean(axis=1)
        else:       # prevalence (n_a + n_b) / n of the pair
            prev = (n_cls[:, a] + n_cls[:, b]) / n_cls.sum(axis=1, keepdims=True).astype(np.float64)
            val = (pair * prev).sum(axis=1) / prev.sum(axis=1)
    else:
        n_cls = r["n_pos"]
        per = r["ap"] if kind == "average_precision" else _auc(r)
        if average == "weighted":
            w = n_cls.astype(np.float64)
            val = (per * w).sum(axis=1) / np.maximum(w.sum(axis=1), 1.0)
        else:
            val = per.mean(axis=1)
    return np.where(np.all(n_cls > 0, axis=1), val, np.nan)


class _RankScores:
    """Ranking scorers of one scoring call: one rank-kernel call per (score, pairs) the scorers need.
    binary_proba: the score that ranks as predict_proba[:, 1] does on binary columns."""

    def __init__(self, eng, coef, codes, label_one=1, binary_proba="proba"):
        self.eng, self.coef, self.codes, self.label_one = eng, coef, codes, label_one
        self.binary_proba = binary_proba
        self.cache = {}

    def value(self, kind, average):
        K = 1 if self.coef.ndim == 2 else self.coef.shape[1]
        score, pos = _RANK_SCORE[kind], None
        if K == 1:
            if score == "proba":
                score = self.binary_proba
            pos = 1
            if kind == "average_precision":     # pos_label=1: classes_[1] as usual, classes_[0] on -decision
                if self.label_one is None:      # scikit-learn: "pos_label=1 is not a valid label"
                    return np.full(len(self.codes), np.nan)
                pos = self.label_one
                score = "decision" if pos == 1 else "neg_decision"
        pairs = kind == "roc_auc_ovo" and K > 1
        key = (score, pairs, pos)
        if key not in self.cache:
            self.cache[key] = self.eng.linear_rank_batch(
                self.coef, self.codes, None if K > 1 else np.full(len(self.codes), pos, dtype=np.int32),
                score=score, pairs=pairs)
        return _rank_average(kind, average, self.cache[key], K)


def _metric_from_confusion(kind, average, conf):
    """scikit-learn's formulas on confusion matrices conf[..., true, predicted]
    (SK/metrics/_classification.py: accuracy_score, balanced_accuracy_score,
    precision_recall_fscore_support with zero_division -> 0.0; labels = classes present in y_true or
    y_pred, as unique_labels gives them)."""
    conf = np.asarray(conf, dtype=np.float64)
    tp = np.diagonal(conf, axis1=-2, axis2=-1)
    support = conf.sum(axis=-1)          # rows per true class
    pred = conf.sum(axis=-2)             # rows per predicted class
    total = support.sum(axis=-1)

    def div(a, b):
        return np.divide(a, b, out=np.zeros(np.broadcast(a, b).shape), where=b != 0)
    if kind == "accuracy" or average == "micro":
        return div(tp.sum(axis=-1), total)
    if kind == "balanced_accuracy":      # mean recall over the classes that occur in y_true
        has = support > 0
        return div((div(tp, support) * has).sum(axis=-1), has.sum(axis=-1).astype(np.float64))
    if kind == "precision":
        per_class = div(tp, pred)
    elif kind == "recall":
        per_class = div(tp, support)
    elif kind == "f1":
        per_class = div(2.0 * tp, support + pred)
    else:
        raise ValueError(kind)
    if average == "macro":
        present = (support + pred) > 0
        return div((per_class * present).sum(axis=-1), present.sum(axis=-1).astype(np.float64))
    if average == "weighted":
        return div((per_class * support).sum(axis=-1), total)
    raise ValueError(average)


def _metric_from_counts(kind, correct, count, pred_pos, actual_pos):
    """scikit-learn's formulas on confusion counts (SK/metrics/_classification.py: accuracy_score,
    precision_recall_fscore_support with zero_division -> 0.0, balanced_accuracy_score)."""
    correct = np.asarray(correct, dtype=np.float64)
    count = np.asarray(count, dtype=np.float64)
    if kind == "accuracy":
        return correct / np.maximum(count, 1)
    pred_pos = np.asarray(pred_pos, dtype=np.float64)
    actual_pos = np.asarray(actual_pos, dtype=np.float64)
    tp = (pred_pos + actual_pos + correct - count) / 2.0
    fp, fn = pred_pos - tp, actual_pos - tp
    tn = count - tp - fp - fn

    def div(a, b):
        return np.divide(a, b, out=np.zeros_like(a), where=b != 0)
    if kind == "precision":
        return div(tp, pred_pos)
    if kind == "recall":
        return div(tp, actual_pos)
    if kind == "f1":
        return div(2.0 * tp, actual_pos + pred_pos)
    if kind == "balanced_accuracy":
        return (div(tp, tp + fn) + div(tn, tn + fp)) / 2.0
    raise ValueError(kind)


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

    def _train(self, f):
        if f < 0:
            return np.arange(len(self.y_class))
        if self.train_rows is not None and self.train_rows[f] is not None:
            return self.train_rows[f]
        return np.flatnonzero(self.fold != f)

    def column(self, class_weight, f):
        """(float32 weight of every class id, sw_sum) of a fit on the training rows of fold f (-1: all rows)."""
        key = (repr(class_weight), int(f))
        if key not in self.cache:
            rows = self._train(f)
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


class _LogRegFamily:
    """(candidate x fold) columns of binary L2 logistic regression."""

    name = "logreg"

    def __init__(self, estimator, candidate_params, X, y, scorers, enc=None):
        self.estimator = estimator
        self.cands = [_check_logreg(q, class_weight=True) for q in _merged_params(estimator, candidate_params)]
        for p in candidate_params:
            extra = set(p) - _LOGREG_SEARCHABLE
            if extra:
                raise NotImplementedError(
                    "searching LogisticRegression over %s has no device path (searchable: %s)"
                    % (sorted(extra), sorted(_LOGREG_SEARCHABLE)))
        self.classes_, self.y_class = _classes_and_ids(y, enc)
        if len(self.classes_) != 2:
            raise NotImplementedError(
                "this family is binary (got %d classes)" % len(self.classes_))
        self.weights = _ClassWeights(self.classes_, self.y_class)
        # every scorer must be a count-based metric (accuracy / precision / recall / f1 / balanced
        # accuracy on predict); scoring=None -> _PassthroughScorer -> estimator.score == accuracy
        self.label_one = _label_one(self.classes_)
        self.metrics = {}
        for name, scorer in scorers.items():
            m = _count_metric(scorer)
            if m is None:
                raise NotImplementedError(
                    "scorer %r has no device path for classifiers (supported: %s)"
                    % (scorer, SUPPORTED_CLASSIFIER_SCORERS))
            # binary averaging keeps the plain name; averaged variants and ranking scorers carry (kind, average)
            self.metrics[name] = m if _is_rank(m) or m[1] not in (None, "binary") else m[0]
        self.needs_pred_pos = any(k not in ("accuracy", "roc_auc", "neg_log_loss") and not _is_rank(k)
                                  for k in self.metrics.values())
        self.engine_entries = _rank_entries(self.metrics)

    def stage(self, eng, X, fold, n_splits, x_staged=False):
        if not x_staged:
            parallel.stage_x_replicated(eng, X)
        eng.stage_labels(self.y_class)
        eng.stage_folds(fold, n_splits)
        self.weights.set_folds(fold)
        if self.needs_pred_pos:     # positives per fold: only the precision / recall / f1 formulas use them
            self.pos_in_fold = np.bincount(np.asarray(fold)[self.y_class == 1], minlength=n_splits).astype(np.int64)
            self.total_pos = int(self.pos_in_fold.sum())
        else:
            self.pos_in_fold = np.zeros(n_splits, dtype=np.int64)
            self.total_pos = 0

    def set_sample_weight(self, sample_weight):
        """float32 sample weight of every row (None: none), indexed by each fit's training rows as the
        reference indexes fit_params (ref search.py:208-211); the refit takes all of them."""
        self.weights.set_sample_weight(sample_weight)

    def set_train_rows(self, train_rows):
        """Training rows of every fold of the staged layout in the splitter's order (None entries: the
        rows outside the fold, ascending): the order sw_sum of a weighted column is summed in."""
        self.weights.set_folds(self.weights.fold, train_rows)

    def _scores(self, eng, coef, codes, pos, actual_pos):
        """{scorer name: per-column value} on the rows selected by the scoring codes."""
        correct, count = eng.linear_score_batch(coef, codes, pos)
        pred_pos = None
        if self.needs_pred_pos:
            # a positive class id that matches no row makes "correct" count the predicted negatives
            neg_correct, _ = eng.linear_score_batch(coef, codes, np.full(len(pos), -7, dtype=np.int32))
            pred_pos = count - neg_correct
        out = {}
        rank = _RankScores(eng, coef, codes, self.label_one)
        for name, kind in self.metrics.items():
            if kind == "roc_auc":
                out[name], _ = eng.linear_auc_batch(coef, codes, pos)
            elif kind == "neg_log_loss":
                out[name] = -eng.linear_logloss_batch(coef, codes, pos)[0]
            elif _is_rank(kind):
                out[name] = rank.value(*kind)
            elif isinstance(kind, tuple):      # micro / macro / weighted: 2 x 2 confusion [true, predicted]
                tp = (pred_pos + actual_pos + correct - count) / 2.0
                fp, fn = pred_pos - tp, actual_pos - tp
                conf = np.stack([np.stack([count - tp - fp - fn, fp], -1), np.stack([fn, tp], -1)], -2)
                out[name] = _metric_from_confusion(kind[0], kind[1], conf)
            else:
                out[name] = _metric_from_counts(kind, correct, count, pred_pos, actual_pos)
        return out, count

    def score_columns(self, eng, coef, codes):
        """{scorer name: per-column value} of fitted coefficients on the rows the scoring codes select."""
        codes = np.asarray(codes, dtype=np.int32)
        f = np.where(codes >= 0, codes, -3 - codes)
        actual = np.where(codes >= 0, self.pos_in_fold[np.clip(f, 0, None)],
                          np.where(codes == -2, self.total_pos, self.total_pos - self.pos_in_fold[np.clip(f, 0, None)]))
        return self._scores(eng, coef, codes, np.ones(len(codes), dtype=np.int32), actual)[0]

    def column_cost(self, n_splits):
        """Expected relative duration of every (candidate, fold) column, for the multi-GPU block deal."""
        from ..parallel import logreg_column_cost
        return np.repeat(logreg_column_cost([p["C"] for p in self.cands]), n_splits)

    def run_columns(self, eng, cols, n_splits, return_train_score):
        """Fit + score the given global column ids (col = cand * n_splits + fold).
        Returns dict of per-column arrays aligned with `cols`."""
        cols = np.asarray(cols, dtype=np.int64)
        out = {
            "n_test": np.zeros(len(cols), dtype=np.int64),
            "fit_time": np.zeros(len(cols)), "score_time": np.zeros(len(cols)),
            "n_iter": np.zeros(len(cols), dtype=np.int32), "status": np.zeros(len(cols), dtype=np.int32),
        }
        for name in self.metrics:           # one array per scorer: "test_<name>" (+ "train_<name>")
            out["test_%s" % name] = np.zeros(len(cols))
            if return_train_score:
                out["train_%s" % name] = np.zeros(len(cols))
        cand = cols // n_splits
        fold = (cols % n_splits).astype(np.int32)
        groups = defaultdict(list)
        for i, c in enumerate(cand):
            p = self.cands[c]
            groups[(bool(p["fit_intercept"]), float(p["tol"]), int(p["max_iter"]))].append(i)
        for (fi, tol, mi), idx in groups.items():
            idx = np.asarray(idx)
            C = np.array([self.cands[c]["C"] for c in cand[idx]], dtype=np.float64)
            pos = np.ones(len(idx), dtype=np.int32)
            t0 = time.time()
            self.weights.stage(eng, [self.cands[c]["class_weight"] for c in cand[idx]], fold[idx])
            res = eng.logreg_fit_batch(C, fold[idx], pos, fit_intercept=fi, tol=tol, max_iter=mi)
            t1 = time.time()
            vals, count = self._scores(eng, res["coef"], fold[idx], pos, self.pos_in_fold[fold[idx]])
            t2 = time.time()
            # a column whose objective went non-finite has no usable coefficients: count-based scores
            # would still be finite numbers, so they are set to NaN here and search.py applies
            # `error_score` to them (ref search.py:226-259); max_iter / line-search stops only warn,
            # as scikit-learn does (SK/linear_model/_logistic.py:599)
            bad = res["status"] == 5
            if np.any(res["status"] == 3) or np.any(res["status"] == 4):
                import warnings
                from sklearn.exceptions import ConvergenceWarning
                warnings.warn("lbfgs failed to converge within max_iter=%d for %d of %d (candidate, fold) fits"
                              % (mi, int(np.sum((res["status"] == 3) | (res["status"] == 4))), len(idx)),
                              ConvergenceWarning)
            for name, v in vals.items():
                v = np.asarray(v, dtype=np.float64).copy()
                v[bad] = np.nan
                out["test_%s" % name][idx] = v
            out["n_test"][idx] = count
            out["fit_time"][idx] = (t1 - t0) / len(idx)
            out["score_time"][idx] = (t2 - t1) / len(idx)
            out["n_iter"][idx] = res["n_iter"]
            out["status"][idx] = res["status"]
            if return_train_score:
                vals, _ = self._scores(eng, res["coef"], _train_codes(fold[idx]), pos,
                                       self.total_pos - self.pos_in_fold[fold[idx]])
                for name, v in vals.items():
                    v = np.asarray(v, dtype=np.float64).copy()
                    v[bad] = np.nan
                    out["train_%s" % name][idx] = v
        return out

    def refit(self, eng, params, X_dtype, n_features):
        p = _check_logreg(_resolve(self.estimator, params), class_weight=True)
        self.weights.stage(eng, [p["class_weight"]], [-1])
        res = eng.logreg_fit_batch(np.array([p["C"]]), np.array([-1], dtype=np.int32),
                                   np.array([1], dtype=np.int32), fit_intercept=p["fit_intercept"],
                                   tol=p["tol"], max_iter=p["max_iter"])
        return self.make_estimator(params, res["coef"][0], res["n_iter"][0], X_dtype, n_features)

    def make_estimator(self, params, coef_row, n_iter, X_dtype, n_features):
        """A genuine fitted sklearn LogisticRegression (attributes as set by
        SK/linear_model/_logistic.py:1561-1593) so inherited predict* work."""
        est = _resolve(self.estimator, params)
        dt = np.float64 if X_dtype == np.float64 else np.float32
        est.coef_ = coef_row[None, :n_features].astype(dt)
        if est.fit_intercept:
            est.intercept_ = coef_row[n_features:n_features + 1].astype(dt)
        else:
            est.intercept_ = np.zeros(1, dtype=dt)
        est.classes_ = self.classes_
        est.n_iter_ = np.array([n_iter], dtype=np.int32)
        est.n_features_in_ = n_features
        return est

    def fold_proba(self, eng, params, fold, n_splits):
        """preds_ support (ref search.py:551-560): per-fold refit of the best params,
        predict_proba on the held-out rows, stacked in fold order."""
        p = _check_logreg(_resolve(self.estimator, params), class_weight=True)
        f = np.arange(n_splits, dtype=np.int32)
        self.weights.stage(eng, [p["class_weight"]] * n_splits, f)
        res = eng.logreg_fit_batch(np.full(n_splits, p["C"]), f, np.ones(n_splits, dtype=np.int32),
                                   fit_intercept=p["fit_intercept"], tol=p["tol"], max_iter=p["max_iter"])
        dec = eng.linear_decision(res["coef"])
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

    def __init__(self, estimator, candidate_params, X, y, scorers, enc=None):
        self.estimator = estimator
        self.cands = [_check_logreg(q, class_weight=True) for q in _merged_params(estimator, candidate_params)]
        for p in candidate_params:
            extra = set(p) - _LOGREG_SEARCHABLE
            if extra:
                raise NotImplementedError(
                    "searching LogisticRegression over %s has no device path (searchable: %s)"
                    % (sorted(extra), sorted(_LOGREG_SEARCHABLE)))
        self.classes_, self.y_class = _classes_and_ids(y, enc)
        self.n_classes = len(self.classes_)
        self.weights = _ClassWeights(self.classes_, self.y_class)
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
        self.needs_pred_pos = False
        self.engine_entries = _rank_entries(self.metrics)

    def stage(self, eng, X, fold, n_splits, x_staged=False):
        if not x_staged:
            parallel.stage_x_replicated(eng, X)
        eng.stage_labels(self.y_class)
        eng.stage_folds(fold, n_splits)
        self.weights.set_folds(fold)

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
            p = self.cands[c]
            groups[(bool(p["fit_intercept"]), float(p["tol"]), int(p["max_iter"]))].append(i)
        for (fi, tol, mi), idx in groups.items():
            idx = np.asarray(idx)
            C = np.array([self.cands[c]["C"] for c in cand[idx]], dtype=np.float64)
            t0 = time.time()
            self.weights.stage(eng, [self.cands[c]["class_weight"] for c in cand[idx]], fold[idx])
            res = eng.logreg_multinomial_fit_batch(C, fold[idx], self.n_classes, fit_intercept=fi, tol=tol,
                                                   max_iter=mi)
            t1 = time.time()
            conf = eng.multinomial_confusion_batch(res["coef"], fold[idx])
            for name, v in self._values(eng, conf, res["coef"], fold[idx]).items():
                out["test_%s" % name][idx] = v
            t2 = time.time()
            out["n_test"][idx] = conf.sum(axis=(1, 2))
            out["fit_time"][idx] = (t1 - t0) / len(idx)
            out["score_time"][idx] = (t2 - t1) / len(idx)
            out["n_iter"][idx] = res["n_iter"]
            out["status"][idx] = res["status"]
            if return_train_score:
                train = _train_codes(fold[idx])
                conf = eng.multinomial_confusion_batch(res["coef"], train)
                for name, v in self._values(eng, conf, res["coef"], train).items():
                    out["train_%s" % name][idx] = v
        return out

    def _values(self, eng, conf, coef, codes):
        """{scorer name: per-problem value} from the confusion counts conf of the rows the codes select."""
        rank = _RankScores(eng, coef, codes)
        out = {}
        for name, (kind, average) in self.metrics.items():
            if kind == "neg_log_loss":
                out[name] = -eng.linear_logloss_batch(coef, codes)[0]
            elif _is_rank((kind, average)):
                out[name] = rank.value(kind, average)
            else:
                out[name] = _metric_from_confusion(kind, average, conf)
        return out

    def score_columns(self, eng, coef, codes):
        """{scorer name: per-problem value} of fitted coefficients on the rows the scoring codes select."""
        return self._values(eng, eng.multinomial_confusion_batch(coef, codes), coef, codes)

    def refit(self, eng, params, X_dtype, n_features):
        p = _check_logreg(_resolve(self.estimator, params), class_weight=True)
        self.weights.stage(eng, [p["class_weight"]], [-1])
        res = eng.logreg_multinomial_fit_batch(np.array([p["C"]]), np.array([-1], dtype=np.int32), self.n_classes,
                                               fit_intercept=p["fit_intercept"], tol=p["tol"],
                                               max_iter=p["max_iter"])
        return self.make_estimator(params, res["coef"][0], res["n_iter"][0], X_dtype, n_features)

    def make_estimator(self, params, coef_rows, n_iter, X_dtype, n_features):
        """Fitted sklearn LogisticRegression with the multiclass attribute shapes
        (SK/linear_model/_logistic.py:1561-1593): coef_ (K, d), intercept_ (K,), n_iter_ (1,)."""
        est = _resolve(self.estimator, params)
        dt = np.float64 if X_dtype == np.float64 else np.float32
        est.coef_ = coef_rows[:, :n_features].astype(dt)
        if est.fit_intercept:
            est.intercept_ = coef_rows[:, n_features].astype(dt)
        else:
            est.intercept_ = np.zeros(self.n_classes, dtype=dt)
        est.classes_ = self.classes_
        est.n_iter_ = np.array([n_iter], dtype=np.int32)
        est.n_features_in_ = n_features
        return est

    def fold_proba(self, eng, params, fold, n_splits):
        from sklearn.utils.extmath import softmax
        p = _check_logreg(_resolve(self.estimator, params), class_weight=True)
        f = np.arange(n_splits, dtype=np.int32)
        self.weights.stage(eng, [p["class_weight"]] * n_splits, f)
        res = eng.logreg_multinomial_fit_batch(np.full(n_splits, p["C"]), f, self.n_classes,
                                               fit_intercept=p["fit_intercept"], tol=p["tol"],
                                               max_iter=p["max_iter"])
        K = self.n_classes
        dec = eng.linear_decision(res["coef"].reshape(n_splits * K, -1))
        return np.vstack([softmax(dec[fold == k, k * K:(k + 1) * K].astype(np.float64)) for k in range(n_splits)])
