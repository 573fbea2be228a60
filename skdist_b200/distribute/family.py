"""What the search families share: the column loop of a search, the classifier scorers and the candidate
bookkeeping.

A family computes, for all (candidate, fold) tasks of a search at once, what one `_fit_and_score` task of
the reference computes (ref search.py:180-288).  `_Family.run_columns` groups the columns into launches and
times, fits and scores every launch; each family supplies

  _launch_key(params)            the parameters every column of one launch shares
  _launch(eng, cands, folds)     one launch: (coef in the scoring layout, n_iter, status, columns whose test
                                 scores become NaN, columns whose train scores become NaN)
  score_columns(eng, coef, codes)   ({scorer name: per-column value}, rows per column) on the rows the scoring
                                 codes select (held-out fold f: f; training rows of fold f: -3 - f)

Classifier scorers are functions of device-side counts / sums: confusion counts (accuracy, balanced accuracy,
precision / recall / f1 with any averaging), ranked counts per segment (csrc/auc.cu: roc_auc on the decision
values, roc_auc_ovr / roc_auc_ovo [_weighted] on float32 predict_proba, average_precision on the decision
values) and a sum of -log p (neg_log_loss)."""
import time
from collections import defaultdict

import numpy as np

from .. import parallel
from .base import _clone
from .folds import _train_codes, _train_rows


def _resolve(estimator, params):
    est = _clone(estimator)
    if params:
        est.set_params(**params)
    return est


def _check_engine_entries(family, eng):
    """Raise NotImplementedError before any fit when the engine lacks an entry the family's scorers call: a
    scorer whose kernel the engine does not provide has no device path (and no CPU fallback)."""
    missing = [e for e in family.engine_entries if not hasattr(eng, e)]
    if missing:
        raise NotImplementedError(
            "scorers %s need %s, which %s does not provide: no device path on this engine"
            % (sorted(family.metrics), ", ".join(missing), type(eng).__name__))


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


class _Family:
    """(candidate x fold) columns of one base estimator.  A column is cand * n_splits + fold."""

    searchable = frozenset()        # the parameters a search may vary
    fold = train_rows = None
    needs_pred_pos = False

    def _check_searchable(self, candidate_params):
        for p in candidate_params:
            extra = set(p) - self.searchable
            if extra:
                raise NotImplementedError(
                    "searching %s over %s has no device path (searchable: %s)"
                    % (type(self.estimator).__name__, sorted(extra), sorted(self.searchable)))

    @property
    def engine_entries(self):
        """Engine entries the scorers call beyond the fit and count kernels."""
        return ("linear_rank_batch",) if any(_is_rank(k) for k in self.metrics.values()) else ()

    # -- layout -------------------------------------------------------------------------------------------
    def prepare(self, fold, n_splits):
        """Host-only statistics of a layout, which the search computes while X is still on its way to the
        device; none by default."""

    def stage(self, eng, X, fold, n_splits, x_staged=False):
        if not x_staged:
            parallel.stage_x_replicated(eng, X)
        eng.stage_labels(self.y_class)
        eng.stage_folds(fold, n_splits)
        self.fold, self.train_rows = np.asarray(fold), None
        if self.needs_pred_pos:     # positives per fold: only the precision / recall / f1 formulas use them
            self.pos_in_fold = np.bincount(self.fold[self.y_class == 1], minlength=n_splits).astype(np.int64)
        else:
            self.pos_in_fold = np.zeros(n_splits, dtype=np.int64)
        self.total_pos = int(self.pos_in_fold.sum())

    def set_train_rows(self, train_rows):
        """Training rows of every fold of the staged layout in the splitter's order (None entries: the rows
        outside the fold, ascending, as KFold / StratifiedKFold give them)."""
        self.train_rows = train_rows

    def _train(self, f):
        return _train_rows(self.fold, self.train_rows, f)

    def column_cost(self, n_splits):
        """Expected relative duration of every (candidate, fold) column, for the multi-GPU block deal: all
        equal unless a family knows better."""
        return np.ones(len(self.cands) * n_splits)

    # -- the column loop ----------------------------------------------------------------------------------
    def run_columns(self, eng, cols, n_splits, return_train_score):
        """Fit + score the given global column ids (col = cand * n_splits + fold), one launch per launch
        key.  Returns dict of per-column arrays aligned with `cols`."""
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
        launches = defaultdict(list)
        for i, c in enumerate(cand):
            launches[self._launch_key(self.cands[c])].append(i)
        for idx in launches.values():
            idx = np.asarray(idx)
            t0 = time.time()
            coef, n_iter, status, bad_test, bad_train = self._launch(eng, [self.cands[c] for c in cand[idx]],
                                                                     fold[idx])
            t1 = time.time()
            vals, count = self.score_columns(eng, coef, fold[idx])
            t2 = time.time()
            # a column without usable coefficients still gets finite count-based scores: NaN here, and
            # search.py applies `error_score` to them (ref search.py:226-259)
            for name, v in vals.items():
                out["test_%s" % name][idx] = np.where(bad_test, np.nan, v)
            out["n_test"][idx] = count
            out["fit_time"][idx] = (t1 - t0) / len(idx)
            out["score_time"][idx] = (t2 - t1) / len(idx)
            out["n_iter"][idx] = n_iter
            out["status"][idx] = status
            if return_train_score:
                vals, _ = self.score_columns(eng, coef, _train_codes(fold[idx]))
                for name, v in vals.items():
                    out["train_%s" % name][idx] = np.where(bad_train, np.nan, v)
        return out

    # -- classifier scorers -------------------------------------------------------------------------------
    def _set_binary_metrics(self, metrics):
        """Scorers {name: (kind, average)} of a binary target: binary averaging keeps the plain kind; averaged
        variants and ranking scorers carry (kind, average)."""
        self.metrics = {name: m if _is_rank(m) or m[1] not in (None, "binary") else m[0]
                        for name, m in metrics.items()}
        self.needs_pred_pos = any(k not in ("accuracy", "roc_auc", "neg_log_loss") and not _is_rank(k)
                                  for k in self.metrics.values())
        self.label_one = _label_one(self.classes_)

    def _binary_scores(self, eng, coef, codes, binary_proba="proba"):
        """({scorer name: per-column value}, rows per column) of binary columns on the rows the scoring codes
        select.  binary_proba: the score that ranks as predict_proba[:, 1] does."""
        codes = np.asarray(codes, dtype=np.int32)
        f = np.clip(np.where(codes >= 0, codes, -3 - codes), 0, None)
        actual_pos = np.where(codes >= 0, self.pos_in_fold[f],
                              np.where(codes == -2, self.total_pos, self.total_pos - self.pos_in_fold[f]))
        pos = np.ones(len(codes), dtype=np.int32)
        correct, count = eng.linear_score_batch(coef, codes, pos)
        pred_pos = None
        if self.needs_pred_pos:
            # a positive class id that matches no row makes "correct" count the predicted negatives
            neg_correct, _ = eng.linear_score_batch(coef, codes, np.full(len(pos), -7, dtype=np.int32))
            pred_pos = count - neg_correct
        out = {}
        rank = _RankScores(eng, coef, codes, self.label_one, binary_proba)
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

    def _multiclass_scores(self, eng, coef, codes):
        """({scorer name: per-column value}, rows per column) of [B, K, d + 1] columns on the rows the scoring
        codes select: confusion counts of the first arg-max, ranked counts and the softmax log loss."""
        conf = eng.multinomial_confusion_batch(coef, codes)
        rank = _RankScores(eng, coef, codes)
        out = {}
        for name, (kind, average) in self.metrics.items():
            if kind == "neg_log_loss":
                out[name] = -eng.linear_logloss_batch(coef, codes)[0]
            elif _is_rank((kind, average)):
                out[name] = rank.value(kind, average)
            else:
                out[name] = _metric_from_confusion(kind, average, conf)
        return out, conf.sum(axis=(1, 2))
