"""Distributed multiclass strategies on H100 GPUs.

Drop-in for /root/reference/skdist/distribute/multiclass.py (class names, constructor
signatures, fitted attributes).  The reference ships one dense 0/1 label vector per class to a
Spark task that runs a full binary fit (`_fit_binary`, multiclass.py:109-152, fan-out
:296-331).  Here the K label columns are K *columns* of one batched solve that shares X: rows
carry an integer class id, column k treats `class id == k` as positive.

  base estimator                         device path
  --------------                         -----------
  LogisticRegression(solver="lbfgs")     Engine.logreg_fit_batch (same kernels as the search path)
  SGDClassifier(loss="hinge"|"log_loss") Engine.sgd_fit_batch (exact-order column-batched SGD)
  anything else                          NotImplementedError (no CPU fallback by design)

Multilabel targets and `max_negatives` give every column its own label vector / row set: bit
matrices on the device (`skd_stage_row_bits`), LogisticRegression base.

`DistOneVsOneClassifier` (ref multiclass.py:365-475) fits the K(K-1)/2 class pairs the same way:
pair (i, j) is a column whose training rows are masked to classes i and j on the device
(`col_neg`), replacing the reference's per-pair `X[cond]` copy (`_fit_ovo_binary`, :155-173).
"""
import warnings

import numpy as np
from sklearn.base import BaseEstimator
from sklearn.linear_model import LogisticRegression, SGDClassifier
from sklearn.multiclass import OneVsOneClassifier, OneVsRestClassifier
from sklearn.preprocessing import LabelBinarizer, normalize
from sklearn.utils.validation import check_is_fitted

from .. import parallel
from ..engine import get_engine
from .base import _clone, _Cloner, _parse_partitions, _ScParamMixin
from .validation import _check_estimator

__all__ = ["DistOneVsRestClassifier", "DistOneVsOneClassifier"]


class _ConstantPredictor(BaseEstimator):
    """Predicts the single label seen in training (ref multiclass.py:175-192)."""

    def fit(self, X, y):
        self.y_ = y
        return self

    def predict(self, X):
        check_is_fitted(self, "y_")
        return np.repeat(self.y_, X.shape[0])

    def decision_function(self, X):
        check_is_fitted(self, "y_")
        return np.repeat(self.y_, X.shape[0])

    def predict_proba(self, X):
        check_is_fitted(self, "y_")
        return np.repeat([np.hstack([1 - self.y_, self.y_])], X.shape[0], axis=0)


def _binary_estimator(template, coef_row, n_features, X_dtype, **extra):
    """A genuine fitted sklearn binary classifier (classes_ = [0, 1]) as `_fit_binary` returns
    (ref multiclass.py:141-152) so the inherited predict / decision_function work."""
    est = template() if isinstance(template, _Cloner) else _clone(template)
    dt = np.float64 if X_dtype == np.float64 else np.float32
    est.coef_ = coef_row[None, :n_features].astype(dt)
    b = coef_row[n_features:n_features + 1]
    # LogisticRegression keeps the intercept in X's dtype, SGDClassifier in float64
    bdt = dt if isinstance(est, LogisticRegression) else np.float64
    est.intercept_ = b.astype(bdt) if est.fit_intercept else np.zeros(1, bdt)
    est.classes_ = np.array([0, 1])
    est.n_features_in_ = n_features
    for k, v in extra.items():
        setattr(est, k, v)
    return est


SGD_DIVERGED = 5        # sgd_fit_batch status: a column's weights or intercept became non-finite


def _check_sgd_status(template, status, n_iter):
    """Report the SGD columns' outcomes as scikit-learn's per-column fits would, in column order: a column whose
    weights or intercept became non-finite raises `_plain_sgd`'s ValueError with its epoch, and a column that ran
    all max_iter epochs with a tolerance set emits `BaseSGDClassifier._fit`'s ConvergenceWarning (once)."""
    from sklearn.exceptions import ConvergenceWarning
    status = np.asarray(status).astype(np.int64)
    n_iter = np.asarray(n_iter).astype(np.int64)
    bad = np.flatnonzero(status == SGD_DIVERGED)
    done = n_iter if bad.size == 0 else n_iter[:bad[0]]       # the columns scikit-learn fits before it raises
    tol = template.tol
    if tol is not None and tol > -np.inf and np.any(done == template.max_iter):
        warnings.warn("Maximum number of iteration reached before convergence. Consider increasing max_iter to "
                      "improve the fit.", ConvergenceWarning)
    if bad.size:
        raise ValueError("Floating-point under-/overflow occurred at epoch #%d. Scaling input data with "
                         "StandardScaler or MinMaxScaler might help." % int(n_iter[bad[0]]))


def _negatives_rows(pos_mask, max_negatives, random_state, method):
    """Training rows of one label column under the reference's negative down-sampling
    (`_negatives_mask`, ref multiclass.py:76-106): every positive row plus the negatives that
    `train_test_split(..., test_size=max_negatives, random_state=random_state)` puts in its test part.
    Returns a boolean row mask (all True where the reference keeps every row).  The reference
    additionally shuffles the kept rows, which does not change a full-batch lbfgs fit beyond the
    summation order."""
    from sklearn.model_selection import train_test_split
    pos_mask = np.asarray(pos_mask, dtype=bool)
    n_pos = int(pos_mask.sum())
    n_neg = int(len(pos_mask) - n_pos)
    if method == "ratio":
        pass
    elif method == "multiplier":
        max_negatives = int(max_negatives * n_pos)
    else:
        raise ValueError("Unknown method. Options are 'ratio' or 'multiplier'.")
    if isinstance(max_negatives, (int, np.integer)) and max_negatives >= n_neg:
        return np.ones(len(pos_mask), bool)
    frac = max_negatives if isinstance(max_negatives, float) else (max_negatives / float(n_neg))
    _, neg_rows = train_test_split(np.flatnonzero(~pos_mask), test_size=frac, random_state=random_state)
    mask = pos_mask.copy()
    mask[neg_rows] = True
    return mask


class DistOneVsRestClassifier(_ScParamMixin, OneVsRestClassifier):
    """One-vs-the-rest with all label columns fitted as one batched GPU solve.
    Constructor mirrors ref multiclass.py:230-253 (``sc`` is the 2nd positional argument)."""

    def __init__(self, estimator, sc=None, norm=None, partitions="auto", max_negatives=None,
                 random_state=None, method="ratio", n_splits=1, mlb_override=False, verbose=False,
                 n_jobs=None):
        self.estimator = estimator
        self.sc = sc
        self.norm = norm
        self.partitions = partitions
        self.max_negatives = max_negatives
        self.random_state = random_state
        self.method = method
        self.n_splits = n_splits
        self.mlb_override = mlb_override
        self.verbose = verbose
        self.n_jobs = n_jobs

    def fit(self, X, y, **fit_params):
        """Fit the K binary estimators (ref multiclass.py:255-335).

        1-d class labels: column k = `class id == k` (the rows carry one integer id).  Multilabel
        targets (indicator matrix, or sequences of labels -> `MultiLabelBinarizer` unless
        `mlb_override`, ref :267-274) and `max_negatives` (ref `_negatives_mask`, :76-106) give every
        column its own 0/1 label vector / training-row set: both go to the device as bit matrices
        (`Engine.stage_row_bits`), no `X[rows]` copies.  `n_splits` only cuts X into broadcast pieces in
        the reference (`_split_X`, :35-50) and has no effect here.

        fit_params: `sample_weight` of a LogisticRegression base.  As in the reference (:145-151), every
        label column's fit takes the full array; with `max_negatives` dropping rows that is a fit on fewer
        rows than weights, which raises the ValueError scikit-learn raises for it."""
        _check_estimator(self, verbose=self.verbose)
        from collections.abc import Sequence
        if (not self.mlb_override and not hasattr(y[0], "__array__") and isinstance(y[0], Sequence)
                and not isinstance(y[0], str)):                          # ref :267-274
            from sklearn.preprocessing import MultiLabelBinarizer
            self.mlb = MultiLabelBinarizer()
            y = self.mlb.fit_transform(y)
        X_arr = np.asarray(X)
        y_arr = np.asarray(y)
        self.label_binarizer_ = LabelBinarizer(sparse_output=True)      # ref :279-281
        self.label_binarizer_.fit(y_arr)
        self.classes_ = self.label_binarizer_.classes_
        K = len(self.classes_)
        n, d = X_arr.shape
        _parse_partitions(self.partitions, K)
        base = self.estimator
        from .logreg_family import _fit_sample_weight
        sample_weight = _fit_sample_weight(base, fit_params, n)
        multilabel = y_arr.ndim == 2
        use_bits = multilabel or self.max_negatives is not None
        if use_bits and type(base) is not LogisticRegression:
            raise NotImplementedError(
                "multilabel targets / max_negatives need per-column row sets: device path for "
                "LogisticRegression(solver='lbfgs') only (SGD walks one shared sample order)")
        if multilabel:
            Y = self.label_binarizer_.transform(y_arr).tocsc()          # ref :289-290
            ycls = np.zeros(n, np.int32)
            counts = np.asarray(Y.sum(axis=0)).ravel().astype(np.int64)
            n_cols = Y.shape[1]
        else:
            ycls = np.searchsorted(self.classes_, y_arr).astype(np.int32)
            counts = np.bincount(ycls, minlength=K)
            n_cols = 1 if K == 2 else K

        rank, world, _ = parallel.dist_info()
        eng = get_engine()
        parallel.stage_x_replicated(eng, X_arr)
        eng.stage_labels(ycls)
        eng.stage_folds(None, 0)
        # constant columns (a label present in every / no row) -> _ConstantPredictor (ref :121-139)
        if multilabel:
            const = (counts == 0) | (counts == n)
            col_ids = np.flatnonzero(~const)
        elif K == 2:
            # LabelBinarizer gives ONE column for binary problems (positive = classes_[1])
            const = np.zeros(K, bool)
            col_ids = np.array([1])
        else:
            const = (counts == 0) | (counts == n)
            col_ids = np.flatnonzero(~const)
        mine = col_ids[parallel.shard_indices(len(col_ids), rank, world)]
        if type(base) is LogisticRegression:
            from .logreg_family import _check_logreg, _fit_class_weights, _stage_columns
            p = _check_logreg(_clone(base), class_weight=True)
            labels = train = None
            if use_bits and len(mine):
                if multilabel:
                    labels = np.ascontiguousarray(Y[:, mine].toarray().T.astype(bool))
                else:
                    labels = ycls[None, :] == mine[:, None].astype(np.int32)
                if self.max_negatives is not None:
                    train = np.stack([_negatives_rows(labels[i], self.max_negatives, self.random_state, self.method)
                                      for i in range(len(mine))])
            # every refusal comes before the first staging call, so that no staged input outlives a refused fit
            if sample_weight is not None and train is not None:
                from sklearn.utils.validation import _check_sample_weight
                for i in range(len(mine)):
                    if not train[i].all():     # the full-length weights of a fit on fewer rows (ref :141-151)
                        _check_sample_weight(sample_weight, np.empty((int(train[i].sum()), 0), np.float32))
            cols = []
            if (p["class_weight"] is not None or sample_weight is not None) and len(mine):
                # every column's binary fit: its 0/1 labels on its training rows (ascending), as _fit_binary
                # hands them to the estimator (ref multiclass.py:141-151), with the sample weights of all rows
                for i, k in enumerate(mine):
                    y01 = labels[i] if labels is not None else ycls == k
                    rows = np.flatnonzero(train[i]) if train is not None else slice(None)
                    cols.append(_fit_class_weights(p["class_weight"], y01[rows].astype(np.intp), np.array([0, 1]),
                                                   None if sample_weight is None else sample_weight[rows]))
            try:
                if labels is not None:
                    eng.stage_row_bits(labels if multilabel else None, train)
                if cols:
                    _stage_columns(eng, cols, sample_weight)
            except Exception:
                eng.stage_row_bits(None, None)     # staged inputs are one-shot: none outlives a failed staging
                raise
            res = eng.logreg_fit_batch(np.full(len(mine), p["C"]), np.full(len(mine), -1, np.int32),
                                       mine.astype(np.int32), fit_intercept=p["fit_intercept"],
                                       tol=p["tol"], max_iter=p["max_iter"])
            packed = np.concatenate([res["coef"], res["n_iter"][:, None].astype(np.float32)], axis=1)
            extra_of = lambda row: {"n_iter_": np.array([int(row[-1])], dtype=np.int32)}
        elif type(base) is SGDClassifier:
            res = eng.sgd_fit_batch(base, mine.astype(np.int32))
            packed = np.concatenate([res["coef"], res["n_iter"][:, None].astype(np.float64),
                                     res["t"][:, None], res["status"][:, None].astype(np.float64)], axis=1)
            extra_of = lambda row: {"n_iter_": int(row[-3]), "t_": float(row[-2])}
        else:
            raise NotImplementedError(
                "%s has no device path; supported base estimators: LogisticRegression(solver='lbfgs'), "
                "SGDClassifier.  (No CPU fallback by design.)" % type(base).__name__)
        full = parallel.all_gather_columns(packed, len(col_ids), rank, world)
        if type(base) is SGDClassifier:
            _check_sgd_status(base, full[:, -1], full[:, -3])
        by_col = {int(c): full[i] for i, c in enumerate(col_ids)}
        ests = []
        cols = [1] if (K == 2 and not multilabel) else range(n_cols)
        make = _Cloner(base)
        for k in cols:
            if k in by_col:
                row = by_col[k]
                ests.append(_binary_estimator(make, row[:d + 1], d, X_arr.dtype, **extra_of(row)))
            else:
                warnings.warn("Label %s is present in all training examples." % str(self.classes_[k]))
                ests.append(_ConstantPredictor().fit(X_arr, np.array([1 if counts[k] == n else 0])))
        self.estimators_ = ests
        self.n_features_in_ = d
        self.__dict__.pop("sc", None)                                                     # ref :283
        if hasattr(self.estimator, "sc"):
            del self.estimator.sc
        return self

    def predict_proba(self, X):
        """Per-class probabilities with optional normalisation (ref multiclass.py:337-362)."""
        probs = np.column_stack([e.predict_proba(X)[:, 1] for e in self.estimators_])
        if self.norm:
            return normalize(probs, norm=self.norm)
        return probs


class DistOneVsOneClassifier(_ScParamMixin, OneVsOneClassifier):
    """One-vs-one: LogisticRegression pairs as one batched GPU solve (row-masked columns), SGDClassifier pairs as
    one exact-order device fit per pair on the pair's rows.
    Constructor mirrors ref multiclass.py:382-386 (``sc`` is the 2nd positional argument)."""

    def __init__(self, estimator, sc=None, partitions="auto", verbose=False, n_jobs=None):
        self.estimator = estimator
        self.sc = sc
        self.partitions = partitions
        self.verbose = verbose
        self.n_jobs = n_jobs

    def fit(self, X, y, **fit_params):
        """Fit the K(K-1)/2 pair estimators (ref multiclass.py:388-475)."""
        if fit_params:
            raise NotImplementedError("fit_params are not supported on the device path")
        _check_estimator(self, verbose=self.verbose)
        X_arr = np.asarray(X)
        y_arr = np.asarray(y)
        if y_arr.ndim != 1:
            raise ValueError("OneVsOneClassifier needs 1-d class labels")
        self.classes_ = np.unique(y_arr)                                 # ref :404
        if len(self.classes_) == 1:
            raise ValueError("OneVsOneClassifier can not be fit when only one class is present.")  # ref :405-408
        K = len(self.classes_)
        n, d = X_arr.shape
        pairs = [(i, j) for i in range(K) for j in range(i + 1, K)]      # ref :410-415 (same order)
        _parse_partitions(self.partitions, len(pairs))
        base = self.estimator
        if type(base) is SGDClassifier:
            return self._fit_sgd_pairs(X_arr, y_arr, pairs)
        if type(base) is not LogisticRegression:
            raise NotImplementedError(
                "%s has no one-vs-one device path; supported base estimators: LogisticRegression(solver='lbfgs'), "
                "SGDClassifier.  (No CPU fallback by design.)" % type(base).__name__)
        from .logreg_family import _check_logreg, _fit_class_weights, _stage_columns
        p = _check_logreg(_clone(base), class_weight=True)
        ycls = np.searchsorted(self.classes_, y_arr).astype(np.int32)
        rank, world, _ = parallel.dist_info()
        eng = get_engine()
        parallel.stage_x_replicated(eng, X_arr)
        eng.stage_labels(ycls)
        eng.stage_folds(None, 0)
        mine = parallel.shard_indices(len(pairs), rank, world)
        neg = np.array([pairs[k][0] for k in mine], dtype=np.int32)      # y_binary: class i -> 0, class j -> 1 (ref :159-161)
        pos = np.array([pairs[k][1] for k in mine], dtype=np.int32)
        if p["class_weight"] is not None and len(mine):
            # the pair's rows (ascending, X[cond] of ref :157-158) labelled 0 / 1
            cols = []
            for i, j in zip(neg, pos):
                yp = ycls[(ycls == i) | (ycls == j)]
                cols.append(_fit_class_weights(p["class_weight"], (yp == j).astype(np.intp), np.array([0, 1])))
            _stage_columns(eng, cols)
        res = eng.logreg_fit_batch(np.full(len(mine), p["C"]), np.full(len(mine), -1, np.int32), pos,
                                   fit_intercept=p["fit_intercept"], tol=p["tol"], max_iter=p["max_iter"],
                                   col_neg=neg)
        packed = np.concatenate([res["coef"], res["n_iter"][:, None].astype(np.float32)], axis=1)
        full = parallel.all_gather_columns(packed, len(pairs), rank, world)
        make = _Cloner(base)
        self.estimators_ = tuple(
            _binary_estimator(make, full[k][:d + 1], d, X_arr.dtype, n_iter_=np.array([int(full[k][-1])], dtype=np.int32))
            for k in range(len(pairs)))
        return self._finish(d)

    def _finish(self, d):
        self.pairwise_indices_ = None                                    # ref :441 (non-pairwise estimators)
        self.n_features_in_ = d
        self.__dict__.pop("sc", None)                                                      # ref :472
        if hasattr(self.estimator, "sc"):
            del self.estimator.sc
        return self

    def _fit_sgd_pairs(self, X_arr, y_arr, pairs):
        """SGD base estimator: `_fit_ovo_binary` (ref multiclass.py:155-173) trains pair (i, j) on the rows of the
        two classes only, and SGD walks ITS OWN shuffled order of those rows -- so a pair is not a masked column of
        the shared matrix (as it is for the full-batch lbfgs fit above) but one exact-order SGD fit on `X[cond]`:
        the pair's rows are staged (the row gather the reference does too) and the one-vs-rest SGD engine fits
        the single label column `y == classes_[j]`; pairs are dealt over the ranks."""
        base = self.estimator
        n, d = X_arr.shape
        Xf = np.ascontiguousarray(X_arr, dtype=np.float32)
        ycls = np.searchsorted(self.classes_, y_arr).astype(np.int32)
        rank, world, _ = parallel.dist_info()
        eng = get_engine()
        mine = parallel.shard_indices(len(pairs), rank, world)
        packed = np.zeros((len(mine), d + 4))
        for r, k in enumerate(mine):
            i, j = pairs[k]
            cond = (ycls == i) | (ycls == j)
            eng.stage_x(Xf[cond])                                        # this rank's pair only: no collective
            eng.stage_labels((ycls[cond] == j).astype(np.int32))         # y_binary: class i -> 0, class j -> 1 (ref :159-161)
            eng.stage_folds(None, 0)
            res = eng.sgd_fit_batch(base, np.array([1], dtype=np.int32))
            packed[r, :d + 1] = res["coef"][0]
            packed[r, d + 1] = res["n_iter"][0]
            packed[r, d + 2] = res["t"][0]
            packed[r, d + 3] = res["status"][0]
        full = parallel.all_gather_columns(packed, len(pairs), rank, world)
        _check_sgd_status(base, full[:, d + 3], full[:, d + 1])
        make = _Cloner(base)
        self.estimators_ = tuple(
            _binary_estimator(make, full[k][:d + 1], d, X_arr.dtype, n_iter_=int(full[k][d + 1]), t_=float(full[k][d + 2]))
            for k in range(len(pairs)))
        return self._finish(d)
