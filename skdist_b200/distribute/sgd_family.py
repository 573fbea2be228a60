"""SGDClassifier family of the search: what one (candidate, fold) task of the reference (`_fit_and_score`,
ref search.py:180-288, with estimator = SGDClassifier) computes, for all tasks of a search at once.

Every (candidate, fold) fit is an exact-order SGD fit on the fold's training rows, X[train] in the
splitter's order, as scikit-learn runs it (csrc/sgd.cu, skd_sgd_fit_groups).  The fits of one fold that
shuffle with the same seed form an order group: they walk the same rows in the same order and differ only
in alpha, so every (candidate, fold, class) column of a launch runs side by side.

  binary target    one column per (candidate, fold); seed = sgd_seed(random_state) as `fit_binary` derives it
  K > 2 classes    K one-vs-rest columns per (candidate, fold); class k shuffles with sgd_seed(seeds[k]),
                   seeds = RandomState(random_state).randint(MAX_INT, size=K) (`_fit_multiclass`)

Only alpha varies within a launch; the other searchable parameters group the launches.  Scores come from the
device scoring kernels: confusion counts of the `decision > 0` rule (binary) or of the first arg-max of the K
decision values (multiclass), exact pair counts (roc_auc) and, for binary log_loss, the expit log loss.  On a
binary target the ranking scorers run on the rank kernel: average_precision on the decision values, and
roc_auc_ovr / roc_auc_ovo [_weighted] (the AUC of predict_proba[:, 1], ranked as the decision values rank) when
every candidate has loss="log_loss"."""
import copy
import warnings

import numpy as np

from ..engine import sgd_config, sgd_seed
from .base import _merged_params
from .family import _count_metric, _Family, _is_rank, _resolve
from .folds import _classes_and_ids

_MAX_INT = np.iinfo(np.int32).max
# parameters that group the launches (one value per launch); alpha varies per column
_SGD_LAUNCH = ("loss", "learning_rate", "eta0", "power_t", "max_iter", "tol", "fit_intercept", "n_iter_no_change",
               "shuffle", "random_state")
SGD_DIVERGED = 5        # sgd_fit_groups / sgd_fit_batch status: a column's weights or intercept became non-finite


def _launch_key(p):
    rs = p["random_state"]
    rs_key = ("int", int(rs)) if isinstance(rs, (int, np.integer)) else ("obj", id(rs))
    return (p["loss"], p["learning_rate"], float(p["eta0"]), float(p["power_t"]), int(p["max_iter"]),
            None if p["tol"] is None else float(p["tol"]), bool(p["fit_intercept"]), int(p["n_iter_no_change"]),
            bool(p["shuffle"]), rs_key)


def _copy_state(random_state):
    """What each (candidate, fold) fit of scikit-learn's search sees: a clone of the estimator, whose
    RandomState instance is a deep copy of the template's; None stays numpy's global state."""
    if isinstance(random_state, np.random.RandomState):
        return copy.deepcopy(random_state)
    return random_state


def sgd_class_seeds(random_state, n_classes):
    """Shuffle seeds of one SGDClassifier fit, one per binary problem: [sgd_seed(random_state)] on a binary
    target; for K > 2 classes `_fit_multiclass`'s seeds = RandomState(random_state).randint(MAX_INT, size=K),
    each then derived as its binary fit derives it (SK/linear_model/_stochastic_gradient.py:804-826)."""
    from sklearn.utils import check_random_state
    rs = _copy_state(random_state)
    if n_classes <= 2:
        return [sgd_seed(rs)]
    draws = check_random_state(rs).randint(_MAX_INT, size=n_classes)
    return [sgd_seed(int(s)) for s in draws]


def _warn_max_iter():
    from sklearn.exceptions import ConvergenceWarning
    warnings.warn("Maximum number of iteration reached before convergence. Consider increasing max_iter to improve "
                  "the fit.", ConvergenceWarning)


class _SGDFamily(_Family):
    """(candidate x fold) columns of SGDClassifier (hinge or log_loss, penalty l2)."""

    name = "sgd"
    searchable = frozenset({"alpha"} | set(_SGD_LAUNCH))

    def __init__(self, estimator, candidate_params, X, y, scorers, enc=None):
        self.estimator = estimator
        self._check_searchable(candidate_params)
        self.cands = _merged_params(estimator, candidate_params)
        for q in self.cands:
            sgd_config(q)
            if not float(q["alpha"]) > 0:
                raise NotImplementedError("SGDClassifier(alpha=%r) has no device path (alpha > 0)" % (q["alpha"],))
        self.classes_, self.y_class = _classes_and_ids(y, enc)
        K = len(self.classes_)
        if K < 2:
            raise ValueError("The number of classes has to be greater than one; got %d class" % K)
        self.n_classes = K
        self.binary = K == 2
        metrics = {}
        for name, scorer in scorers.items():
            m = _count_metric(scorer)
            ok = m is not None
            if ok and self.binary and (m[0] == "neg_log_loss" or m[0] in ("roc_auc_ovr", "roc_auc_ovo")):
                # predict_proba of log_loss is _predict_proba_lr's expit; hinge has none
                ok = all(q["loss"] == "log_loss" for q in self.cands)
            elif ok and not self.binary:
                # scikit-learn rejects binary averaging and roc_auc on a multiclass target; SGD's multiclass
                # probabilities are one-vs-rest normalised, not the softmax the device forms, and its
                # average_precision stays with them
                ok = m[1] != "binary" and m[0] not in ("roc_auc", "neg_log_loss") and not _is_rank(m)
            if not ok:
                raise NotImplementedError(
                    "scorer %r has no device path for SGDClassifier (supported: accuracy, balanced_accuracy, "
                    "precision / recall / f1 with average binary (binary target), micro, macro or weighted, "
                    "roc_auc and average_precision (binary target), neg_log_loss, roc_auc_ovr, "
                    "roc_auc_ovr_weighted, roc_auc_ovo and roc_auc_ovo_weighted (binary target, "
                    "loss='log_loss'))" % (scorer,))
            metrics[name] = m
        if self.binary:
            self._set_binary_metrics(metrics)
        else:
            self.metrics = metrics

    # -- fits ---------------------------------------------------------------------------------------------
    def _fit(self, eng, p, alphas, folds):
        """One launch: SGD fits with the shared parameters `p`, alpha alphas[i] on the training rows of fold
        folds[i] (-1: all rows).  Returns (engine result, K') with K' engine columns per fit (class-major
        within a fit: column i * K' + k is class k of fit i)."""
        Kc = 1 if self.binary else self.n_classes
        group_of, rows, seeds = {}, [], []
        seed_of_fold = {}
        col_group = np.empty(len(alphas) * Kc, dtype=np.int32)
        for i, f in enumerate(folds):
            f = int(f)
            if f not in seed_of_fold:       # every (candidate, fold) fit of scikit-learn draws from its own clone
                seed_of_fold[f] = sgd_class_seeds(p["random_state"], self.n_classes)
            for k in range(Kc):
                key = (f, k)
                if key not in group_of:
                    group_of[key] = len(rows)
                    rows.append(self._train(f))
                    seeds.append(seed_of_fold[f][k])
                col_group[i * Kc + k] = group_of[key]
        col_pos = np.tile(np.arange(Kc, dtype=np.int32) if Kc > 1 else np.array([1], np.int32), len(alphas))
        col_alpha = np.repeat(np.asarray(alphas, dtype=np.float64), Kc)
        res = eng.sgd_fit_groups(p, col_pos, col_group, col_alpha, rows, np.array(seeds, dtype=np.uint32))
        return res, Kc

    _launch_key = staticmethod(_launch_key)

    def _launch(self, eng, cands, folds):
        """One launch through `_fit`: float32 [B, d + 1] (binary) or [B, K, d + 1] coefficients, intercept last,
        for the scoring kernels; a fit's epochs are the most of its class columns, and its status is
        SGD_DIVERGED when a class column diverged (scikit-learn's _plain_sgd raises there), else the least of
        theirs."""
        res, Kc = self._fit(eng, cands[0], [p["alpha"] for p in cands], folds)
        coef = np.concatenate([res["coef32"], res["intercept"].astype(np.float32)[:, None]], axis=1)
        coef = coef if Kc == 1 else coef.reshape(-1, Kc, coef.shape[1])
        status = res["status"].reshape(len(cands), Kc)
        n_iter = res["n_iter"].reshape(len(cands), Kc).max(axis=1)
        bad = np.any(status == SGD_DIVERGED, axis=1)
        return coef, n_iter, np.where(bad, SGD_DIVERGED, status.min(axis=1)), bad, bad

    def score_columns(self, eng, coef, codes):
        if not self.binary:
            return self._multiclass_scores(eng, coef, codes)
        # binary SGDClassifier's predict_proba is expit of a float64 decision (float64 intercept_): strictly
        # increasing in z until float64 saturates (|z| > 36), so it ranks the rows as the decision values do
        return self._binary_scores(eng, coef, codes, binary_proba="decision")

    def run_columns(self, eng, cols, n_splits, return_train_score):
        """The base loop, and scikit-learn's ConvergenceWarning once when a fit that did not diverge ran
        max_iter epochs with tol set."""
        out = super().run_columns(eng, cols, n_splits, return_train_score)
        cand = np.asarray(cols, dtype=np.int64) // n_splits
        live = out["status"] != SGD_DIVERGED
        if any(self.cands[c]["tol"] is not None and n == int(self.cands[c]["max_iter"])
               for c, n in zip(cand[live], out["n_iter"][live])):
            _warn_max_iter()
        return out

    # -- refit --------------------------------------------------------------------------------------------
    def refit(self, eng, params, X_dtype, n_features):
        p = _resolve(self.estimator, params).get_params(deep=False)
        res, Kc = self._fit(eng, p, [p["alpha"]], [-1])
        status = res["status"]
        if np.any(status == SGD_DIVERGED):
            raise ValueError("Floating-point under-/overflow occurred at epoch #%d. Scaling input data with "
                             "StandardScaler or MinMaxScaler might help."
                             % int(res["n_iter"][np.flatnonzero(status == SGD_DIVERGED)[0]]))
        n_iter = int(res["n_iter"].max())
        if p["tol"] is not None and n_iter == int(p["max_iter"]):
            _warn_max_iter()
        return self.make_estimator(params, res["coef32"], res["intercept"], n_iter, X_dtype, n_features)

    def make_estimator(self, params, coef32, intercept, n_iter, X_dtype, n_features):
        """A genuine fitted SGDClassifier with the attributes BaseSGDClassifier._fit_binary / _fit_multiclass
        set (SK/linear_model/_stochastic_gradient.py:760-850): coef_ (1 or K, d) in X's dtype, intercept_
        float64 (binary) or in X's dtype (K > 2), n_iter_ = the largest of the binary fits' epochs and
        t_ = 1 + n_iter_ * n."""
        est = _resolve(self.estimator, params)
        dt = np.float64 if X_dtype == np.float64 else np.float32
        est.coef_ = np.asarray(coef32)[:, :n_features].astype(dt)
        est.intercept_ = np.asarray(intercept, dtype=np.float64).astype(np.float64 if self.binary else dt)
        est.classes_ = self.classes_
        est.n_iter_ = int(n_iter)
        est.t_ = 1.0 + float(n_iter) * len(self.y_class)
        est.n_features_in_ = n_features
        est._loss_function_ = est._get_loss_function(est.loss)
        est._expanded_class_weight = np.ones(self.n_classes, dtype=np.float64)
        return est
