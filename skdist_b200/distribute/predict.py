"""Batched model inference on H100 GPUs.

Counterpart of /root/reference/skdist/distribute/predict.py.  The reference wraps
``model.predict`` / ``model.predict_proba`` in a Spark pandas UDF that is called once per Arrow
batch (`get_prediction_udf`, ref predict.py:74-179; `_get_vals` transposes the column batch,
:59-71).  Here the same callable streams its batch through the device: the rows are staged
through pinned bounce buffers and one kernel pass evaluates

  linear models     out = X . coef^T + intercept         (csrc/predict.cu predict_kernel)
  forests           soft vote over the `Tree` arrays       (csrc/predict.cu forest_predict_kernel)

and the cheap label / probability post-processing follows scikit-learn's own formulas on the
host.  `get_prediction_udf` returns the vectorised function the reference hands to
``F.pandas_udf`` (INTEGRATION.md shows the one-line Spark wrapper); `batch_predict` is the same
thing on a 2-d array.  Models without a device path raise NotImplementedError (no CPU fallback).
"""
import numpy as np
from scipy.special import expit
from sklearn.utils.extmath import softmax

from ..engine import get_engine

__all__ = ["get_prediction_udf", "batch_predict"]


# ----------------------------------------------------------------------------------------
# model -> device representation
# ----------------------------------------------------------------------------------------
def _linear_pack(coef, intercept):
    """[B, d+1] float32 rows (weights, intercept) from sklearn's coef_ / intercept_."""
    coef = np.atleast_2d(np.asarray(coef, dtype=np.float64))
    b = np.broadcast_to(np.asarray(intercept, dtype=np.float64).reshape(-1), (coef.shape[0],))
    return np.concatenate([coef, b[:, None]], axis=1).astype(np.float32)


class _LinearPlan:
    def __init__(self, model, kind, packed, post):
        self.model, self.kind, self.packed, self.post = model, kind, packed, post

    def decision(self, X):
        return get_engine().predict_linear(X, self.packed)


def _forest_arrays(estimators):
    """Concatenate the `Tree` arrays of fitted sklearn trees (SK/tree/_tree.pyx:688-748)."""
    off = np.zeros(len(estimators) + 1, dtype=np.int64)
    left, right, feat, thr, val = [], [], [], [], []
    for i, e in enumerate(estimators):
        t = e.tree_
        if t.value.shape[1] != 1:
            raise NotImplementedError("multi-output forests have no device inference path")
        off[i + 1] = off[i] + t.node_count
        left.append(t.children_left.astype(np.int32))
        right.append(t.children_right.astype(np.int32))
        feat.append(np.where(t.children_left == -1, 0, t.feature).astype(np.int32))
        thr.append(t.threshold.astype(np.float64))
        val.append(t.value[:, 0, :].astype(np.float64))
    return (off, np.concatenate(left), np.concatenate(right), np.concatenate(feat), np.concatenate(thr),
            np.ascontiguousarray(np.concatenate(val, axis=0)))


class _ForestPlan:
    def __init__(self, model, classifier):
        self.model, self.classifier = model, classifier
        self.arrays = _forest_arrays(model.estimators_)

    def values(self, X):
        return get_engine().forest_predict(X, *self.arrays)


def _plan(model):
    from sklearn.ensemble import (ExtraTreesClassifier, ExtraTreesRegressor, RandomForestClassifier,
                                  RandomForestRegressor)
    from sklearn.linear_model import (LinearRegression, LogisticRegression, Ridge, SGDClassifier,
                                      SGDRegressor)
    from sklearn.multiclass import OneVsRestClassifier
    if isinstance(model, (RandomForestClassifier, ExtraTreesClassifier)):
        return _ForestPlan(model, True)
    if isinstance(model, (RandomForestRegressor, ExtraTreesRegressor)):
        return _ForestPlan(model, False)
    if isinstance(model, OneVsRestClassifier):
        ests = model.estimators_
        if not all(hasattr(e, "coef_") and np.atleast_2d(e.coef_).shape[0] == 1 for e in ests):
            raise NotImplementedError("OneVsRest inference on the device needs linear binary estimators")
        packed = np.concatenate([_linear_pack(e.coef_, e.intercept_) for e in ests], axis=0)
        return _LinearPlan(model, "ovr", packed, None)
    if isinstance(model, (LogisticRegression, SGDClassifier)):
        return _LinearPlan(model, "classifier", _linear_pack(model.coef_, model.intercept_), None)
    if isinstance(model, (Ridge, LinearRegression, SGDRegressor)):
        return _LinearPlan(model, "regressor", _linear_pack(model.coef_, model.intercept_), None)
    raise NotImplementedError(
        "%s has no device inference path; supported: LogisticRegression, SGDClassifier, Ridge, "
        "LinearRegression, SGDRegressor, OneVsRest of linear models, RandomForest / ExtraTrees "
        "classifiers and regressors.  (No CPU fallback by design.)" % type(model).__name__)


# ----------------------------------------------------------------------------------------
# post-processing: scikit-learn's own formulas on the decision values
# ----------------------------------------------------------------------------------------
def _classifier_predict(model, dec):
    # LinearClassifierMixin.predict (SK/linear_model/_base.py:351-374)
    if dec.shape[1] == 1:
        idx = (dec[:, 0] > 0).astype(np.intp)
    else:
        idx = dec.argmax(axis=1)
    return np.asarray(model.classes_)[idx]


def _classifier_proba(model, dec):
    from sklearn.linear_model import LogisticRegression
    dec = dec.astype(np.float64)
    if isinstance(model, LogisticRegression):
        if dec.shape[1] == 1:           # _predict_proba_lr binary (SK/linear_model/_base.py:376-397)
            p1 = expit(dec[:, 0])
            return np.column_stack([1.0 - p1, p1])
        return softmax(dec, copy=False)  # SK/linear_model/_logistic.py:1621-1625
    if getattr(model, "loss", None) == "log_loss":   # SGDClassifier._predict_proba (log loss branch)
        if dec.shape[1] == 1:
            p1 = expit(dec[:, 0])
            return np.column_stack([1.0 - p1, p1])
        prob = expit(dec)
        s = prob.sum(axis=1)
        zero = s == 0
        prob[zero] = 1.0
        s[zero] = prob.shape[1]
        return prob / s[:, None]
    raise NotImplementedError("predict_proba on the device needs LogisticRegression or SGDClassifier(loss='log_loss')")


def batch_predict(model, X, method="predict"):
    """`model.<method>(X)` for a 2-d float array X, evaluated on the device."""
    if method not in ("predict", "predict_proba"):
        raise ValueError("Unknown method: {0}".format(method))
    plan = model if isinstance(model, (_LinearPlan, _ForestPlan)) else _plan(model)
    model = plan.model
    X = np.asarray(X)
    if X.ndim != 2:
        raise ValueError("expected a 2-d feature array")
    if isinstance(plan, _ForestPlan):
        vals = plan.values(X)
        if not plan.classifier:
            if method != "predict":
                raise AttributeError("regressors have no predict_proba")
            return vals[:, 0]
        if method == "predict_proba":
            return vals
        return np.asarray(model.classes_).take(np.argmax(vals, axis=1), axis=0)   # SK/ensemble/_forest.py:904-906
    dec = plan.decision(X)
    if plan.kind == "regressor":
        if method != "predict":
            raise AttributeError("regressors have no predict_proba")
        return dec[:, 0].astype(np.float64 if np.asarray(model.coef_).dtype == np.float64 else np.float32) \
            if dec.shape[1] == 1 else dec
    if plan.kind == "ovr":
        if len(model.estimators_) == 1:     # binary problem: one column, positive = classes_[1]
            if method == "predict":
                return np.asarray(model.classes_)[(dec[:, 0] > 0).astype(np.intp)]
            p1 = expit(dec[:, 0].astype(np.float64))
            return np.column_stack([1.0 - p1, p1])
        if method == "predict":             # SK/multiclass.py:498-508 (== first arg max)
            return np.asarray(model.classes_)[dec.argmax(axis=1)]
        prob = expit(dec.astype(np.float64))
        norm = getattr(model, "norm", None)
        if norm:                            # ref multiclass.py:337-362
            from sklearn.preprocessing import normalize
            return normalize(prob, norm=norm)
        if type(model).__name__ == "DistOneVsRestClassifier":
            return prob
        return prob / prob.sum(axis=1)[:, None]   # SK/multiclass.py predict_proba, multiclass branch
    if method == "predict":
        return _classifier_predict(model, dec)
    return _classifier_proba(model, dec)


def _get_vals(*cols, feature_type="numpy", names=None):
    """Feature block of one column batch (ref predict.py:59-71)."""
    if feature_type == "numpy":
        return np.transpose([np.asarray(getattr(a, "values", a)) for a in cols])
    if feature_type in ("pandas", "text"):
        raise NotImplementedError(
            "feature_type=%r feeds a text / mixed-type pipeline, which has no device path" % feature_type)
    raise ValueError("Unknown feature_type: {0}".format(feature_type))


def get_prediction_udf(model, method="predict", feature_type="numpy", names=None):
    """Vectorised prediction function over feature columns (ref predict.py:74-179).

    Returns ``f(*cols) -> pandas.Series`` — the function the reference passes to
    ``pyspark.sql.functions.pandas_udf`` — with the model evaluated on the device.  ``method`` is
    'predict' or 'predict_proba'; 'predict_proba' rows are lists of floats as in the reference
    (ArrayType(DoubleType())).
    """
    import pandas as pd
    if method not in ("predict", "predict_proba"):
        raise ValueError("Unknown method: {0}".format(method))
    if feature_type not in ("numpy", "pandas", "text"):
        raise ValueError("Unknown feature_type: {0}".format(feature_type))
    plan = _plan(model)

    if method == "predict":
        def predict_func(*cols):
            vals = _get_vals(*cols, feature_type=feature_type, names=names)
            return pd.Series(batch_predict(plan, vals, "predict"))
    else:
        def predict_func(*cols):
            vals = _get_vals(*cols, feature_type=feature_type, names=names)
            return pd.Series(list(batch_predict(plan, vals, "predict_proba")))
    predict_func.method = method
    predict_func.model = model
    return predict_func
