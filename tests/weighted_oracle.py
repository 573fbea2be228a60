"""numpy restatement of LogisticRegression(lbfgs, class_weight=...).fit -- TEST INFRASTRUCTURE ONLY.

The weighted counterpart of oracle/logreg_oracle.py.  Citations are to site-packages/sklearn (``SK/``):
  * per-row weights   SK/linear_model/_logistic.py:409-436 (compute_class_weight on the fit's own labels,
                      cast to X's dtype, times a float32 vector of ones)
  * sw_sum            SK/linear_model/_logistic.py:474 (float of the float32 sum), l2 = 1 / (C sw_sum) :580
  * objective         SK/linear_model/_linear_loss.py:291-379 with sample_weight: sum(loss_i) / sw_sum in
                      float32, pointwise gradients divided by the float32 sw_sum
  * pointwise terms   SK/_loss/_loss.pyx.tp:1083-1084 (binary: weight times the double results, stored as
                      float32), :1348-1350 (multinomial: float32 products)
tests/test_class_weight_host.py checks that these fits are bit-identical to scikit-learn's."""
import numpy as np
from scipy import optimize
from sklearn.utils.class_weight import compute_class_weight

from oracle import logreg_oracle as lo


def row_weights(class_weight, y, dtype=np.float32):
    """The per-row sample weights LogisticRegression.fit forms from `class_weight` on the labels `y` of
    its training rows (classes = np.unique(y)), and sw_sum."""
    sw = np.ones(len(y), dtype=dtype)
    if class_weight is not None:
        classes = np.unique(y)
        cw = compute_class_weight(class_weight, classes=classes, y=y)
        sw *= np.asarray(cw[np.searchsorted(classes, y)], dtype=dtype)
    return sw, float(np.sum(sw))


def loss_gradient(coef, X, y, sw, l2_reg_strength, fit_intercept=True):
    """LinearModelLoss.loss_gradient, binary, with sample weights."""
    n, d = X.shape
    if fit_intercept:
        weights, intercept = coef[:-1], coef[-1]
    else:
        weights, intercept = coef, 0.0
    raw = X @ np.asarray(weights, dtype=X.dtype) + np.asarray(intercept, dtype=X.dtype)
    loss64, grad64 = lo.loss_grad_pointwise(y, raw.astype(np.float64))
    sw64 = sw.astype(np.float64)
    loss_i = (sw64 * loss64).astype(raw.dtype)
    g_i = (sw64 * grad64).astype(raw.dtype)
    sw_sum = np.sum(sw)
    loss = float(np.sum(loss_i) / sw_sum)
    loss += float(0.5 * l2_reg_strength * (weights @ weights))
    g_i /= sw_sum
    grad = np.empty_like(coef, dtype=weights.dtype)
    grad[:d] = X.T @ g_i + l2_reg_strength * weights
    if fit_intercept:
        grad[-1] = np.sum(g_i)
    return loss, grad


def fit_binary_lbfgs(X, y01, sw, C=1.0, tol=1e-4, max_iter=100, fit_intercept=True):
    """Weighted _logistic_regression_path, solver='lbfgs', binary.  Returns (coef, intercept, n_iter)."""
    n, d = X.shape
    w0 = np.zeros(d + int(fit_intercept), dtype=X.dtype)
    l2 = 1.0 / (C * float(np.sum(sw)))
    res = optimize.minimize(lambda w: loss_gradient(w, X, y01, sw, l2, fit_intercept), w0, method="L-BFGS-B",
                            jac=True, options={"maxiter": max_iter, "maxls": 50, "gtol": tol,
                                               "ftol": 64 * np.finfo(float).eps})
    w = np.asarray(res.x, dtype=X.dtype)
    if fit_intercept:
        return w[:d], w[-1], min(res.nit, max_iter)
    return w, X.dtype.type(0), min(res.nit, max_iter)


def multinomial_loss_gradient(coef, X, y, sw, l2_reg_strength, n_classes, fit_intercept=True):
    """LinearModelLoss.loss_gradient, multiclass, with sample weights."""
    n, d = X.shape
    W = coef.reshape((n_classes, -1), order="F")
    if fit_intercept:
        intercept, weights = W[:, -1], W[:, :-1]
    else:
        intercept, weights = 0.0, W
    raw = X @ np.asarray(weights, dtype=X.dtype).T + np.asarray(intercept, dtype=X.dtype)
    loss_i, g_i = lo.multinomial_loss_grad_pointwise(y, raw)
    g_i = (g_i * sw[:, None]).astype(raw.dtype)
    loss_i = (loss_i * sw).astype(raw.dtype)
    sw_sum = np.sum(sw)
    loss = float(np.sum(loss_i) / sw_sum)
    loss += float(0.5 * l2_reg_strength * np.dot(weights.ravel(order="K"), weights.ravel(order="K")))
    g_i /= sw_sum
    grad = np.empty((n_classes, d + int(fit_intercept)), dtype=weights.dtype, order="F")
    grad[:, :d] = g_i.T @ X + l2_reg_strength * weights
    if fit_intercept:
        grad[:, -1] = np.sum(g_i, axis=0)
    return loss, grad.ravel(order="F")


def fit_multinomial_lbfgs(X, y_cls, sw, n_classes, C=1.0, tol=1e-4, max_iter=100, fit_intercept=True):
    """Weighted _logistic_regression_path, solver='lbfgs', n_classes > 2."""
    n, d = X.shape
    w0 = np.zeros((n_classes, d + int(fit_intercept)), dtype=X.dtype, order="F").ravel(order="F")
    y = np.asarray(y_cls, dtype=X.dtype)
    l2 = 1.0 / (C * float(np.sum(sw)))
    res = optimize.minimize(lambda w: multinomial_loss_gradient(w, X, y, sw, l2, n_classes, fit_intercept),
                            w0, method="L-BFGS-B", jac=True,
                            options={"maxiter": max_iter, "maxls": 50, "gtol": tol,
                                     "ftol": 64 * np.finfo(float).eps})
    W = np.asarray(np.reshape(res.x, (n_classes, -1), order="F"), dtype=X.dtype)
    n_iter = min(res.nit, max_iter)
    if fit_intercept:
        return W[:, :d], W[:, d], n_iter
    return W, np.zeros(n_classes, dtype=X.dtype), n_iter
