"""Accumulation scheme of csrc/ridge.cu, restated in numpy (no GPU): the fp32 chunk sums of the Gram and
cross products, float64 across chunks and folds, float64 centring and the fp32 Cholesky solve reach a
normwise backward error far below tests/test_ridge_gpu.py's bound (1e-6) at every target offset, and they do
so only because y is shifted by its global mean before the fp32 products: the same scheme on the raw
targets violates the bound once |mean y| is a few thousand standard deviations.
"""
import numpy as np
import pytest

from skdist_b200.datasets import make_g1_regression
from tests.ridge_reference import ETA_BOUND, RidgeRef, cholesky_solve32, emulate_statistics, eta

ALPHAS = np.array([1e-3, 1.0, 1e3])


def _data(c):
    X, y = make_g1_regression(12000, 70, seed=21)
    y = (y.astype(np.float64) + c * y.std()).astype(np.float32)
    fold = np.repeat(np.arange(5), 2400)             # two chunks per fold (2048 + 352 rows)
    return X, y, fold


def _worst_eta(X, y, fold, shift_y, fit_intercept=True, h=2):
    ref = RidgeRef(X, y, fold, 5, fit_intercept)
    A, b, _, _ = ref.stats(h)
    A32, b32, _, _ = emulate_statistics(X, y, fold, 5, h, fit_intercept, shift_y=shift_y)
    W = np.array([cholesky_solve32(A32, b32, a)[0] for a in ALPHAS])
    return eta(A, b, ALPHAS, W).max()


@pytest.mark.parametrize("c", [0.0, 1e2, 1e4, 1e6])
def test_shifted_targets_meet_the_backward_error_bound(c):
    X, y, fold = _data(c)
    e = _worst_eta(X, y, fold, shift_y=True)
    assert e <= ETA_BOUND / 5, e


def test_uncentred_targets_violate_the_bound():
    """What xty_kernel computed before the target shift: sum (x - mu) y over fp32 chunks, cancelled in float64."""
    X, y, fold = _data(1e4)
    e = _worst_eta(X, y, fold, shift_y=False)
    assert e > ETA_BOUND, e
    X, y, fold = _data(0.0)
    assert _worst_eta(X, y, fold, shift_y=False) <= ETA_BOUND / 5       # harmless on centred targets


def test_no_intercept_shifts_nothing():
    """Without an intercept the statistics are the raw products: on centred data the scheme is as accurate."""
    X, y, fold = _data(0.0)
    X = (X - X.mean(0)).astype(np.float32)
    y = (y - y.mean()).astype(np.float32)
    assert _worst_eta(X, y, fold, shift_y=True, fit_intercept=False) <= ETA_BOUND / 5


def test_emulated_statistics_match_float64():
    """The restatement itself: its fp32 statistics agree with the float64 ones to fp32 accumulation accuracy,
    and its intercept pieces (xbar, ybar) are the training means."""
    X, y, fold = _data(1e2)
    ref = RidgeRef(X, y, fold, 5)
    A, b, xbar, ybar = ref.stats(1)
    A32, b32, xb32, yb = emulate_statistics(X, y, fold, 5, 1)
    assert np.abs(A32 - A).max() <= 1e-5 * np.abs(A).max()
    assert np.abs(b32 - b).max() <= 1e-5 * np.abs(b).max()
    tr = fold != 1
    np.testing.assert_allclose(xb32, X[tr].astype(np.float64).mean(0), rtol=0, atol=1e-6)
    assert abs(yb - y[tr].astype(np.float64).mean()) <= 1e-9 * abs(ybar)
