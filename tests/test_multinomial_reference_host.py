"""Host rehearsal of tests/test_multinomial_eval_gpu.py: its float64 reference and error bound
(tests/multinomial_reference.py) against the oracle and scikit-learn, its closed form at W = 0 against the
reference, and a numpy fp32 restatement of the kernel's order of operations inside the bound at every float-tier
shape -- so the constants are checked before any device runs them."""
import numpy as np
import pytest
from sklearn._loss.loss import HalfMultinomialLoss
from sklearn.linear_model._linear_loss import LinearModelLoss

from oracle.logreg_oracle import multinomial_loss_gradient
from tests import multinomial_reference as mr
from tests.test_multinomial_eval_gpu import (N_FLOAT_MAX, OPTIONS, SHAPE_IDS, SHAPES, _columns, _float_data,
                                             _float_points, _folds, _int_data)


def _case(seed, n, d, K, B, fi=True):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((n, d)).astype(np.float32)
    y = rng.integers(0, K, n).astype(np.int32)
    W = (rng.standard_normal((B, K, d + 1)) * 0.3).astype(np.float32).astype(np.float64)   # fp32-representable
    if not fi:
        W[:, :, d] = 0.0
    return rng, X, y, W


@pytest.mark.parametrize("fi", [True, False], ids=["intercept", "no_intercept"])
def test_reference_matches_oracle_unweighted(fi):
    n, d, K, B = 300, 7, 4, 3
    _, X, y, W = _case(1, n, d, K, B, fi)
    C = np.array([0.1, 1.0, 10.0])
    ref = mr.loss_grad(X, y, np.ones((n, B), bool), W, C, fit_intercept=fi, bounds=False)
    for b in range(B):
        Wb = W[b] if fi else W[b, :, :d]
        f, g = multinomial_loss_gradient(Wb.ravel(order="F"), X.astype(np.float64), y.astype(np.float64),
                                         1.0 / (C[b] * n), K, fi)
        g = g.reshape((K, -1), order="F")
        assert abs(f - ref["f"][b]) <= 1e-12 * abs(f)
        np.testing.assert_allclose(ref["g"][b, :, :g.shape[1]], g, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("fi", [True, False], ids=["intercept", "no_intercept"])
def test_reference_matches_sklearn_weighted_with_folds(fi):
    n, d, K, B = 400, 6, 5, 4
    rng, X, y, W = _case(2, n, d, K, B, fi)
    fold = (np.arange(n) * 3 // n).astype(np.int8)
    cf = np.array([0, 1, 2, -1], np.int32)
    M = mr.row_mask(n, fold, cf)
    cw = rng.uniform(0.3, 3.0, (B, K)).astype(np.float32)
    C = np.array([0.01, 0.5, 3.0, 100.0])
    ref = mr.loss_grad(X, y, M, W, C, cw, fit_intercept=fi, bounds=False)
    lml = LinearModelLoss(base_loss=HalfMultinomialLoss(n_classes=K), fit_intercept=fi)
    for b in range(B):
        sw = M[:, b] * cw[b, y].astype(np.float64)
        coef = W[b] if fi else W[b, :, :d]
        f, g = lml.loss_gradient(coef.copy(), X.astype(np.float64), y.astype(np.float64), sample_weight=sw,
                                 l2_reg_strength=1.0 / (C[b] * sw.sum()))
        assert abs(f - ref["f"][b]) <= 1e-12 * abs(f)
        np.testing.assert_allclose(ref["g"][b, :, :g.shape[1]], g, rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("K", [3, 4, 128])
def test_closed_form_at_zero_matches_reference(K):
    n, d, B = 700, 9, 3
    rng = np.random.default_rng(3)
    X, _ = _int_data(rng, n, d)
    y = rng.integers(0, K, n).astype(np.int32)
    fold = (np.arange(n) * 3 // n).astype(np.int8)
    cf = np.array([0, 2, -1], np.int32)
    M = mr.row_mask(n, fold, cf)
    cw = np.exp2(rng.integers(-1, 2, (B, K))).astype(np.float32)
    for w in (None, cw):
        want, ntr = mr.grad_at_zero(X, y, M, K, w)
        ref = mr.loss_grad(X, y, M, np.zeros((B, K, d + 1)), np.ones(B), w, bounds=False)
        np.testing.assert_allclose(ref["g"], want, rtol=1e-12, atol=1e-300)
        np.testing.assert_allclose(ref["f"], np.log(K), rtol=1e-14)
        np.testing.assert_allclose(ref["ntr"], ntr, rtol=0)


def test_chunking_matches_the_kernel():
    """multi_chunks restated: the chunk regimes the GPU shape matrix names."""
    assert mr.multi_chunks(50) == (1, 64)
    assert mr.multi_chunks(4096) == (64, 64)
    assert mr.multi_chunks(4097) == (33, 128)
    assert mr.multi_chunks(5000) == (40, 128)
    assert mr.multi_chunks(70001) == (61, 1152)
    nz = mr.multi_chunks(200_000)[0]
    assert mr.candidates_per_pass(200_000, 16, 128, nz) == 58


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_fp32_restatement_inside_bound(shape):
    """The kernel's order of operations in numpy fp32 lands inside the bound at every float-tier shape, and the
    bound still sees one training row."""
    K, d, n, fk, B = shape
    n = min(n, N_FLOAT_MAX)
    use_cw, use_mask, fi = OPTIONS[shape]
    rng = np.random.default_rng(K * 1000 + d + 2)
    X, scale = _float_data(rng, n, d)
    y = rng.integers(0, K, n).astype(np.int32)
    fold, nf = _folds(fk, n, y, K + d)
    cf = _columns(nf, B)
    M = mr.row_mask(n, fold, cf)
    cw = rng.uniform(0.2, 3.0, (B, K)).astype(np.float32) if use_cw else None
    W = _float_points(rng, B, K, d, scale, fi)
    C = np.exp(rng.uniform(np.log(1e-2), np.log(1e2), B))
    ref = mr.loss_grad(X, y, M, W, C, cw, None, fi)
    f, g = mr.emulate(X, y, M, W, C, cw, fi)
    rf, rg = mr.check_float(X, ref, f, g, "fp32 restatement %s" % "-".join(map(str, shape)), fi)
    assert rg > 0.0 or rf > 0.0      # the restatement does round
