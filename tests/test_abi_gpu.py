"""Argument handling of the C-ABI entry points on the device.

  * one-shot staged inputs (column masks, row bit matrices, class weights) are taken off the context by
    the call that reads them even when that call fails its argument checks, so they cannot make a later,
    correct call with another batch size fail;
  * skd_logreg_loss_grad and skd_logreg_multinomial_loss_grad reject C <= 0 and an empty training set, as the
    fits do, and the multinomial one staged class weights or masks that do not match the batch;
  * every entry that takes n_classes rejects staged class ids outside 0..n_classes-1, naming them: such a row
    would count in n_train while the kernels leave it out of the objective and the scores;
  * every scoring entry rejects code -1 and a code that names an unstaged fold, with the same message.
"""
import numpy as np
import pytest

from skdist_b200._lib import SkdError

pytestmark = pytest.mark.gpu

N, D = 512, 12


@pytest.fixture
def eng():
    from skdist_b200.engine import Engine
    rng = np.random.default_rng(3)
    e = Engine(0)
    e.stage_x(rng.standard_normal((N, D)).astype(np.float32))
    e.stage_labels((np.arange(N) % 3).astype(np.int32))
    e.stage_targets(rng.standard_normal(N).astype(np.float32))
    e.stage_folds((np.arange(N) % 2).astype(np.int8), 2)
    yield e
    e.close()


def _fails_bad_arguments(eng):
    """skd_logreg_fit_batch with B = 0: rejected by its first argument check."""
    rc = eng._lib.skd_logreg_fit_batch(eng._h, 0, None, None, None, None, 1, 1e-4, 100, None, None, None, None,
                                       None, None)
    assert rc != 0
    assert "bad arguments" in eng._lib.skd_last_error(eng._h).decode()


def test_failed_binary_fit_leaves_nothing_staged(eng):
    B = 3
    eng.stage_column_masks(np.ones((B, D), np.uint8))
    eng.stage_row_bits(labels=np.ones((B, N), np.uint8), train=np.ones((B, N), np.uint8))
    eng.stage_class_weights(np.ones((B, 2), np.float32), np.full(B, float(N)))
    _fails_bad_arguments(eng)
    C = np.ones(2)
    res = eng.logreg_fit_batch(C, np.zeros(2, np.int32), np.ones(2, np.int32), max_iter=5)
    assert res["coef"].shape == (2, D + 1)


def test_failed_multinomial_fit_leaves_nothing_staged(eng):
    B, K = 3, 3
    eng.stage_column_masks(np.ones((B, D), np.uint8))
    eng.stage_class_weights(np.ones((B, K), np.float32), np.full(B, N / 2.0))
    with pytest.raises(SkdError, match="max_iter"):
        eng.logreg_multinomial_fit_batch(np.ones(B), np.zeros(B, np.int32), K, max_iter=0)
    res = eng.logreg_multinomial_fit_batch(np.ones(2), np.zeros(2, np.int32), K, max_iter=5)
    assert res["coef"].shape == (2, K, D + 1)


def test_loss_grad_checks_c_and_training_set(eng):
    w = np.zeros((1, D + 1))
    for C in (0.0, -1.0):
        with pytest.raises(SkdError, match="skd_logreg_loss_grad: C must be positive"):
            eng.logreg_loss_grad(w, np.array([C]), np.zeros(1, np.int32), np.ones(1, np.int32))
    eng.stage_folds(np.zeros(N, np.int8), 1)     # fold 0 holds every row: nothing is left to train on
    with pytest.raises(SkdError, match="skd_logreg_loss_grad: empty training set"):
        eng.logreg_loss_grad(w, np.ones(1), np.zeros(1, np.int32), np.ones(1, np.int32))


SCORERS = {
    "skd_linear_score_batch": lambda e, codes: e.linear_score_batch(np.zeros((1, D + 1)), codes, np.ones(1, np.int32)),
    "skd_linear_r2_batch": lambda e, codes: e.linear_r2_batch(np.zeros((1, D + 1)), codes),
    "skd_linear_auc_batch": lambda e, codes: e.linear_auc_batch(np.zeros((1, D + 1)), codes, np.ones(1, np.int32)),
    "skd_linear_logloss_batch": lambda e, codes: e.linear_logloss_batch(np.zeros((1, D + 1)), codes, np.ones(1, np.int32)),
    "skd_multinomial_score_batch": lambda e, codes: e.multinomial_score_batch(np.zeros((1, 3, D + 1)), codes),
    "skd_multinomial_confusion_batch": lambda e, codes: e.multinomial_confusion_batch(np.zeros((1, 3, D + 1)), codes),
}


@pytest.mark.parametrize("entry", sorted(SCORERS))
def test_scoring_entries_reject_bad_codes(eng, entry):
    score = SCORERS[entry]
    with pytest.raises(SkdError, match="^%s: col_fold -1 is not a scoring code$" % entry):
        score(eng, np.array([-1], np.int32))
    for code in (2, -3 - 2):          # fold 2 is not staged (two folds)
        with pytest.raises(SkdError, match="^%s: col_fold refers to an unstaged fold$" % entry):
            score(eng, np.array([code], np.int32))
    for code in (0, -2, -3 - 1):      # valid codes score
        score(eng, np.array([code], np.int32))


MULTI_ENTRIES = {
    "skd_logreg_multinomial_fit_batch":
        lambda e, K: e.logreg_multinomial_fit_batch(np.ones(1), np.zeros(1, np.int32), K, max_iter=5),
    "skd_logreg_multinomial_loss_grad":
        lambda e, K: e.logreg_multinomial_loss_grad(np.zeros((1, K, D + 1)), np.ones(1), np.zeros(1, np.int32)),
    "skd_multinomial_score_batch": lambda e, K: e.multinomial_score_batch(np.zeros((1, K, D + 1)), np.zeros(1, np.int32)),
    "skd_multinomial_confusion_batch":
        lambda e, K: e.multinomial_confusion_batch(np.zeros((1, K, D + 1)), np.zeros(1, np.int32)),
    "skd_linear_logloss_batch": lambda e, K: e.linear_logloss_batch(np.zeros((1, K, D + 1)), np.zeros(1, np.int32)),
}


@pytest.mark.parametrize("entry", sorted(MULTI_ENTRIES))
def test_multinomial_entries_reject_class_ids_out_of_range(eng, entry):
    call = MULTI_ENTRIES[entry]
    K = 3
    call(eng, K)                                              # staged ids 0..2
    eng.stage_labels((np.arange(N) % (K + 1)).astype(np.int32))     # ids 0..K
    with pytest.raises(SkdError, match="^%s: staged class ids span 0..3, outside 0..n_classes-1 = 0..2$" % entry):
        call(eng, K)
    call(eng, K + 1)
    y = (np.arange(N) % K).astype(np.int32)
    y[7] = -1
    eng.stage_labels(y)
    with pytest.raises(SkdError, match="^%s: staged class ids span -1..2, outside" % entry):
        call(eng, K)


def test_multinomial_fit_takes_two_classes(eng):
    eng.stage_labels((np.arange(N) % 2).astype(np.int32))
    res = eng.logreg_multinomial_fit_batch(np.ones(1), np.full(1, -1, np.int32), 2, max_iter=5)
    assert res["coef"].shape == (1, 2, D + 1)


def test_multinomial_loss_grad_checks_arguments(eng):
    K = 3
    w = np.zeros((2, K, D + 1))
    cf = np.zeros(2, np.int32)
    who = "skd_logreg_multinomial_loss_grad"
    for C in (0.0, -1.0):
        with pytest.raises(SkdError, match="%s: C must be positive" % who):
            eng.logreg_multinomial_loss_grad(w, np.array([1.0, C]), cf)
    eng.stage_class_weights(np.ones((3, K), np.float32), np.full(3, N / 2.0))          # B = 3, not 2
    with pytest.raises(SkdError, match="%s: staged class weights do not match this batch" % who):
        eng.logreg_multinomial_loss_grad(w, np.ones(2), cf)
    eng.stage_class_weights(np.ones((2, K + 1), np.float32), np.full(2, N / 2.0))      # K + 1 classes
    with pytest.raises(SkdError, match="%s: staged class weights do not match this batch" % who):
        eng.logreg_multinomial_loss_grad(w, np.ones(2), cf)
    eng.stage_column_masks(np.ones((3, D), np.uint8))
    with pytest.raises(SkdError, match="%s: staged column masks do not match the batch" % who):
        eng.logreg_multinomial_loss_grad(w, np.ones(2), cf)
    eng.stage_folds(np.zeros(N, np.int8), 1)     # fold 0 holds every row: nothing is left to train on
    with pytest.raises(SkdError, match="%s: empty training set" % who):
        eng.logreg_multinomial_loss_grad(w, np.ones(2), cf)


def test_failed_multinomial_loss_grad_leaves_nothing_staged(eng):
    B, K = 3, 3
    eng.stage_column_masks(np.ones((B, D), np.uint8))
    eng.stage_class_weights(np.full((B, K), 2.0, np.float32), np.full(B, float(N)))
    with pytest.raises(SkdError, match="C must be positive"):
        eng.logreg_multinomial_loss_grad(np.zeros((B, K, D + 1)), np.zeros(B), np.zeros(B, np.int32))
    f, g = eng.logreg_multinomial_loss_grad(np.zeros((2, K, D + 1)), np.ones(2), np.zeros(2, np.int32))
    assert np.allclose(f, np.log(K), rtol=1e-6)     # unweighted: the staged weights of 2 are gone
