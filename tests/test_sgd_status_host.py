"""How the one-vs-rest and one-vs-one SGD paths report the device's per-column status (no GPU).

scikit-learn's SGDClassifier raises ValueError when a fit's weights or intercept become non-finite
(`_plain_sgd`, "Floating-point under-/overflow occurred at epoch #N ..."), and warns with a
ConvergenceWarning when a fit with a tolerance runs all max_iter epochs.  The device returns a status and
n_iter per column; a stub engine returns chosen ones here, and both classifiers must react as
scikit-learn's per-column fits would, in column order."""
import warnings

import numpy as np
import pytest
from sklearn.exceptions import ConvergenceWarning
from sklearn.linear_model import SGDClassifier

from skdist.distribute.multiclass import DistOneVsOneClassifier, DistOneVsRestClassifier
from skdist_b200 import engine

DONE, MAX_ITER, DIVERGED = 1, 3, 5          # sgd_fit_batch status: stopping rule met, max_iter reached, non-finite


class _StubEngine:
    """Answers every sgd_fit_batch call with the next (status, n_iter) of `outcomes`, indexed by column."""

    def __init__(self, outcomes):
        self.outcomes = list(outcomes)
        self.calls = 0

    def stage_x(self, X):
        self.d = np.asarray(X).shape[1]

    def stage_labels(self, y):
        pass

    def stage_folds(self, fold, n_folds):
        pass

    def sgd_fit_batch(self, est, col_pos):
        status, n_iter = self.outcomes[self.calls]
        self.calls += 1
        B = len(col_pos)
        status = np.broadcast_to(np.asarray(status, np.int32), (B,)).copy()
        n_iter = np.broadcast_to(np.asarray(n_iter, np.int32), (B,)).copy()
        return {"coef": np.zeros((B, self.d + 1)), "coef32": np.zeros((B, self.d), np.float32),
                "intercept": np.zeros(B), "n_iter": n_iter, "t": 1.0 + 10.0 * n_iter, "status": status,
                "gpu_seconds": 0.0}


@pytest.fixture
def stub(request):
    eng = _StubEngine(request.param)
    engine.set_engine_factory(lambda: eng)
    yield eng
    engine.set_engine_factory(None)


def _data(k, n=60, d=3):
    rng = np.random.default_rng(0)
    return rng.standard_normal((n, d)).astype(np.float32), np.arange(n) % k


def _fit(cls, k, **params):
    X, y = _data(k)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        cls(SGDClassifier(**params), None).fit(X, y)
    return [w for w in rec if issubclass(w.category, ConvergenceWarning)]


MSG = ("Floating-point under-/overflow occurred at epoch #%d. Scaling input data with StandardScaler or MinMaxScaler "
       "might help.")


@pytest.mark.parametrize("stub", [[([DONE, DIVERGED, DIVERGED, DONE], [4, 7, 2, 9])]], indirect=True)
def test_ovr_overflow_raises_with_the_first_column_epoch(stub):
    """Columns 1 and 2 diverge: scikit-learn fits column 1 first and stops there, so its epoch is reported."""
    with pytest.raises(ValueError) as e:
        _fit(DistOneVsRestClassifier, 4, max_iter=10)
    assert str(e.value) == MSG % 7


@pytest.mark.parametrize("stub", [[(DONE, 4), (DONE, 4), (DIVERGED, 3), (DIVERGED, 1), (DONE, 4), (DONE, 4)]],
                         indirect=True)
def test_ovo_overflow_raises_with_the_first_pair_epoch(stub):
    with pytest.raises(ValueError) as e:
        _fit(DistOneVsOneClassifier, 4, max_iter=10)
    assert str(e.value) == MSG % 3
    assert stub.calls == 6


@pytest.mark.parametrize("stub", [[([DONE, MAX_ITER, DONE], [4, 10, 6])]], indirect=True)
def test_ovr_max_iter_warns(stub):
    rec = _fit(DistOneVsRestClassifier, 3, max_iter=10)
    assert len(rec) == 1
    assert str(rec[0].message).startswith("Maximum number of iteration reached before convergence.")


@pytest.mark.parametrize("stub", [[(DONE, 4), (MAX_ITER, 10), (DONE, 5)]], indirect=True)
def test_ovo_max_iter_warns(stub):
    rec = _fit(DistOneVsOneClassifier, 3, max_iter=10)
    assert len(rec) == 1
    assert str(rec[0].message).startswith("Maximum number of iteration reached before convergence.")


@pytest.mark.parametrize("stub", [[([DONE, DONE, DONE], [10, 4, 6])]], indirect=True)
def test_ovr_stopping_at_the_last_epoch_still_warns(stub):
    """scikit-learn's test is n_iter_ == max_iter, so a fit whose stopping rule fires in the last epoch warns too."""
    assert len(_fit(DistOneVsRestClassifier, 3, max_iter=10)) == 1


@pytest.mark.parametrize("stub", [[([MAX_ITER, MAX_ITER, MAX_ITER], [10, 10, 10])]], indirect=True)
def test_ovr_max_iter_without_tol_is_silent(stub):
    assert _fit(DistOneVsRestClassifier, 3, max_iter=10, tol=None) == []


@pytest.mark.parametrize("stub", [[([DONE, DONE, DONE], [4, 9, 6])]], indirect=True)
def test_ovr_converged_is_silent(stub):
    assert _fit(DistOneVsRestClassifier, 3, max_iter=10) == []


@pytest.mark.parametrize("stub", [[([MAX_ITER, DIVERGED, DONE], [10, 2, 4])]], indirect=True)
def test_ovr_warning_of_earlier_column_comes_before_the_overflow(stub):
    """scikit-learn fits column 0 (warns) before column 1 (raises)."""
    X, y = _data(3)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        with pytest.raises(ValueError, match="epoch #2"):
            DistOneVsRestClassifier(SGDClassifier(max_iter=10), None).fit(X, y)
    assert [w.category for w in rec if issubclass(w.category, ConvergenceWarning)] == [ConvergenceWarning]
