"""FakeEngine plus the class-weight staging call -- TEST DOUBLE, CPU only.

Weighted fits run tests/weighted_oracle.py on the column's training rows (ascending order) with the
staged per-class weights; every weighted fit's staged arrays are recorded in `staged`."""
import numpy as np

from tests import weighted_oracle as wo
from tests.fake_engine import FakeEngine


class WeightedFakeEngine(FakeEngine):
    def __init__(self, device=0):
        super().__init__(device)
        self._cw = None
        self.staged = []        # (weights [B, K], sw_sum [B], col_fold [B]) of every weighted fit

    def stage_class_weights(self, w, sw_sum):
        self._cw = None if w is None else (np.asarray(w, np.float32), np.asarray(sw_sum, np.float64))

    def _take(self, B, K, col_fold):
        cw, self._cw = self._cw, None
        if cw is not None:
            assert cw[0].shape == (B, K) and cw[1].shape == (B,)
            self.staged.append((cw[0], cw[1], np.asarray(col_fold).copy()))
        return cw

    def logreg_fit_batch(self, C, col_fold, col_pos, fit_intercept=True, tol=1e-4, max_iter=100, col_neg=None):
        cw = self._take(len(C), 2, col_fold)
        if cw is None:
            return super().logreg_fit_batch(C, col_fold, col_pos, fit_intercept, tol, max_iter, col_neg)
        fmask, self._fmask = getattr(self, "_fmask", None), None
        ybits, mbits = getattr(self, "_ybits", None), getattr(self, "_mbits", None)
        self._ybits = self._mbits = None
        B = len(C)
        coef = np.zeros((B, self.d + 1), np.float32)
        n_iter = np.zeros(B, np.int32)
        for j in range(B):
            m = self._train_mask(int(col_fold[j]))
            if col_neg is not None and col_neg[j] >= 0:
                m = m & ((self.y == col_pos[j]) | (self.y == col_neg[j]))
            if mbits is not None:
                m = m & mbits[j]
            yb = (self.y[m] == col_pos[j]) if ybits is None else ybits[j][m]
            yb = yb.astype(np.intp)
            keep = np.arange(self.d) if fmask is None else np.flatnonzero(fmask[j])
            Xm = np.ascontiguousarray(self.X[m][:, keep])
            w, b, it = wo.fit_binary_lbfgs(Xm, yb.astype(np.float32), cw[0][j][yb], C=float(C[j]), tol=tol,
                                           max_iter=max_iter, fit_intercept=fit_intercept)
            coef[j, keep], coef[j, self.d], n_iter[j] = w, b, it
        return {"coef": coef, "n_iter": n_iter, "status": np.ones(B, np.int32), "loss": np.zeros(B),
                "n_evals": n_iter + 1, "gpu_seconds": 0.0}

    def logreg_multinomial_fit_batch(self, C, col_fold, n_classes, fit_intercept=True, tol=1e-4, max_iter=100):
        cw = self._take(len(C), n_classes, col_fold)
        if cw is None:
            return super().logreg_multinomial_fit_batch(C, col_fold, n_classes, fit_intercept, tol, max_iter)
        fmask, self._fmask = getattr(self, "_fmask", None), None
        B = len(C)
        coef = np.zeros((B, n_classes, self.d + 1), np.float32)
        n_iter = np.zeros(B, np.int32)
        for j in range(B):
            m = self._train_mask(int(col_fold[j]))
            keep = np.arange(self.d) if fmask is None else np.flatnonzero(fmask[j])
            Xm = np.ascontiguousarray(self.X[m][:, keep])
            W, b, it = wo.fit_multinomial_lbfgs(Xm, self.y[m], cw[0][j][self.y[m]], n_classes, C=float(C[j]),
                                                tol=tol, max_iter=max_iter, fit_intercept=fit_intercept)
            coef[j][:, keep], coef[j, :, self.d], n_iter[j] = W, b, it
        return {"coef": coef, "n_iter": n_iter, "status": np.ones(B, np.int32), "loss": np.zeros(B),
                "n_evals": n_iter + 1, "gpu_seconds": 0.0}
