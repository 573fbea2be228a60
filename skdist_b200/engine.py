"""Host-side handle on one GPU's staged dataset + batched solvers (ctypes over the C-ABI)."""
import ctypes

import numpy as np

from . import _lib
from ._lib import check, ptr


class Engine:
    """One context per process / GPU.  Replaces the reference's SparkContext
    (ref skdist/distribute/search.py:309-313, `sc`): data is staged once in
    HBM instead of being shipped with every task."""

    def __init__(self, device=0):
        self._lib = _lib.load()
        h = ctypes.c_void_p()
        check(self._lib.skd_ctx_create(int(device), ctypes.byref(h)))
        self._h = h
        self.device = int(device)
        self.n = self.d = 0

    # -- lifetime -------------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self._lib.skd_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- staging ----------------------------------------------------------------
    def stage_x(self, X):
        X = np.asarray(X)
        ok = (X.ndim == 2 and X.dtype == np.float32 and X.shape[1] > 0 and X.strides[1] == 4
              and X.strides[0] % 4 == 0 and X.strides[0] >= 4 * X.shape[1])
        if not ok:      # row-strided fp32 views are staged in place; anything else is converted first
            X = np.ascontiguousarray(X, dtype=np.float32)
        n, d = X.shape
        check(self._lib.skd_stage_x(self._h, ptr(X), n, d, X.strides[0] // 4), self._h)
        self.n, self.d = n, d

    def stage_x_device(self, dev_ptr, n, d, ldx=None):
        check(self._lib.skd_stage_x_device(self._h, ctypes.c_void_p(int(dev_ptr)), n, d, ldx or d), self._h)
        self.n, self.d = n, d

    def stage_x_sliced(self, X, row0, row1, n_alloc, gather):
        """Stage X when several ranks hold it: this rank copies rows [row0, row1) to its GPU,
        `gather(dev_ptr, ldx)` completes the buffer in place (all-gather over NVLink), then the
        matrix is validated and becomes the staged X."""
        X = np.asarray(X)
        ok = (X.ndim == 2 and X.dtype == np.float32 and X.shape[1] > 0 and X.strides[1] == 4
              and X.strides[0] % 4 == 0 and X.strides[0] >= 4 * X.shape[1])
        n, d = X.shape
        sl = X[row0:row1]
        if not ok:
            sl = np.ascontiguousarray(sl, dtype=np.float32)
        p, ldx = ctypes.c_void_p(), ctypes.c_int64()
        check(self._lib.skd_stage_x_begin(self._h, n, d, int(n_alloc), ctypes.byref(p), ctypes.byref(ldx)), self._h)
        err = None
        try:
            if row1 > row0:
                check(self._lib.skd_stage_x_rows(self._h, ptr(sl), sl.strides[0] // 4, int(row0), int(row1 - row0)), self._h)
        except Exception as e:      # noqa: BLE001 - the collective below must still be entered by every rank
            err = e
        gather(p.value, ldx.value)
        if err is not None:
            raise err
        check(self._lib.skd_stage_x_commit(self._h), self._h)
        self.n, self.d = n, d

    def staged_x(self):
        """(device pointer, n, d, ldx) of the staged matrix."""
        p = ctypes.c_void_p()
        n, d, ldx = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
        check(self._lib.skd_staged_x(self._h, ctypes.byref(p), ctypes.byref(n), ctypes.byref(d),
                                     ctypes.byref(ldx)), self._h)
        return p.value, n.value, d.value, ldx.value

    def stage_labels(self, y_class):
        y = np.ascontiguousarray(y_class, dtype=np.int32)
        check(self._lib.skd_stage_labels(self._h, ptr(y), y.shape[0]), self._h)

    def stage_targets(self, y):
        y = np.ascontiguousarray(y, dtype=np.float32)
        check(self._lib.skd_stage_targets(self._h, ptr(y), y.shape[0]), self._h)

    def stage_folds(self, fold_id, n_folds):
        if fold_id is None:
            check(self._lib.skd_stage_folds(self._h, None, 0, 0), self._h)
            return
        f = np.ascontiguousarray(fold_id, dtype=np.int8)
        check(self._lib.skd_stage_folds(self._h, ptr(f), f.shape[0], int(n_folds)), self._h)

    def set_kernel(self, which):
        return self._lib.skd_set_kernel(self._h, int(which))

    def counters(self):
        a, b, c = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
        check(self._lib.skd_get_counters(self._h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c)), self._h)
        return {"launches": a.value, "h2d_bytes": b.value, "d2h_bytes": c.value}

    def profile(self, enable=-1):
        """Read (and with enable in {0,1} reset + switch) the evaluation-kernel timers."""
        ms, fl = ctypes.c_double(), ctypes.c_double()
        nl, nr = ctypes.c_int64(), ctypes.c_int64()
        check(self._lib.skd_profile(self._h, int(enable), ctypes.byref(ms), ctypes.byref(fl),
                                    ctypes.byref(nl), ctypes.byref(nr)), self._h)
        return {"eval_ms": ms.value, "eval_flops": fl.value, "eval_launches": nl.value,
                "rounds": nr.value}

    def timer_start(self):
        check(self._lib.skd_timer_start(self._h), self._h)

    def timer_stop(self):
        """Elapsed device time (seconds) on the library's stream since timer_start()."""
        ms = ctypes.c_double()
        check(self._lib.skd_timer_stop(self._h, ctypes.byref(ms)), self._h)
        return ms.value * 1e-3

    # -- solvers ------------------------------------------------------------------
    def stage_column_masks(self, mask):
        """[B, d] 0/1 feature masks consumed by the next logreg_fit_batch (None clears)."""
        if mask is None:
            check(self._lib.skd_stage_column_masks(self._h, 0, None), self._h)
            return
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        assert m.ndim == 2 and m.shape[1] == self.d
        check(self._lib.skd_stage_column_masks(self._h, m.shape[0], ptr(m)), self._h)

    def stage_row_bits(self, labels=None, train=None):
        """[B, n] 0/1 matrices consumed by the next logreg_fit_batch: `labels[j, r]` = binary label of
        row r in column j (multilabel targets), `train[j, r]` = row r takes part in column j's fit
        (sampled negatives).  None clears."""
        if labels is None and train is None:
            check(self._lib.skd_stage_row_bits(self._h, 0, None, None, 0), self._h)
            return
        packed = []
        B = None
        for m in (labels, train):
            if m is None:
                packed.append(None)
                continue
            m = np.asarray(m)
            assert m.ndim == 2 and m.shape[1] == self.n
            B = m.shape[0] if B is None else B
            assert m.shape[0] == B
            packed.append(np.ascontiguousarray(np.packbits(m.astype(bool), axis=1, bitorder="little")))
        bpc = next(p for p in packed if p is not None).shape[1]
        check(self._lib.skd_stage_row_bits(self._h, B, ptr(packed[0]) if packed[0] is not None else None,
                                           ptr(packed[1]) if packed[1] is not None else None, bpc), self._h)

    def stage_class_weights(self, w, sw_sum):
        """[B, K] class weights and [B] sums of the per-row weights consumed by the next logreg_fit_batch /
        logreg_loss_grad (K = 2: label 0, label 1) or logreg_multinomial_fit_batch (K = n_classes).
        None clears."""
        if w is None:
            check(self._lib.skd_stage_class_weights(self._h, 0, 0, None, None), self._h)
            return
        w = np.ascontiguousarray(w, dtype=np.float32)
        sw_sum = np.ascontiguousarray(sw_sum, dtype=np.float64)
        assert w.ndim == 2 and sw_sum.shape == (w.shape[0],)
        check(self._lib.skd_stage_class_weights(self._h, w.shape[0], w.shape[1], ptr(w), ptr(sw_sum)), self._h)

    def stage_sample_weights(self, w):
        """[n] float32 per-row sample weights consumed by the next logreg_fit_batch / logreg_loss_grad /
        logreg_multinomial_fit_batch / logreg_multinomial_loss_grad, together with the class weights staged for
        that call (whose sw_sum must include them).  Scores stay unweighted.  None clears."""
        if w is None:
            check(self._lib.skd_stage_sample_weights(self._h, None, 0), self._h)
            return
        w = np.ascontiguousarray(w, dtype=np.float32)
        assert w.ndim == 1
        check(self._lib.skd_stage_sample_weights(self._h, ptr(w), w.shape[0]), self._h)

    def logreg_fit_batch(self, C, col_fold, col_pos, fit_intercept=True, tol=1e-4, max_iter=100, col_neg=None):
        """B binary lbfgs fits sharing the staged X.  col_neg[j] >= 0 restricts column j to the rows
        of class col_pos[j] / col_neg[j] (one-vs-one pair); None or < 0 = one-vs-rest."""
        C = np.ascontiguousarray(C, dtype=np.float64)
        B = C.shape[0]
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        assert col_fold.shape == (B,) and col_pos.shape == (B,)
        if col_neg is not None:
            col_neg = np.ascontiguousarray(col_neg, dtype=np.int32)
            assert col_neg.shape == (B,)
        coef = np.empty((B, self.d + 1), dtype=np.float32)
        n_iter = np.empty(B, dtype=np.int32)
        status = np.empty(B, dtype=np.int32)
        loss = np.empty(B, dtype=np.float64)
        n_evals = np.empty(B, dtype=np.int32)
        secs = ctypes.c_double(0.0)
        check(self._lib.skd_logreg_fit_batch(
            self._h, B, ptr(C), ptr(col_fold), ptr(col_pos), ptr(col_neg) if col_neg is not None else None,
            int(bool(fit_intercept)), float(tol), int(max_iter), ptr(coef), ptr(n_iter), ptr(status), ptr(loss), ptr(n_evals),
            ctypes.byref(secs)), self._h)
        return {"coef": coef, "n_iter": n_iter, "status": status, "loss": loss,
                "n_evals": n_evals, "gpu_seconds": secs.value}

    def logreg_loss_grad(self, w, C, col_fold, col_pos, fit_intercept=True):
        w = np.ascontiguousarray(w, dtype=np.float64)
        B = w.shape[0]
        assert w.shape[1] == self.d + 1
        C = np.ascontiguousarray(C, dtype=np.float64)
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        loss = np.empty(B, dtype=np.float64)
        grad = np.empty((B, self.d + 1), dtype=np.float64)
        check(self._lib.skd_logreg_loss_grad(self._h, B, ptr(w), ptr(C), ptr(col_fold), ptr(col_pos),
                                             int(bool(fit_intercept)), ptr(loss), ptr(grad)), self._h)
        return loss, grad

    def linear_score_batch(self, coef, col_fold, col_pos):
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B = coef.shape[0]
        assert coef.shape[1] == self.d + 1
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        correct = np.empty(B, dtype=np.int64)
        count = np.empty(B, dtype=np.int64)
        check(self._lib.skd_linear_score_batch(self._h, B, ptr(coef), ptr(col_fold), ptr(col_pos),
                                               ptr(correct), ptr(count)), self._h)
        return correct, count

    def logreg_multinomial_fit_batch(self, C, col_fold, n_classes, fit_intercept=True, tol=1e-4, max_iter=100):
        """B multinomial lbfgs fits (class ids 0..n_classes-1 staged) sharing the staged X.
        coef is [B, n_classes, d + 1] (weights, intercept last)."""
        C = np.ascontiguousarray(C, dtype=np.float64)
        B = C.shape[0]
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        assert col_fold.shape == (B,)
        K = int(n_classes)
        coef = np.empty((B, K, self.d + 1), dtype=np.float32)
        n_iter = np.empty(B, dtype=np.int32)
        status = np.empty(B, dtype=np.int32)
        loss = np.empty(B, dtype=np.float64)
        n_evals = np.empty(B, dtype=np.int32)
        secs = ctypes.c_double(0.0)
        check(self._lib.skd_logreg_multinomial_fit_batch(
            self._h, B, K, ptr(C), ptr(col_fold), int(bool(fit_intercept)), float(tol), int(max_iter), ptr(coef),
            ptr(n_iter), ptr(status), ptr(loss), ptr(n_evals), ctypes.byref(secs)), self._h)
        return {"coef": coef, "n_iter": n_iter, "status": status, "loss": loss,
                "n_evals": n_evals, "gpu_seconds": secs.value}

    def logreg_multinomial_loss_grad(self, w, C, col_fold, fit_intercept=True):
        """Objective [B] and gradient [B, K, d + 1] of B multinomial candidates at the points w [B, K, d + 1],
        by the evaluation of logreg_multinomial_fit_batch (class ids 0..K-1 staged)."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        B, K = w.shape[0], w.shape[1]
        assert w.shape[2] == self.d + 1
        C = np.ascontiguousarray(C, dtype=np.float64)
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        assert C.shape == (B,) and col_fold.shape == (B,)
        loss = np.empty(B, dtype=np.float64)
        grad = np.empty_like(w)
        check(self._lib.skd_logreg_multinomial_loss_grad(self._h, B, K, ptr(w), ptr(C), ptr(col_fold),
                                                         int(bool(fit_intercept)), ptr(loss), ptr(grad)), self._h)
        return loss, grad

    def multinomial_score_batch(self, coef, col_fold):
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B, K = coef.shape[0], coef.shape[1]
        assert coef.shape[2] == self.d + 1
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        correct = np.empty(B, dtype=np.int64)
        count = np.empty(B, dtype=np.int64)
        check(self._lib.skd_multinomial_score_batch(self._h, B, K, ptr(coef), ptr(col_fold), ptr(correct),
                                                    ptr(count)), self._h)
        return correct, count

    def multinomial_confusion_batch(self, coef, col_fold):
        """[B, K, K] confusion counts (true class, predicted class) on the rows selected by the fold codes."""
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B, K = coef.shape[0], coef.shape[1]
        assert coef.shape[2] == self.d + 1
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        conf = np.empty((B, K, K), dtype=np.int64)
        check(self._lib.skd_multinomial_confusion_batch(self._h, B, K, ptr(coef), ptr(col_fold), ptr(conf)), self._h)
        return conf

    def linear_auc_batch(self, coef, col_fold, col_pos):
        """ROC-AUC of B linear binary classifiers on the rows selected by the fold codes (NaN where a
        class is missing), from exact integer pair counts."""
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B = coef.shape[0]
        assert coef.shape[1] == self.d + 1
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        u2 = np.empty(B, dtype=np.int64)
        n_pos = np.empty(B, dtype=np.int64)
        n_neg = np.empty(B, dtype=np.int64)
        check(self._lib.skd_linear_auc_batch(self._h, B, ptr(coef), ptr(col_fold), ptr(col_pos), ptr(u2), ptr(n_pos),
                                             ptr(n_neg)), self._h)
        den = 2.0 * n_pos.astype(np.float64) * n_neg.astype(np.float64)
        return np.divide(u2.astype(np.float64), den, out=np.full(B, np.nan), where=den > 0), n_pos + n_neg

    RANK_SCORES = {"decision": 0, "neg_decision": 1, "proba": 2}

    def linear_rank_batch(self, coef, col_fold, col_pos=None, score="decision", pairs=False):
        """Ranked counts per segment on the rows selected by the fold codes: {"u2", "n_pos", "n_neg", "ap"},
        each [B, S].  coef [B, d+1] with col_pos: one binary segment per column; coef [B, K, d+1]: K
        one-vs-rest segments per column, or K (K - 1) ordered one-vs-one pairs when `pairs`.  score:
        "decision", "neg_decision" or "proba" (float32 predict_proba)."""
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B = coef.shape[0]
        K = 1 if coef.ndim == 2 else coef.shape[1]
        assert coef.shape[-1] == self.d + 1
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        if K == 1:
            col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        S = 1 if K == 1 else (K * (K - 1) if pairs else K)
        out = {k: np.empty((B, S), dtype=np.int64) for k in ("u2", "n_pos", "n_neg")}
        out["ap"] = np.empty((B, S), dtype=np.float64)
        check(self._lib.skd_linear_rank_batch(self._h, B, K, ptr(coef), ptr(col_fold),
                                              ptr(col_pos) if K == 1 else None, self.RANK_SCORES[score],
                                              int(bool(pairs)), ptr(out["u2"]), ptr(out["n_pos"]),
                                              ptr(out["n_neg"]), ptr(out["ap"])), self._h)
        return out

    def linear_logloss_batch(self, coef, col_fold, col_pos=None):
        """Mean log loss of the predicted probabilities per column on the rows selected by the fold codes.
        coef [B, d+1] with col_pos: binary columns; coef [B, K, d+1]: multiclass."""
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B = coef.shape[0]
        K = 1 if coef.ndim == 2 else coef.shape[1]
        assert coef.shape[-1] == self.d + 1
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        if K == 1:
            col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        loss = np.empty(B, dtype=np.float64)
        count = np.empty(B, dtype=np.int64)
        check(self._lib.skd_linear_logloss_batch(self._h, B, K, ptr(coef), ptr(col_fold),
                                                 ptr(col_pos) if K == 1 else None, ptr(loss), ptr(count)), self._h)
        return loss / np.maximum(count, 1), count

    def sgd_fit_batch(self, est, col_pos):
        """Fit one binary SGDClassifier per entry of col_pos (one-vs-rest label columns).
        `est` is the template SGDClassifier; host-side constants are derived exactly as
        SK/linear_model/_stochastic_gradient.py:455-473 and _sgd_fast.pyx.tp:447-452 do."""
        p = est.get_params(deep=False)
        loss, lr = sgd_config(p)
        seed = sgd_seed(p["random_state"])
        alpha = float(p["alpha"])
        col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        B = col_pos.shape[0]
        out = _sgd_outputs(B, self.d)
        secs = ctypes.c_double(0.0)
        tol = -np.inf if p["tol"] is None else float(p["tol"])
        check(self._lib.skd_sgd_fit_batch(
            self._h, B, ptr(col_pos), loss, alpha, int(bool(p["fit_intercept"])), int(p["max_iter"]), tol,
            int(bool(p["shuffle"])), seed, lr, float(p["eta0"]), float(p["power_t"]), sgd_optimal_init(loss, alpha),
            int(p["n_iter_no_change"]), ptr(out["coef32"]), ptr(out["intercept"]), ptr(out["n_iter"]), ptr(out["t"]),
            ptr(out["status"]), ctypes.byref(secs)), self._h)
        return _sgd_result(out, secs.value)

    def sgd_fit_groups(self, params, col_pos, col_group, col_alpha, group_rows, group_seeds):
        """Binary SGDClassifier fits in order groups: column j fits the rows group_rows[col_group[j]] (int row ids,
        in the order the fit walks them before its first shuffle) with alpha col_alpha[j] and positives y_class ==
        col_pos[j]; group g shuffles with its own seed group_seeds[g] (the `seed` _plain_sgd receives, see
        sgd_seed).  `params` are the SGDClassifier parameters shared by every column (their alpha is unused)."""
        loss, lr = sgd_config(params)
        p = params
        col_pos = np.ascontiguousarray(col_pos, dtype=np.int32)
        col_group = np.ascontiguousarray(col_group, dtype=np.int32)
        col_alpha = np.ascontiguousarray(col_alpha, dtype=np.float64)
        B = col_pos.shape[0]
        assert col_group.shape == (B,) and col_alpha.shape == (B,)
        if self.n >= 2 ** 31:
            raise NotImplementedError("sgd_fit_groups: the device path supports n < 2^31 rows (int32 row ids)")
        col_oi = np.array([sgd_optimal_init(loss, a) if a > 0 else 1.0 for a in col_alpha], dtype=np.float64)
        sizes = np.array([len(r) for r in group_rows], dtype=np.int64)
        offsets = np.ascontiguousarray(np.concatenate([[0], np.cumsum(sizes)]), dtype=np.int64)
        rows = np.ascontiguousarray(np.concatenate([np.asarray(r, dtype=np.int64) for r in group_rows])
                                    if len(group_rows) else np.zeros(0, np.int64))
        if rows.size and (rows.min() < 0 or rows.max() >= self.n):
            raise ValueError("sgd_fit_groups: row ids outside [0, %d)" % self.n)
        rows = rows.astype(np.int32)
        seeds = np.ascontiguousarray(group_seeds, dtype=np.uint32)
        assert seeds.shape == (len(group_rows),)
        out = _sgd_outputs(B, self.d)
        secs = ctypes.c_double(0.0)
        tol = -np.inf if p["tol"] is None else float(p["tol"])
        check(self._lib.skd_sgd_fit_groups(
            self._h, B, ptr(col_pos), ptr(col_group), ptr(col_alpha), ptr(col_oi), len(group_rows), ptr(offsets),
            ptr(rows), ptr(seeds), loss, int(bool(p["fit_intercept"])), int(p["max_iter"]), tol,
            int(bool(p["shuffle"])), lr, float(p["eta0"]), float(p["power_t"]), int(p["n_iter_no_change"]),
            ptr(out["coef32"]), ptr(out["intercept"]), ptr(out["n_iter"]), ptr(out["t"]), ptr(out["status"]),
            ctypes.byref(secs)), self._h)
        return _sgd_result(out, secs.value)

    def stage_forest_class_weights(self, n_classes, w=None, balanced_subsample=False, min_weight_fraction_leaf=0.0):
        """Class weights of the next forest_fit: w [n_classes] float64 (the same for every tree), or
        balanced_subsample=True (per tree from its bootstrap class counts; w unused).  min_weight_fraction_leaf
        replaces that fit's min_weight_leaf (per tree: fraction * its sum of weights).  n_classes = 0 clears."""
        if balanced_subsample or not n_classes:
            check(self._lib.skd_stage_forest_class_weights(self._h, int(n_classes), None, int(bool(balanced_subsample)),
                                                           float(min_weight_fraction_leaf)), self._h)
            return
        w = np.ascontiguousarray(w, dtype=np.float64)
        assert w.shape == (n_classes,)
        check(self._lib.skd_stage_forest_class_weights(self._h, int(n_classes), ptr(w), 0,
                                                       float(min_weight_fraction_leaf)), self._h)

    def stage_forest_criterion(self, criterion):
        """Split criterion of the next forest_fit: 0 Gini / squared error, 1 entropy (classification only;
        the general tree builder, impurity in bits formed on the host as scikit-learn forms it)."""
        check(self._lib.skd_stage_forest_criterion(self._h, int(criterion)), self._h)

    def forest_fit(self, sample_counts, rand_states, n_classes, max_features, max_depth, min_samples_split,
                   min_samples_leaf, min_weight_leaf, min_impurity_decrease, splitter=0, y_regression=None):
        """Build len(rand_states) classifier trees.  sample_counts [n_trees, n] uint8 (bootstrap
        multiplicities = the reference's sample_weight; None = every row once), rand_states [n_trees]
        uint32 splitter seeds, splitter 0 = best (RandomForest) / 1 = random (ExtraTrees) / 2 = best, also on
        features with more than 256 distinct values (sorts their raw values; otherwise the same as 0).
        y_regression: float64 targets [n] -> regression trees (MSE), one value per node.
        Returns a list of dicts with the sklearn Tree arrays of every tree."""
        yreg = None
        if y_regression is not None:
            yreg = np.ascontiguousarray(y_regression, dtype=np.float64)
            assert yreg.shape == (self.n,)
            n_classes = 1
        rs = np.ascontiguousarray(rand_states, dtype=np.uint32)
        T = rs.shape[0]
        counts = None
        if sample_counts is not None:
            counts = np.ascontiguousarray(sample_counts, dtype=np.uint8)
            assert counts.shape == (T, self.n)
        h = ctypes.c_void_p()
        secs = ctypes.c_double(0.0)
        check(self._lib.skd_forest_fit(self._h, T, ptr(counts) if counts is not None else None, ptr(rs),
                                       int(n_classes), int(max_features),
                                       int(max_depth), int(min_samples_split), int(min_samples_leaf),
                                       float(min_weight_leaf), float(min_impurity_decrease), int(splitter),
                                       ptr(yreg) if yreg is not None else None,
                                       ctypes.byref(h), ctypes.byref(secs)), self._h)
        self.last_forest_seconds = secs.value
        ks = ctypes.c_double(0.0)
        check(self._lib.skd_forest_kernel_seconds(self._h, ctypes.byref(ks)), self._h)
        self.last_forest_kernel_seconds = ks.value
        from sklearn.tree._tree import NODE_DTYPE
        node_records = (NODE_DTYPE.itemsize == 64 and
                        [NODE_DTYPE.fields[k][1] for k in NODE_DTYPE.names] == [0, 8, 16, 24, 32, 40, 48, 56])

        def fetch(t):
            m, md = ctypes.c_int32(), ctypes.c_int32()
            check(self._lib.skd_forest_tree_size(h, t, ctypes.byref(m), ctypes.byref(md)))
            m = m.value
            if node_records:      # scikit-learn's node struct filled by the library: no per-field passes in Python
                nodes = np.empty(m, dtype=NODE_DTYPE)
                value = np.empty((m, n_classes), np.float64)
                check(self._lib.skd_forest_tree_nodes(h, t, ptr(nodes), ptr(value)))
                return {"nodes": nodes, "value": value, "max_depth": md.value, "left": nodes["left_child"],
                        "n_node_samples": nodes["n_node_samples"]}
            a = {"left": np.empty(m, np.int32), "right": np.empty(m, np.int32), "feature": np.empty(m, np.int32),
                 "threshold": np.empty(m, np.float64), "impurity": np.empty(m, np.float64),
                 "n_node_samples": np.empty(m, np.int32), "weighted_n_node_samples": np.empty(m, np.float64),
                 "missing_go_to_left": np.empty(m, np.uint8), "value": np.empty((m, n_classes), np.float64)}
            check(self._lib.skd_forest_tree_copy(h, t, ptr(a["left"]), ptr(a["right"]), ptr(a["feature"]),
                                                 ptr(a["threshold"]), ptr(a["impurity"]), ptr(a["n_node_samples"]),
                                                 ptr(a["weighted_n_node_samples"]), ptr(a["missing_go_to_left"]),
                                                 ptr(a["value"])))
            a["max_depth"] = md.value
            return a

        try:
            # the copies (and, for the compact records of the throughput builder, the float64 fields formed
            # from the integer class sums) run in the library without the GIL: one host thread per tree
            import os
            from concurrent.futures import ThreadPoolExecutor
            nthr = max(1, min(32, T, (os.cpu_count() or 8) // 2))
            if nthr > 1:
                with ThreadPoolExecutor(max_workers=nthr) as ex:
                    trees = list(ex.map(fetch, range(T)))
            else:
                trees = [fetch(t) for t in range(T)]
        finally:
            self._lib.skd_forest_free(h)
        return trees

    def ridge_fit_batch(self, alpha, col_fold, fit_intercept=True):
        alpha = np.ascontiguousarray(alpha, dtype=np.float64)
        B = alpha.shape[0]
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        coef = np.empty((B, self.d + 1), dtype=np.float32)
        status = np.empty(B, dtype=np.int32)
        secs = ctypes.c_double(0.0)
        check(self._lib.skd_ridge_fit_batch(self._h, B, ptr(alpha), ptr(col_fold), int(bool(fit_intercept)),
                                            ptr(coef), ptr(status), ctypes.byref(secs)), self._h)
        return {"coef": coef, "status": status, "gpu_seconds": secs.value}

    def linear_r2_batch(self, coef, col_fold):
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B = coef.shape[0]
        col_fold = np.ascontiguousarray(col_fold, dtype=np.int32)
        sse = np.empty(B, dtype=np.float64)
        count = np.empty(B, dtype=np.int64)
        check(self._lib.skd_linear_r2_batch(self._h, B, ptr(coef), ptr(col_fold), ptr(sse), ptr(count)), self._h)
        return sse, count

    def predict_linear(self, Xnew, coef):
        """out[m, B] for NEW host rows (streamed); coef [B, d+1] with the intercept last."""
        Xnew = np.ascontiguousarray(Xnew, dtype=np.float32)
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        m, d = Xnew.shape
        B = coef.shape[0]
        assert coef.shape[1] == d + 1
        out = np.empty((m, B), dtype=np.float32)
        secs = ctypes.c_double(0.0)
        check(self._lib.skd_predict_linear(self._h, ptr(Xnew), m, d, d, B, ptr(coef), ptr(out),
                                           ctypes.byref(secs)), self._h)
        self.last_predict_seconds = secs.value
        return out

    def forest_predict(self, Xnew, tree_offset, left, right, feature, threshold, value):
        """Soft-vote forest inference on NEW host rows: [m, C] float64 mean of the leaf values of
        every tree (class fractions for classifiers, C = 1 for regressors)."""
        Xnew = np.ascontiguousarray(Xnew, dtype=np.float32)
        m, d = Xnew.shape
        off = np.ascontiguousarray(tree_offset, dtype=np.int64)
        left = np.ascontiguousarray(left, dtype=np.int32)
        right = np.ascontiguousarray(right, dtype=np.int32)
        feature = np.ascontiguousarray(feature, dtype=np.int32)
        threshold = np.ascontiguousarray(threshold, dtype=np.float64)
        value = np.ascontiguousarray(value, dtype=np.float64)
        C = value.shape[1]
        out = np.empty((m, C), dtype=np.float64)
        secs = ctypes.c_double(0.0)
        check(self._lib.skd_forest_predict(self._h, ptr(Xnew), m, d, d, len(off) - 1, ptr(off), ptr(left),
                                           ptr(right), ptr(feature), ptr(threshold), ptr(value), C, ptr(out),
                                           ctypes.byref(secs)), self._h)
        self.last_predict_seconds = secs.value
        return out

    def linear_decision(self, coef):
        coef = np.ascontiguousarray(coef, dtype=np.float32)
        B = coef.shape[0]
        out = np.empty((self.n, B), dtype=np.float32)
        check(self._lib.skd_linear_decision(self._h, B, ptr(coef), ptr(out)), self._h)
        return out


# -- SGDClassifier on the device ------------------------------------------------------------------
SGD_LOSSES = {"hinge": 0, "log_loss": 1}
SGD_LEARNING_RATES = {"optimal": 0, "constant": 1, "invscaling": 2}
_MAX_INT = np.iinfo(np.int32).max


def sgd_config(p):
    """(loss code, learning-rate code) of SGDClassifier parameters `p` (get_params(deep=False)), or
    NotImplementedError naming every setting the exact-order SGD kernels do not reproduce."""
    bad = []
    loss = SGD_LOSSES.get(p["loss"])
    if loss is None:
        bad.append("loss=%r" % p["loss"])
    if p["penalty"] != "l2":
        bad.append("penalty=%r" % (p["penalty"],))
    lr = SGD_LEARNING_RATES.get(p["learning_rate"])
    if lr is None:
        bad.append("learning_rate=%r" % p["learning_rate"])
    for k in ("average", "early_stopping", "warm_start"):
        if p.get(k):
            bad.append("%s=%r" % (k, p[k]))
    if p.get("class_weight") is not None:
        bad.append("class_weight")
    if bad:
        raise NotImplementedError("SGDClassifier configuration without a device path: " + ", ".join(bad))
    return loss, lr


def sgd_seed(random_state):
    """The shuffle seed one binary fit hands to _plain_sgd (SK/linear_model/_stochastic_gradient.py:455-473):
    make_dataset() draws the dataset seed first, then seed = randint(MAX_INT)."""
    from sklearn.utils import check_random_state
    rs = check_random_state(random_state)
    rs.randint(1, _MAX_INT)
    return int(rs.randint(_MAX_INT))


def sgd_optimal_init(loss, alpha):
    """optimal_init of the "optimal" schedule for loss code `loss` (SK/linear_model/_sgd_fast.pyx.tp:447-452)."""
    typw = np.sqrt(1.0 / np.sqrt(alpha))
    if loss == 0:
        g0 = -1.0 if -typw <= 1.0 else 0.0      # Hinge.cy_gradient(1.0, -typw)
    else:
        g0 = -1.0 / (1.0 + np.exp(-typw))       # CyHalfBinomialLoss.cy_gradient(1.0, -typw) < 0
    return float(1.0 / ((typw / max(1.0, g0)) * alpha))


def _sgd_outputs(B, d):
    return {"coef32": np.empty((B, d), dtype=np.float32), "intercept": np.empty(B, dtype=np.float64),
            "n_iter": np.empty(B, dtype=np.int32), "t": np.empty(B, dtype=np.float64),
            "status": np.empty(B, dtype=np.int32)}


def _sgd_result(out, secs):
    out["coef"] = np.concatenate([out["coef32"].astype(np.float64), out["intercept"][:, None]], axis=1)
    out["gpu_seconds"] = secs
    return out


# -- per-process singleton -------------------------------------------------------------------
_ENGINE = None
_FACTORY = None


def set_engine_factory(factory):
    """Test hook: replace the object returned by get_engine() (e.g. with an oracle-backed
    stand-in so host logic can be exercised without a GPU).  Pass None to restore."""
    global _FACTORY, _ENGINE
    _FACTORY = factory
    _ENGINE = None


def get_engine():
    """The process-wide Engine, bound to cuda:LOCAL_RANK (one process per GPU)."""
    global _ENGINE
    if _ENGINE is None:
        if _FACTORY is not None:
            _ENGINE = _FACTORY()
        else:
            import os
            _ENGINE = Engine(int(os.environ.get("LOCAL_RANK", 0)))
    return _ENGINE


def reset_engine():
    global _ENGINE
    if _ENGINE is not None and hasattr(_ENGINE, "close"):
        _ENGINE.close()
    _ENGINE = None
