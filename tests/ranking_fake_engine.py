"""FakeEngine plus the rank-kernel call -- TEST DOUBLE, CPU only.

linear_rank_batch forms the scores as scikit-learn's scorers see them (float32 decision_function, float32
predict_proba) and counts every segment with tests/ranking_reference.py."""
import numpy as np

from tests import ranking_reference as rr
from tests.fake_engine import FakeEngine


class RankingFakeEngine(FakeEngine):
    def linear_rank_batch(self, coef, col_fold, col_pos=None, score="decision", pairs=False):
        coef = np.asarray(coef, dtype=np.float32)
        B = coef.shape[0]
        K = 1 if coef.ndim == 2 else coef.shape[1]
        W = coef[:, None, :] if K == 1 else coef
        self.calls.append(("rank", B, score, bool(pairs)))
        rows = []
        for j in range(B):
            m = self._rows(int(col_fold[j]))
            Z = self.X[m] @ W[j, :, :self.d].T + W[j, :, self.d]       # decision_function, float32
            Z = Z[:, 0] if K == 1 else Z
            S = rr.f32_proba(Z) if score == "proba" else (-Z if score == "neg_decision" else Z)
            rows.append(rr.rank_counts(S, self.y[m], K, pairs, None if K > 1 else int(col_pos[j])))
        return {k: np.stack([r[k] for r in rows]) for k in ("u2", "n_pos", "n_neg", "ap")}
