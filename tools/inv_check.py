"""Batch invariance of the tensor-core fit: one (C, fold) column fitted alone and inside batches of
4 / 32 / 148 / 160 groups of 128 columns must give bit-identical coefficients (more groups than SMs
exercises the weight reload of a CTA that spans several groups)."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sklearn.model_selection import StratifiedKFold
from skdist_b200.datasets import make_g1_classification
from skdist_b200.engine import Engine
e = Engine(0); e.set_kernel(2)
X, y = make_g1_classification(6000, 32, seed=77)
fold = np.zeros(len(y), np.int8)
for k, (_, te) in enumerate(StratifiedKFold(4).split(X, y)):
    fold[te] = k
e.stage_x(X); e.stage_labels(y.astype(np.int32)); e.stage_folds(fold, 4)
def run(ncand):
    Cs = np.repeat(np.logspace(-4, -1, ncand), 4); fs = np.tile(np.arange(4, dtype=np.int32), ncand)
    return Cs, fs, e.logreg_fit_batch(Cs, fs, np.ones(len(Cs), np.int32))
ref = {}
for ncand in (32, 1024, 4736, 5120):          # 4, 32, 148, 160 groups
    Cs, fs, r = run(ncand)
    one = e.logreg_fit_batch(Cs[[5]], fs[[5]], np.ones(1, np.int32))
    last = e.logreg_fit_batch(Cs[[-1]], fs[[-1]], np.ones(1, np.int32))
    print(ncand, "groups", len(Cs) // 128, "col5 equal", np.array_equal(one["coef"][0], r["coef"][5]), r["n_iter"][5], one["n_iter"][0],
          "last equal", np.array_equal(last["coef"][0], r["coef"][-1]), r["n_iter"][-1], last["n_iter"][0],
          "max diff", np.abs(last["coef"][0] - r["coef"][-1]).max())
