"""Rank kernel (csrc/auc.cu, skd_linear_rank_batch) and the ranking scorers on the device.

(a) exact tier: integer X and coefficients make every fp32 decision value exact, so 2U / n_pos / n_neg of
    every binary, one-vs-rest and one-vs-one segment equal the integer reference (tests/ranking_reference.py)
    and the average precision matches it to 1e-12 relative: ties inside and across classes, a class absent
    from a fold, every scoring code (held-out, train -3 - f, all rows -2), B = 1, and one-vs-one over more
    than one block of fits;
(b) probability tier: 2U lies inside the reference's interval when pairs closer than the kernel's stated
    bound may rank either way; saturated / well separated probabilities give roc_auc_score(y,
    est.predict_proba(X)) exactly;
(c) public tier: DistGridSearchCV(LogisticRegression()) on digits with each new scorer and a multi-metric dict,
    binary average_precision for LogisticRegression and SGDClassifier(loss="log_loss"), and the eliminator on a
    covtype-shaped multiclass set with f1_weighted, against scikit-learn's scorers."""
import numpy as np
import pytest
from sklearn.linear_model import LogisticRegression, SGDClassifier
from sklearn.metrics import get_scorer, roc_auc_score

from tests import ranking_reference as rr

pytestmark = pytest.mark.gpu

RAN = set()
NEW = ["roc_auc_ovr", "roc_auc_ovr_weighted", "roc_auc_ovo", "roc_auc_ovo_weighted", "average_precision"]


@pytest.fixture(scope="module")
def eng():
    from skdist_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def _rows(code, fold):
    if code == -2:
        return np.ones(len(fold), bool)
    return fold == code if code >= 0 else fold != (-3 - code)


def _int_problem(rng, n, d, K, nf):
    X = rng.integers(-3, 4, (n, d)).astype(np.float32)
    y = rng.integers(0, K, n).astype(np.int32)
    fold = rng.permutation(np.arange(n) % nf).astype(np.int8)
    return X, y, fold


def _check(eng, X, y, fold, coef, codes, pos, score, pairs, label):
    K = 1 if coef.ndim == 2 else coef.shape[1]
    got = eng.linear_rank_batch(coef, codes, pos, score=score, pairs=pairs)
    W = coef[:, None, :] if K == 1 else coef
    for j in range(len(codes)):
        m = _rows(int(codes[j]), fold)
        Z = X[m].astype(np.float64) @ W[j, :, :-1].T.astype(np.float64) + W[j, :, -1]
        Z = Z[:, 0] if K == 1 else Z
        S = -Z if score == "neg_decision" else Z
        want = rr.rank_counts(S, y[m], K, pairs, None if K > 1 else int(pos[j]))
        for k in ("u2", "n_pos", "n_neg"):
            assert np.array_equal(got[k][j], want[k]), (label, j, k)
        np.testing.assert_allclose(got["ap"][j], want["ap"], rtol=1e-12, atol=0, err_msg="%s %d" % (label, j))
    return got


def test_exact_segments(eng):
    rng = np.random.default_rng(0)
    n, d, K, nf = 20000, 5, 5, 4
    X, y, fold = _int_problem(rng, n, d, K, nf)
    y[(fold == 0) & (y == 4)] = 0                                      # class 4 absent from fold 0
    eng.stage_x(X)
    eng.stage_labels(y)
    eng.stage_folds(fold, nf)
    codes = np.array([0, 1, 2, 3, -2, -3, -4, -5, -6, 0], np.int32)
    coef = np.zeros((len(codes), K, d + 1), np.float32)
    coef[..., :d] = rng.integers(-2, 3, (len(codes), K, d))
    coef[..., d] = rng.integers(-2, 3, (len(codes), K))
    coef[-1, 1:] = coef[-1, 0]                                         # every class scores alike: ties across classes
    for pairs in (False, True):
        got = _check(eng, X, y, fold, coef, codes, None, "decision", pairs, "pairs=%s" % pairs)
        RAN.add(("ovo" if pairs else "ovr", "all codes"))
        assert np.any(got["n_pos"][0] == 0)                             # the absent class
        RAN.add(("ovo" if pairs else "ovr", "absent class"))
        _check(eng, X, y, fold, coef[5:6], codes[5:6], None, "decision", pairs, "B=1")
        RAN.add(("ovo" if pairs else "ovr", "B=1"))
    ycls2 = (y % 2).astype(np.int32)
    eng.stage_labels(ycls2)
    bcoef = coef[:, 0, :].copy()
    pos = np.array([1, 0, 1, 0, 1, 1, 0, 1, 3, 1], np.int32)           # 3: no positives
    for score in ("decision", "neg_decision"):
        _check(eng, X, ycls2, fold, bcoef, codes, pos, score, False, score)
        _check(eng, X, ycls2, fold, bcoef[:1], codes[:1], pos[:1], score, False, score + " B=1")
        RAN.add(("binary", score))


def test_exact_ovo_over_fit_blocks(eng):
    """K = 10 one-vs-one has 90 segments per fit: 120 fits run as three blocks of at most 4096 segments."""
    rng = np.random.default_rng(1)
    n, d, K, nf = 300, 4, 10, 3
    X, y, fold = _int_problem(rng, n, d, K, nf)
    y[:K] = np.arange(K)
    eng.stage_x(X)
    eng.stage_labels(y)
    eng.stage_folds(fold, nf)
    B = 120
    codes = rng.choice(np.array([0, 1, 2, -2, -3, -4, -5], np.int32), B).astype(np.int32)
    coef = np.zeros((B, K, d + 1), np.float32)
    coef[..., :d] = rng.integers(-2, 3, (B, K, d))
    coef[..., d] = rng.integers(-3, 4, (B, K))
    assert B * K * (K - 1) > 2 * 4096
    _check(eng, X, y, fold, coef, codes, None, "decision", True, "blocks")
    RAN.add(("ovo", "two blocks"))


def _estimator(coef, K):
    est = LogisticRegression()
    est.coef_ = coef[:, :-1].astype(np.float32) if K > 1 else coef[None, :-1].astype(np.float32)
    est.intercept_ = coef[:, -1].astype(np.float32) if K > 1 else coef[None, -1].astype(np.float32)
    est.classes_ = np.arange(max(K, 2))
    return est


@pytest.mark.parametrize("K", [1, 4, 10])
def test_probability_tier(eng, K):
    rng = np.random.default_rng(10 + K)
    n, d = 4000, 6
    # small integers times dyadic weights: every fp32 decision value is exact, whatever the summation order
    X = rng.integers(-3, 4, (n, d)).astype(np.float32)
    Kc = max(K, 2)
    y = rng.integers(0, Kc, n).astype(np.int32)
    eng.stage_x(X)
    eng.stage_labels(y)
    eng.stage_folds(None, 0)
    B = 6
    shape = (B, d + 1) if K == 1 else (B, K, d + 1)
    scale = np.array([0.5, 2, 8, 16, 32, 64]).reshape((B,) + (1,) * (len(shape) - 1))
    coef = (rng.integers(-1024, 1025, shape) / 1024.0 * scale).astype(np.float32)
    codes = np.full(B, -2, np.int32)
    pos = np.ones(B, np.int32)
    W = coef[:, None, :] if K == 1 else coef
    for pairs in ((False,) if K == 1 else (False, True)):
        got = eng.linear_rank_batch(coef, codes, pos if K == 1 else None, score="proba", pairs=pairs)
        for j in range(B):
            Z = (X.astype(np.float64) @ W[j, :, :-1].T.astype(np.float64) + W[j, :, -1]).astype(np.float32)
            P = rr.f32_proba(Z[:, 0] if K == 1 else Z)
            for s, (sc, pm) in enumerate(rr.segments(P, y, K, pairs)):
                lo, hi = rr.u2_interval(sc, pm, rr.proba_rel_tol(K))
                assert lo <= got["u2"][j, s] <= hi, (K, pairs, j, s, lo, got["u2"][j, s], hi)
        RAN.add(("proba", K, pairs))
    # saturated or well separated: z in multiples of 24 gives probabilities exactly 1.0f / 0 or far apart
    Xs = rng.integers(-2, 3, (n, d)).astype(np.float32)
    eng.stage_x(Xs)
    scoef = (rng.integers(-1, 2, shape) * 24).astype(np.float32)
    got = eng.linear_rank_batch(scoef, codes, pos if K == 1 else None, score="proba")
    for j in range(B):
        est = _estimator(scoef[j], K)
        P = est.predict_proba(Xs)
        if K == 1:
            want = roc_auc_score(y, P[:, 1])
            auc = got["u2"][j, 0] / (2.0 * got["n_pos"][j, 0] * got["n_neg"][j, 0])
        else:
            want = roc_auc_score(y, P, multi_class="ovr", average="macro")
            auc = np.mean(got["u2"][j] / (2.0 * got["n_pos"][j] * got["n_neg"][j]))
        assert auc == pytest.approx(want, rel=1e-14, abs=1e-15), (K, j)
    RAN.add(("saturated", K))


def _digits():
    from sklearn.datasets import load_digits
    X, y = load_digits(return_X_y=True)
    return (X / 16.0).astype(np.float32), y


@pytest.mark.filterwarnings("ignore")
def test_public_digits_search(eng):
    """Every split score of the search against scikit-learn's scorer on the device-fitted estimator of the
    same (C, fold) on the same test rows."""
    from skdist.distribute.search import DistGridSearchCV
    from skdist_b200.distribute.folds import _fold_ids
    from skdist_b200.distribute.logreg_family import _MultinomialFamily
    from sklearn.model_selection import StratifiedKFold
    from skdist_b200 import engine as E
    X, y = _digits()
    grid = {"C": [0.1, 1.0]}
    splits = list(StratifiedKFold(3).split(X, y))
    fold = _fold_ids(splits, len(y))
    worst = 0.0
    scorings = [[n] for n in NEW] + [{"ovr": "roc_auc_ovr", "ovo_w": "roc_auc_ovo_weighted", "ap": "average_precision",
                                      "f1w": "f1_weighted"}]
    e = E.get_engine()
    for scoring in scorings:
        names = scoring if isinstance(scoring, dict) else {"score": scoring[0]}
        gs = DistGridSearchCV(LogisticRegression(), grid, None, cv=3, scoring=scoring if isinstance(scoring, dict)
                              else scoring[0], refit=list(names)[0] if isinstance(scoring, dict) else True).fit(X, y)
        fam = _MultinomialFamily(LogisticRegression(), list(gs.cv_results_["params"]), X, y,
                                 {k: get_scorer(v) for k, v in names.items()})
        fam.stage(e, X, fold, 3)
        C = np.repeat([p["C"] for p in gs.cv_results_["params"]], 3)
        f = np.tile(np.arange(3, dtype=np.int32), len(grid["C"]))
        res = e.logreg_multinomial_fit_batch(C, f, 10)
        for i in range(len(C)):
            est = fam.make_estimator({"C": C[i]}, res["coef"][i], res["n_iter"][i], np.float32, X.shape[1])
            te = splits[f[i]][1]
            for key, sname in names.items():
                want = get_scorer(sname)(est, X[te], y[te])
                got = gs.cv_results_["split%d_test_%s" % (f[i], key)][i // 3]
                worst = max(worst, abs(got - want))
                assert got == pytest.approx(want, abs=1e-4), (sname, i)
        RAN.add(("public", "digits", tuple(sorted(names.values()))))
    print("largest |device - scikit-learn| split score on digits: %.3g" % worst)


@pytest.mark.filterwarnings("ignore")
def test_public_binary_average_precision(eng):
    from skdist.distribute.search import DistGridSearchCV
    from sklearn.model_selection import GridSearchCV
    from skdist_b200.datasets import make_g1_classification
    X, y = make_g1_classification(3000, 12, seed=4)
    y = y + 1                                                           # label 1 is classes_[0]
    grid = {"alpha": [1e-4, 1e-3]}
    est = SGDClassifier(loss="log_loss", random_state=0)
    names = ["average_precision", "roc_auc_ovr"]
    ours = DistGridSearchCV(est, grid, None, cv=3, scoring=names, refit=names[0]).fit(X, y)
    ref = GridSearchCV(est, grid, cv=3, scoring=names, refit=names[0]).fit(X, y)
    worst = 0.0
    for m in names:
        for s in range(3):
            k = "split%d_test_%s" % (s, m)
            worst = max(worst, np.max(np.abs(ours.cv_results_[k] - ref.cv_results_[k])))
            np.testing.assert_allclose(ours.cv_results_[k], ref.cv_results_[k], atol=1e-6, err_msg=k)
    RAN.add(("public", "sgd binary"))
    lr = DistGridSearchCV(LogisticRegression(), {"C": [0.1, 1.0]}, None, cv=3, scoring="average_precision").fit(X, y)
    sk = GridSearchCV(LogisticRegression(), {"C": [0.1, 1.0]}, cv=3, scoring="average_precision").fit(X, y)
    np.testing.assert_allclose(lr.cv_results_["mean_test_score"], sk.cv_results_["mean_test_score"], atol=1e-3)
    RAN.add(("public", "logreg binary"))
    print("largest |device - scikit-learn| binary split score: %.3g" % worst)


@pytest.mark.filterwarnings("ignore")
def test_public_eliminator_f1_weighted(eng):
    from skdist.distribute.eliminate import DistFeatureEliminator
    rng = np.random.default_rng(5)
    n, d, K = 6000, 12, 7
    X = rng.normal(size=(n, d)).astype(np.float32)
    W = rng.normal(size=(K, 6))
    y = np.argmax(X[:, :6] @ W.T + rng.normal(scale=1.0, size=(n, K)), axis=1)
    fe = DistFeatureEliminator(LogisticRegression(), None, step=2, cv=3, min_features_to_select=6,
                               scoring="f1_weighted").fit(X, y)
    assert len(fe.scores_) == 4 and np.all(np.isfinite(fe.scores_)) and fe.n_features_ >= 6
    from sklearn.model_selection import StratifiedKFold
    sc = get_scorer("f1_weighted")
    full = np.mean([sc(LogisticRegression().fit(X[tr], y[tr]), X[te], y[te]) for tr, te in StratifiedKFold(3).split(X, y)])
    assert fe.scores_[0] == pytest.approx(full, abs=5e-3)
    RAN.add(("public", "eliminator"))


def test_every_variant_ran():
    want = {("ovr", "all codes"), ("ovr", "absent class"), ("ovr", "B=1"), ("ovo", "all codes"),
            ("ovo", "absent class"), ("ovo", "B=1"), ("ovo", "two blocks"), ("binary", "decision"),
            ("binary", "neg_decision"), ("proba", 1, False), ("proba", 4, False), ("proba", 4, True),
            ("proba", 10, False), ("proba", 10, True), ("saturated", 1), ("saturated", 4), ("saturated", 10),
            ("public", "sgd binary"), ("public", "logreg binary"), ("public", "eliminator")}
    want |= {("public", "digits", (n,)) for n in NEW}
    want.add(("public", "digits", tuple(sorted(["roc_auc_ovr", "roc_auc_ovo_weighted", "average_precision",
                                                "f1_weighted"]))))
    assert RAN == want, sorted(map(str, want - RAN))
