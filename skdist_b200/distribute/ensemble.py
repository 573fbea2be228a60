"""Distributed tree ensembles on H100 GPUs.

Drop-in for /root/reference/skdist/distribute/ensemble.py (class name, constructor signature with
``sc`` FIRST, fitted attributes).  The reference fans `_build_trees` (ensemble.py:68-109) out over
Spark, one task per tree seed (ensemble.py:278-322).  Here every tree is built by one persistent
CTA of `forest_build_kernel` (csrc/forest.cu); the host draws exactly the random numbers the
reference draws (per-tree seeds ensemble.py:278, bootstrap indices ensemble.py:51-55, splitter seed
SK/tree/_splitter.pyx:155) and wraps the returned node arrays into genuine scikit-learn
`DecisionTreeClassifier` objects, so `estimators_`, `predict`, `predict_proba` behave as before and
the tree structure is bit-identical under a fixed `random_state`.
"""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from sklearn.ensemble import (ExtraTreesClassifier, ExtraTreesRegressor, RandomForestClassifier, RandomTreesEmbedding,
                              RandomForestRegressor)
from sklearn.tree import (DecisionTreeClassifier, DecisionTreeRegressor, ExtraTreeClassifier,
                          ExtraTreeRegressor)
from sklearn.tree._tree import NODE_DTYPE, Tree
from sklearn.utils import check_random_state

from .. import parallel
from ..bootstrap import bootstrap_counts
from ..engine import get_engine
from .base import _parse_partitions, _ScParamMixin
from .validation import _check_estimator

__all__ = ["DistRandomForestClassifier", "DistExtraTreesClassifier", "DistRandomForestRegressor",
           "DistExtraTreesRegressor", "DistRandomTreesEmbedding", "get_single_oof", "get_oof"]

MAX_RAND_SEED = np.iinfo(np.int32).max     # ref ensemble.py:38
RAND_R_MAX = 2147483647                    # SK/tree/_utils.pxd


def _tree_inputs(state, n_samples, bootstrap):
    """What `_build_trees` (ref ensemble.py:68-109) derives from one tree seed: the bootstrap
    multiplicities used as sample_weight and the splitter's xorshift seed."""
    if bootstrap:
        indices = check_random_state(state).randint(0, n_samples, n_samples)      # ref :51-55
        counts = np.bincount(indices, minlength=n_samples)
        if counts.max() > 255:
            raise NotImplementedError("a bootstrap multiplicity above 255 does not fit the device format")
        counts = counts.astype(np.uint8)
    else:
        counts = np.ones(n_samples, np.uint8)
    rand_r_state = check_random_state(state).randint(0, RAND_R_MAX)                 # SK/tree/_splitter.pyx:155
    return counts, np.uint32(rand_r_state)


def _make_sklearn_tree(template_params, state, arrays, n_features, n_classes, max_features_,
                       tree_cls=DecisionTreeClassifier):
    """A fitted DecisionTreeClassifier / ExtraTreeClassifier holding the device-built tree (same
    attributes as SK/tree/_classes.py:_fit leaves behind)."""
    m = arrays["left"].shape[0]
    if "nodes" in arrays:       # the library filled scikit-learn's node records directly
        t = Tree(n_features, np.array([n_classes], dtype=np.intp), 1)
        t.__setstate__({"max_depth": int(arrays["max_depth"]), "node_count": m, "nodes": arrays["nodes"],
                        "values": np.ascontiguousarray(arrays["value"].reshape(m, 1, n_classes))})
        return _finish_tree(t, template_params, state, n_features, n_classes, max_features_, tree_cls)
    nodes = np.zeros(m, dtype=NODE_DTYPE)
    nodes["left_child"] = arrays["left"]
    nodes["right_child"] = arrays["right"]
    nodes["feature"] = arrays["feature"]
    nodes["threshold"] = arrays["threshold"]
    nodes["impurity"] = arrays["impurity"]
    nodes["n_node_samples"] = arrays["n_node_samples"]
    nodes["weighted_n_node_samples"] = arrays["weighted_n_node_samples"]
    nodes["missing_go_to_left"] = arrays["missing_go_to_left"]
    t = Tree(n_features, np.array([n_classes], dtype=np.intp), 1)
    t.__setstate__({"max_depth": int(arrays["max_depth"]), "node_count": m, "nodes": nodes,
                    "values": np.ascontiguousarray(arrays["value"].reshape(m, 1, n_classes))})
    return _finish_tree(t, template_params, state, n_features, n_classes, max_features_, tree_cls)


def _rows(X, idx):
    return X.iloc[idx] if hasattr(X, "iloc") else X[idx]


def get_single_oof(clf, X, y, train_index, test_index):
    """Out-of-fold probabilities of one split (ref ensemble.py:112-127): fit on the train rows, `predict_proba`
    on the test rows; `clf` is any classifier -- a Dist* forest fits on the device."""
    clf.fit(_rows(X, train_index), y[train_index])
    return test_index, clf.predict_proba(_rows(X, test_index))


def get_oof(clf, X, y, n_splits=5):
    """Out-of-fold probabilities over an unshuffled KFold, then a fit on everything (ref ensemble.py:130-151).
    Returns (clf fitted on all rows, [n, n_classes] out-of-fold probabilities)."""
    from sklearn.model_selection import KFold
    oof = np.zeros((y.shape[0], len(np.unique(y))))
    for train_index, test_index in KFold(n_splits=n_splits).split(X):
        _, oof[test_index] = get_single_oof(clf, X, y, train_index, test_index)
    clf.fit(X, y)
    return clf, oof


def _quantile_codes(X, max_bins):
    """Opt-in histogram mode for continuous features (env SKDIST_B200_FOREST_MAX_BINS = 2 ... 256).

    The exact splitter of the device path needs features with at most 256 distinct values.  Every feature
    with more than `max_bins` distinct values is replaced by its equal-count bin code 0 .. B-1 (ties stay in
    one bin), the forest is built on the codes -- exactly the trees scikit-learn builds on the coded matrix --
    and `_remap_thresholds` then moves every threshold back to raw units (the midpoint between the largest
    value of the left bin and the smallest of the right bin, scikit-learn's own rule for two adjacent values),
    so the fitted trees route raw rows exactly as they route the coded ones.  This is the usual histogram
    approximation (the candidate thresholds of such a feature are the B-1 bin boundaries, not every pair of
    adjacent values): NOT bit-identical to the reference on such data, hence opt-in.

    Returns (X with the coded columns, table [d x max_bins] float64 of raw thresholds after code c -- NaN
    rows for untouched features) or (X, None) when no feature needs it."""
    n, d = X.shape
    table = None
    out = X
    for f in range(d):
        srt = np.sort(X[:, f])
        n_distinct = 1 + int(np.count_nonzero(srt[1:] != srt[:-1]))
        if n_distinct <= max_bins:
            continue
        pos = (np.arange(1, max_bins, dtype=np.int64) * n) // max_bins
        edges = np.unique(srt[pos])                                  # inclusive upper edges; the last bin is open
        code = np.searchsorted(edges, X[:, f], side="left")
        present, code = np.unique(code, return_inverse=True)         # dense codes (the top edge can be the maximum)
        cnt = np.bincount(code, minlength=len(present))
        end = np.cumsum(cnt)
        hi = srt[end - 1].astype(np.float64)                         # codes are monotone in the value
        lo = srt[end - cnt].astype(np.float64)
        thr = hi[:-1] / 2.0 + lo[1:] / 2.0                           # SK/tree/_splitter.pyx: midpoint in float64 ...
        thr = np.where(thr == lo[1:], hi[:-1], thr)                  # ... that falls back to the left value
        if table is None:
            table = np.full((d, max_bins), np.nan)
            out = X.copy()
        table[f, :len(thr)] = thr
        out[:, f] = code.astype(np.float32)
    return out, table


def _remap_thresholds(arrays, table):
    """Thresholds of the coded features (any cut between two codes a < b present in the node: the device
    reports their midpoint, the random splitter a uniform draw in [a, b)) back to raw units: the boundary
    after code floor(t), which lies in [a, b)."""
    if "nodes" in arrays:
        feat, thr = arrays["nodes"]["feature"], arrays["nodes"]["threshold"]
    else:
        feat, thr = arrays["feature"], arrays["threshold"]
    coded = ~np.isnan(table[:, 0])
    sel = np.flatnonzero((feat >= 0) & coded[np.maximum(feat, 0)])
    if len(sel):
        c = np.clip(np.floor(thr[sel]).astype(np.int64), 0, table.shape[1] - 1)
        thr[sel] = table[feat[sel], c]
    return arrays


def _sort_switch():
    """SKDIST_B200_FOREST_SORT: unset (the best splitter refuses a feature with more than 256 distinct values)
    or 1 (such features are split by sorting their values on the device: scikit-learn's trees)."""
    v = os.environ.get("SKDIST_B200_FOREST_SORT")
    if v is None:
        return False
    if v != "1":
        raise ValueError("SKDIST_B200_FOREST_SORT must be unset or 1, not %r" % v)
    return True


def _finish_tree(t, template_params, state, n_features, n_classes, max_features_, tree_cls):
    est = tree_cls(**template_params)
    est.set_params(random_state=int(state))
    est.n_features_in_ = n_features
    est.n_outputs_ = 1
    if issubclass(tree_cls, DecisionTreeClassifier):
        est.classes_ = np.arange(n_classes, dtype=np.float64)
        est.n_classes_ = n_classes
    est.max_features_ = max_features_
    est.tree_ = t
    return est


# classifier criteria with a device path -> the library's criterion code (skd_stage_forest_criterion)
_CLASS_CRITERIA = {"gini": 0, "entropy": 1, "log_loss": 1}

_LIMITS = """

    Limits of the device path (checked when the trees are built; `NotImplementedError` otherwise, there
    is no CPU fallback): by default the best splitter (RandomForest) takes features with at most 256 distinct
    values (it works on per-feature value histograms: data on a lattice, counts, categorical codes, quantised
    measurements).  `SKDIST_B200_FOREST_SORT=1` lets it take continuous float features too: a feature with
    more distinct values is split by sorting the node's raw float32 values on the device, which gives
    scikit-learn's trees (features with at most 256 distinct values still take the histograms).  The
    histogram mode `SKDIST_B200_FOREST_MAX_BINS=<2..256>` instead replaces such features by equal-count bin
    codes and maps the thresholds back to raw units -- the trees scikit-learn builds on the coded matrix, not
    bit-identical to the reference on the raw one; the two switches exclude each other.  The random splitter (ExtraTrees, RandomTreesEmbedding)
    reads the raw float32 values and takes any finite X (with the switch set it, too, is fitted on the coded
    matrix), at most 16 classes, at most
    384 features, bootstrap multiplicities up to 255, no missing values, `criterion` gini, entropy or
    log_loss (classifiers; the entropy alias, fitted by the general tree builder, whose `impurity` arrays are
    formed on the host with scikit-learn's log) or squared error (regressors), no `max_leaf_nodes`, `sample_weight` or multi-output targets; `class_weight` (classifiers) may
    be a dict, "balanced" or "balanced_subsample", not "subsample" or a list of dicts."""

_CLASS_WEIGHT = """

    `class_weight` follows the reference's per-tree task (ref ensemble.py:68-109): tree t is fitted with
    sample_weight = (bootstrap multiplicity) * cw[y], cw from scikit-learn's `compute_class_weight` on all of
    y ("balanced", dict: absent classes 1.0) or, for "balanced_subsample" with bootstrap, on the tree's
    bootstrap sample (absent classes 0).  Rows of weight 0 leave the tree.  scikit-learn 1.9's own
    RandomForestClassifier differs for a dict or "balanced" with bootstrap=True: it draws the bootstrap
    with the class weights as sampling probabilities and fits on plain multiplicities; with
    "balanced_subsample", or bootstrap=False, the two agree.  The trees equal the reference's bit for bit
    when the weighted sums are exact (integer or dyadic weights); otherwise node statistics agree to
    rounding and a split can differ only between candidates whose Gini proxies lie within rounding of
    each other (DESIGN.md §4)."""


class _DistForestClassifier(_ScParamMixin):
    """Shared fit of the forest classifiers (ref DistBaseForest.fit, ensemble.py:177-336).
    Subclasses set `_splitter` (0 best / 1 random) and `_tree_cls`."""

    _splitter = 0
    _tree_cls = DecisionTreeClassifier
    _regression = False

    def _init_params(self, sc, partitions, n_estimators, criterion, max_depth, min_samples_split,
                     min_samples_leaf, min_weight_fraction_leaf, max_features, max_leaf_nodes,
                     min_impurity_decrease, min_impurity_split, bootstrap, oob_score, n_jobs, random_state,
                     verbose, warm_start, class_weight):
        self.sc = sc
        self.partitions = partitions
        self.n_estimators = n_estimators
        self.criterion = criterion
        self.max_depth = max_depth
        self.min_samples_split = min_samples_split
        self.min_samples_leaf = min_samples_leaf
        self.min_weight_fraction_leaf = min_weight_fraction_leaf
        self.max_features = max_features
        self.max_leaf_nodes = max_leaf_nodes
        self.min_impurity_decrease = min_impurity_decrease
        self.min_impurity_split = min_impurity_split
        self.bootstrap = bootstrap
        self.oob_score = oob_score
        self.n_jobs = n_jobs
        self.random_state = random_state
        self.verbose = verbose
        self.warm_start = warm_start
        self.class_weight = class_weight
        # attributes newer scikit-learn forests expect on the instance
        self.ccp_alpha = 0.0
        self.max_samples = None
        self.monotonic_cst = None
        self.estimator = self._tree_cls()
        self.estimator_params = ("criterion", "max_depth", "min_samples_split", "min_samples_leaf",
                                 "min_weight_fraction_leaf", "max_features", "max_leaf_nodes",
                                 "min_impurity_decrease", "random_state", "ccp_alpha", "monotonic_cst")

    @classmethod
    def _get_param_names(cls):
        return sorted(["sc", "partitions", "n_estimators", "criterion", "max_depth", "min_samples_split",
                       "min_samples_leaf", "min_weight_fraction_leaf", "max_features", "max_leaf_nodes",
                       "min_impurity_decrease", "min_impurity_split", "bootstrap", "oob_score", "n_jobs",
                       "random_state", "verbose", "warm_start", "class_weight"])

    def _resolved(self, n_features):
        bad = []
        if self._regression:
            if self.criterion not in ("mse", "squared_error"):   # "mse" is the reference era's name
                bad.append("criterion=%r (only 'squared_error' / 'mse')" % self.criterion)
        elif not (isinstance(self.criterion, str) and self.criterion in _CLASS_CRITERIA):
            bad.append("criterion=%r (only 'gini', 'entropy' / 'log_loss')" % (self.criterion,))
        if self.max_leaf_nodes is not None:
            bad.append("max_leaf_nodes (best-first builder)")
        cw = self.class_weight
        if cw is not None and not (isinstance(cw, dict) or cw in ("balanced", "balanced_subsample")):
            bad.append("class_weight=%r (dict, 'balanced' or 'balanced_subsample'; 'subsample' is a removed "
                       "scikit-learn mode, a list of dicts is multi-output)" % (cw,))
        if self.min_impurity_split is not None:
            bad.append("min_impurity_split")
        if bad:
            raise NotImplementedError("forest configuration without a device path: " + ", ".join(bad))
        mf = self.max_features
        if mf == "auto" and self._regression:            # 'auto' meant all features for regressors (ref era)
            mf_i = n_features
        elif mf in ("auto", "sqrt"):                     # ... and sqrt for classifiers
            mf_i = max(1, int(np.sqrt(n_features)))
        elif mf == "log2":
            mf_i = max(1, int(np.log2(n_features)))
        elif mf is None:
            mf_i = n_features
        elif isinstance(mf, (int, np.integer)):
            mf_i = int(mf)
        else:
            mf_i = max(1, int(mf * n_features))
        max_depth = np.iinfo(np.int32).max if self.max_depth is None else int(self.max_depth)
        mss = self.min_samples_split
        msl = self.min_samples_leaf
        return mf_i, max_depth, mss, msl

    def _class_weights(self, y):
        """(per-class weights or None, balanced_subsample) of the reference's per-tree sample_weight
        (ref ensemble.py:68-109, 229-238)."""
        cw = self.class_weight
        if cw is None:
            return None, False
        if isinstance(cw, str) and cw == "balanced_subsample":
            if self.bootstrap:
                return None, True                     # per tree, on the device, from its bootstrap class counts
            cw = "balanced"                           # no bootstrap: the sample is all of y
        from sklearn.utils.class_weight import compute_class_weight
        w = np.asarray(compute_class_weight(cw, classes=self.classes_, y=y), dtype=np.float64)
        if not (np.all(np.isfinite(w)) and np.all(w >= 0)):
            raise ValueError("class_weight must be finite and >= 0")
        if not np.any(w > 0):
            raise ValueError("class_weight gives every class weight 0")
        return w, False

    def fit(self, X, y, sample_weight=None):
        """Build the forest (ref ensemble.py:177-336)."""
        if sample_weight is not None:
            raise NotImplementedError("sample_weight is not supported on the device path")
        _check_estimator(self, verbose=self.verbose)
        X = np.ascontiguousarray(X, dtype=np.float32)                 # ref :200 (check_array dtype=float32)
        y = np.asarray(y)
        if y.ndim != 1:
            raise NotImplementedError("multi-output forests have no device path")
        n, d = X.shape
        self.n_features_in_ = d
        self.n_features_ = d                                           # ref :210 (the attribute's pre-1.0 name)
        self.n_outputs_ = 1
        if self._regression:
            y_reg = np.ascontiguousarray(y, dtype=np.float64)          # SK/ensemble/_forest.py: y = DOUBLE
            y_enc = np.zeros(len(y), np.int32)
            self.n_classes_ = 1
        else:
            y_reg = None
            self.classes_, y_enc = np.unique(y, return_inverse=True)   # ref :229 (_validate_y_class_weight)
            self.n_classes_ = len(self.classes_)
        mf_i, max_depth, mss, msl = self._resolved(d)
        cw, cw_subsample = (None, False) if self._regression else self._class_weights(y)
        weighted = cw is not None or cw_subsample
        if not isinstance(mss, (int, np.integer)):
            mss = max(2, int(np.ceil(mss * n)))
        if not isinstance(msl, (int, np.integer)):
            msl = max(1, int(np.ceil(msl * n)))
        mss = max(int(mss), 2 * int(msl))
        min_weight_leaf = self.min_weight_fraction_leaf * n
        random_state = check_random_state(self.random_state)
        # warm start (ref :250-272): keep the fitted trees, draw past their seeds, grow only the new ones
        kept = list(self.estimators_) if (self.warm_start and hasattr(self, "estimators_")) else []
        n_more = self.n_estimators - len(kept)
        if n_more < 0:
            raise ValueError("n_estimators=%d must be larger or equal to len(estimators_)=%d when warm_start==True"
                             % (self.n_estimators, len(kept)))
        if n_more == 0:
            import warnings
            warnings.warn("Warm-start fitting without increasing n_estimators does not fit new trees.")
            self.__dict__.pop("sc", None)
            return self
        if kept:
            random_state.randint(MAX_RAND_SEED, size=len(kept))                   # ref :267-269
        states = list(random_state.randint(MAX_RAND_SEED, size=n_more))         # ref :278
        _parse_partitions(self.partitions, n_more)

        rank, world, _ = parallel.dist_info()
        eng = get_engine()
        max_bins = int(os.environ.get("SKDIST_B200_FOREST_MAX_BINS", "0"))
        if max_bins and not 2 <= max_bins <= 256:
            raise ValueError("SKDIST_B200_FOREST_MAX_BINS must be between 2 and 256")
        exact_sort = _sort_switch()
        if exact_sort and max_bins:
            raise ValueError("SKDIST_B200_FOREST_SORT and SKDIST_B200_FOREST_MAX_BINS ask for different trees "
                             "(scikit-learn's exact ones, the histogram approximation); set one of them")
        # the best splitter also takes features with more than 256 distinct values (sort-based splitter)
        splitter = 2 if exact_sort and self._splitter == 0 else self._splitter
        X_dev, bin_table = _quantile_codes(X, max_bins) if max_bins else (X, None)
        try:
            parallel.stage_x_replicated(eng, X_dev)
            eng.stage_labels(y_enc.astype(np.int32))
            eng.stage_folds(None, 0)
        finally:
            del X_dev
        mine = parallel.shard_indices(n_more, rank, world)
        my_states = [states[i] for i in mine]
        crit = "squared_error" if self._regression else self.criterion
        tmpl = dict(criterion=crit, max_depth=self.max_depth, min_samples_split=self.min_samples_split,
                    min_samples_leaf=self.min_samples_leaf, min_weight_fraction_leaf=self.min_weight_fraction_leaf,
                    max_features=(1.0 if self._regression else "sqrt") if self.max_features == "auto"
                    else self.max_features,
                    max_leaf_nodes=self.max_leaf_nodes, min_impurity_decrease=self.min_impurity_decrease)

        # Trees go to the device in chunks (two resident tree builders per SM).  While chunk k is
        # being built, the host draws the bootstrap samples of chunk k+1 and wraps the node arrays
        # of chunk k-1 into scikit-learn trees (ctypes releases the GIL during the device call).
        # (the throughput builder of csrc/forest_fast.cu keeps seven trees per SM resident, the general
        # one two: a chunk is one full wave of the builder that will run)
        # criterion code of the library: 1 = entropy ("log_loss" is scikit-learn's other name for it), which
        # only the general builder runs
        entropy = not self._regression and _CLASS_CRITERIA[self.criterion] == 1
        fast = (not self._regression and not entropy and self._splitter == 0 and self.n_classes_ <= 4
                and d <= 255)
        if cw is not None and fast:       # the library keeps positive dict weights within 2^40 on the throughput builder
            pos = cw[cw > 0]
            fast = bool(pos.max() <= 2.0 ** 40 * pos.min())
        chunk = int(os.environ.get("SKDIST_B200_FOREST_CHUNK", "1036" if fast else "296"))
        chunks = [my_states[i:i + chunk] for i in range(0, len(my_states), chunk)]

        host_threads = max(1, min(64, (os.cpu_count() or 8) // max(world, 1)))

        def prepare(sts):
            # bootstrap multiplicities + splitter seeds of a chunk: the library's host threads restate
            # numpy's legacy generator bit for bit (csrc/bootstrap.cu; `_tree_inputs` is the numpy form)
            return bootstrap_counts(sts, n, bootstrap=self.bootstrap, n_threads=host_threads)

        def build(counts, rs):
            try:
                if weighted:      # one-shot: staged for each chunk's fit (min_weight_leaf per tree: fraction * sum w)
                    eng.stage_forest_class_weights(self.n_classes_, cw, cw_subsample, self.min_weight_fraction_leaf)
                if entropy:       # one-shot as well; Gini fits stage nothing (the library's default)
                    eng.stage_forest_criterion(1)
                return eng.forest_fit(counts, rs, self.n_classes_, mf_i, max_depth, int(mss), int(msl),
                                      float(min_weight_leaf), float(self.min_impurity_decrease),
                                      splitter=splitter, y_regression=y_reg)
            except NotImplementedError as e:
                if "distinct values" in str(e) and not max_bins:
                    raise NotImplementedError(str(e) + "; SKDIST_B200_FOREST_SORT=1 selects scikit-learn's exact "
                                              "trees (sort-based splitter), SKDIST_B200_FOREST_MAX_BINS=256 the "
                                              "histogram approximation (equal-count bins, see the class "
                                              "docstring)") from None
                raise

        def wrap(sts, arrays):
            with ThreadPoolExecutor(max_workers=min(32, max(8, host_threads))) as ex:   # strided field copies release the GIL
                return list(ex.map(lambda sa: _make_sklearn_tree(
                    tmpl, sa[0], sa[1] if bin_table is None else _remap_thresholds(sa[1], bin_table), d,
                    self.n_classes_, mf_i, self._tree_cls), zip(sts, arrays)))

        local = []
        self.device_seconds_ = 0.0
        self.kernel_seconds_ = 0.0
        if chunks:
            with ThreadPoolExecutor(max_workers=1) as dev, ThreadPoolExecutor(max_workers=1) as side:
                nxt = side.submit(prepare, chunks[0])
                pending = None                      # (states, arrays) of the previous chunk, not yet wrapped
                for k, sts in enumerate(chunks):
                    counts, rs = nxt.result()
                    fut = dev.submit(build, counts, rs)
                    if k + 1 < len(chunks):
                        nxt = side.submit(prepare, chunks[k + 1])
                    if pending is not None:
                        local.extend(wrap(*pending))
                    arrays = fut.result()
                    self.device_seconds_ += getattr(eng, "last_forest_seconds", 0.0)
                    self.kernel_seconds_ = getattr(self, "kernel_seconds_", 0.0) + getattr(eng, "last_forest_kernel_seconds", 0.0)
                    pending = (sts, arrays)
                local.extend(wrap(*pending))
        if world > 1:
            # the trees of the other ranks arrive as raw node / value arrays in bounded pieces and are wrapped
            # here (parallel.all_gather_trees: no pickle of the whole forest, optional rank-0-only collection)
            def rebuild(i, depth, nodes, values):
                t = Tree(d, np.array([self.n_classes_], dtype=np.intp), 1)
                t.__setstate__({"max_depth": depth, "node_count": nodes.shape[0], "nodes": nodes,
                                "values": np.ascontiguousarray(values.reshape(nodes.shape[0], 1, -1))})
                return _finish_tree(t, tmpl, states[i], d, self.n_classes_, mf_i, self._tree_cls)
            ests = parallel.all_gather_trees(local, n_more, rank, world, rebuild)
            if any(e is None for e in ests):        # rank-0-only collection: this rank keeps the trees it built
                ests = [e for e in ests if e is not None]
        else:
            ests = local
        self.estimators_ = kept + ests
        self.estimator_ = self._tree_cls()
        self.__dict__.pop("sc", None)                                                     # ref :335
        return self

    def _set_oob_score(self, X, y):
        """The reference overrides this to a no-op (ref ensemble.py:338-340)."""
        return


class DistRandomForestClassifier(_DistForestClassifier, RandomForestClassifier):
    __doc__ = """Same as sklearn `RandomForestClassifier` with every tree built on an H100.
    Constructor mirrors ref ensemble.py:378-422 (``sc`` is the FIRST positional argument).""" + _LIMITS + _CLASS_WEIGHT

    _splitter = 0
    _tree_cls = DecisionTreeClassifier

    def __init__(self, sc=None, partitions="auto", n_estimators=100, criterion="gini", max_depth=None,
                 min_samples_split=2, min_samples_leaf=1, min_weight_fraction_leaf=0.0, max_features="auto",
                 max_leaf_nodes=None, min_impurity_decrease=0.0, min_impurity_split=None, bootstrap=True,
                 oob_score=False, n_jobs=None, random_state=None, verbose=0, warm_start=False,
                 class_weight=None):
        self._init_params(sc, partitions, n_estimators, criterion, max_depth, min_samples_split, min_samples_leaf,
                          min_weight_fraction_leaf, max_features, max_leaf_nodes, min_impurity_decrease,
                          min_impurity_split, bootstrap, oob_score, n_jobs, random_state, verbose, warm_start,
                          class_weight)


class DistExtraTreesClassifier(_DistForestClassifier, ExtraTreesClassifier):
    __doc__ = """Same as sklearn `ExtraTreesClassifier` with every tree built on an H100 (random splitter:
    one uniformly drawn threshold per drawn feature over the raw float32 values, no bootstrap by default;
    continuous features are fitted exactly, scikit-learn's trees bit for bit).
    Constructor mirrors ref ensemble.py:437-478 (``sc`` is the FIRST positional argument).""" + _LIMITS + _CLASS_WEIGHT

    _splitter = 1
    _tree_cls = ExtraTreeClassifier

    def __init__(self, sc=None, partitions="auto", n_estimators=100, criterion="gini", max_depth=None,
                 min_samples_split=2, min_samples_leaf=1, min_weight_fraction_leaf=0.0, max_features="auto",
                 max_leaf_nodes=None, min_impurity_decrease=0.0, min_impurity_split=None, bootstrap=False,
                 oob_score=False, n_jobs=None, random_state=None, verbose=0, warm_start=False,
                 class_weight=None):
        self._init_params(sc, partitions, n_estimators, criterion, max_depth, min_samples_split, min_samples_leaf,
                          min_weight_fraction_leaf, max_features, max_leaf_nodes, min_impurity_decrease,
                          min_impurity_split, bootstrap, oob_score, n_jobs, random_state, verbose, warm_start,
                          class_weight)


class _DistForestRegressor(_DistForestClassifier):
    """Regression flavour of the shared fit: float64 targets, MSE criterion, no class bookkeeping
    (ref DistForestRegressor, ensemble.py:481-517)."""

    _regression = True
    _tree_cls = DecisionTreeRegressor

    def _init_reg(self, sc, partitions, n_estimators, criterion, max_depth, min_samples_split, min_samples_leaf,
                  min_weight_fraction_leaf, max_features, max_leaf_nodes, min_impurity_decrease,
                  min_impurity_split, bootstrap, oob_score, n_jobs, random_state, verbose, warm_start):
        self._init_params(sc, partitions, n_estimators, criterion, max_depth, min_samples_split, min_samples_leaf,
                          min_weight_fraction_leaf, max_features, max_leaf_nodes, min_impurity_decrease,
                          min_impurity_split, bootstrap, oob_score, n_jobs, random_state, verbose, warm_start, None)
        del self.class_weight

    @classmethod
    def _get_param_names(cls):
        return sorted(["sc", "partitions", "n_estimators", "criterion", "max_depth", "min_samples_split",
                       "min_samples_leaf", "min_weight_fraction_leaf", "max_features", "max_leaf_nodes",
                       "min_impurity_decrease", "min_impurity_split", "bootstrap", "oob_score", "n_jobs",
                       "random_state", "verbose", "warm_start"])

    class_weight = None      # read by the shared validation; regressors have no such parameter


class DistRandomForestRegressor(_DistForestRegressor, RandomForestRegressor):
    __doc__ = """Same as sklearn `RandomForestRegressor` with every tree built on an H100.
    Constructor mirrors ref ensemble.py:531-572 (``sc`` FIRST; criterion "mse" = squared error).""" + _LIMITS

    _splitter = 0
    _tree_cls = DecisionTreeRegressor

    def __init__(self, sc=None, partitions="auto", n_estimators=100, criterion="mse", max_depth=None,
                 min_samples_split=2, min_samples_leaf=1, min_weight_fraction_leaf=0.0, max_features="auto",
                 max_leaf_nodes=None, min_impurity_decrease=0.0, min_impurity_split=None, bootstrap=True,
                 oob_score=False, n_jobs=None, random_state=None, verbose=0, warm_start=False):
        self._init_reg(sc, partitions, n_estimators, criterion, max_depth, min_samples_split, min_samples_leaf,
                       min_weight_fraction_leaf, max_features, max_leaf_nodes, min_impurity_decrease,
                       min_impurity_split, bootstrap, oob_score, n_jobs, random_state, verbose, warm_start)


class DistExtraTreesRegressor(_DistForestRegressor, ExtraTreesRegressor):
    __doc__ = """Same as sklearn `ExtraTreesRegressor` with every tree built on an H100 (random splitter over
    the raw float32 values: continuous features need no binning).
    Constructor mirrors ref ensemble.py:584-616.""" + _LIMITS

    _splitter = 1
    _tree_cls = ExtraTreeRegressor

    def __init__(self, sc=None, partitions="auto", n_estimators=100, criterion="mse", max_depth=None,
                 min_samples_split=2, min_samples_leaf=1, min_weight_fraction_leaf=0.0, max_features="auto",
                 max_leaf_nodes=None, min_impurity_decrease=0.0, min_impurity_split=None, bootstrap=False,
                 oob_score=False, n_jobs=None, random_state=None, verbose=0, warm_start=False):
        self._init_reg(sc, partitions, n_estimators, criterion, max_depth, min_samples_split, min_samples_leaf,
                       min_weight_fraction_leaf, max_features, max_leaf_nodes, min_impurity_decrease,
                       min_impurity_split, bootstrap, oob_score, n_jobs, random_state, verbose, warm_start)


class DistRandomTreesEmbedding(_DistForestRegressor, RandomTreesEmbedding):
    __doc__ = """Same as sklearn `RandomTreesEmbedding` with every tree built on an H100: totally random trees
    (`ExtraTreeRegressor`, one drawn feature per node, uniformly drawn threshold) fitted on uniform random
    targets, then the one-hot code of the leaf every row lands in.  Constructor and `fit` / `fit_transform` /
    `transform` mirror ref ensemble.py:619-708 (``sc`` is the FIRST positional argument).  With one feature
    drawn per node the split does not depend on the criterion, so the trees -- and the embedding -- are
    scikit-learn's bit for bit.""" + _LIMITS

    _splitter = 1
    _tree_cls = ExtraTreeRegressor
    criterion = "squared_error"        # ref :633 ("mse")
    max_features = 1                   # ref :634

    def __init__(self, sc=None, partitions="auto", n_estimators=100, max_depth=5, min_samples_split=2,
                 min_samples_leaf=1, min_weight_fraction_leaf=0.0, max_leaf_nodes=None, min_impurity_decrease=0.0,
                 min_impurity_split=None, sparse_output=True, n_jobs=None, random_state=None, verbose=0,
                 warm_start=False):
        self._init_reg(sc, partitions, n_estimators, "squared_error", max_depth, min_samples_split, min_samples_leaf,
                       min_weight_fraction_leaf, 1, max_leaf_nodes, min_impurity_decrease, min_impurity_split,
                       False, False, n_jobs, random_state, verbose, warm_start)
        # class attributes in the reference, not constructor parameters
        del self.criterion, self.max_features, self.bootstrap, self.oob_score
        self.sparse_output = sparse_output

    bootstrap = False
    oob_score = False

    @classmethod
    def _get_param_names(cls):
        return sorted(["sc", "partitions", "n_estimators", "max_depth", "min_samples_split", "min_samples_leaf",
                       "min_weight_fraction_leaf", "max_leaf_nodes", "min_impurity_decrease", "min_impurity_split",
                       "sparse_output", "n_jobs", "random_state", "verbose", "warm_start"])

    def _set_oob_score(self, X, y):
        raise NotImplementedError("OOB score not supported by tree embedding")      # ref :685-686

    def fit(self, X, y=None, sample_weight=None):
        self.fit_transform(X, y, sample_weight=sample_weight)                        # ref :688-691
        return self

    def fit_transform(self, X, y=None, sample_weight=None):
        """ref :693-710: uniform random targets from `random_state`, the forest fit, one-hot of the leaves."""
        from sklearn.preprocessing import OneHotEncoder
        X = np.ascontiguousarray(X, dtype=np.float32)
        rnd = check_random_state(self.random_state)
        y = rnd.uniform(size=X.shape[0])
        _DistForestClassifier.fit(self, X, y, sample_weight=sample_weight)
        self.one_hot_encoder_ = OneHotEncoder(sparse_output=self.sparse_output)
        out = self.one_hot_encoder_.fit_transform(self.apply(X))
        self._n_features_out = out.shape[1]
        return out
