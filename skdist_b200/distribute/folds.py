"""Cross-validation layout of the device path: one int8 fold id per row instead of the reference's
per-task (train, test) index arrays (ref search.py:378-383), and the class encoding of the target
shared by the fold allocation and the estimator families."""
import numpy as np

def _fold_ids(cv_splitted, n_samples):
    """Turn the list of (train, test) index arrays (ref search.py:379) into one fold id per
    row.  Requires what KFold / StratifiedKFold / GroupKFold / LeaveOneGroupOut produce: test
    sets partition the rows and each train set is the complement of its test set."""
    if len(cv_splitted) > 127:
        raise NotImplementedError("more than 127 cv splits are not supported on the device path")
    fold = np.full(n_samples, -1, dtype=np.int8)
    for k, (train, test) in enumerate(cv_splitted):
        test = np.asarray(test)
        if np.any(fold[test] != -1):
            raise NotImplementedError(
                "cv splits with overlapping test sets (e.g. ShuffleSplit, RepeatedKFold) are not "
                "supported on the device path")
        fold[test] = k
        if len(train) + len(test) != n_samples:
            raise NotImplementedError(
                "cv splits whose train set is not the complement of the test set are not "
                "supported on the device path")
    if np.any(fold < 0):
        raise NotImplementedError("cv splits must cover every row exactly once on the device path")
    for k, (train, test) in enumerate(cv_splitted):
        if np.any(fold[np.asarray(train)] == k):
            raise NotImplementedError("cv train/test sets overlap")
    return fold


def _train_codes(fold):
    """Scoring codes of the device scoring calls that select the training rows of every column (the rows
    outside its held-out fold `fold`): -3 - fold, as int32."""
    return (-3 - fold).astype(np.int32)


def _train_rows(fold, train_rows, f):
    """Training rows of fold f of a layout (-1: all rows) in the order a fit takes them: train_rows[f], the
    splitter's order, when given, else the rows outside fold f in ascending order."""
    if f < 0:
        return np.arange(len(fold))
    if train_rows is not None and train_rows[f] is not None:
        return np.asarray(train_rows[f])
    return np.flatnonzero(fold != f)


class _TargetCodes:
    """One hash pass over a 1-d integer / bool target: `codes` numbers the classes by order of first
    appearance (what StratifiedKFold's `_make_test_folds` works on), `classes` are the sorted labels and
    `y_class` the index of every row's label in them (what `np.unique` + `searchsorted` give, without
    the sort over the rows)."""

    def __init__(self, y):
        import pandas as pd
        self.y = y
        self.codes, uniques = pd.factorize(y)
        uniques = np.asarray(uniques, dtype=y.dtype)
        order = np.argsort(uniques, kind="stable")
        self.classes = uniques[order]
        rank = np.empty(len(order), dtype=np.int32)
        rank[order] = np.arange(len(order), dtype=np.int32)
        self.y_class = rank[self.codes]


def _encode_target(y):
    """_TargetCodes for targets the fast path covers (1-d integer / bool arrays), else None."""
    y1 = np.asarray(y) if y is not None else None
    if y1 is None or y1.ndim != 1 or y1.dtype.kind not in "biu" or len(y1) == 0:
        return None
    return _TargetCodes(y1)


def _classes_and_ids(y, enc=None):
    """(sorted class labels, int32 class id per row)."""
    if enc is not None and enc.y is y:
        return enc.classes, enc.y_class
    classes = np.unique(y)
    return classes, np.searchsorted(classes, y).astype(np.int32)


def _cv_fold_ids(cv, X, y, groups, n_samples, enc=None, train_orders=None):
    """(fold id per row, n_splits) of a cross-validator.  The generic route materialises every
    (train, test) index pair like the reference does (search.py:379) and converts them; the two
    splitters `check_cv` produces for an integer `cv` -- unshuffled `StratifiedKFold` / `KFold` -- are
    restated directly (no per-split index arrays, no sorts over the rows), fold for fold what
    SK/model_selection/_split.py:774-841 (`_make_test_folds`) and :531-547 (`_iter_test_indices`) give.
    `enc` (a _TargetCodes of y) saves the hash pass when the caller already has it.  A list passed as
    `train_orders` receives the train index arrays of the splits when the splits were materialised (else
    every split's train rows are its complement in ascending order, as the two restated splitters give)."""
    from sklearn.model_selection import KFold, StratifiedKFold
    if type(cv) is KFold and not cv.shuffle and groups is None:
        k = cv.n_splits
        if k > n_samples or k > 127:      # scikit-learn's own error / the int8 fold-id limit of _fold_ids
            return _fold_ids(list(cv.split(X, y, groups)), n_samples), k
        sizes = np.full(k, n_samples // k, dtype=np.int64)
        sizes[: n_samples % k] += 1
        return np.repeat(np.arange(k, dtype=np.int8), sizes), k
    if type(cv) is StratifiedKFold and not cv.shuffle and groups is None and y is not None:
        k = cv.n_splits
        if enc is None or enc.y is not y:
            enc = _encode_target(y)
        if enc is not None and k <= 127:
            y_encoded = enc.codes                             # classes numbered by order of appearance
            counts = np.bincount(y_encoded)
            if counts.min() >= k:                             # otherwise: scikit-learn's own warnings / errors
                # y_order = sorted codes: class c occupies positions [start_c, start_c + counts[c]); fold i
                # takes the positions congruent to i modulo k, class by class in original row order:
                # alloc[i] = #{p in [start, start + count): p mod k == i}, in closed form
                starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
                fold = np.empty(n_samples, dtype=np.int8)
                folds = np.arange(k, dtype=np.int64)
                for c in range(len(counts)):
                    s0, cnt = int(starts[c]), int(counts[c])
                    alloc = (s0 + cnt - 1 - folds) // k - (s0 - 1 - folds) // k
                    fold[np.flatnonzero(y_encoded == c)] = np.repeat(np.arange(k, dtype=np.int8), alloc)
                return fold, k
    cv_splitted = list(cv.split(X, y, groups))
    if train_orders is not None:
        train_orders[:] = [np.asarray(train) for train, _ in cv_splitted]
    return _fold_ids(cv_splitted, n_samples), len(cv_splitted)


def _cv_fold_groups(cv, X, y, groups, n_samples, enc=None, train_orders=None):
    """Fold-id layouts for ANY cross-validator whose train sets are the complements of its test sets
    (ShuffleSplit, StratifiedShuffleSplit, RepeatedKFold, RepeatedStratifiedKFold, LeavePOut,
    PredefinedSplit, Group* ... as well as the partitions `_cv_fold_ids` handles directly).

    Returns (layouts, n_splits): every layout is (fold id per row int8, n_folds, split indices) -- a
    set of splits with pairwise disjoint test sets; split `split indices[k]` holds out the rows with
    fold id k, rows in none of the layout's test sets carry the extra id `n_folds - 1` that no column
    holds out.  A partition is one layout (no extra id); ShuffleSplit(n) is n layouts of one split.
    The search re-stages the fold ids (n bytes) per layout; X stays staged.  Splitters whose train set
    is not the complement of the test set (TimeSeriesSplit) have no device path.  `train_orders`: as in
    `_cv_fold_ids`."""
    try:
        fold, n_splits = _cv_fold_ids(cv, X, y, groups, n_samples, enc, train_orders)
        return [(fold, n_splits, list(range(n_splits)))], n_splits
    except NotImplementedError:
        pass
    cv_splitted = list(cv.split(X, y, groups))
    if train_orders is not None:
        train_orders[:] = [np.asarray(train) for train, _ in cv_splitted]
    n_splits = len(cv_splitted)
    layouts = []       # [used mask, fold ids, split indices]
    for s, (train, test) in enumerate(cv_splitted):
        train, test = np.asarray(train), np.asarray(test)
        if len(train) + len(test) != n_samples or len(np.intersect1d(train, test, assume_unique=False)):
            raise NotImplementedError(
                "cv splits whose train set is not the complement of the test set (e.g. TimeSeriesSplit) "
                "are not supported on the device path")
        for lay in layouts:
            if len(lay[2]) < 126 and not np.any(lay[0][test]):
                break
        else:
            lay = [np.zeros(n_samples, bool), np.full(n_samples, -1, dtype=np.int8), []]
            layouts.append(lay)
        lay[1][test] = len(lay[2])
        lay[0][test] = True
        lay[2].append(s)
    out = []
    for used, fold, idx in layouts:
        k = len(idx)
        if np.all(used):
            out.append((fold, k, idx))
        else:
            fold = fold.copy()
            fold[~used] = k            # never held out
            out.append((fold, k + 1, idx))
    return out, n_splits
