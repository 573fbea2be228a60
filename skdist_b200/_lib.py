"""ctypes binding of libskdist_b200.so (the C-ABI in include/skdist_b200.h).

There is NO CPU fallback: if the library is missing or no H100 is visible the
calls raise.  The library is built in-tree by ``skdist_b200._build`` /
``__graft_entry__.build()``.
"""
import ctypes
import os

import numpy as np

from . import _build

_c = ctypes
_LIB = None


class SkdError(RuntimeError):
    pass


def _p(dtype):
    return np.ctypeslib.ndpointer(dtype=dtype, flags="C_CONTIGUOUS")


SYMBOLS = {
    # name: (restype, argtypes)
    "skd_version": (_c.c_int, []),
    "skd_device_count": (_c.c_int, []),
    "skd_ctx_create": (_c.c_int, [_c.c_int, _c.POINTER(_c.c_void_p)]),
    "skd_ctx_destroy": (_c.c_int, [_c.c_void_p]),
    "skd_last_error": (_c.c_char_p, [_c.c_void_p]),
    "skd_stage_x": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_int64, _c.c_int64]),
    "skd_stage_x_device": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_int64, _c.c_int64]),
    "skd_staged_x": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    "skd_stage_x_begin": (_c.c_int, [_c.c_void_p, _c.c_int64, _c.c_int64, _c.c_int64, _c.c_void_p, _c.c_void_p]),
    "skd_stage_x_rows": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_int64, _c.c_int64]),
    "skd_stage_x_commit": (_c.c_int, [_c.c_void_p]),
    "skd_stage_labels": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64]),
    "skd_stage_targets": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64]),
    "skd_stage_folds": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_int32]),
    "skd_stage_column_masks": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p]),
    "skd_stage_row_bits": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_int64]),
    "skd_stage_class_weights": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p]),
    "skd_stage_forest_class_weights": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_int32, _c.c_double]),
    "skd_stage_forest_criterion": (_c.c_int, [_c.c_void_p, _c.c_int32]),
    "skd_logreg_fit_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                        _c.c_void_p, _c.c_int32, _c.c_double, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                        _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_logreg_loss_grad": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                        _c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p]),
    "skd_linear_score_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                          _c.c_void_p, _c.c_void_p]),
    "skd_logreg_multinomial_fit_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                                    _c.c_int32, _c.c_double, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                                    _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_logreg_multinomial_loss_grad": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                                    _c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p]),
    "skd_multinomial_score_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                               _c.c_void_p, _c.c_void_p]),
    "skd_multinomial_confusion_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                                   _c.c_void_p]),
    "skd_linear_auc_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                        _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    "skd_linear_rank_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                         _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    "skd_linear_logloss_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                            _c.c_void_p, _c.c_void_p, _c.c_void_p]),
    "skd_ridge_fit_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_int32,
                                       _c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_sgd_fit_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_int32, _c.c_double, _c.c_int32,
                                     _c.c_int32, _c.c_double, _c.c_int32, _c.c_uint32, _c.c_int32, _c.c_double,
                                     _c.c_double, _c.c_double, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                     _c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_sgd_fit_groups": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                      _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_int32, _c.c_int32,
                                      _c.c_int32, _c.c_double, _c.c_int32, _c.c_int32, _c.c_double, _c.c_double,
                                      _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                      _c.POINTER(_c.c_double)]),
    "skd_bootstrap_counts": (_c.c_int, [_c.c_int32, _c.c_void_p, _c.c_int64, _c.c_int32, _c.c_void_p, _c.c_void_p,
                                        _c.c_int32]),
    "skd_forest_fit": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_int32, _c.c_int32,
                                  _c.c_int32, _c.c_int32, _c.c_int32, _c.c_double, _c.c_double, _c.c_int32, _c.c_void_p,
                                  _c.POINTER(_c.c_void_p), _c.POINTER(_c.c_double)]),
    "skd_forest_kernel_seconds": (_c.c_int, [_c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_forest_tree_size": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.POINTER(_c.c_int32), _c.POINTER(_c.c_int32)]),
    "skd_forest_tree_copy": (_c.c_int, [_c.c_void_p, _c.c_int32] + [_c.c_void_p] * 9),
    "skd_forest_tree_nodes": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p]),
    "skd_forest_free": (None, [_c.c_void_p]),
    "skd_linear_r2_batch": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                       _c.c_void_p]),
    "skd_predict_linear": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_int64, _c.c_int64,
                                      _c.c_int32, _c.c_void_p, _c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_forest_predict": (_c.c_int, [_c.c_void_p, _c.c_void_p, _c.c_int64, _c.c_int64, _c.c_int64, _c.c_int32]
                           + [_c.c_void_p] * 6 + [_c.c_int32, _c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_linear_decision": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.c_void_p, _c.c_void_p]),
    "skd_set_kernel": (_c.c_int, [_c.c_void_p, _c.c_int32]),
    "skd_profile": (_c.c_int, [_c.c_void_p, _c.c_int32, _c.POINTER(_c.c_double), _c.POINTER(_c.c_double),
                               _c.POINTER(_c.c_int64), _c.POINTER(_c.c_int64)]),
    "skd_timer_start": (_c.c_int, [_c.c_void_p]),
    "skd_timer_stop": (_c.c_int, [_c.c_void_p, _c.POINTER(_c.c_double)]),
    "skd_get_counters": (_c.c_int, [_c.c_void_p, _c.POINTER(_c.c_int64), _c.POINTER(_c.c_int64),
                                    _c.POINTER(_c.c_int64)]),
    "skd_lbfgs_create": (_c.c_void_p, [_c.c_int32, _c.c_int32, _c.c_int32, _c.c_int32, _c.c_double,
                                       _c.c_double]),
    "skd_lbfgs_x": (_c.POINTER(_c.c_double), [_c.c_void_p]),
    "skd_lbfgs_g": (_c.POINTER(_c.c_double), [_c.c_void_p]),
    "skd_lbfgs_advance": (_c.c_int, [_c.c_void_p, _c.c_double]),
    "skd_lbfgs_nit": (_c.c_int, [_c.c_void_p]),
    "skd_lbfgs_nfev": (_c.c_int, [_c.c_void_p]),
    "skd_lbfgs_state": (None, [_c.c_void_p, _c.c_void_p]),
    "skd_lbfgs_set_state": (None, [_c.c_void_p, _c.c_void_p]),
    "skd_lbfgs_state_bytes": (_c.c_int, []),
    "skd_lbfgs_free": (None, [_c.c_void_p]),
    "skd_lbfgs_dev_create": (_c.c_void_p, [_c.c_void_p, _c.c_int32, _c.c_int32, _c.c_int32, _c.c_int32, _c.c_int32,
                                           _c.c_void_p, _c.c_int32, _c.c_int32, _c.c_int32, _c.c_int32, _c.c_double,
                                           _c.c_double, _c.c_void_p, _c.c_void_p, _c.c_void_p, _c.c_void_p,
                                           _c.c_void_p]),
    "skd_lbfgs_dev_step": (_c.c_int, [_c.c_void_p, _c.c_int32] + [_c.c_void_p] * 8),
    "skd_lbfgs_dev_finish": (_c.c_int, [_c.c_void_p] + [_c.c_void_p] * 4),
    "skd_lbfgs_dev_free": (None, [_c.c_void_p]),
}


def lib_path():
    # SKDIST_B200_LIBPATH: A/B experiments against another build of the same C-ABI
    return os.environ.get("SKDIST_B200_LIBPATH") or _build.LIBPATH


def load(build_if_missing=True):
    """Load the shared library (building it first if the source is newer)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if build_if_missing and _build.needs_build():
        try:
            _build.build()
        except Exception as e:  # no nvcc on the box: use the prebuilt file if any
            if not os.path.exists(path):
                raise SkdError("libskdist_b200.so is missing and could not be built: %s" % e)
            import warnings
            warnings.warn("libskdist_b200.so is older than its sources and could not be rebuilt (%s); "
                          "loading the existing file" % e)
    if not os.path.exists(path):
        raise SkdError("libskdist_b200.so not found at %s (run __graft_entry__.build())" % path)
    lib = ctypes.CDLL(path)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def check(rc, ctx=None):
    if rc != 0:
        msg = load().skd_last_error(ctx)
        text = msg.decode() if msg else "libskdist_b200 call failed (rc=%d)" % rc
        if text.startswith("Input X contains NaN"):     # what scikit-learn's check_array raises
            raise ValueError(text)
        if text.startswith("forest: feature") or "device path supports" in text:   # input outside the device path's limits
            raise NotImplementedError(text)
        raise SkdError(text)


def ptr(a):
    return a.ctypes.data_as(_c.c_void_p)
