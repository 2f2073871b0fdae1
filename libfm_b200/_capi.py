"""ctypes binding of include/fmb200.h (the C ABI of libfmb200.so).

This is the same stub a maintainer of the reference would write to reach the
library from Python; the C++ command line (host/) links the library directly.
There is no fallback: if the shared object is missing, loading raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# FMB200_LIB: an alternative build of the same ABI (A/B timing of kernel variants; development aid)
LIB_PATH = os.environ.get("FMB200_LIB") or os.path.join(_HERE, "lib", "libfmb200.so")

# every symbol include/fmb200.h declares, with (restype, argtypes)
_u64p = C.POINTER(C.c_uint64)
_u32p = C.POINTER(C.c_uint32)
_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_intp = C.POINTER(C.c_int)
_ctx = C.c_void_p

# fmb200_xt_blocks: a data set given as blocks of its .xt file (fmb200_mcmc_begin_xt)
XT_FETCH = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p), C.POINTER(_u32p))
XT_RELEASE = C.CFUNCTYPE(None, C.c_void_p, C.c_uint64)


class XtBlocksC(C.Structure):
    _fields_ = [("n_cases", C.c_uint64), ("target", _f32p), ("n_blocks", C.c_uint64), ("col_lo", _u32p),
                ("nnz", _u64p), ("slot", C.c_int * 2), ("user", C.c_void_p), ("fetch", XT_FETCH),
                ("release", XT_RELEASE)]


class RelationC(C.Structure):
    """fmb200_relation (fmb200_mcmc_set_relations)"""
    _fields_ = [("num_cases", C.c_uint32), ("num_feature", C.c_uint32), ("attr_offset", C.c_uint32),
                ("col_ptr", _u64p), ("row", _u32p), ("val", _f32p), ("n_train", C.c_uint64), ("n_test", C.c_uint64),
                ("train_join", _u32p), ("test_join", _u32p)]

SYMBOLS = {
    "fmb200_create": (C.c_int, [C.POINTER(_ctx), C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_int]),
    "fmb200_destroy": (None, [_ctx]),
    "fmb200_last_error": (C.c_char_p, []),
    "fmb200_set_hparams": (C.c_int, [_ctx, C.c_int] + [C.c_double] * 6),
    "fmb200_set_mode": (C.c_int, [_ctx, C.c_int]),
    "fmb200_upload_data": (C.c_int, [_ctx, C.c_int, C.c_uint64, C.c_uint64, _u64p, _u32p, _f32p, _f32p]),
    "fmb200_upload_data_async": (C.c_int, [_ctx, C.c_int, C.c_uint64, C.c_uint64, _u64p, _u32p, _f32p, _f32p]),
    "fmb200_upload_data_aos": (C.c_int, [_ctx, C.c_int, C.c_uint64, C.c_void_p, _f32p]),
    "fmb200_upload_onehot": (C.c_int, [_ctx, C.c_int, C.c_uint64, C.c_uint32, _u32p, _f32p]),
    "fmb200_upload_onehot_async": (C.c_int, [_ctx, C.c_int, C.c_uint64, C.c_uint32, _u32p, _f32p]),
    "fmb200_upload_xblock": (C.c_int, [_ctx, C.c_int, C.c_uint64, C.c_uint64, C.c_void_p, _u32p, _f32p]),
    "fmb200_upload_xblock_async": (C.c_int, [_ctx, C.c_int, C.c_uint64, C.c_uint64, C.c_void_p, _u32p, _f32p]),
    "fmb200_free_data": (C.c_int, [_ctx, C.c_int]),
    "fmb200_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_uint64]),
    "fmb200_host_free": (C.c_int, [C.c_void_p]),
    "fmb200_set_params": (C.c_int, [_ctx, C.c_double, _f64p, _f64p]),
    "fmb200_get_params": (C.c_int, [_ctx, _f64p, _f64p, _f64p]),
    "fmb200_sgd_epoch": (C.c_int, [_ctx, C.c_int, _f64p]),
    "fmb200_sgd_epoch_async": (C.c_int, [_ctx, C.c_int]),
    "fmb200_sync": (C.c_int, [_ctx]),
    "fmb200_evaluate": (C.c_int, [_ctx, C.c_int, _f64p, _f64p, _u64p]),
    "fmb200_predict": (C.c_int, [_ctx, C.c_int, C.c_int, _f64p]),
    "fmb200_sgda_begin": (C.c_int, [_ctx, C.c_uint32, _u32p]),
    "fmb200_sgda_epoch": (C.c_int, [_ctx, C.c_int, C.c_int, C.c_int, _f64p]),
    "fmb200_sgda_epoch_x": (C.c_int, [_ctx, C.c_int, C.POINTER(XtBlocksC), C.c_int, C.POINTER(XtBlocksC), C.c_int,
                                      _f64p]),
    "fmb200_sgda_get_reg": (C.c_int, [_ctx, _f64p, _f64p]),
    "fmb200_sgda_get_moments": (C.c_int, [_ctx, _f64p, _f64p]),
    "fmb200_mcmc_eterms": (C.c_int, [_ctx, C.c_int, _f64p]),
    "fmb200_mcmc_begin": (C.c_int, [_ctx, C.c_int, C.c_int, C.c_int, C.c_int, C.c_uint32, _u32p, _u32p, C.c_double,
                                    _f64p, _f64p]),
    "fmb200_mcmc_begin_xt": (C.c_int, [_ctx, C.c_int, C.POINTER(XtBlocksC), C.c_int, C.POINTER(XtBlocksC), C.c_int,
                                       C.c_int, C.c_uint32, _u32p, _u32p, C.c_double, _f64p, _f64p]),
    "fmb200_mcmc_set_relations": (C.c_int, [_ctx, C.c_int, C.c_int, C.c_uint32, C.POINTER(RelationC)]),
    "fmb200_mcmc_iteration": (C.c_int, [_ctx, _f64p, _u32p]),
    "fmb200_mcmc_get_hyper": (C.c_int, [_ctx] + [_f64p] * 5),
    "fmb200_mcmc_get_pred": (C.c_int, [_ctx] + [_f64p] * 3),
    "fmb200_mcmc_runs": (C.c_int, [_ctx, _u32p]),
    "fmb200_params_device": (C.c_int, [_ctx, C.POINTER(C.c_void_p), _u64p]),
    "fmb200_scale_params": (C.c_int, [_ctx, C.c_double]),
    "fmb200_params_layout": (C.c_int, [_ctx, _u64p, _intp, _u64p, _intp]),
    "fmb200_stream": (C.c_int, [_ctx, C.POINTER(C.c_void_p)]),
    "fmb200_peer_export": (C.c_int, [_ctx, C.c_void_p]),
    "fmb200_peer_attach_ipc": (C.c_int, [_ctx, C.c_int, C.c_int, C.c_void_p]),
    "fmb200_peer_attach_local": (C.c_int, [_ctx, C.c_int, C.c_int, C.POINTER(_ctx)]),
    "fmb200_allreduce_mean": (C.c_int, [_ctx]),
    "fmb200_allreduce_meanfield": (C.c_int, [_ctx]),
    "fmb200_peer_barrier": (C.c_int, [_ctx]),
    "fmb200_download_data": (C.c_int, [_ctx, C.c_int, _u64p, _u64p, _u64p, _u32p, _f32p, _f32p]),
    "fmb200_kernel_launches": (C.c_int, [_ctx, _u64p]),
    "fmb200_last_epoch_config": (C.c_int, [_ctx] + [_intp] * 7),
    "fmb200_last_epoch_dealt": (C.c_int, [_ctx, _intp]),
    "fmb200_set_tuning": (C.c_int, [_ctx, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "fmb200_set_reproducible": (C.c_int, [_ctx, C.c_int, C.c_int, C.c_int]),
    "fmb200_ordered_index": (C.c_int, [_ctx, C.c_int, _u32p, _u32p]),
}

_lib = None


def load() -> C.CDLL:
    """dlopen libfmb200.so and type every entry point.  Raises if absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m libfm_b200.build` "
                "(libfm_b200 has no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the export is missing
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib
