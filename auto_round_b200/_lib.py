"""ctypes binding of libar_b200.so (the C ABI declared in include/ar_b200.h).

There is NO fallback: if the CUDA library is missing or a call fails, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libar_b200.so")

DT_INT_SYM, DT_INT_ASYM, DT_MX_FP4, DT_NV_FP4 = 0, 1, 2, 3


class QSpec(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("bits", C.c_int32), ("group_size", C.c_int32), ("n", C.c_int32),
                ("k", C.c_int32), ("q_scale_thresh", C.c_float), ("scale_bound_hi", C.c_float),
                ("init_scale", C.c_void_p)]          # device fp32 [G] or NULL (enable_alg_ext)


_P, _I, _L, _F, _D = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double
_QS = C.POINTER(QSpec)

# name -> argtypes (every function returns int status); kept in one table so the symbol test can walk it
SIGNATURES = {
    "ar_group_minmax": [_QS, _P, _P, _P, _P],
    "ar_absmax": [_P, _L, _P, _P],
    "ar_nv_global_scale": [_P, _P, _P],
    "ar_qdq_fwd": [_QS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "ar_qdq_bwd": [_QS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P],
    "ar_gemm_bf16": [_P, _P, _P, _I, _I, _I, _I, _I, _L, _L, _L, _P, _P],
    "ar_gemm_bf16_grouped": [_P, _P, _P, _I, _I, _I, _I, _I, _I, _L, _L, _L, _I, _I, _P, _P, _I, _I, _P],
    "ar_moe_route": [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "ar_moe_gather": [_P, _P, _P, _I, _I, _I, _P, _P],
    "ar_moe_combine": [_P, _P, _P, _P, _I, _I, _I, _P, _P],
    "ar_moe_rowdot": [_P, _P, _P, _I, _I, _I, _P, _P],
    "ar_fq_linear_bwd_dx": [_QS, _P, _L, _P, _P, _P],
    "ar_fq_update": [_QS, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _I, _P, _F, _P, _P, _P, _P, _P, _P, _P, _P],
    "ar_wq_decode": [_QS, _P, _L, _I, _P, _P],
    "ar_mse_fwd_bwd": [_P, _P, _P, _L, _L, _F, _F, _P, _P, _P],
    "ar_best_update": [_P, _D, _D, _I, _P, _P, _P, _P, _P, _P],
    "ar_sched_load": [_P, _P, _P, _I, _P, _P, _P, _P],
    "ar_iter_advance": [_P, _P],
    "ar_rmsnorm_fwd": [_P, _P, _F, _L, _I, _P, _P, _P],
    "ar_rmsnorm_bwd": [_P, _P, _P, _P, _L, _I, _P, _I, _P],
    "ar_rope": [_P, _P, _P, _L, _I, _I, _I, _I, _I, _P, _P],
    "ar_swiglu_fwd": [_P, _P, _L, _P, _P],
    "ar_swiglu_bwd": [_P, _P, _P, _L, _P, _P, _P],
    "ar_gather_rows": [_P, _P, _I, _L, _P, _P],
    "ar_pack_int": [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P],
    "ar_unpack_int": [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P],
    "ar_pack_awq": [_P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P],
    "ar_unpack_awq": [_P, _P, _P, _I, _I, _I, _P, _P, _P],
    "ar_pack_fp4_nv": [_P, _P, _P, _I, _I, _P, _P, _P],
    "ar_pack_fp4_mx": [_P, _P, _I, _I, _P, _P, _P],
    "ar_unpack_fp4": [_P, _I, _I, _P, _P],
    "ar_search_scale_int": [_P, _P, _L, _P, _I, _QS, _P, _P, _P],
    "ar_search_scale_nv": [_P, _P, _L, _P, _P, _I, _QS, _P, _P],
    "ar_search_scale_mx": [_P, _P, _L, _P, _I, _QS, _P, _P],
    "ar_imatrix_accum": [_P, _L, _I, _P, _P],
    "ar_absdiff_hist": [_P, _P, _L, _P, _P],
    "ar_topk_threshold": [_P, _L, _P, _P],
    "ar_topk_threshold_ranks": [_P, _I, _I, _P, _L, _P, _P],
    "ar_mse_outlier_fwd_bwd": [_P, _P, _P, _L, _L, _L, _F, _P, _P, _P, _P],
}

_lib = None


def load() -> C.CDLL:
    """Load the library (once).  Raises if it has not been built: no CPU fallback exists."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} not found: run `python -m auto_round_b200.build` (nvcc, sm_90a). "
                           "auto_round_b200 has no CPU or eager-PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    lib.ar_version.restype = C.c_int
    lib.ar_last_error.restype = C.c_char_p
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().ar_last_error().decode(errors="replace")
        raise RuntimeError(f"{what} failed (status {rc}): {msg}")
