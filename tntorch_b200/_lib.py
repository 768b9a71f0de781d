"""ctypes binding of libtnb200.so (the C-ABI in include/tnb200.h).

There is no CPU fallback: if the shared library is missing, or a compute entry point is called
without a CUDA device, this module raises.  Build the library with
``python tntorch_b200/csrc/build.py`` (or ``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtnb200.so")

TNB_F32, TNB_F64, TNB_BF16, TNB_F16 = 0, 1, 2, 3
FLAG_NO_TENSORCORE = 1
FLAG_BATCH_MODE = 2
FLAG_PROFILE = 4
FLAG_CONCURRENT = 8
FLAG_NO_SPECULATE = 16

ERR_INVALID, ERR_CUDA, ERR_WORKSPACE, ERR_UNSUPPORTED, ERR_NOCONV = 1, 2, 3, 4, 5


class TnbError(RuntimeError):
    pass


_lib = None

_i64p = C.POINTER(C.c_int64)
_i32p = C.POINTER(C.c_int32)
_f64p = C.POINTER(C.c_double)
_vp = C.c_void_p

# name -> (restype, argtypes); must list every symbol declared in include/tnb200.h
SIGNATURES = {
    "tnb_version": (C.c_int, []),
    "tnb_last_error": (C.c_char_p, []),
    "tnb_launch_count": (C.c_uint64, []),
    "tnb_has_tensorcore_path": (C.c_int, []),
    "tnb_set_reserved_sms": (None, [C.c_int32]),
    "tnb_ttsvd_cores_capacity": (C.c_int64, [C.c_int, _i64p, _i32p, _i64p]),
    "tnb_ttsvd_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, _i64p, _i32p, C.c_uint32]),
    "tnb_ttsvd": (C.c_int, [C.c_int, _vp, C.c_int, _i64p, _i32p, C.c_double, C.c_uint32, _vp, C.c_size_t, _vp,
                            C.c_int64, _i32p, _f64p, _vp]),
    "tnb_ttsvd_batch_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, _i64p, _i32p, C.c_uint32, C.POINTER(C.c_size_t)]),
    "tnb_ttsvd_batch": (C.c_int, [C.c_int, C.POINTER(_vp), C.c_int, C.c_int, _i64p, _i32p, C.c_double, C.c_uint32, _vp,
                                  C.c_size_t, C.POINTER(_vp), C.c_int64, _i32p, _f64p, _i32p, _vp]),
    "tnb_ttsvd_host": (C.c_int, [C.c_int, _vp, C.c_int, _i64p, _i32p, C.c_double, C.c_uint32, _vp, _vp, C.c_size_t,
                                 _vp, C.c_int64, _vp, _i32p, _f64p, _vp]),
    "tnb_tt_round_cores_capacity": (C.c_int64, [C.c_int, _i64p, _i32p, _i32p, _i64p]),
    "tnb_tt_round_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, _i64p, _i32p, _i32p]),
    "tnb_tt_round": (C.c_int, [C.c_int, C.POINTER(_vp), C.c_int, _i64p, _i32p, _i32p, C.c_double, C.c_uint32, _vp,
                               C.c_size_t, _vp, C.c_int64, _i32p, _vp]),
    "tnb_tt_round_batch_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, _i64p, _i32p, _i32p, C.POINTER(C.c_size_t)]),
    "tnb_tt_round_batch": (C.c_int, [C.c_int, C.POINTER(_vp), C.c_int, C.c_int, _i64p, _i32p, _i32p, C.c_double, C.c_uint32, _vp,
                                     C.c_size_t, C.POINTER(_vp), C.c_int64, _i32p, _i32p, _vp]),
    "tnb_tt_sum_cores_capacity": (C.c_int64, [C.c_int, C.c_int, _i64p, _i32p, _i32p, _i64p]),
    "tnb_tt_sum": (C.c_int, [C.c_int, C.POINTER(_vp), C.c_int, _f64p, C.c_int, _i64p, _i32p, _vp, C.c_int64, _vp]),
    "tnb_tt_sum_round_cores_capacity": (C.c_int64, [C.c_int, C.c_int, _i64p, _i32p, _i32p, _i64p]),
    "tnb_tt_sum_round_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, _i64p, _i32p, _i32p]),
    "tnb_tt_sum_round": (C.c_int, [C.c_int, C.POINTER(_vp), C.c_int, _f64p, C.c_int, _i64p, _i32p, _i32p, C.c_double,
                                   C.c_uint32, _vp, C.c_size_t, _vp, C.c_int64, _i32p, _vp]),
    "tnb_tt_hadamard": (C.c_int, [C.c_int, C.POINTER(_vp), C.POINTER(_vp), C.c_int, _i64p, _i32p, _i32p, C.POINTER(_vp), _vp]),
    "tnb_truncated_svd_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64]),
    "tnb_truncated_svd": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, C.c_double, C.c_double, C.c_int32, C.c_int,
                                    _vp, C.c_size_t, _vp, _vp, _i32p, _vp]),
    "tnb_cp_als_factors_capacity": (C.c_int64, [C.c_int, _i64p, C.c_int32, _i64p]),
    "tnb_cp_als_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, _i64p, C.c_int32]),
    "tnb_cp_als": (C.c_int, [C.c_int, _vp, C.c_int, _i64p, C.c_int32, C.c_int32, C.c_double, _vp, C.c_size_t, _vp, C.c_int64,
                             _f64p, _i32p, _vp]),
    "tnb_cp_als_from": (C.c_int, [C.c_int, _vp, C.c_int, _i64p, C.c_int32, C.c_int32, C.c_double, _vp, C.c_size_t, _vp, C.c_int64,
                                  _f64p, _i32p, _vp]),
    "tnb_maxvol_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "tnb_maxvol": (C.c_int, [_vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32, _vp, C.c_size_t, _vp, _vp, _i32p, _vp]),
    "tnb_rect_maxvol_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "tnb_rect_maxvol": (C.c_int, [_vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.c_int32, C.c_int32, _vp,
                                  C.c_size_t, _vp, _vp, _vp, _vp]),
    "tnb_cross_gather_coords": (C.c_int, [_vp, _vp, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                          C.c_int32, _vp, _vp]),
    "tnb_cross_update_lsets": (C.c_int, [_vp, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, _vp]),
    "tnb_cross_update_rsets": (C.c_int, [_vp, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _vp, _vp,
                                         _vp]),
    "tnb_cross_tt_eval": (C.c_int, [C.POINTER(_vp), C.c_int32, _i32p, _i32p, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp]),
    "tnb_measure_tf32_peak": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _f64p, _f64p, _vp]),
    "tnb_measure_wgmma_tf32_peak": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, _f64p, _f64p, _vp]),
    "tnb_matmul": (C.c_int, [C.c_int, _vp, _vp, _vp, C.c_int64, C.c_int64, C.c_int64, _vp]),
    "tnb_qr_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "tnb_qr_householder": (C.c_int, [_vp, C.c_int32, C.c_int32, C.c_int32, _vp, C.c_size_t, _vp, _vp, _vp]),
    "tnb_gram_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int64, C.c_int64]),
    "tnb_gram": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, C.c_size_t, _vp]),
    "tnb_gram_tc_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "tnb_gram_tc_f32": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, _vp, C.c_size_t, _vp]),
    "tnb_gram_tc_kblocked_f32": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, _vp, C.c_size_t, _vp]),
    "tnb_gram_tc_bf16_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "tnb_gram_noise_level": (C.c_double, [C.c_int]),
    "tnb_gram_tc_bf16": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, _vp, C.c_size_t, _vp]),
    "tnb_project_tc_bf16": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int32, C.c_int64, _vp, _vp, C.c_size_t, _vp]),
    "tnb_gram_tc_f16_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64]),
    "tnb_gram_tc_f16": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, _vp, C.c_size_t, _vp]),
    "tnb_project_tc_f16": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int32, C.c_int64, _vp, _vp, C.c_size_t, _vp]),
    "tnb_atb_tc_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int64, C.c_int64]),
    "tnb_atb_tc_f32": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int64, _vp, C.c_float, _vp, C.c_float, _vp,
                                 C.c_size_t, _vp]),
    "tnb_cheb_filter_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "tnb_cheb_filter_f32": (C.c_int, [_vp, C.c_int32, C.c_int32, _vp, _vp, _vp, C.c_int32, _vp, _vp, _vp, _vp, C.c_size_t,
                                      _vp]),
    "tnb_project": (C.c_int, [C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_int32, _vp, _vp]),
    "tnb_project_tc_workspace_bytes": (C.c_size_t, [C.c_int64, C.c_int32]),
    "tnb_project_tc_f32": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int32, _vp, _vp, C.c_size_t, _vp]),
    "tnb_project_tc_kblocked_out_f32": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int32, C.c_int64, _vp, _vp,
                                                  C.c_size_t, _vp]),
    "tnb_project_tc_kblocked_in_f32": (C.c_int, [_vp, C.c_int64, C.c_int64, _vp, C.c_int32, _vp, _vp, C.c_size_t, _vp]),
    "tnb_eigh_workspace_bytes": (C.c_size_t, [C.c_int32]),
    "tnb_eigh_jacobi": (C.c_int, [_vp, C.c_int32, _vp, _vp, _vp, C.c_size_t, _vp]),
    "tnb_eig_topk_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32, C.c_int32]),
    "tnb_eig_topk": (C.c_int, [_vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, _vp, _vp, _vp, C.c_size_t, _f64p, _vp]),
    "tnb_tt_relative_error_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, _i64p, _i32p]),
    "tnb_tt_relative_error": (C.c_int, [C.c_int, _vp, C.POINTER(_vp), C.c_int, _i64p, _i32p, _vp, C.c_size_t, _f64p, _vp]),
}


def lib():
    """Load (once) and return the ctypes handle; raises if the extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise TnbError(
                f"{LIB_PATH} not found: build the CUDA extension first "
                "(python tntorch_b200/csrc/build.py). tntorch_b200 has no CPU fallback."
            )
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(rc: int):
    """Map a C-ABI status to the Python exception the reference would raise at this boundary."""
    if rc == 0:
        return
    msg = lib().tnb_last_error().decode("utf-8", "replace")
    if rc == ERR_INVALID:
        raise ValueError(msg)
    if rc == ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise TnbError(f"tnb200 error {rc}: {msg}")


def i64(seq):
    return (C.c_int64 * len(seq))(*[int(x) for x in seq])


def i32(seq):
    return (C.c_int32 * len(seq))(*[int(x) for x in seq])
