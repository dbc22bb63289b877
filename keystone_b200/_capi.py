"""ctypes binding of libkeystone_b200.so (include/keystone_b200.h) -- the same C ABI a JNI shim binds.

The library is the product: if it is missing or a call fails, this module raises; there is no
Python/NumPy fallback for any compute entry point.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from typing import List

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libkeystone_b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "keystone_b200.h")

KS_NCCL_ID_BYTES = 128
KS_PRECISION_TF32 = 0
KS_PRECISION_F16 = 1
KS_PRECISION_F16X2 = 2  # split-operand parity mode
KS_PRECISION_DEFAULT = -1
PRECISIONS = {"tf32": KS_PRECISION_TF32, "f16": KS_PRECISION_F16, "f16x2": KS_PRECISION_F16X2, "parity": KS_PRECISION_F16X2,
              "default": KS_PRECISION_DEFAULT}


class KeystoneError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"keystone_b200 error {code}: {msg}")
        self.code = code


def declared_symbols() -> List[str]:
    """Every function the public header declares (used by the export test)."""
    with open(HEADER_PATH) as fh:
        return re.findall(r"KS_API\s+(?:int32_t|const char\*)\s+(ks_[a-z0-9_]+)\s*\(", fh.read())


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise KeystoneError(-100, f"{LIB_PATH} not built; run `python -m keystone_b200.build` (no fallback exists)")
        _lib = C.CDLL(LIB_PATH)
        _declare(_lib)
    return _lib


i32, i64, u64, f64 = C.c_int32, C.c_int64, C.c_uint64, C.c_double
p_i32, p_i64, p_f64, p_f32 = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_float)
p_u8 = C.POINTER(C.c_uint8)
pp_f64 = C.POINTER(C.POINTER(C.c_double))


def _declare(L: C.CDLL) -> None:
    def sig(name, *argtypes, restype=i32):
        fn = getattr(L, name)
        fn.argtypes = list(argtypes)
        fn.restype = restype

    sig("ks_version")
    sig("ks_nccl_unique_id", p_u8)
    sig("ks_ctx_create", i32, i32, i32, p_u8, p_i64)
    sig("ks_ctx_destroy", i64)
    sig("ks_last_error", i64, restype=C.c_char_p)
    sig("ks_ctx_synchronize", i64)
    sig("ks_ctx_set_option", i64, C.c_char_p, i64)
    sig("ks_ctx_launch_count", i64, p_i64)
    sig("ks_matrix_from_host_f64", i64, C.c_void_p, i64, i64, i64, p_i64)
    sig("ks_matrix_from_host_f32", i64, C.c_void_p, i64, i64, i64, p_i64)
    sig("ks_matrix_create", i64, i64, i64, p_i64)
    sig("ks_matrix_write_rows_f64", i64, i64, i64, C.c_void_p, i64, i64)
    sig("ks_matrix_write_rows_f32", i64, i64, i64, C.c_void_p, i64, i64)
    sig("ks_matrix_synthetic_normal", i64, i64, i64, u64, i64, f64, f64, p_i64)
    sig("ks_labels_from_classes", i64, C.c_void_p, i64, i32, p_i64)
    sig("ks_matrix_shape", i64, i64, p_i64, p_i64)
    sig("ks_matrix_to_host_f64", i64, i64, C.c_void_p, i64)
    sig("ks_matrix_to_host_f32", i64, i64, C.c_void_p, i64)
    sig("ks_matrix_destroy", i64, i64)
    sig("ks_cosine_rf_create", i64, C.c_void_p, C.c_void_p, i64, i64, p_i64)
    sig("ks_cosine_rf_apply", i64, i64, i64, p_i64)
    sig("ks_cosine_rf_destroy", i64, i64)
    sig("ks_convolver_create", i64, C.c_void_p, i32, i32, i32, i32, i32, C.c_void_p, i32, f64, p_i64)
    sig("ks_convolver_apply", i64, i64, i64, i32, i32, f64, f64, p_i64)
    sig("ks_convolver_destroy", i64, i64)
    sig("ks_padded_fft_create", i64, C.c_void_p, i64, i32, f64, f64, p_i64)
    sig("ks_matrix_map", i64, i64, i32, C.c_void_p, f64, f64, p_i64)
    sig("ks_blockls_fit", i64, i64, i64, p_i64, i32, i64, i32, i32, f64, i64, i32, p_i64)
    sig("ks_blockwls_fit", i64, i64, i64, p_i64, i32, i64, i32, i32, f64, f64, i64, i32, p_i64)
    sig("ks_linear_map_fit", i64, i64, i64, i32, f64, p_i64)
    sig("ks_lbfgs_fit", i64, i64, i64, p_i64, i32, i64, i32, i32, f64, i32, f64, i32, p_i64)
    sig("ks_model_from_host", i64, pp_f64, p_i64, i32, i64, C.c_void_p, pp_f64, i32, p_i64)
    sig("ks_model_num_blocks", i64, i64, p_i32, p_i64, p_i32)
    sig("ks_model_block_rows", i64, i64, i32, p_i64)
    sig("ks_model_get_block", i64, i64, i32, C.c_void_p, C.c_void_p, p_i32)
    sig("ks_model_get_intercept", i64, i64, C.c_void_p, p_i32)
    sig("ks_model_host_view", i64, i64, i32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p))
    sig("ks_model_apply", i64, i64, i64, i64, p_i64, i32, p_i64)
    sig("ks_model_apply_argmax", i64, i64, i64, i64, p_i64, i32, C.c_void_p)
    sig("ks_model_apply_partial", i64, i64, i64, i64, p_i64, i32, i32, p_i64)
    sig("ks_model_cost", i64, i64, i64, i64, p_i64, i32, i64, f64, p_f64)
    sig("ks_model_confusion_matrix", i64, i64, i64, i64, p_i64, i32, i64, C.c_void_p)
    sig("ks_model_destroy", i64, i64)
    sig("ks_model_save", i64, i64, C.c_char_p)
    sig("ks_model_load", i64, C.c_char_p, p_i64)
    sig("ks_gaussian_kernel_create", i64, i64, f64, p_i64)
    sig("ks_gaussian_kernel_block", i64, i64, i64, i64, i64, p_i64)
    sig("ks_gaussian_kernel_shape", i64, i64, p_i64, p_i64)
    sig("ks_gaussian_kernel_destroy", i64, i64)
    sig("ks_krr_fit", i64, i64, i64, f64, i32, i32, C.c_void_p, p_i64)
    sig("ks_kernel_model_from_host", i64, i64, pp_f64, p_i64, i32, i64, i32, p_i64)
    sig("ks_io_last_error", restype=C.c_char_p)
    sig("ks_csv_dims", C.c_char_p, p_i64, p_i64)
    sig("ks_csv_read_f64", C.c_char_p, C.c_void_p, i64, i64, i64)
    sig("ks_csv_read_f32", C.c_char_p, C.c_void_p, i64, i64, i64)
    sig("ks_timit_labels_read", C.c_char_p, C.c_void_p, i64)
    sig("ks_cifar_read", C.c_char_p, C.c_void_p, C.c_void_p, i64, p_i64)
    sig("ks_last_fit_stats_json", i64, C.c_char_p, i64)
    sig("ks_last_fit_stats_json_size", i64, p_i64)
    sig("ks_debug_gram", i64, i64, i64, C.c_void_p, i64, C.c_void_p, i64)
    sig("ks_debug_time_gram", i64, i64, i64, i32, p_f64)
    sig("ks_debug_chol_solve", i64, C.c_void_p, i32, C.c_void_p, i32, i32, C.c_void_p, p_f64)


def check(ctx: int, rc: int) -> None:
    if rc != 0:
        msg = lib().ks_last_error(ctx)
        raise KeystoneError(rc, msg.decode("utf-8", "replace") if msg else "unknown error")
