"""Loader for libdbx.so (the CUDA implementation behind include/dbx.h).

There is NO CPU fallback: if the shared library is missing, or no CUDA device is usable,
every operator fails loudly (DbxError).  Nothing in this package imports `oracle/`.
"""
from __future__ import annotations

import ctypes as C
import os

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdbx.so")


class DbxError(RuntimeError):
    """ErrorCode of the reference (src/common/exception): status + message."""

    def __init__(self, status: int, message: str):
        self.status = status
        self.message = message
        super().__init__(f"dbx status {status}: {message}")


_lib = None


def load():
    """Load libdbx.so and declare the C signatures of every export in include/dbx.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise DbxError(abi.ERR_NO_DEVICE, f"{LIB_PATH} is missing: build it with `python -m databend_b200.build` "
                                          "(no CPU fallback exists)")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, u64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
    P = C.POINTER
    sig = {
        "dbx_abi_version": (i32, []),
        "dbx_device_count": (i32, [P(i32)]),
        "dbx_last_error": (C.c_char_p, [vp]),
        "dbx_host_alloc": (i32, [C.c_size_t, P(vp)]),
        "dbx_host_free": (i32, [vp]),
        "dbx_host_register": (i32, [vp, C.c_size_t]),
        "dbx_host_unregister": (i32, [vp]),
        "dbx_device_alloc": (i32, [i32, C.c_size_t, P(vp)]),
        "dbx_device_free": (i32, [i32, vp]),
        "dbx_memcpy_h2d": (i32, [i32, vp, vp, C.c_size_t]),
        "dbx_memcpy_d2h": (i32, [i32, vp, vp, C.c_size_t]),
        "dbx_memcpy_d2d": (i32, [i32, vp, vp, C.c_size_t]),
        "dbx_device_synchronize": (i32, [i32]),
        "dbx_op_create": (i32, [i32, vp, P(i32), i32, i32, P(vp)]),
        "dbx_op_destroy": (i32, [vp]),
        "dbx_op_push": (i32, [vp, P(abi.Block)]),
        "dbx_op_finish": (i32, [vp]),
        "dbx_op_pull": (i32, [vp, i32, P(abi.Block), P(i32)]),
        "dbx_block_release": (i32, [P(abi.Block)]),
        "dbx_op_reset": (i32, [vp]),
        "dbx_op_synchronize": (i32, [vp]),
        "dbx_join_probe": (i32, [vp, P(abi.Block)]),
        "dbx_join_final_probe": (i32, [vp]),
        "dbx_agg_final_merge_partial": (i32, [vp, vp]),
        "dbx_agg_partial_partition": (i32, [vp, i32, P(vp), P(i64), P(i32)]),
        "dbx_agg_final_merge_rows": (i32, [vp, vp, i64]),
        "dbx_agg_exchange_create": (i32, [vp, i32, i32, i64, P(vp), vp]),
        "dbx_agg_exchange_local_buffer": (i32, [vp, P(vp), P(i64), P(i32)]),
        "dbx_agg_exchange_connect": (i32, [vp, vp, P(vp)]),
        "dbx_agg_exchange_scatter": (i32, [vp, vp]),
        "dbx_agg_exchange_merge": (i32, [vp, vp]),
        "dbx_agg_exchange_destroy": (i32, [vp]),
        "dbx_agg_exchange_last_error": (C.c_char_p, [vp]),
        "dbx_hash_partition": (i32, [i32, P(abi.Block), i32, i32, P(vp), P(i64)]),
        "dbx_eval_distance": (i32, [i32, i32, P(abi.Column), P(abi.Column), P(abi.Column)]),
        "dbx_knn_create": (i32, [i32, i32, P(abi.Column), P(vp)]),
        "dbx_knn_search": (i32, [vp, P(abi.Column), i32, i32, vp, vp]),
        "dbx_knn_destroy": (i32, [vp]),
        "dbx_knn_last_error": (C.c_char_p, [vp]),
        "dbx_knn_last_gemm_ms": (i32, [vp, P(C.c_float), P(i64)]),
        "dbx_knn_last_stats": (i32, [vp, P(i64)]),
        "dbx_synth_fill": (i32, [i32, i32, u64, i64, i64, i64, vp]),
        "dbx_kernel_launch_count": (i64, []),
        "dbx_op_last_kernel_ms": (i32, [vp, P(C.c_float)]),
        "dbx_op_stream": (i32, [vp, P(vp)]),
        "dbx_op_kernel_ms": (i32, [vp, i32, P(C.c_float)]),
        "dbx_agg_partial_serialize": (i32, [vp, i32, P(abi.Block), P(i32)]),
        "dbx_agg_final_merge_serialized": (i32, [vp, P(abi.Block)]),
        "dbx_op_inputs_consumed": (i32, [vp]),
        "dbx_op_kernel_variant": (i32, [vp, C.c_char_p, i32]),
        "dbx_agg_jit_selftest": (i32, [C.c_char_p, i32]),
        "dbx_eval_jit_selftest": (i32, [C.c_char_p, i32]),
        "dbx_agg_exchange_phase_ms": (i32, [vp, P(C.c_float)]),
        "dbx_shuffle_create": (i32, [i32, i32, i32, P(i32), i32, i32, i64, P(vp), vp]),
        "dbx_shuffle_local_buffer": (i32, [vp, P(vp)]),
        "dbx_shuffle_connect": (i32, [vp, vp, P(vp)]),
        "dbx_shuffle_send": (i32, [vp, P(abi.Block)]),
        "dbx_shuffle_recv": (i32, [vp, P(abi.Block), P(abi.Column)]),
        "dbx_shuffle_last_ms": (i32, [vp, P(C.c_float), P(C.c_float)]),
        "dbx_shuffle_destroy": (i32, [vp]),
        "dbx_shuffle_last_error": (C.c_char_p, [vp]),
        "dbx_block_take": (i32, [i32, P(abi.Block), vp, i64, i32, i32, P(abi.Block)]),
        "dbx_block_take_ranges": (i32, [i32, P(abi.Block), vp, vp, i64, i32, P(abi.Block)]),
        "dbx_block_scatter": (i32, [i32, P(abi.Block), vp, i32, i32, i32, P(abi.Block)]),
        "dbx_block_concat": (i32, [i32, P(abi.Block), i32, i32, P(abi.Block)]),
        "dbx_eval_scalar": (i32, [i32, P(abi.Expr), P(abi.Block), i32, P(abi.Block), P(i32), P(i64)]),
        "dbx_join_runtime_filter": (i32, [vp, P(abi.RuntimeFilterParams), P(vp)]),
        "dbx_runtime_filter_info": (i32, [vp, P(abi.RfInfo)]),
        "dbx_runtime_filter_export": (i32, [vp, i32, P(C.c_uint32), i64, P(i64), i64]),
        "dbx_runtime_filter_apply": (i32, [vp, P(abi.Block), P(i32), i32, P(abi.Block), P(i64)]),
        "dbx_runtime_filter_destroy": (i32, [vp]),
        "dbx_op_create_computed": (i32, [i32, vp, P(i32), i32, P(abi.Expr), i32, i32, P(vp)]),
        "dbx_agg_expr_jit_selftest": (i32, [C.c_char_p, i32]),
        "dbx_op_create_join": (i32, [P(abi.JoinParams), P(i32), i32, P(abi.Expr), i32, P(vp)]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)  # AttributeError = the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if L.dbx_abi_version() != abi.ABI_VERSION:
        raise DbxError(abi.ERR_INVALID, "libdbx.so ABI version differs from databend_b200.abi")
    _lib = L
    return L


def check(status: int, handle=None):
    """Raise DbxError with dbx_last_error(handle) when status != DBX_OK."""
    if status != abi.OK:
        msg = load().dbx_last_error(handle)
        raise DbxError(status, (msg or b"").decode("utf-8", "replace"))


def device_count() -> int:
    n = C.c_int32(0)
    check(load().dbx_device_count(C.byref(n)))
    return n.value


def require_device() -> int:
    """Fail loudly when there is no GPU (the product has no CPU path)."""
    return device_count()
