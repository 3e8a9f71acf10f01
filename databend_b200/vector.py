"""Host-side mirror of the reference's vector-distance scalar functions and of the
`ORDER BY distance(col, q) LIMIT k` pipeline (SURVEY 3.5).

  cosine_distance / l2_distance     src/common/vector/src/distance.rs:19-35,65-80
  calculate_distance (row driver)   src/query/functions/src/scalars/vector.rs:497-556
  registration / NULL passthrough   src/query/functions/src/scalars/vector.rs:263-281
  EvalScalar -> TopN                src/query/service/src/pipelines/builders/builder_sort.rs + top_n/*.rs

Everything forwards to libdbx (`dbx_eval_distance`, `dbx_knn_*`); there is no CPU path here.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np

from . import abi
from .block import Column
from .lib import DbxError, check, load

_KINDS = {"cosine_distance": abi.DIST_COSINE, "l2_distance": abi.DIST_L2}


def _kind(name_or_kind) -> int:
    if isinstance(name_or_kind, str):
        if name_or_kind not in _KINDS:
            raise DbxError(abi.ERR_UNSUPPORTED, f"Unknown vector function {name_or_kind}")
        return _KINDS[name_or_kind]
    return int(name_or_kind)


def eval_distance(fn: str, lhs: Column, rhs: Column, device: int = 0) -> Column:
    """ScalarFunction::eval for `cosine_distance(lhs, rhs)` / `l2_distance(lhs, rhs)`.
    Either side may be a const column (one vector); NULL on either side gives NULL.  Vector(Int8)
    sides are widened to f32 as in the reference; a Vector(Int8) / Vector(Float32) pair gives 0.0 on
    every row (NULL when the result is Nullable).
    Returns a Float32 column (Nullable when an input is)."""
    kind = _kind(fn)
    rows = rhs.length if lhs.is_const else lhs.length
    out = np.zeros(max(rows, 1), dtype=np.float32)[:rows]
    nullable = any(c.validity is not None or c.dev_validity or (c.is_const and c.const_value is None) for c in (lhs, rhs))
    oc = abi.Column()
    oc.dtype, oc.mem, oc.len, oc.data = abi.F32, abi.MEM_HOST, rows, out.ctypes.data
    vbits = None
    if nullable:
        vbits = np.zeros((rows + 7) // 8 + 1, dtype=np.uint8)
        oc.validity = vbits.ctypes.data
    lc, rc = _vector_as_c(lhs), _vector_as_c(rhs)
    st = load().dbx_eval_distance(kind, device, C.byref(lc[0]), C.byref(rc[0]), C.byref(oc))
    check(st)
    col = Column(abi.F32, rows, data=out)
    if nullable:
        col.validity = vbits
    return col


def _vector_as_c(col: Column):
    """dbx_column of a Vector(Float32) / Vector(Int8) entry; a const side carries its single vector in
    `data`, in the column's element type."""
    if col.is_const:
        c = abi.Column()
        c.dtype, c.is_const, c.len, c.mem = col.dtype, 1, col.length, abi.MEM_HOST
        keep = None
        if col.const_value is None:
            c.konst.is_null = 1
            c.vec_dim = col.vec_dim
        else:
            keep = np.ascontiguousarray(col.const_value, dtype=np.int8 if col.dtype == abi.VEC_I8 else np.float32)
            c.vec_dim = keep.shape[-1]
            c.data = keep.ctypes.data
        return c, keep
    return col.as_c(), None


def const_vector(value, n: int, dim: Optional[int] = None, dtype: Optional[int] = None) -> Column:
    """BlockEntry::Const(Scalar::Vector(..), DataType::Vector, n).  An int8 array gives a Vector(Int8)
    constant (kept int8), anything else a Vector(Float32) one; `dtype` (abi.VEC_F32 / abi.VEC_I8)
    picks the type of a NULL constant."""
    if value is None:
        return Column(abi.VEC_F32 if dtype is None else dtype, n, is_const=True, const_value=None, vec_dim=dim)
    if dtype is None:
        dtype = abi.VEC_I8 if np.asarray(value).dtype == np.int8 else abi.VEC_F32
    if dtype == abi.VEC_I8 and np.asarray(value).dtype != np.int8:
        raise TypeError("const_vector: a Vector(Int8) constant takes int8 values")
    v = np.ascontiguousarray(value, dtype=np.int8 if dtype == abi.VEC_I8 else np.float32)
    return Column(dtype, n, is_const=True, const_value=v, vec_dim=v.shape[-1])


class VectorTopN:
    """`SELECT row, distance(c, q) ... ORDER BY distance(c, q) LIMIT k` for a batch of query
    vectors over one resident corpus column.  Returned rows are ordered by (distance, row id)
    with the OrderedFloat total order (NaN last); distances are bit-identical to eval_distance."""

    def __init__(self, fn: str, corpus: Column, device: int = 0):
        self.kind = _kind(fn)
        self.device = device
        self._h = C.c_void_p()
        self._corpus = corpus  # keep device/host buffers alive
        c = corpus.as_c()
        st = load().dbx_knn_create(self.kind, device, C.byref(c), C.byref(self._h))
        if st != abi.OK:
            msg = load().dbx_knn_last_error(None)
            raise DbxError(st, (msg or b"").decode("utf-8", "replace"))

    def search(self, queries: Column, k: int) -> Tuple[np.ndarray, np.ndarray]:
        nq = queries.length
        idx = np.empty((nq, k), dtype=np.int64)
        dist = np.empty((nq, k), dtype=np.float32)
        q = queries.as_c()
        st = load().dbx_knn_search(self._h, C.byref(q), k, abi.MEM_HOST, idx.ctypes.data, dist.ctypes.data)
        if st != abi.OK:
            msg = load().dbx_knn_last_error(self._h)
            raise DbxError(st, (msg or b"").decode("utf-8", "replace"))
        return idx, dist

    def search_into(self, queries: Column, k: int, out_idx_dev_ptr: int, out_dist_dev_ptr: int):
        """Same search, results written to caller-provided DEVICE buffers ([nq, k] int64 row ids and
        [nq, k] float32 distances): the multi-GPU merge then never leaves HBM."""
        q = queries.as_c()
        st = load().dbx_knn_search(self._h, C.byref(q), k, abi.MEM_DEVICE, out_idx_dev_ptr, out_dist_dev_ptr)
        if st != abi.OK:
            msg = load().dbx_knn_last_error(self._h)
            raise DbxError(st, (msg or b"").decode("utf-8", "replace"))

    def last_gemm_ms(self) -> Tuple[float, int]:
        ms, n = C.c_float(0), C.c_int64(0)
        load().dbx_knn_last_gemm_ms(self._h, C.byref(ms), C.byref(n))
        return ms.value, n.value

    def stats(self) -> dict:
        s = (C.c_int64 * 8)()
        load().dbx_knn_last_stats(self._h, s)
        return {"certified": s[0], "exact_fallback": s[1], "candidates": s[2], "passes": s[3], "cluster": s[4], "grid": s[5], "us_passes": s[6], "us_rerank": s[7]}

    def close(self):
        if self._h:
            load().dbx_knn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
