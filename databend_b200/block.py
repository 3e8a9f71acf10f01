"""Host-side mirror of the reference's DataBlock / BlockEntry / Column / Bitmap.

Reference types (paths relative to the databend source tree):
  DataBlock{entries, num_rows, meta}      src/query/expression/src/block.rs:49-60
  BlockEntry::{Const, Column}             src/query/expression/src/block.rs:62-80
  Column::Number / Nullable / Vector      src/query/expression/src/values.rs:192-215
  Buffer<T>                               src/common/column/src/buffer/immutable.rs:60-73
  Bitmap{bytes, offset, length}           src/common/column/src/bitmap/immutable.rs

Columns hold numpy arrays (host) or raw device pointers; `as_c()` produces the
`dbx_column` descriptor that crosses the C-ABI.  No compute happens here.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import abi

_NP2DBX = {
    np.dtype(np.int8): abi.I8, np.dtype(np.int16): abi.I16, np.dtype(np.int32): abi.I32, np.dtype(np.int64): abi.I64,
    np.dtype(np.uint8): abi.U8, np.dtype(np.uint16): abi.U16, np.dtype(np.uint32): abi.U32, np.dtype(np.uint64): abi.U64,
    np.dtype(np.float32): abi.F32, np.dtype(np.float64): abi.F64,
}
_DBX2NP = {v: k for k, v in _NP2DBX.items()}
DTYPE_NAMES = {
    abi.BOOL: "Boolean", abi.I8: "Int8", abi.I16: "Int16", abi.I32: "Int32", abi.I64: "Int64",
    abi.U8: "UInt8", abi.U16: "UInt16", abi.U32: "UInt32", abi.U64: "UInt64",
    abi.F32: "Float32", abi.F64: "Float64", abi.VEC_F32: "Vector(Float32)", abi.VEC_I8: "Vector(Int8)",
}
_VEC_ELEM = {abi.VEC_F32: np.dtype(np.float32), abi.VEC_I8: np.dtype(np.int8)}


def np_dtype(dbx_dtype: int) -> np.dtype:
    return _DBX2NP[dbx_dtype]


def dbx_dtype_of(arr: np.ndarray) -> int:
    return _NP2DBX[arr.dtype]


def make_scalar(dtype: int, value) -> abi.Scalar:
    """Scalar (values.rs:122-190) -> dbx_scalar."""
    s = abi.Scalar()
    s.dtype = dtype
    if value is None:
        s.is_null = 1
        return s
    s.is_null = 0
    if dtype in (abi.F32, abi.F64):
        s.v.f64 = float(value)
    elif dtype in (abi.U8, abi.U16, abi.U32, abi.U64, abi.BOOL):
        s.v.u64 = int(value)
    else:
        s.v.i64 = int(value)
    return s


def pack_bitmap(bits: Sequence[bool], bit_offset: int = 0) -> np.ndarray:
    """MutableBitmap (bitmap/mutable.rs): LSB-first packing, optionally starting at a bit offset
    (as produced by Bitmap::slice)."""
    b = np.asarray(bits, dtype=bool)
    if bit_offset:
        b = np.concatenate([np.zeros(bit_offset, dtype=bool), b])
    return np.packbits(b, bitorder="little")


@dataclass
class Column:
    """One BlockEntry. Exactly one of (`data` host array, `dev_ptr`, `const`) is the payload."""

    dtype: int
    length: int
    data: Optional[np.ndarray] = None          # host Buffer<T>
    dev_ptr: int = 0                            # device Buffer<T>
    validity: Optional[np.ndarray] = None       # packed LSB-first bitmap (host) or None
    dev_validity: int = 0
    validity_bit_offset: int = 0
    is_const: bool = False
    const_value: object = None
    vec_dim: int = 0
    data_bit_offset: int = 0
    _keep: list = field(default_factory=list, repr=False)

    # -- constructors mirroring `XType::from_data` / `from_data_with_validity` / new_const_column
    @staticmethod
    def from_data(values, dtype: Optional[int] = None, validity: Optional[Sequence[bool]] = None,
                  validity_bit_offset: int = 0) -> "Column":
        if dtype is None:
            arr = np.ascontiguousarray(values)
            dtype = dbx_dtype_of(arr)
        elif dtype == abi.BOOL:
            bits = np.asarray(values, dtype=bool)
            col = Column(abi.BOOL, len(bits), data=pack_bitmap(bits))
            if validity is not None:
                col.validity = pack_bitmap(validity, validity_bit_offset)
                col.validity_bit_offset = validity_bit_offset
            return col
        else:
            arr = np.ascontiguousarray(np.asarray(values, dtype=np_dtype(dtype)))
        col = Column(dtype, len(arr), data=arr)
        if validity is not None:
            col.validity = pack_bitmap(validity, validity_bit_offset)
            col.validity_bit_offset = validity_bit_offset
        return col

    @staticmethod
    def from_opt_data(values: Sequence, dtype: int) -> "Column":
        """`from_opt_data`: None entries become NULL (value slot 0)."""
        valid = [v is not None for v in values]
        filled = [0 if v is None else v for v in values]
        return Column.from_data(filled, dtype, validity=valid)

    @staticmethod
    def new_const(dtype: int, value, n: int) -> "Column":
        """BlockEntry::new_const_column (block.rs): value repeated n times, not materialised."""
        return Column(dtype, n, is_const=True, const_value=value)

    @staticmethod
    def vector(values: np.ndarray) -> "Column":
        """VectorColumn::Float32((Buffer<F32>, dim)) (types/vector.rs:377-380)."""
        arr = np.ascontiguousarray(values, dtype=np.float32)
        assert arr.ndim == 2
        return Column(abi.VEC_F32, arr.shape[0], data=arr, vec_dim=arr.shape[1])

    @staticmethod
    def vector_int8(values: np.ndarray) -> "Column":
        """VectorColumn::Int8((Buffer<i8>, dim)) (types/vector.rs:377-380).  The values must already be
        int8: nothing is rounded or clipped here."""
        arr = np.asarray(values)
        if arr.dtype != np.int8 or arr.ndim != 2:
            raise TypeError("Column.vector_int8 takes a 2-d int8 array")
        arr = np.ascontiguousarray(arr)
        return Column(abi.VEC_I8, arr.shape[0], data=arr, vec_dim=arr.shape[1])

    @staticmethod
    def device(dtype: int, length: int, dev_ptr: int, vec_dim: int = 0, dev_validity: int = 0) -> "Column":
        return Column(dtype, length, dev_ptr=dev_ptr, vec_dim=vec_dim, dev_validity=dev_validity)

    # -- helpers
    def slice(self, start: int, end: int) -> "Column":
        """Column::slice: zero-copy; the validity keeps its bytes and gains a bit offset."""
        n = end - start
        if self.is_const:
            return Column(self.dtype, n, is_const=True, const_value=self.const_value)
        c = Column(self.dtype, n, vec_dim=self.vec_dim)
        if self.dtype == abi.BOOL:
            c.data = self.data
            c.data_bit_offset = self.data_bit_offset + start
        elif self.data is not None:
            c.data = self.data[start:end]
        else:
            width = _VEC_ELEM[self.dtype].itemsize * self.vec_dim if self.dtype in _VEC_ELEM else np_dtype(self.dtype).itemsize
            c.dev_ptr = self.dev_ptr + start * width
        if self.validity is not None:
            c.validity = self.validity
            c.validity_bit_offset = self.validity_bit_offset + start
        if self.dev_validity:
            c.dev_validity = self.dev_validity
            c.validity_bit_offset = self.validity_bit_offset + start
        return c

    def valid_mask(self) -> np.ndarray:
        if self.is_const:
            return np.full(self.length, self.const_value is not None)
        if self.validity is None:
            return np.ones(self.length, dtype=bool)
        bits = np.unpackbits(self.validity, bitorder="little")
        return bits[self.validity_bit_offset:self.validity_bit_offset + self.length].astype(bool)

    def values(self) -> np.ndarray:
        if self.is_const:
            v = 0 if self.const_value is None else self.const_value
            return np.full(self.length, v, dtype=np_dtype(self.dtype))
        if self.dtype == abi.BOOL:
            bits = np.unpackbits(self.data, bitorder="little")
            return bits[self.data_bit_offset:self.data_bit_offset + self.length].astype(bool)
        return self.data

    def as_c(self) -> abi.Column:
        c = abi.Column()
        c.dtype = self.dtype
        c.len = self.length
        c.vec_dim = self.vec_dim
        c.is_const = 1 if self.is_const else 0
        c.data_bit_offset = self.data_bit_offset
        c.null_count = -1
        c.validity_bit_offset = self.validity_bit_offset
        if self.is_const:
            c.konst = make_scalar(self.dtype, self.const_value)
            c.mem = abi.MEM_HOST
            return c
        if self.data is not None:
            c.mem = abi.MEM_HOST
            c.data = self.data.ctypes.data
            if self.validity is not None:
                c.validity = self.validity.ctypes.data
        else:
            c.mem = abi.MEM_DEVICE
            c.data = self.dev_ptr
            if self.dev_validity:
                c.validity = self.dev_validity
        return c


@dataclass
class DataBlock:
    """DataBlock::new(entries, num_rows) (block.rs:84-120)."""

    columns: List[Column]
    num_rows: int = -1

    def __post_init__(self):
        if self.num_rows < 0:
            self.num_rows = self.columns[0].length if self.columns else 0
        for c in self.columns:
            assert c.length == self.num_rows, "DataBlock::check_valid: column length mismatch"

    def num_columns(self) -> int:
        return len(self.columns)

    def slice(self, start: int, end: int) -> "DataBlock":
        return DataBlock([c.slice(start, end) for c in self.columns], end - start)

    def split_by_rows(self, max_rows: int) -> List["DataBlock"]:
        """DataBlock::split_by_rows_no_tail-like helper used by TransformFilter."""
        return [self.slice(s, min(s + max_rows, self.num_rows)) for s in range(0, self.num_rows, max_rows)] or [self]

    def freeze(self) -> "DataBlock":
        """Build the C descriptors once and reuse them on every as_c() (the block must not change
        afterwards): what a compiled caller does anyway — only the Python mirror rebuilds them per call."""
        self._frozen = None
        self._frozen = self.as_c()
        return self

    def as_c(self):
        """Returns (dbx_block, keepalive)."""
        fz = getattr(self, "_frozen", None)
        if fz is not None:
            return fz
        arr = (abi.Column * max(1, len(self.columns)))()
        for i, c in enumerate(self.columns):
            arr[i] = c.as_c()
        b = abi.Block()
        b.num_rows = self.num_rows
        b.num_cols = len(self.columns)
        b.cols = C.cast(arr, C.POINTER(abi.Column))
        return b, arr
