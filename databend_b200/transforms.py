"""Host-side mirror of the reference's operator interface for the hot path.

Each class corresponds to a reference Processor / Transform and forwards to one `dbx_op`
handle of libdbx through the C-ABI (include/dbx.h).  Names, argument meaning and error
behaviour follow the reference so the parity tests read like the reference's own tests:

  TransformFilter             src/query/pipeline/transforms/src/processors/transforms/filters/filter_predicate.rs:35-104
  AggregatorParams            src/query/service/src/pipelines/processors/transforms/aggregator/aggregator_params.rs:30-78
  TransformPartialAggregate   .../aggregator/transform_aggregate_partial.rs:117-304  (AccumulatingTransform)
  TransformFinalAggregate     .../aggregator/transform_aggregate_final.rs:67-330
  (no GROUP BY)               .../aggregator/transform_single_key.rs:42-279

In the reference a worker thread calls Processor::process(); here the caller drives
transform()/on_finish() directly (the adaptor contract of transform_accumulating.rs:30-37).
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import abi, expr as E, scalar_expr as S
from .block import Column, DataBlock, np_dtype
from .lib import DbxError, check, load

_AGG_NAMES = {"sum": abi.AGG_SUM, "count": abi.AGG_COUNT, "avg": abi.AGG_AVG, "min": abi.AGG_MIN, "max": abi.AGG_MAX}


class DeviceBuffer:
    """A cudaMalloc'ed buffer owned by Python (tests / bench)."""

    def __init__(self, nbytes: int, device: int = 0):
        self.device, self.nbytes = device, nbytes
        p = C.c_void_p()
        check(load().dbx_device_alloc(device, nbytes, C.byref(p)))
        self.ptr = p.value

    def free(self):
        if self.ptr:
            load().dbx_device_free(self.device, self.ptr)
            self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def upload(self, arr: np.ndarray):
        arr = np.ascontiguousarray(arr)
        assert arr.nbytes <= self.nbytes
        check(load().dbx_memcpy_h2d(self.device, self.ptr, arr.ctypes.data, arr.nbytes))

    def download(self, dtype, count: int) -> np.ndarray:
        out = np.empty(count, dtype=dtype)
        check(load().dbx_memcpy_d2h(self.device, out.ctypes.data, self.ptr, out.nbytes))
        return out


def to_device(col: Column, device: int = 0) -> Column:
    """Copy a host column into HBM (device-resident pipelines)."""
    if col.is_const or col.data is None:
        return col
    buf = DeviceBuffer(max(1, col.data.nbytes), device)
    buf.upload(col.data)
    out = Column(col.dtype, col.length, dev_ptr=buf.ptr, vec_dim=col.vec_dim, data_bit_offset=col.data_bit_offset)
    out._keep.append(buf)
    if col.validity is not None:
        vb = DeviceBuffer(max(1, col.validity.nbytes), device)
        vb.upload(col.validity)
        out.dev_validity = vb.ptr
        out.validity_bit_offset = col.validity_bit_offset
        out._keep.append(vb)
    return out


def _block_from_c(b: abi.Block, device: int) -> DataBlock:
    """Copy a library-owned HOST output block into numpy-backed columns, then release it."""
    cols = []
    for i in range(b.num_cols):
        c = b.cols[i]
        n = c.len
        if c.is_const:  # BlockEntry::Const stays const
            k = c.konst
            if k.is_null:
                v = None
            elif c.dtype in (abi.F32, abi.F64):
                v = k.v.f64
            elif c.dtype in (abi.U8, abi.U16, abi.U32, abi.U64, abi.BOOL):
                v = k.v.u64
            else:
                v = k.v.i64
            cols.append(Column.new_const(c.dtype, v, n))
            continue
        assert c.mem == abi.MEM_HOST
        if c.dtype == abi.BOOL:
            nb = (c.data_bit_offset + n + 7) // 8
            arr = np.zeros(max(nb, 1), dtype=np.uint8)
            if nb:
                C.memmove(arr.ctypes.data, c.data, nb)
            col = Column(abi.BOOL, n, data=arr, data_bit_offset=c.data_bit_offset)
        elif c.dtype in (abi.VEC_F32, abi.VEC_I8):
            arr = np.empty((n, c.vec_dim), dtype=np.float32 if c.dtype == abi.VEC_F32 else np.int8)
            if n:
                C.memmove(arr.ctypes.data, c.data, arr.nbytes)
            col = Column(c.dtype, n, data=arr, vec_dim=c.vec_dim)
        else:
            nd = np_dtype(c.dtype)
            arr = np.empty(n, dtype=nd)
            if n:
                C.memmove(arr.ctypes.data, c.data, arr.nbytes)
            col = Column(c.dtype, n, data=arr)
        if c.validity:
            nb = (c.validity_bit_offset + n + 7) // 8
            v = np.empty(max(nb, 1), dtype=np.uint8)
            if nb:
                C.memmove(v.ctypes.data, c.validity, nb)
            col.validity = v
            col.validity_bit_offset = c.validity_bit_offset
        cols.append(col)
    rows = b.num_rows
    check(load().dbx_block_release(C.byref(b)))
    return DataBlock(cols, rows)


class _Op:
    """Owns one dbx_op handle."""

    def __init__(self, kind: int, params, input_types: Sequence[int], device: int, computed=None):
        self._h = C.c_void_p()
        self.device = device
        types = (C.c_int32 * max(1, len(input_types)))(*input_types)
        self._params = params
        if computed is not None and computed.exprs:
            self._computed = computed.to_c()
            check(load().dbx_op_create_computed(kind, C.cast(C.byref(params), C.c_void_p), types, len(input_types), self._computed,
                                                len(computed.exprs), device, C.byref(self._h)))
            return
        check(load().dbx_op_create(kind, C.cast(C.byref(params), C.c_void_p), types, len(input_types), device,
                                   C.byref(self._h)))

    @property
    def handle(self):
        return self._h

    def push(self, block: DataBlock):
        b, keep = block.as_c()
        check(load().dbx_op_push(self._h, C.byref(b)), self._h)

    def finish(self):
        check(load().dbx_op_finish(self._h), self._h)

    def pull_c(self, out_mem: int = abi.MEM_HOST) -> Optional[abi.Block]:
        b = abi.Block()
        has = C.c_int32(0)
        check(load().dbx_op_pull(self._h, out_mem, C.byref(b), C.byref(has)), self._h)
        return b if has.value else None

    def reset(self):
        check(load().dbx_op_reset(self._h), self._h)

    def synchronize(self):
        check(load().dbx_op_synchronize(self._h), self._h)

    def last_kernel_ms(self) -> float:
        ms = C.c_float(0)
        check(load().dbx_op_last_kernel_ms(self._h, C.byref(ms)), self._h)
        return ms.value

    def kernel_ms(self, back: int = 0) -> float:
        """Device time of the dominant kernel(s) of an earlier push (0 = last, 1 = the one before ...)."""
        ms = C.c_float(0)
        check(load().dbx_op_kernel_ms(self._h, back, C.byref(ms)), self._h)
        return ms.value

    def kernel_variant(self) -> str:
        """"specialised" (kernel compiled for this plan) or "precompiled kernels (<why>)"."""
        buf = C.create_string_buffer(2048)
        check(load().dbx_op_kernel_variant(self._h, buf, 2048), self._h)
        return buf.value.decode("utf-8", "replace")

    def inputs_consumed(self):
        """Block until every pushed block has been read completely (pinned/device inputs may be reused)."""
        check(load().dbx_op_inputs_consumed(self._h), self._h)

    def close(self):
        if self._h:
            load().dbx_op_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TransformFilter(_Op):
    """TransformFilter (filters/filter_predicate.rs:35-104) = FilterExecutor::filter
    (filter_executor.rs:82-160): `transform(block)` returns the rows for which the predicate is
    true, in input order, for every column.  NULL predicate values count as false."""

    def __init__(self, predicate: Optional[E.Node], input_types: Sequence[int], device: int = 0):
        """Predicate operands may be scalar_expr.SExpr: evaluated inside the filter kernel."""
        computed = S.Computed(len(input_types))
        super().__init__(abi.OP_FILTER, E.build_predicate(predicate, computed), input_types, device, computed)

    def transform(self, block: DataBlock) -> DataBlock:
        self.push(block)
        b = self.pull_c(abi.MEM_HOST)
        return _block_from_c(b, self.device)


@dataclass
class AggregatorParams:
    """AggregatorParams::try_create (aggregator_params.rs:44-78): group column offsets and the
    aggregate functions with their argument offsets.  `aggregate_functions` entries are
    (factory name, argument column offset or None for count())."""

    group_columns: List[int]
    aggregate_functions: List[Tuple[str, Optional[int]]]
    expected_groups: int = 0

    # A group column or an aggregate argument may also be a scalar_expr.SExpr: the operators evaluate it
    # as a computed column inside their kernels.

    def computed(self, n_inputs: int, filter_expr: Optional[E.Node] = None) -> S.Computed:
        """The operator's computed columns: the expressions of the group columns and arguments first (so a
        final operator built from the same params numbers them alike), then the predicate's."""
        c = S.Computed(n_inputs)
        for g in self.group_columns:
            c.column(g)
        for _, arg in self.aggregate_functions:
            if arg is not None:
                c.column(arg)
        for e in E.sexprs(filter_expr):
            c.column(e)
        return c

    def to_c(self, filter_expr: Optional[E.Node] = None, computed: Optional[S.Computed] = None) -> abi.AggParams:
        def colno(x):
            if isinstance(x, S.SExpr):
                if computed is None:
                    raise ValueError("parameters with scalar expressions need the operator's computed-column list")
                return computed.column(x)
            return x
        p = abi.AggParams()
        p.n_group_cols = len(self.group_columns)
        for i, g in enumerate(self.group_columns):
            p.group_cols[i] = colno(g)
        p.n_aggs = len(self.aggregate_functions)
        for i, (name, arg) in enumerate(self.aggregate_functions):
            if name not in _AGG_NAMES:
                raise DbxError(abi.ERR_UNSUPPORTED, f"Unknown aggregate function {name}")  # factory.get error
            p.aggs[i].kind = _AGG_NAMES[name]
            p.aggs[i].arg_col = -1 if arg is None else colno(arg)
        p.filter = E.build_predicate(filter_expr, computed)
        p.expected_groups = self.expected_groups
        return p


def schema_types(block_or_types, nullable: Optional[Sequence[bool]] = None) -> List[int]:
    """DataSchema -> input_types[] with the DBX_NULLABLE flag for Nullable(T) columns."""
    if isinstance(block_or_types, DataBlock):
        out = []
        for c in block_or_types.columns:
            nul = c.validity is not None or c.dev_validity != 0 or (c.is_const and c.const_value is None)
            out.append(c.dtype | (abi.NULLABLE if nul else 0))
        return out
    types = list(block_or_types)
    if nullable:
        types = [t | (abi.NULLABLE if n else 0) for t, n in zip(types, nullable)]
    return types


class TransformPartialAggregate(_Op):
    """[TransformFilter ->] TransformPartialAggregate fused into one device pass.

    transform(block) accumulates (AccumulatingTransform::transform returns no blocks while
    the hash table has room); on_finish() yields the payload reference that
    TransformFinalAggregate consumes (AggregateMeta::AggregatePayload)."""

    def __init__(self, params: AggregatorParams, input_types: Sequence[int], filter_expr: Optional[E.Node] = None,
                 device: int = 0):
        self.params = params
        computed = params.computed(len(input_types), filter_expr)
        super().__init__(abi.OP_AGG_PARTIAL, params.to_c(filter_expr, computed), input_types, device, computed)

    def transform(self, block: DataBlock) -> List[DataBlock]:
        self.push(block)
        return []

    def finish(self):
        """A computed column that failed on a row the predicate kept raises scalar_expr.EvalError with
        the first failing row (rows counted from the first row pushed since create / reset)."""
        st = load().dbx_op_finish(self._h)
        if st == abi.ERR_BAD_ARGUMENTS:
            msg = (load().dbx_last_error(self._h) or b"").decode("utf-8", "replace")
            m = re.search(r"first failing row (\d+)", msg)
            raise S.EvalError(st, msg, int(m.group(1)) if m else -1)
        check(st, self._h)

    def on_finish(self):
        self.finish()
        return self  # the payload stays in HBM; the handle is the AggregateMeta

    def serialize(self):
        """The partial's groups in the reference's spill / wire layout (AggregatorParams::spill_schema):
        (block with every `agg_i` Tuple flattened into consecutive columns followed by the group
        columns, [arity of agg_0, ...])."""
        out = abi.Block()
        arity = (C.c_int32 * abi.MAX_AGGS)()
        check(load().dbx_agg_partial_serialize(self._h, abi.MEM_HOST, C.byref(out), arity), self._h)
        return _block_from_c(out, self.device), list(arity[:len(self.params.aggregate_functions)])


class TransformFinalAggregate(_Op):
    def __init__(self, params: AggregatorParams, input_types: Sequence[int], device: int = 0):
        self.params = params
        computed = params.computed(len(input_types))
        super().__init__(abi.OP_AGG_FINAL, params.to_c(None, computed), input_types, device, computed)

    def transform(self, partial: TransformPartialAggregate) -> List[DataBlock]:
        """handle_meta -> combine_payload (transform_aggregate_final.rs:201-303)."""
        check(load().dbx_agg_final_merge_partial(self._h, partial.handle), self._h)
        return []

    def merge_serialized(self, block: DataBlock):
        """Merge a spill-schema block (flattened tuples + group columns) produced by a CPU partial
        aggregate or by TransformPartialAggregate.serialize() elsewhere."""
        b, keep = block.as_c()
        check(load().dbx_agg_final_merge_serialized(self._h, C.byref(b)), self._h)
        del keep

    def merge_rows(self, dev_rows_ptr: int, n_rows: int):
        check(load().dbx_agg_final_merge_rows(self._h, dev_rows_ptr, n_rows), self._h)

    def on_finish(self, out_mem: int = abi.MEM_HOST):
        """merge_result: returns the result blocks [aggs..., group keys...]."""
        self.finish()
        if out_mem == abi.MEM_HOST:
            b = self.pull_c(abi.MEM_HOST)
            return [] if b is None else [_block_from_c(b, self.device)]
        b = self.pull_c(abi.MEM_DEVICE)
        return [] if b is None else [b]


class TransformTopN(_Op):
    """ORDER BY key LIMIT k: TransformSortPartial + limit-aware merge / TransformPartialTopN+FinalTopN
    (sorts/sort_partial.rs:24-60, top_n/transform_partial_top_n.rs:73-130) as one streaming device
    top-k.  SortColumnDescription{offset, asc, nulls_first} + LimitType::LimitRows(k)
    (kernels/sort.rs:41-63).  The result block is [key column, row_id Int64] in output order; ties
    are broken by ascending row id."""

    def __init__(self, offset: int, asc: bool, nulls_first: bool, limit: int, input_types: Sequence[int], device: int = 0,
                 extra_keys: Sequence[Tuple[int, bool, bool]] = ()):
        """extra_keys: further SortColumnDescriptions (offset, asc, nulls_first) that break ties of the
        earlier keys (ORDER BY a, b, c); the result still is [first key column, row_id]."""
        p = abi.TopkParams()
        p.key_col, p.asc, p.nulls_first, p.limit = offset, int(asc), int(nulls_first), limit
        p.n_extra_keys = len(extra_keys)
        for i, (c, a, nf) in enumerate(extra_keys):
            p.extra_key_cols[i], p.extra_asc[i], p.extra_nulls_first[i] = c, int(a), int(nf)
        super().__init__(abi.OP_TOPK, p, input_types, device)

    def transform(self, block: DataBlock) -> List[DataBlock]:
        self.push(block)
        return []

    def on_finish(self) -> DataBlock:
        self.finish()
        b = self.pull_c(abi.MEM_HOST)
        return _block_from_c(b, self.device)


_WIN_KINDS = {"row_number": abi.WIN_ROW_NUMBER, "rank": abi.WIN_RANK, "dense_rank": abi.WIN_DENSE_RANK,
              "percent_rank": abi.WIN_PERCENT_RANK, "cume_dist": abi.WIN_CUME_DIST, "ntile": abi.WIN_NTILE, "lag": abi.WIN_LAG,
              "lead": abi.WIN_LEAD, "nth_value": abi.WIN_NTH_VALUE, "last_value": abi.WIN_NTH_VALUE}
_WIN_AGGS = {"sum": abi.AGG_SUM, "count": abi.AGG_COUNT, "avg": abi.AGG_AVG, "min": abi.AGG_MIN, "max": abi.AGG_MAX}
_BOUNDS = {"unbounded_preceding": abi.BOUND_UNBOUNDED_PRECEDING, "preceding": abi.BOUND_PRECEDING, "current_row": abi.BOUND_CURRENT_ROW,
           "following": abi.BOUND_FOLLOWING, "unbounded_following": abi.BOUND_UNBOUNDED_FOLLOWING}


@dataclass
class WindowFunc:
    """One Window node: `name` is a ranking function, ntile, lag, lead, nth_value, last_value or an
    aggregate (sum, count, avg, min, max; arg = -1 is count(*)).  `n`: ntile buckets, lag / lead offset,
    nth_value index.  `default`: lag / lead default column (-1: NULL).  `frame` (aggregates and
    nth_value only): (units "rows" | "range", start, end), a bound being "unbounded_preceding",
    ("preceding", k), "current_row", ("following", k) or "unbounded_following"."""
    name: str
    arg: int = -1
    n: int = 0
    default: int = -1
    frame: Optional[Tuple] = None
    ignore_nulls: bool = False
    distinct: bool = False

    def to_c(self, out: abi.WindowFunc):
        if self.name in _WIN_AGGS:
            out.kind, out.agg_kind = abi.WIN_AGGREGATE, _WIN_AGGS[self.name]
        else:
            out.kind = _WIN_KINDS[self.name]
        out.arg_col, out.default_col, out.n = self.arg, self.default, self.n
        out.ignore_nulls, out.distinct = int(self.ignore_nulls), int(self.distinct)
        if self.frame is not None:
            units, start, end = self.frame
            out.frame.units = abi.FRAME_RANGE if units == "range" else abi.FRAME_ROWS
            for b, kind_f, off_f in ((start, "start", "start_offset"), (end, "end", "end_offset")):
                name, off = (b, 0) if isinstance(b, str) else b
                setattr(out.frame, kind_f, _BOUNDS[name])
                setattr(out.frame, off_f, off)


class TransformWindow(_Op):
    """WindowPartition + its chain of Window nodes (physical_window{,_partition}.rs, TransformWindow
    transform_window.rs) as one DBX_OP_WINDOW.  `transform(block)` buffers the block on the device;
    `on_finish()` returns one block: every input column in window order (grouped by partition, sorted
    by the order keys inside it, ties in input order), then one column per function."""

    def __init__(self, partition_by: Sequence[int], order_by: Sequence[Tuple[int, bool, bool]], funcs: Sequence[WindowFunc],
                 input_types: Sequence[int], device: int = 0):
        """order_by: (offset, asc, nulls_first) per ORDER BY key."""
        p = abi.WindowParams()
        p.n_partition_cols, p.n_order_cols, p.n_funcs = len(partition_by), len(order_by), len(funcs)
        for i, c in enumerate(partition_by[:abi.MAX_SORT_KEYS]):
            p.partition_cols[i] = c
        for i, (c, a, nf) in enumerate(order_by[:abi.MAX_SORT_KEYS]):
            p.order_cols[i], p.order_asc[i], p.order_nulls_first[i] = c, int(a), int(nf)
        for i, f in enumerate(funcs[:abi.MAX_WINDOW_FUNCS]):
            f.to_c(p.funcs[i])
        super().__init__(abi.OP_WINDOW, p, input_types, device)

    def transform(self, block: DataBlock) -> List[DataBlock]:
        self.push(block)
        return []

    def on_finish(self, out_mem: int = abi.MEM_HOST):
        """The result as a host DataBlock, or (out_mem = MEM_DEVICE) the library-owned abi.Block."""
        self.finish()
        b = self.pull_c(out_mem)
        return _block_from_c(b, self.device) if out_mem == abi.MEM_HOST else b


def _key_list(key) -> List[int]:
    return [int(key)] if isinstance(key, (int, np.integer)) else [int(k) for k in key]


_SIGNED = (abi.I8, abi.I16, abi.I32, abi.I64)
_KEY_BYTES = {abi.I8: 1, abi.U8: 1, abi.I16: 2, abi.U16: 2, abi.I32: 4, abi.U32: 4, abi.I64: 8, abi.U64: 8}


def join_key_layout(build_dtypes: Sequence[int], probe_dtypes: Sequence[int]) -> Tuple[List[Tuple[int, int]], int]:
    """The composite join key's bit fields as the operator packs them: [(shift, width in bits)] per key
    pair and the total bits, with a field never straddling bit 64.  A pair's width is its common
    type's: the larger size for equal signedness, max(S, 2 U) bytes for signed S with unsigned U.
    Up to 64 bits the table key is one word, up to 128 bits two; wider layouts are refused."""
    fields, bits = [], 0
    for b, p in zip(build_dtypes, probe_dtypes):
        b, p = b & 0xFF, p & 0xFF
        if b not in _KEY_BYTES or p not in _KEY_BYTES:
            raise DbxError(abi.ERR_UNSUPPORTED, "join: keys must be integer columns")
        bs, ps, bz, pz = b in _SIGNED, p in _SIGNED, _KEY_BYTES[b], _KEY_BYTES[p]
        if (b == abi.U64 and ps) or (p == abi.U64 and bs):
            raise DbxError(abi.ERR_UNSUPPORTED, "join: a signed key cannot be compared with a UInt64 key without a cast")
        w = 8 * (max(bz, pz) if bs == ps else max(bz, 2 * pz) if bs else max(pz, 2 * bz))
        if bits < 64 < bits + w:
            bits = 64
        fields.append((bits, w))
        bits += w
    return fields, bits


class HashJoin(_Op):
    """Hash join behind the reference's `Join` trait (new_hash_join/join.rs:26-53):
    add_block(build block) / final_build() / probe_block(block) -> joined blocks /
    final_probe() -> the build rows a build-side join keeps.
    Output columns = probe columns then build columns (inner_join.rs:236-245); output row order is
    unspecified (compare as multisets)."""

    def __init__(self, build_types: Sequence[int], probe_types: Sequence[int], build_key: Union[int, Sequence[int]],
                 probe_key: Union[int, Sequence[int]], device: int = 0, kind: int = abi.JOIN_INNER, expected_build_rows: int = 0,
                 other_predicate: Optional[S.SExpr] = None):
        """kind (probe side = left, build side = right):
          JOIN_INNER, JOIN_LEFT (probe rows kept), JOIN_LEFT_SEMI / JOIN_LEFT_ANTI (probe columns only:
          left_join_semi.rs / left_join_anti.rs);
          JOIN_RIGHT (build rows kept: final_probe emits the unmatched ones with NULL probe columns),
          JOIN_RIGHT_SEMI / JOIN_RIGHT_ANTI (build columns only, all from final_probe), JOIN_FULL
          (LEFT during the probe, then RIGHT's final stream).
        build_key / probe_key: one column index each, or equally long sequences of up to
        abi.MAX_JOIN_KEYS indices (ON b[0] = p[0] AND b[1] = p[1] ...; a NULL in any key column never
        matches).  The keys are packed into 64 or 128 bits (join_key_layout).
        other_predicate: the ON clause's non-equi conditions ANDed together (HashJoinDesc::other_predicate), a
        Boolean scalar_expr.SExpr whose column i is build column i for i < len(build_types) and probe column
        i - len(build_types) above.  It is evaluated on every pair of equal keys inside the probe; a pair on
        which it is NULL or false is no match, for every kind (include/dbx.h: dbx_op_create_join)."""
        bkeys, pkeys = _key_list(build_key), _key_list(probe_key)
        if len(bkeys) != len(pkeys) or not 1 <= len(bkeys) <= abi.MAX_JOIN_KEYS:
            raise DbxError(abi.ERR_INVALID, f"join: build and probe keys must be 1 .. {abi.MAX_JOIN_KEYS} columns each, as many on both sides")
        p = abi.JoinParams()
        p.kind, p.build_key_col, p.probe_key_col, p.n_build_cols = kind, bkeys[0], pkeys[0], len(build_types)
        p.expected_build_rows = expected_build_rows
        p.n_extra_keys = len(bkeys) - 1
        for i in range(1, len(bkeys)):
            p.extra_build_key_cols[i - 1], p.extra_probe_key_cols[i - 1] = bkeys[i], pkeys[i]
        types = list(build_types) + list(probe_types)
        if other_predicate is None:
            super().__init__(abi.OP_JOIN, p, types, device)
            return
        self._h = C.c_void_p()
        self.device = device
        self._params = p
        self._predicate = S.flatten(other_predicate)
        ctypes_ = (C.c_int32 * len(types))(*types)
        check(load().dbx_op_create_join(C.byref(p), ctypes_, len(types), C.byref(self._predicate), device, C.byref(self._h)))

    def add_block(self, block: DataBlock):
        self.push(block)

    def final_build(self):
        self.finish()

    def probe_block(self, block: DataBlock, out_mem: int = abi.MEM_HOST) -> List[DataBlock]:
        b, keep = block.as_c()
        check(load().dbx_join_probe(self._h, C.byref(b)), self._h)
        out = []
        while True:
            ob = self.pull_c(out_mem)
            if ob is None:
                break
            out.append(_block_from_c(ob, self.device) if out_mem == abi.MEM_HOST else ob)
        return out

    def runtime_filter(self, enable_inlist: bool = True, enable_bloom: bool = True, enable_min_max: bool = True,
                       in_probe: bool = False, inlist_threshold: int = 1024, bloom_threshold: int = 3_000_000,
                       min_max_threshold: int = 2**64 - 1, build_table_rows: int = 0,
                       selectivity_threshold: int = 10) -> RuntimeFilter:
        """The runtime filter of the finished build side (defaults = the reference's settings).
        build_table_rows = 0 means unknown, so no bloom.  in_probe: the probe kernel also tests min-max
        and bloom until reset() (single-key joins)."""
        p = abi.RuntimeFilterParams()
        p.enable_inlist, p.enable_bloom, p.enable_min_max, p.in_probe = int(enable_inlist), int(enable_bloom), int(enable_min_max), int(in_probe)
        p.inlist_threshold, p.bloom_threshold, p.min_max_threshold = inlist_threshold, bloom_threshold, min_max_threshold
        p.build_table_rows, p.selectivity_threshold = build_table_rows, selectivity_threshold
        h = C.c_void_p()
        check(load().dbx_join_runtime_filter(self._h, C.byref(p), C.byref(h)), self._h)
        return RuntimeFilter(h, self.device)

    def final_probe(self, out_mem: int = abi.MEM_HOST) -> List[DataBlock]:
        """Join::final_probe, called once after the last probe_block: the build rows that RIGHT,
        RIGHT ANTI and FULL keep unmatched, or that RIGHT SEMI matched (each once).  Empty for the
        other kinds and on a second call.  probe_block fails after it until reset()."""
        check(load().dbx_join_final_probe(self._h), self._h)
        out = []
        while True:
            ob = self.pull_c(out_mem)
            if ob is None:
                break
            out.append(_block_from_c(ob, self.device) if out_mem == abi.MEM_HOST else ob)
        return out


@dataclass
class RuntimeFilterPartInfo:
    """One key pair's filters: which exist, the bounds and sizes (common type `key_dtype`)."""
    has_min_max: bool
    has_inlist: bool
    has_bloom: bool
    key_dtype: int
    min: Optional[int]
    max: Optional[int]
    inlist_len: int
    bloom_bytes: int


@dataclass
class RuntimeFilterInfo:
    """RuntimeFilterInfo + RuntimeFilterStats (catalog/src/runtime_filter_info.rs)."""
    build_rows: int
    in_probe: bool
    apply_rows_checked: int
    apply_rows_rejected: int
    probe_rows_checked: int
    probe_rows_rejected: int
    parts: List[RuntimeFilterPartInfo]


class RuntimeFilter:
    """A join's runtime filter (dbx_runtime_filter): min-max, IN-list and bloom per key pair, built on
    the device from the build keys.  Valid after the join is reset or closed."""

    def __init__(self, handle: C.c_void_p, device: int):
        self._h, self.device = handle, device

    def info(self) -> RuntimeFilterInfo:
        r = abi.RfInfo()
        check(load().dbx_runtime_filter_info(self._h, C.byref(r)))
        parts = []
        for i in range(r.n_parts):
            pi = r.parts[i]
            signed = pi.key_dtype in _SIGNED

            def val(s):
                return None if s.is_null else (s.v.i64 if signed else s.v.u64)
            parts.append(RuntimeFilterPartInfo(bool(pi.has_min_max), bool(pi.has_inlist), bool(pi.has_bloom), pi.key_dtype,
                                               val(pi.min), val(pi.max), pi.inlist_len, pi.bloom_bytes))
        return RuntimeFilterInfo(r.build_rows, bool(r.in_probe), r.apply_rows_checked, r.apply_rows_rejected,
                                 r.probe_rows_checked, r.probe_rows_rejected, parts)

    def bloom_words(self, part: int = 0) -> np.ndarray:
        """The bloom filter of key pair `part` as uint32 words (8 per 32-byte block); empty if none."""
        n = self.info().parts[part].bloom_bytes // 4
        out = np.zeros(n, dtype=np.uint32)
        if n:
            check(load().dbx_runtime_filter_export(self._h, part, out.ctypes.data_as(C.POINTER(C.c_uint32)), n, None, 0))
        return out

    def inlist(self, part: int = 0) -> np.ndarray:
        """The distinct build keys of pair `part`, ascending, as the common type (empty if none)."""
        pi = self.info().parts[part]
        out = np.zeros(pi.inlist_len, dtype=np.int64)
        if pi.inlist_len:
            check(load().dbx_runtime_filter_export(self._h, part, None, 0, out.ctypes.data_as(C.POINTER(C.c_int64)), pi.inlist_len))
        return out.view(np_dtype(abi.I64 if pi.key_dtype in _SIGNED else abi.U64)).astype(np_dtype(pi.key_dtype))

    def apply(self, block: DataBlock, key_cols: Union[int, Sequence[int]]) -> Column:
        """ExprBloomFilter::apply ANDed over the parts: a Boolean column, true where the probe row may
        match.  key_cols: the probe key column of each key pair in `block`."""
        cols = _key_list(key_cols)
        kc = (C.c_int32 * len(cols))(*cols)
        b, keep = block.as_c()
        out = abi.Block()
        passed = C.c_int64(0)
        check(load().dbx_runtime_filter_apply(self._h, C.byref(b), kc, abi.MEM_HOST, C.byref(out), C.byref(passed)))
        del keep
        col = _block_from_c(out, self.device).columns[0]
        self.last_passed = passed.value
        return col

    def close(self):
        if self._h:
            load().dbx_runtime_filter_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def filter_group_aggregate(blocks: Sequence[DataBlock], params: AggregatorParams, filter_expr: Optional[E.Node] = None,
                           input_types: Optional[Sequence[int]] = None, device: int = 0,
                           n_partials: int = 1) -> DataBlock:
    """Convenience pipeline: Filter -> Partial x n_partials -> Final, like
    PipelineBuilder::build_aggregate_partial/final would wire it."""
    types = list(input_types) if input_types is not None else schema_types(blocks[0])
    partials = [TransformPartialAggregate(params, types, filter_expr, device) for _ in range(n_partials)]
    for i, b in enumerate(blocks):
        partials[i % n_partials].transform(b)
    final = TransformFinalAggregate(params, types, device)
    for p in partials:
        final.transform(p.on_finish())
    out = final.on_finish()
    for p in partials:
        p.close()
    final.close()
    return out[0]
