"""CPU ORACLE (test infrastructure only) for DBX_OP_WINDOW.

A straight restatement of TransformWindow's row loop (src/query/pipeline/transforms/src/processors/
transforms/window/transform_window.rs: add_block :1003-1153, apply_aggregate :481-526,
merge_result_of_current_row :529-660) over ONE sorted input.  The order is sort_oracle.sort_permutation
over the partition keys (ascending, NULLS LAST) then the order keys; ties keep input order.  Partition
and peer boundaries use ScalarRef equality: NULL == NULL, floats as OrderedFloat (NaN == NaN, -0 == +0).

Aggregates keep one state per function and, like apply_aggregate, either extend it by the rows between
the previous and the new frame end (the frame start did not move) or reset it and add the whole frame,
in row order.  Sums are 64-bit wrapping for integers and Float64 (f32 widened) for floats, avg is the
sum over the count in Float64, min / max compare OrderedFloat images in which -0 < +0 and every NaN is
one greatest value (the aggregate path's rule), count counts non-NULL arguments (count(*): rows).
Meant for up to about 1e5 rows."""
from __future__ import annotations

import struct
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

from databend_b200 import abi
from oracle.sort_oracle import sort_permutation

RESULT_NP = {abi.I8: np.int8, abi.I16: np.int16, abi.I32: np.int32, abi.I64: np.int64, abi.U8: np.uint8, abi.U16: np.uint16,
             abi.U32: np.uint32, abi.U64: np.uint64, abi.F32: np.float32, abi.F64: np.float64}
SIGNED = (abi.I8, abi.I16, abi.I32, abi.I64)
FLOATS = (abi.F32, abi.F64)
M64 = (1 << 64) - 1


@dataclass
class Col:
    values: np.ndarray
    valid: Optional[np.ndarray]  # None: no NULLs
    dtype: int
    nullable: bool = False


def f64_ordered(x: float) -> int:
    """common.cuh f64_to_ordered: NaN greatest, -0 below +0."""
    if x != x:
        return M64
    b = struct.unpack("<Q", struct.pack("<d", x))[0]
    return (~b & M64) if b >> 63 else b | (1 << 63)


def ordered_f64(o: int) -> float:
    if o == M64:
        return float("nan")
    b = (o & ~(1 << 63) & M64) if o >> 63 else (~o & M64)
    return struct.unpack("<d", struct.pack("<Q", b))[0]


def result_type(f, cols: Sequence[Col]) -> Tuple[int, bool]:
    """(dtype, nullable) of a function's column (WindowFunction::data_type)."""
    if f.name in ("percent_rank", "cume_dist"):
        return abi.F64, False
    if f.name in ("row_number", "rank", "dense_rank", "ntile"):
        return abi.U64, False
    if f.name in ("lag", "lead"):
        a = cols[f.arg]
        return a.dtype, f.default < 0 or cols[f.default].nullable or a.nullable
    if f.name in ("nth_value", "last_value"):
        return cols[f.arg].dtype, True
    if f.name == "count":
        return abi.U64, False
    if f.name == "avg":
        return abi.F64, True
    dt = cols[f.arg].dtype
    if f.name == "sum":
        return (abi.F64 if dt in FLOATS else abi.I64 if dt in SIGNED else abi.U64), True
    return dt, True


def _bound(b):
    return (b, 0) if isinstance(b, str) else (b[0], int(b[1]))


def _bound_key(b):
    name, off = _bound(b)
    order = ["unbounded_preceding", "preceding", "current_row", "following", "unbounded_following"]
    return order.index(name), (-off if name == "preceding" else off if name == "following" else 0)


def _key_equal(col: Col, a: int, b: int) -> bool:
    va = col.valid is None or col.valid[a]
    vb = col.valid is None or col.valid[b]
    if not va or not vb:
        return va == vb
    x, y = col.values[a], col.values[b]
    if col.dtype in FLOATS and x != x:
        return y != y
    return x == y


class _Agg:
    def __init__(self, name: str, col: Optional[Col]):
        self.name, self.col = name, col
        self.reset()

    def reset(self):
        self.count = 0
        self.acc = 0.0 if self.col is not None and self.col.dtype in FLOATS and self.name in ("sum", "avg") else 0
        self.ext = None

    def add(self, r: int):
        c = self.col
        if c is None:
            self.count += 1
            return
        if c.valid is not None and not c.valid[r]:
            return
        self.count += 1
        v = c.values[r]
        if self.name in ("sum", "avg"):
            if c.dtype in FLOATS:
                self.acc = self.acc + float(v)
            else:
                self.acc = (self.acc + int(v)) & M64
        elif self.name in ("min", "max"):
            img = f64_ordered(float(v)) if c.dtype in FLOATS else int(v)
            if self.ext is None or (img < self.ext if self.name == "min" else img > self.ext):
                self.ext = img

    def result(self):
        c = self.col
        if self.name == "count":
            return self.count, True
        if self.count == 0:
            return 0, False
        if self.name in ("sum", "avg"):
            if c.dtype in FLOATS:
                s = self.acc
            elif c.dtype in SIGNED:
                s = self.acc - (1 << 64) if self.acc >> 63 else self.acc
            else:
                s = self.acc
            if self.name == "avg":
                return float(s) / float(self.count), True
            return s, True
        return (ordered_f64(self.ext) if c.dtype in FLOATS else self.ext), True


def window(cols: Sequence[Col], partition_by: Sequence[int], order_by: Sequence[Tuple[int, bool, bool]], funcs) -> Tuple[np.ndarray, List]:
    """-> (permutation: sorted position -> input row, [(values, valid) per function in window order])."""
    n = len(cols[0].values) if cols else 0
    keys = [(cols[c].values, cols[c].valid, True, False) for c in partition_by]
    keys += [(cols[c].values, cols[c].valid, asc, nf) for c, asc, nf in order_by]
    perm = sort_permutation(keys) if keys and n else np.arange(n)
    sc = [Col(c.values[perm], None if c.valid is None else np.asarray(c.valid, bool)[perm], c.dtype, c.nullable) for c in cols]
    # partition and peer boundaries
    ps = np.zeros(n, np.int64)
    pe = np.zeros(n, np.int64)
    gs = np.zeros(n, np.int64)
    ge = np.zeros(n, np.int64)
    dense = np.zeros(n, np.int64)
    start = 0
    for i in range(n):
        new_part = i == 0 or not all(_key_equal(sc[c], i, i - 1) for c in partition_by)
        new_peer = new_part or not all(_key_equal(sc[c], i, i - 1) for c, _, _ in order_by)
        if new_part:
            start, d = i, 0
        if new_peer:
            gstart, d = i, d + 1
        ps[i], gs[i], dense[i] = start, gstart, d
    end = n
    gend = n
    for i in range(n - 1, -1, -1):
        pe[i] = end
        ge[i] = gend
        if ps[i] == i:
            end = i
        if gs[i] == i:
            gend = i
    out = []
    for f in funcs:
        dt, _ = result_type(f, cols)
        vals = np.zeros(n, RESULT_NP[dt])
        valid = np.ones(n, bool)
        arg = sc[f.arg] if f.arg >= 0 else None
        if f.name in ("sum", "count", "avg", "min", "max", "nth_value", "last_value"):
            units, sb, eb = f.frame
            empty_static = _bound_key(sb) > _bound_key(eb)
            agg = _Agg(f.name, arg) if f.name not in ("nth_value", "last_value") else None
            prev_s = prev_e = 0
            for i in range(n):
                p0, p1 = ps[i], pe[i]
                if i == p0:  # a new partition: reset function and frames
                    if agg:
                        agg.reset()
                    prev_s = prev_e = p0
                if empty_static:
                    s = e = p0 if i == p0 else prev_s
                    if agg:
                        agg.reset()
                else:
                    s, e = _frame(units, sb, eb, i, p0, p1, gs[i], ge[i])
                    if agg:
                        if s == prev_s:
                            for r in range(prev_e, e):
                                agg.add(r)
                        else:
                            agg.reset()
                            for r in range(s, e):
                                agg.add(r)
                if agg:
                    v, ok = agg.result()
                else:
                    k = f.n if f.name == "nth_value" else 0
                    t = (e - 1) if k == 0 else s + k - 1
                    if empty_static or s >= e or t >= e:
                        v, ok = 0, False
                    else:
                        v, ok = arg.values[t], arg.valid is None or bool(arg.valid[t])
                vals[i] = v if ok else 0
                valid[i] = ok
                prev_s, prev_e = s, e
        else:
            for i in range(n):
                p0, p1 = ps[i], pe[i]
                size = p1 - p0
                ok = True
                if f.name == "row_number":
                    v = i - p0 + 1
                elif f.name == "rank":
                    v = gs[i] - p0 + 1
                elif f.name == "dense_rank":
                    v = dense[i]
                elif f.name == "percent_rank":
                    v = 0.0 if size <= 1 else float(gs[i] - p0) / float(size - 1)
                elif f.name == "cume_dist":
                    v = float(ge[i] - p0) / float(size)
                elif f.name == "ntile":
                    v = _ntile(f.n, i - p0 + 1, size)
                else:  # lag / lead
                    t = i - f.n if f.name == "lag" else i + f.n
                    if p0 <= t < p1:
                        v, ok = arg.values[t], arg.valid is None or bool(arg.valid[t])
                    elif f.default >= 0:
                        d = sc[f.default]
                        v, ok = d.values[i], d.valid is None or bool(d.valid[i])
                    else:
                        v, ok = 0, False
                vals[i] = v if ok else 0
                valid[i] = ok
        out.append((vals, valid))
    return perm, out


def _frame(units, sb, eb, i, p0, p1, g0, g1):
    """[start, end) of row i's frame (advance_frame_start / advance_frame_end, ROWS and RANGE without offsets)."""
    sn, so = _bound(sb)
    en, eo = _bound(eb)
    rng = units == "range"
    if sn == "unbounded_preceding":
        s = p0
    elif sn == "current_row":
        s = g0 if rng else i
    elif sn == "preceding":
        s = p0 if i - p0 <= so else i - so
    else:
        s = min(i + so, p1)
    if en == "unbounded_following":
        e = p1
    elif en == "current_row":
        e = g1 if rng else i + 1
    elif en == "preceding":
        e = p0 if i - p0 < eo else i - eo + 1
    else:
        e = min(i + eo + 1, p1)
    return s, max(s, e)


def _ntile(n, row, rows):
    """WindowFuncNtileImpl::compute_nitle (window_function.rs:129-177)."""
    if n > rows:
        return row
    per, extra = rows // n, rows % n
    boundary = (per + 1) * extra
    r = row - 1
    return r // (per + 1) + 1 if r < boundary else (r - extra) // per + 1


# ---------------------------------------------------------------- the reference's own cases (tests/golden/window.json)
def golden_inputs(case):
    """-> (column names, oracle Cols, partition_by, order_by, WindowFuncs) of one case.  A constant lag /
    lead default becomes one more column, named `const:<value>`."""
    from databend_b200.transforms import WindowFunc
    names = list(case["table"])
    values = {k: case["table"][k] for k in names}
    for f in case["funcs"]:
        if isinstance(f["default"], list):
            name = f"const:{f['default'][1]}"
            if name not in values:
                names.append(name)
                values[name] = [f["default"][1]] * len(values[names[0]])
    cols = []
    for k in names:
        v = values[k]
        valid = np.asarray([x is not None for x in v])
        cols.append(Col(np.asarray([0 if x is None else x for x in v], np.int64), None if valid.all() else valid, abi.I64,
                        not valid.all()))
    idx = lambda c: -1 if c is None else names.index(c if isinstance(c, str) else f"const:{c[1]}")
    funcs = [WindowFunc(f["name"], arg=idx(f["arg"]), n=f["n"], default=idx(f["default"]),
                        frame=None if f["frame"] is None else tuple(f["frame"])) for f in case["funcs"]]
    return names, cols, [names.index(c) for c in case["partition_by"]], [(names.index(c), a, nf) for c, a, nf in case["order_by"]], funcs


def golden_mismatch(case, names, cols, perm, results):
    """None when the window result (perm: window position -> input row; results: [(values, valid)] per
    function) gives the reference's rows for the case's select list, comparing rows as multisets inside
    each run of equal final ORDER BY keys (one run when the query has no ORDER BY; a key named
    `-name` is descending); else a message."""
    def norm(v):
        if v is None:
            return (0, 0)
        v = v.item() if hasattr(v, "item") else v
        return (1, round(float(v), 9))

    rows = []
    for i, r in enumerate(perm):
        val = {k: cols[j].values[r] if cols[j].valid is None or cols[j].valid[r] else None for j, k in enumerate(names)}
        for k, (v, ok) in enumerate(results):
            val[f"${k}"] = v[i] if ok[i] else None
        key = []
        for c in case["final_order"] or []:  # "-name": descending
            f, x = norm(val[c.lstrip("-")])
            key.append((-f, -x) if c.startswith("-") else (f, x))
        rows.append((tuple(key), tuple(norm(val[c]) for c in case["select"])))
    rows.sort()
    exp = [tuple(norm(v) for v in r) for r in case["expected"]]
    if len(exp) != len(rows):
        return f"{case['name']}: {len(rows)} rows, the reference has {len(exp)}"
    at = 0
    while at < len(rows):
        end = at
        while end < len(rows) and rows[end][0] == rows[at][0]:
            end += 1
        if sorted(r[1] for r in rows[at:end]) != sorted(exp[at:end]):
            return f"{case['name']}: rows {at}..{end - 1} differ: {[r[1] for r in rows[at:end]]} vs {exp[at:end]}"
        at = end
    return None
