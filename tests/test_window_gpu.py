"""DBX_OP_WINDOW on the device against tests/window_oracle.py (a restatement of TransformWindow's row
loop): every output column bit for bit, every input column against its permuted input."""
import ctypes as C
import math

import numpy as np
import pytest

from databend_b200 import abi, lib
from databend_b200.block import Column, DataBlock, np_dtype
from databend_b200.lib import DbxError
from databend_b200.transforms import TransformWindow, WindowFunc, to_device

from window_oracle import Col, result_type, window

pytestmark = pytest.mark.gpu

INT_TYPES = [abi.I8, abi.I16, abi.I32, abi.I64, abi.U8, abi.U16, abi.U32, abi.U64]
SPECIAL_F = [float("nan"), -0.0, 0.0, 1.5, -2.0, 3.0]


def make_values(rng, dtype, n, card):
    if dtype in (abi.F32, abi.F64):
        v = rng.integers(-card, card, n).astype(np_dtype(dtype)) / 2
        sp = rng.random(n) < 0.2
        v[sp] = np.asarray(SPECIAL_F, np_dtype(dtype))[rng.integers(0, len(SPECIAL_F), sp.sum())]
        return v
    info = np.iinfo(np_dtype(dtype))
    lo, hi = max(info.min, -card), min(info.max, card)
    v = rng.integers(lo, hi + 1, n).astype(np_dtype(dtype))
    ext = rng.random(n) < 0.05
    v[ext] = np.asarray([info.min, info.max], np_dtype(dtype))[rng.integers(0, 2, ext.sum())]
    return v


def make_table(rng, n, spec):
    """spec: list of (dtype, nullable, cardinality) -> (oracle Cols, host Columns)."""
    cols, hcols = [], []
    for dtype, nullable, card in spec:
        v = make_values(rng, dtype, n, card)
        valid = (rng.random(n) > 0.15) if nullable else None
        cols.append(Col(v, valid, dtype, nullable))
        hcols.append(Column.from_data(v, dtype, validity=None if valid is None else valid.tolist()))
    return cols, hcols


def bits(a):
    a = np.asarray(a)
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def check(out: DataBlock, cols, partition_by, order_by, funcs, nan_sums_loose=True):
    perm, exp = window(cols, partition_by, order_by, funcs)
    n = len(perm)
    assert out.num_rows == n
    assert len(out.columns) == len(cols) + len(funcs)
    for j, c in enumerate(cols):  # input columns in window order
        g = out.columns[j]
        ok = np.ones(n, bool) if c.valid is None else np.asarray(c.valid, bool)[perm]
        np.testing.assert_array_equal(g.valid_mask(), ok, err_msg=f"input column {j} validity")
        np.testing.assert_array_equal(bits(g.values()[ok]), bits(np.asarray(c.values)[perm][ok]), err_msg=f"input column {j}")
    for k, f in enumerate(funcs):
        g = out.columns[len(cols) + k]
        dt, nullable = result_type(f, cols)
        assert g.dtype == dt, f
        ev, eok = exp[k]
        gok = g.valid_mask()
        np.testing.assert_array_equal(gok, eok, err_msg=f"{f} validity")
        gv, ev = g.values()[eok], ev[eok]
        if nan_sums_loose and f.name in ("sum", "avg") and dt == abi.F64:  # a NaN's payload depends on the unit that made it
            gn, en = np.isnan(gv), np.isnan(ev)
            np.testing.assert_array_equal(gn, en, err_msg=f"{f} NaN rows")
            gv, ev = gv[~gn], ev[~en]
        np.testing.assert_array_equal(bits(gv), bits(np.asarray(ev, gv.dtype)), err_msg=str(f))


def run(hcols, types, partition_by, order_by, funcs, split=0, device=False):
    op = TransformWindow(partition_by, order_by, funcs, types)
    blk = DataBlock(hcols)
    blocks = blk.split_by_rows(split) if split else [blk]
    for b in blocks:
        if device:
            b = DataBlock([to_device(c) for c in b.columns], b.num_rows)
        op.transform(b)
    out = op.on_finish()
    op.close()
    return out


SPEC = [(abi.I16, True, 4), (abi.U8, False, 3), (abi.F64, True, 6), (abi.I32, False, 50), (abi.I64, True, 1000),
        (abi.F64, True, 64), (abi.F32, False, 64), (abi.I64, False, 1000)]
P0, P1, T0, T1, V, X, F, D = range(8)

GROUP_RANK = [WindowFunc("row_number"), WindowFunc("rank"), WindowFunc("dense_rank"), WindowFunc("percent_rank"),
              WindowFunc("cume_dist"), WindowFunc("ntile", n=3), WindowFunc("lag", arg=V, n=2), WindowFunc("lead", arg=X, n=1)]
GROUP_VALUE = [WindowFunc("lag", arg=V, n=1, default=D), WindowFunc("lead", arg=D, n=3, default=D), WindowFunc("lag", arg=F, n=0),
               WindowFunc("lead", arg=T0, n=2), WindowFunc("ntile", n=1000), WindowFunc("ntile", n=1), WindowFunc("lag", arg=P0, n=100)]

FRAMES = [("rows", "unbounded_preceding", "current_row"), ("rows", ("preceding", 3), "current_row"),
          ("rows", ("preceding", 2), ("following", 2)), ("rows", "current_row", "unbounded_following"),
          ("rows", ("following", 1), ("following", 4)), ("rows", "unbounded_preceding", "unbounded_following"),
          ("rows", ("preceding", 5), ("preceding", 2)), ("range", "unbounded_preceding", "current_row"),
          ("range", "current_row", "unbounded_following"), ("range", "current_row", "current_row"),
          ("rows", ("following", 1), ("preceding", 1)), ("rows", "unbounded_preceding", ("preceding", 1)),
          ("rows", ("following", 2), "unbounded_following"), ("rows", ("preceding", 0), ("following", 0)),
          ("range", "unbounded_preceding", "unbounded_following"), ("rows", "current_row", ("preceding", 1))]

KEYS = [([], []), ([], [(T0, True, False)]), ([P0], [(T0, False, True)]), ([P0, P1], [(T1, True, True), (T0, True, False)]),
        ([P0, P1, T1], [(T0, False, False)]), ([], [(T0, True, True), (P0, False, False), (T1, True, False)]),
        ([P1, P0, T0], []), ([P0], [])]


@pytest.mark.parametrize("keys", range(len(KEYS)))
def test_ranking_and_offsets_against_the_oracle(gpu, keys):
    rng = np.random.default_rng(100 + keys)
    cols, hcols = make_table(rng, 3000, SPEC)
    types = [d | (abi.NULLABLE if nl else 0) for d, nl, _ in SPEC]
    pb, ob = KEYS[keys]
    for funcs in (GROUP_RANK, GROUP_VALUE):
        out = run(hcols, types, pb, ob, funcs, split=777)
        check(out, cols, pb, ob, funcs)


@pytest.mark.parametrize("frame", range(len(FRAMES)))
@pytest.mark.parametrize("keys", [2, 3, 5])
def test_aggregates_and_nth_value_over_every_frame(gpu, frame, keys):
    """Integer-valued doubles: every Float sum is exact, so every path must match the oracle bit for bit."""
    rng = np.random.default_rng(frame * 7 + keys)
    cols, hcols = make_table(rng, 2500, SPEC)
    types = [d | (abi.NULLABLE if nl else 0) for d, nl, _ in SPEC]
    fr = FRAMES[frame]
    funcs = [WindowFunc("sum", arg=V, frame=fr), WindowFunc("count", arg=X, frame=fr), WindowFunc("avg", arg=V, frame=fr),
             WindowFunc("min", arg=X, frame=fr), WindowFunc("max", arg=F, frame=fr), WindowFunc("sum", arg=X, frame=fr),
             WindowFunc("nth_value", arg=X, n=2, frame=fr), WindowFunc("last_value", arg=V, frame=fr)]
    pb, ob = KEYS[keys]
    out = run(hcols, types, pb, ob, funcs, split=1000)
    check(out, cols, pb, ob, funcs)
    funcs2 = [WindowFunc("count", frame=fr), WindowFunc("avg", arg=F, frame=fr), WindowFunc("min", arg=T1, frame=fr),
              WindowFunc("max", arg=V, frame=fr), WindowFunc("sum", arg=P1, frame=fr), WindowFunc("nth_value", arg=F, n=1, frame=fr),
              WindowFunc("min", arg=D, frame=fr), WindowFunc("max", arg=T0, frame=fr)]
    out = run(hcols, types, pb, ob, funcs2, device=True)
    check(out, cols, pb, ob, funcs2)


@pytest.mark.parametrize("dtype", INT_TYPES + [abi.F32, abi.F64])
@pytest.mark.parametrize("nulls_first", [False, True])
def test_key_types_with_nan_zeros_and_nulls(gpu, dtype, nulls_first):
    rng = np.random.default_rng(dtype * 2 + nulls_first)
    spec = [(dtype, True, 5), (dtype, True, 8), (abi.I64, True, 100)]
    cols, hcols = make_table(rng, 4000, spec)
    types = [d | abi.NULLABLE for d, _, _ in spec]
    funcs = [WindowFunc("row_number"), WindowFunc("rank"), WindowFunc("dense_rank"), WindowFunc("cume_dist"),
             WindowFunc("lag", arg=1, n=1), WindowFunc("sum", arg=2, frame=("range", "unbounded_preceding", "current_row")),
             WindowFunc("min", arg=1, frame=("range", "current_row", "current_row")),
             WindowFunc("max", arg=0, frame=("rows", ("preceding", 3), ("following", 3)))]
    for pb, ob in (([0], [(1, True, nulls_first)]), ([], [(0, False, nulls_first), (1, True, not nulls_first)])):
        out = run(hcols, types, pb, ob, funcs, split=999)
        check(out, cols, pb, ob, funcs)


def test_blocks_from_host_pinned_and_device_with_const_columns(gpu):
    rng = np.random.default_rng(5)
    n = 6000
    L = lib.load()
    k = rng.integers(0, 30, n).astype(np.int64)
    t = rng.integers(0, 200, n).astype(np.int32)
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    ptrs = []
    try:
        p = C.c_void_p()
        lib.check(L.dbx_host_alloc(n * 8, C.byref(p)))
        ptrs.append(p)
        pinned = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int64)), shape=(n,))
        pinned[:] = v
        vcol = Column.from_data(pinned)
        funcs = [WindowFunc("row_number"), WindowFunc("sum", arg=2, frame=("rows", "unbounded_preceding", "current_row")),
                 WindowFunc("lag", arg=3, n=1), WindowFunc("max", arg=4, frame=("rows", ("preceding", 1), "current_row")),
                 WindowFunc("count", arg=3, frame=("rows", "unbounded_preceding", "unbounded_following"))]
        types = [abi.I64, abi.I32, abi.I64, abi.I64 | abi.NULLABLE, abi.I32 | abi.NULLABLE]
        op = TransformWindow([0], [(1, True, False), (4, False, True)], funcs, types)
        bounds = [0, 1000, 1001, 2500, 2501, 4000, n]
        const_vals, kinds = [], []
        for b, (s, e) in enumerate(zip(bounds[:-1], bounds[1:])):
            m = e - s
            cv = None if b % 3 == 2 else 7  # Const column 3: equal in some blocks, NULL in others
            kv = b * 10 if b % 2 else 5      # Const key column 4: differs between blocks
            const_vals += [cv] * m
            kinds += [kv] * m
            cols = [Column.from_data(k[s:e]), Column.from_data(t[s:e]), vcol.slice(s, e), Column.new_const(abi.I64, cv, m),
                    Column.new_const(abi.I32, kv, m)]
            blk = DataBlock(cols, m)
            if b % 3 == 1:
                blk = DataBlock([to_device(c) for c in cols], m)
            op.transform(blk)
        out = op.on_finish()
        op.close()
        cvals = np.asarray([0 if x is None else x for x in const_vals], np.int64)
        cvalid = np.asarray([x is not None for x in const_vals])
        ocols = [Col(k, None, abi.I64), Col(t, None, abi.I32), Col(v, None, abi.I64), Col(cvals, cvalid, abi.I64, True),
                 Col(np.asarray(kinds, np.int32), None, abi.I32, True)]
        check(out, ocols, [0], [(1, True, False), (4, False, True)], funcs)
    finally:
        for p in ptrs:
            L.dbx_host_free(p)


def test_empty_input_one_row_partitions_and_one_partition(gpu):
    types = [abi.I64, abi.F64 | abi.NULLABLE]
    funcs = [WindowFunc("row_number"), WindowFunc("percent_rank"), WindowFunc("lag", arg=1, n=1),
             WindowFunc("avg", arg=1, frame=("rows", ("preceding", 1), ("following", 1)))]
    op = TransformWindow([0], [(1, True, False)], funcs, types)
    out = op.on_finish()
    op.close()
    assert out.num_rows == 0 and len(out.columns) == 6
    rng = np.random.default_rng(9)
    n = 5000
    x = rng.integers(-50, 50, n).astype(np.float64)
    valid = rng.random(n) > 0.1
    for keys in (np.arange(n, dtype=np.int64), np.zeros(n, np.int64)):
        cols = [Col(keys, None, abi.I64), Col(x, valid, abi.F64, True)]
        hcols = [Column.from_data(keys), Column.from_data(x, abi.F64, validity=valid.tolist())]
        out = run(hcols, types, [0], [(1, True, False)], funcs, split=333)
        check(out, cols, [0], [(1, True, False)], funcs)


def test_float_sums_over_bounded_frames_are_bit_exact_and_unbounded_ones_within_the_bound(gpu):
    rng = np.random.default_rng(11)
    n = 20000
    k = rng.integers(0, 20, n).astype(np.int64)
    x = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n)).astype(np.float64)
    cols = [Col(k, None, abi.I64), Col(x, None, abi.F64)]
    hcols = [Column.from_data(k), Column.from_data(x)]
    types = [abi.I64, abi.F64]
    bounded = [WindowFunc("sum", arg=1, frame=("rows", ("preceding", 7), ("following", 3))),
               WindowFunc("avg", arg=1, frame=("rows", ("preceding", 100), "current_row")),
               WindowFunc("sum", arg=1, frame=("range", "current_row", "current_row"))]
    out = run(hcols, types, [0], [], bounded)
    check(out, cols, [0], [], bounded, nan_sums_loose=False)
    open_frames = [WindowFunc("sum", arg=1, frame=("rows", "unbounded_preceding", "current_row")),
                   WindowFunc("sum", arg=1, frame=("rows", ("preceding", 2), "unbounded_following")),
                   WindowFunc("avg", arg=1, frame=("rows", "unbounded_preceding", "unbounded_following"))]
    out = run(hcols, types, [0], [], open_frames)
    perm = np.argsort(k, kind="stable")
    xs, ks = x[perm], k[perm]
    u = 2.0 ** -53
    for f_i, f in enumerate(open_frames):
        got = out.columns[2 + f_i].values()
        for i in range(0, n, 97):  # exact per-row reference: fsum over the frame, |error| <= gamma(m + 1) * sum |x|
            p0 = np.searchsorted(ks, ks[i], "left")
            p1 = np.searchsorted(ks, ks[i], "right")
            s, e = (p0, i + 1) if f_i == 0 else ((max(p0, i - 2), p1) if f_i == 1 else (p0, p1))
            fr = xs[s:e]
            m = len(fr)
            exact = math.fsum(fr)
            bound = (m + 1) * u / (1 - (m + 1) * u) * math.fsum(np.abs(fr))
            if f.name == "avg":
                exact, bound = exact / m, bound / m + 3 * u * abs(exact) / m
            assert abs(got[i] - exact) <= bound, (f, i, got[i], exact, bound)


def test_refusals(gpu):
    types = [abi.I64, abi.F64, abi.BOOL, abi.VEC_F32]
    L = lib.load()

    def create(pb, ob, funcs):
        with pytest.raises(DbxError) as e:
            TransformWindow(pb, ob, funcs, types)
        return e.value, (L.dbx_last_error(None) or b"").decode()

    def expect(code, pb, ob, funcs):
        err, msg = create(pb, ob, funcs)
        assert err.status == code, (err, msg)
        assert msg, "no message in dbx_last_error(NULL)"

    unb = ("rows", "unbounded_preceding", "current_row")
    expect(abi.ERR_UNSUPPORTED, [], [(0, True, False)], [WindowFunc("sum", arg=1, frame=("range", ("preceding", 10), "current_row"))])
    expect(abi.ERR_UNSUPPORTED, [], [(0, True, False)], [WindowFunc("nth_value", arg=1, n=1, frame=unb, ignore_nulls=True)])
    expect(abi.ERR_UNSUPPORTED, [], [(0, True, False)], [WindowFunc("sum", arg=1, frame=unb, distinct=True)])
    expect(abi.ERR_INVALID, [], [], [WindowFunc("sum", arg=2, frame=unb)])
    expect(abi.ERR_INVALID, [], [], [WindowFunc("max", arg=3, frame=unb)])
    expect(abi.ERR_INVALID, [7], [], [WindowFunc("row_number")])
    expect(abi.ERR_INVALID, [], [], [WindowFunc("lag", arg=9, n=1)])
    expect(abi.ERR_INVALID, [], [], [WindowFunc("ntile", n=0)])
    expect(abi.ERR_INVALID, [], [], [WindowFunc("rank", frame=unb)])
    expect(abi.ERR_INVALID, [0, 1], [(0, True, False), (1, True, False), (0, True, True)], [WindowFunc("row_number")])
    # the row limit: one Int8 column pushed as two 2^29-row device blocks; the second push is refused
    n = 1 << 29
    buf = C.c_void_p()
    lib.check(L.dbx_device_alloc(0, n, C.byref(buf)))
    try:
        op = TransformWindow([], [(0, True, False)], [WindowFunc("row_number")], [abi.I8])
        blk = DataBlock([Column.device(abi.I8, n, buf.value)], n)
        op.transform(blk)
        with pytest.raises(DbxError) as e:
            op.transform(blk)
        assert e.value.status == abi.ERR_UNSUPPORTED
        assert "2^30" in L.dbx_last_error(op.handle).decode()
        op.close()
    finally:
        L.dbx_device_free(0, buf)


# ---------------------------------------------------------------- scale (closed-form expectations)
def _segments(keys_sorted):
    n = len(keys_sorted)
    start = np.ones(n, bool)
    start[1:] = keys_sorted[1:] != keys_sorted[:-1]
    idx = np.arange(n)
    ps = np.maximum.accumulate(np.where(start, idx, 0))
    return start, ps


def _device_block(arrays):
    cols = [to_device(Column.from_data(a)) for a in arrays]
    return DataBlock(cols, len(arrays[0]))


@pytest.mark.parametrize("n_keys", [1 << 20, 1])
def test_scale_2_26_rows(gpu, n_keys):
    """2^26 rows: 2^20 partitions of ~64 rows that straddle the 2048-row scan tiles, and one partition
    holding every row."""
    n = 1 << 26
    rng = np.random.default_rng(n_keys)
    k = rng.integers(0, n_keys, n).astype(np.int64)
    t = rng.permutation(n).astype(np.int64)
    v = rng.integers(-(1 << 40), 1 << 40, n).astype(np.int64)
    funcs = [WindowFunc("row_number"), WindowFunc("rank"), WindowFunc("sum", arg=2, frame=("rows", "unbounded_preceding", "current_row")),
             WindowFunc("lag", arg=2, n=1), WindowFunc("count", frame=("rows", "unbounded_preceding", "unbounded_following"))]
    op = TransformWindow([0], [(1, True, False)], funcs, [abi.I64, abi.I64, abi.I64])
    for s in range(0, n, 1 << 24):
        op.transform(_device_block([k[s:s + (1 << 24)], t[s:s + (1 << 24)], v[s:s + (1 << 24)]]))
    out = op.on_finish()
    op.close()
    perm = np.lexsort((t, k))
    ks, vs = k[perm], v[perm]
    start, ps = _segments(ks)
    idx = np.arange(n)
    np.testing.assert_array_equal(out.columns[0].values(), ks)
    np.testing.assert_array_equal(out.columns[1].values(), t[perm])
    np.testing.assert_array_equal(out.columns[3].values(), idx - ps + 1)
    np.testing.assert_array_equal(out.columns[4].values(), idx - ps + 1)  # t is unique: rank = row_number
    cs = np.cumsum(vs)
    np.testing.assert_array_equal(out.columns[5].values(), cs - np.where(ps > 0, cs[ps - 1], 0))
    lag_ok = ~start
    np.testing.assert_array_equal(out.columns[6].valid_mask(), lag_ok)
    np.testing.assert_array_equal(out.columns[6].values()[lag_ok], vs[idx[lag_ok] - 1])
    pe = np.empty(n, np.int64)
    ends = np.flatnonzero(np.r_[start[1:], True]) + 1
    pe[:] = np.repeat(ends, np.diff(np.r_[0, ends]))
    np.testing.assert_array_equal(out.columns[7].values(), (pe - ps).astype(np.uint64))


def test_integer_sums_wrap_near_2_63(gpu):
    n = 100000
    rng = np.random.default_rng(3)
    k = rng.integers(0, 10, n).astype(np.int64)
    v = rng.integers(1 << 61, (1 << 62), n).astype(np.int64) * np.where(rng.random(n) < 0.3, -1, 1)
    u = (v.astype(np.uint64) | np.uint64(1 << 63))
    funcs = [WindowFunc("sum", arg=1, frame=("rows", "unbounded_preceding", "current_row")),
             WindowFunc("sum", arg=2, frame=("rows", ("preceding", 3), ("following", 5))),
             WindowFunc("avg", arg=1, frame=("rows", "current_row", "unbounded_following"))]
    out = run([Column.from_data(k), Column.from_data(v), Column.from_data(u)], [abi.I64, abi.I64, abi.U64], [0], [], funcs)
    cols = [Col(k, None, abi.I64), Col(v, None, abi.I64), Col(u, None, abi.U64)]
    check(out, cols, [0], [], funcs)


def test_reference_cases_on_the_device():
    """The reference's own window_bound / window_basic / window_ntile cases, run on the device; a constant
    lag / lead default is pushed as a Const column."""
    import json
    import os
    from window_oracle import golden_inputs, golden_mismatch
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "window.json")) as f:
        cases = json.load(f)["cases"]
    for case in cases:
        names, cols, pb, ob, funcs = golden_inputs(case)
        n = len(cols[0].values)
        hcols = [Column.new_const(abi.I64, int(c.values[0]), n) if k.startswith("const:") else Column.from_data(c.values, abi.I64)
                 for k, c in zip(names, cols)]
        out = run(hcols, [abi.I64] * len(cols), pb, ob, funcs, split=3)
        perm = np.asarray(window(cols, pb, ob, funcs)[0])
        for j, c in enumerate(cols):  # the device's window order, as the oracle's, is stable
            if not names[j].startswith("const:"):
                np.testing.assert_array_equal(out.columns[j].values(), c.values[perm], err_msg=case["name"])
        res = [(out.columns[len(cols) + k].values(), out.columns[len(cols) + k].valid_mask()) for k in range(len(funcs))]
        msg = golden_mismatch(case, names, cols, perm, res)
        assert msg is None, msg
