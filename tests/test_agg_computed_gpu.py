"""Computed columns inside the fused filter / aggregate kernels (dbx_op_create_computed): aggregate
arguments, GROUP BY expressions and predicate operands evaluated in registers, against numpy restatements
of the same expressions on the rows the predicate keeps (Filter -> EvalScalar -> Aggregate)."""
import numpy as np
import pytest

from computed_oracle import OracleEvalError, composed
from helpers import assert_group_results_equal, sorted_group_result_from_block, sorted_group_result_from_oracle
from float_agg_ref import avg_violations, exact_reference, sum_violations
from databend_b200 import abi, expr as E, scalar_expr as S
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError
from databend_b200.transforms import (AggregatorParams, TransformFilter, TransformFinalAggregate, TransformPartialAggregate,
                                      filter_group_aggregate, to_device)

pytestmark = pytest.mark.gpu

JIT = ["0", "1"]


@pytest.fixture(params=JIT, ids=["precompiled", "specialised"])
def jit(request, monkeypatch):
    monkeypatch.setenv("DBX_AGG_JIT", request.param)
    return request.param


def _data(n, seed=0):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 5000, n).astype(np.int64)
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    b = rng.integers(-1000, 1000, n).astype(np.int32)
    v = rng.integers(0, 1 << 20, n).astype(np.int64)
    return k, a, b, v


def _grouped(keys, vals, fn):
    order = np.argsort(keys, kind="stable")
    ks, vs = keys[order], vals[order]
    uk, start = np.unique(ks, return_index=True)
    return uk, np.array([fn(x) for x in np.split(vs, start[1:])]) if len(uk) else np.array([])


def _result(out, n_aggs):
    keys = out.columns[n_aggs].values()
    order = np.argsort(keys)
    return keys[order], [out.columns[i].values()[order] for i in range(n_aggs)]


@pytest.mark.parametrize("blocks", ["one", "split65536", "device"])
def test_int_args_and_key(jit, blocks):
    n = 300_000
    k, a, b, v = _data(n)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    params = AggregatorParams([0], [("sum", S.col(1) * S.col(2)), ("min", S.col(1) + S.col(2)), ("max", S.col(1) - S.col(2)),
                                    ("avg", S.col(1) * S.col(2)), ("count", None)])
    filt = E.eq(E.col(3) % E.lit(3), E.lit(0))
    if blocks == "one":
        bl = [blk]
    elif blocks == "split65536":
        bl = blk.split_by_rows(65536)
    else:
        bl = [DataBlock([to_device(c) for c in blk.columns], n)]
    out = filter_group_aggregate(bl, params, filt, input_types=[abi.I64, abi.I64, abi.I32, abi.I64])
    keep = v % 3 == 0
    kk, prod, s, d = k[keep], a[keep] * b[keep].astype(np.int64), a[keep] + b[keep], a[keep] - b[keep]
    gk, got = _result(out, 5)
    uk, want_sum = _grouped(kk, prod, np.sum)
    np.testing.assert_array_equal(gk, uk)
    np.testing.assert_array_equal(got[0], want_sum)
    np.testing.assert_array_equal(got[1], _grouped(kk, s, np.min)[1])
    np.testing.assert_array_equal(got[2], _grouped(kk, d, np.max)[1])
    np.testing.assert_array_equal(got[3], _grouped(kk, prod, lambda x: x.sum() / len(x))[1])
    np.testing.assert_array_equal(got[4], _grouped(kk, prod, len)[1])


@pytest.mark.parametrize("path", ["one-pass", "partitioned", "growth"])
def test_computed_key(jit, path, monkeypatch):
    n = 400_000
    k, a, b, v = _data(n, 1)
    expected = 0
    if path == "partitioned":
        monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "4096")
        monkeypatch.setenv("DBX_AGG_PARTITION_ALWAYS", "1")
    if path == "growth":
        expected = 1
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    key = S.col(3) % S.lit(1000, abi.U16)
    params = AggregatorParams([key], [("sum", S.col(1) * S.col(2)), ("count", None)], expected_groups=expected)
    filt = E.gt(E.col(1), E.lit(-500))
    out, variant = run_ops([blk], params, filt, [abi.I64, abi.I64, abi.I32, abi.I64])
    if path == "partitioned":
        assert "two-pass (partitioned by table slice) chunks: 1" in variant, variant
    else:
        assert "two-pass" not in variant, variant
    keep = a > -500
    gk, got = _result(out, 2)
    uk, want = _grouped(v[keep] % 1000, a[keep] * b[keep].astype(np.int64), np.sum)
    np.testing.assert_array_equal(gk, uk)
    np.testing.assert_array_equal(got[0], want)


def test_float_key_and_computed_predicate(jit):
    n = 200_000
    k, a, b, v = _data(n, 2)
    x = (v % 64).astype(np.float64)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(x)])
    params = AggregatorParams([S.col(3) * S.lit(0.5, abi.F64)], [("sum", S.col(1)), ("count", None)])
    filt = E.gt(S.col(1) + S.col(2), E.lit(0))  # computed operand in a CMP
    out = filter_group_aggregate([blk], params, filt, input_types=[abi.I64, abi.I64, abi.I32, abi.F64])
    keep = a + b > 0
    gk, got = _result(out, 2)
    uk, want = _grouped(x[keep] * 0.5, a[keep], np.sum)
    np.testing.assert_array_equal(gk, uk)
    np.testing.assert_array_equal(got[0], want)


@pytest.mark.parametrize("shape", ["packed64", "packed128"])
def test_packed_keys(jit, shape):
    n = 200_000
    k, a, b, v = _data(n, 3)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    second = S.col(3) % S.lit(7, abi.U8) if shape == "packed64" else S.col(3) * S.lit(3, abi.I64)
    params = AggregatorParams([S.col(0) % S.lit(50, abi.U8), second], [("sum", S.col(1) + S.col(2))])
    out = filter_group_aggregate([blk], params, None, input_types=[abi.I64, abi.I64, abi.I32, abi.I64])
    k1 = k % 50
    k2 = v % 7 if shape == "packed64" else v * 3
    want = {}
    for x, y, s in zip(k1.tolist(), k2.tolist(), (a + b).tolist()):
        want[(x, y)] = want.get((x, y), 0) + s
    got = {(int(x), int(y)): int(s) for x, y, s in zip(out.columns[1].values(), out.columns[2].values(), out.columns[0].values())}
    assert got == want


def test_q6_shape_no_group_by(jit):
    """Q6 at 1e7 rows with general floats: the sum against the order-independent exact bound."""
    n = 10_000_000
    rng = np.random.default_rng(6)
    price = rng.uniform(900.0, 105000.0, n)
    disc = rng.integers(0, 11, n) / 100.0
    qty = rng.integers(1, 51, n).astype(np.float64)
    blk = DataBlock([Column.from_data(price), Column.from_data(disc), Column.from_data(qty)])
    params = AggregatorParams([], [("sum", S.col(0) * S.col(1)), ("avg", S.col(0) * S.col(1))])
    filt = E.lt(E.col(2), E.lit(24.0))
    out = filter_group_aggregate([blk], params, filt, input_types=[abi.F64, abi.F64, abi.F64])
    keep = qty < 24
    ref = exact_reference(np.zeros(n, dtype=np.int64), price * disc, keep)
    assert sum_violations(ref, {0: float(out.columns[0].values()[0])}) == []
    assert avg_violations(ref, {0: float(out.columns[1].values()[0])}) == []


def test_q1_shape_slot_reuse(jit):
    """Q1 at 1e7 rows: 7 inputs, 2 computed columns and 8 aggregates fit 8 slots only through reuse;
    general floats checked against the exact bounds of float_agg_ref."""
    n = 10_000_000
    rng = np.random.default_rng(1)
    flag = rng.integers(0, 3, n).astype(np.uint8)
    status = rng.integers(0, 2, n).astype(np.uint8)
    qty = rng.integers(1, 51, n).astype(np.float64)
    price = rng.uniform(900.0, 105000.0, n)
    disc = rng.integers(0, 11, n) / 100.0
    tax = rng.integers(0, 9, n) / 100.0
    ship = rng.integers(8000, 10600, n).astype(np.int32)
    blk = DataBlock([Column.from_data(c) for c in (flag, status, qty, price, disc, tax, ship)])
    one = S.lit(1.0, abi.F64)
    disc_price = S.col(3) * (one - S.col(4))
    charge = disc_price * (one + S.col(5))
    params = AggregatorParams([0, 1], [("sum", 2), ("sum", 3), ("sum", disc_price), ("sum", charge), ("avg", 2), ("avg", 3),
                                       ("avg", 4), ("count", None)])
    filt = E.le(E.col(6), E.lit(10471, abi.I32))
    types = [abi.U8, abi.U8, abi.F64, abi.F64, abi.F64, abi.F64, abi.I32]
    out = filter_group_aggregate([blk], params, filt, input_types=types)
    keep = ship <= 10471
    key = flag.astype(np.int64) * 2 + status
    dp = price * (1 - disc)
    ch = dp * (1 + tax)
    gkey = out.columns[8].values().astype(np.int64) * 2 + out.columns[9].values()
    for col, vals, check in ((2, dp, sum_violations), (3, ch, sum_violations), (1, price, sum_violations), (6, disc, avg_violations)):
        ref = exact_reference(key, vals, keep)
        got = {int(k): float(v) for k, v in zip(gkey, out.columns[col].values())}
        assert check(ref, got) == [], col
    cnt = {int(k): int(c) for k, c in zip(gkey, out.columns[7].values())}
    assert cnt == {int(k): int(c) for k, c in zip(*np.unique(key[keep], return_counts=True))}


def test_equivalence_with_materialised(jit):
    n = 250_000
    k, a, b, v = _data(n, 4)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    e = (S.col(1) * S.col(2)) % S.lit(97, abi.U8)
    fused = filter_group_aggregate([blk], AggregatorParams([0], [("sum", e), ("max", e)]), E.lt(E.col(3), E.lit(1 << 19)),
                                   input_types=[abi.I64, abi.I64, abi.I32, abi.I64])
    col, dt = S.eval_scalar(blk, e)
    blk2 = DataBlock(list(blk.columns) + [col])
    mat = filter_group_aggregate([blk2], AggregatorParams([0], [("sum", 4), ("max", 4)]), E.lt(E.col(3), E.lit(1 << 19)),
                                 input_types=[abi.I64, abi.I64, abi.I32, abi.I64, dt])
    for i in range(3):
        fo, mo = np.argsort(fused.columns[2].values()), np.argsort(mat.columns[2].values())
        np.testing.assert_array_equal(fused.columns[i].values()[fo], mat.columns[i].values()[mo])


def test_errors(jit):
    n = 100_000
    k, a, b, v = _data(n, 5)
    b = np.where(np.arange(n) % 1000 == 7, 0, b).astype(np.int32)  # zero divisors on rows 7, 1007, ...
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    types = [abi.I64, abi.I64, abi.I32, abi.I64]
    params = AggregatorParams([0], [("sum", S.col(1) % S.col(2))])
    # zero divisors only on rows the predicate drops: no error
    out = filter_group_aggregate([blk], params, E.ne(E.col(2), E.lit(0)), input_types=types)
    assert out.num_rows > 0
    # a zero divisor on a kept row: finish raises with the first failing row, then STATE until reset
    part = TransformPartialAggregate(params, types)
    for blk_i in blk.split_by_rows(30_000):
        part.transform(blk_i)
    with pytest.raises(S.EvalError) as ei:
        part.on_finish()
    assert ei.value.row == 7 and "Division by zero" in ei.value.message
    with pytest.raises(DbxError) as e2:
        part.finish()
    assert e2.value.status == abi.ERR_STATE
    with pytest.raises(DbxError) as e3:
        part.push(blk)
    assert e3.value.status == abi.ERR_STATE
    part.reset()
    part.transform(DataBlock([Column.from_data(c[:5]) for c in (k, a, b, v)]))
    part.on_finish()
    part.close()
    # a NULL divisor does not raise
    nb = Column.from_data(b)
    nb.validity = np.packbits(b != 0, bitorder="little")
    blk_n = DataBlock([Column.from_data(k), Column.from_data(a), nb, Column.from_data(v)])
    out = filter_group_aggregate([blk_n], params, None, input_types=[abi.I64, abi.I64, abi.I32 | abi.NULLABLE, abi.I64])
    assert out.num_rows > 0
    # an expression that can raise is refused in the predicate
    with pytest.raises(DbxError) as e4:
        TransformPartialAggregate(AggregatorParams([0], [("count", None)]), types, E.gt(S.col(1) % S.col(2), E.lit(0)))
    assert e4.value.status == abi.ERR_UNSUPPORTED


def test_hand_off_serialize_and_final(jit):
    n = 200_000
    k, a, b, v = _data(n, 7)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    types = [abi.I64, abi.I64, abi.I32, abi.I64]
    params = AggregatorParams([S.col(0) % S.lit(100, abi.U8)], [("sum", S.col(1) * S.col(2)), ("avg", S.col(2) + S.lit(1, abi.U8))])
    filt = E.gt(S.col(3) - S.col(1), E.lit(1000))
    part = TransformPartialAggregate(params, types, filt)
    part.transform(blk)
    part.on_finish()
    ser, _ = part.serialize()
    fin = TransformFinalAggregate(params, types)
    fin.merge_serialized(ser)
    via_ser = fin.on_finish()[0]
    ref = filter_group_aggregate([blk], params, filt, input_types=types)
    keep = v - a > 1000
    uk, want = _grouped(k[keep] % 100, a[keep] * b[keep].astype(np.int64), np.sum)
    assert [c.dtype for c in via_ser.columns] == [abi.I64, abi.F64, abi.I16]  # sum(Int64), avg, Int64 % UInt8 = Int16
    assert [c.dtype for c in ref.columns] == [abi.I64, abi.F64, abi.I16]
    for out in (via_ser, ref):
        gk, got = _result(out, 2)
        np.testing.assert_array_equal(gk, uk)
        np.testing.assert_array_equal(got[0], want)
    part.close()
    fin.close()


def test_filter_operator(jit):
    n = 100_000
    k, a, b, v = _data(n, 8)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    f = TransformFilter(E.and_(E.gt(S.col(1) * S.col(2), E.lit(1000)), E.bool_column(S.call("lt", S.col(0), S.col(3)))),
                        [abi.I64, abi.I64, abi.I32, abi.I64])
    out = f.transform(blk)
    keep = (a * b.astype(np.int64) > 1000) & (k < v)
    np.testing.assert_array_equal(out.columns[0].values(), k[keep])
    f.close()


def test_refusals():
    types = [abi.I64, abi.I64]
    cp = AggregatorParams([0], [("count", None)]).to_c()
    ex = (abi.Expr * 1)()
    ex[0] = S.flatten(S.col(1) + S.col(2))  # references computed column 2
    from databend_b200.lib import load
    import ctypes as C
    h = C.c_void_p()
    t = (C.c_int32 * 2)(*types)
    assert load().dbx_op_create_computed(abi.OP_AGG_PARTIAL, C.cast(C.byref(cp), C.c_void_p), t, 2, ex, 1, 0, C.byref(h)) == abi.ERR_INVALID
    ex[0] = S.flatten(S.col(5) + S.col(1))
    assert load().dbx_op_create_computed(abi.OP_AGG_PARTIAL, C.cast(C.byref(cp), C.c_void_p), t, 2, ex, 1, 0, C.byref(h)) == abi.ERR_INVALID
    ex[0] = S.flatten(S.col(0) + S.col(1))
    assert load().dbx_op_create_computed(abi.OP_AGG_PARTIAL, C.cast(C.byref(cp), C.c_void_p), t, 2, ex, 5, 0, C.byref(h)) == abi.ERR_INVALID
    tp = abi.TopkParams()
    tp.limit = 10
    assert load().dbx_op_create_computed(abi.OP_TOPK, C.cast(C.byref(tp), C.c_void_p), t, 2, ex, 1, 0, C.byref(h)) == abi.ERR_UNSUPPORTED
    jp = abi.JoinParams()
    assert load().dbx_op_create_computed(abi.OP_JOIN, C.cast(C.byref(jp), C.c_void_p), t, 2, ex, 1, 0, C.byref(h)) == abi.ERR_UNSUPPORTED
    # more than 8 values per row
    types9 = [abi.I64] * 9
    params = AggregatorParams([0], [("sum", i) for i in range(1, 8)] + [("sum", S.col(8) + S.col(1))])
    with pytest.raises(DbxError) as e:
        TransformPartialAggregate(params, types9)
    assert e.value.status == abi.ERR_UNSUPPORTED


def run_ops(blocks, params, filt, types):
    """Partial -> final through the operator classes: (result block, the partial's kernel_variant())."""
    part = TransformPartialAggregate(params, types, filt)
    for b in blocks:
        part.transform(b)
    part.on_finish()
    fin = TransformFinalAggregate(params, types)
    fin.transform(part)
    variant = part.kernel_variant()
    out = fin.on_finish()[0]
    part.close()
    fin.close()
    return out, variant


def check_against_oracle(out, blk, types, params, filt):
    n_aggs, n_keys = len(params.aggregate_functions), len(params.group_columns)
    res, _ = composed(blk, types, params, filt)
    key_dtypes = [out.columns[n_aggs + j].dtype for j in range(n_keys)]
    gpu = sorted_group_result_from_block(out, n_aggs, n_keys)
    orc = sorted_group_result_from_oracle(res, key_dtypes)
    assert_group_results_equal(gpu, orc)


def _values(t, n, rng):
    if t in (abi.F32, abi.F64):
        return rng.integers(-100, 100, n).astype(np.float32 if t == abi.F32 else np.float64)
    if t in (abi.U8, abi.U16, abi.U32, abi.U64):
        return rng.integers(0, 200, n).astype({abi.U8: np.uint8, abi.U16: np.uint16, abi.U32: np.uint32, abi.U64: np.uint64}[t])
    return rng.integers(-100, 100, n).astype({abi.I8: np.int8, abi.I16: np.int16, abi.I32: np.int32, abi.I64: np.int64}[t])


PAIRS = [(abi.I8, abi.U8), (abi.I16, abi.U16), (abi.I32, abi.U32), (abi.I64, abi.U64), (abi.U8, abi.I64), (abi.U16, abi.F32),
         (abi.U32, abi.F64), (abi.F32, abi.I8), (abi.F64, abi.I16), (abi.U64, abi.U64), (abi.F32, abi.F64), (abi.I32, abi.I32)]


@pytest.mark.parametrize("ta,tb", PAIRS, ids=[f"{a}x{b}" for a, b in PAIRS])
def test_type_pairs_against_composed_oracle(jit, ta, tb):
    """plus / minus / multiply of every numeric input type into sum / min / max / avg / count, the left
    argument Nullable with NULLs on kept rows."""
    n = 20_000
    rng = np.random.default_rng(ta * 16 + tb)
    k = rng.integers(0, 40, n).astype(np.int64)
    a, b = _values(ta, n, rng), _values(tb, n, rng)
    v = rng.integers(0, 1 << 20, n).astype(np.int64)
    blk = DataBlock([Column.from_data(k), Column.from_data(a, ta, validity=rng.random(n) > 0.15), Column.from_data(b, tb),
                     Column.from_data(v)])
    types = [abi.I64, ta | abi.NULLABLE, tb, abi.I64]
    params = AggregatorParams([0], [("sum", S.col(1) + S.col(2)), ("min", S.col(1) - S.col(2)), ("max", S.col(1) * S.col(2)),
                                    ("avg", S.col(1) + S.col(2)), ("count", S.col(1) * S.col(2))])
    filt = E.ne(E.col(3) % E.lit(3), E.lit(0))
    out, _ = run_ops(blk.split_by_rows(7_001), params, filt, types)
    check_against_oracle(out, blk, types, params, filt)


@pytest.mark.parametrize("part", [0, 1])
def test_nulls_consts_try_cast_null_literal(jit, part):
    """Nullable inputs with NULLs on kept rows, a Const and a NULL Const input, try_cast, a NULL literal
    and a nullable computed GROUP BY key (its NULL group included)."""
    n = 30_000
    rng = np.random.default_rng(11)
    k = rng.integers(0, 40, n).astype(np.int64)
    a = rng.integers(-50, 50, n).astype(np.int32)
    x = rng.integers(-300, 300, n).astype(np.int64)
    v = rng.integers(0, 1 << 20, n).astype(np.int64)
    blk = DataBlock([Column.from_data(k), Column.from_data(a, validity=rng.random(n) > 0.2), Column.new_const(abi.I64, 7, n),
                     Column.new_const(abi.I64, None, n), Column.from_data(x), Column.from_data(v)])
    types = [abi.I64, abi.I32 | abi.NULLABLE, abi.I64, abi.I64 | abi.NULLABLE, abi.I64, abi.I64]
    key = S.col(1) % S.lit(10, abi.U8)
    if part == 0:  # at most DBX_MAX_COMPUTED_COLS distinct expressions per operator
        aggs = [("sum", S.col(1) + S.col(2)), ("count", S.col(1) + S.col(3)), ("sum", S.col(1) * S.lit(None, abi.I32)),
                ("avg", S.col(1) + S.col(2)), ("count", None)]
    else:
        aggs = [("min", S.cast(S.col(4), abi.I8, try_cast=True)), ("max", S.col(1) - S.col(2)), ("count", None)]
    params = AggregatorParams([key], aggs)
    filt = E.ne(E.col(5) % E.lit(4), E.lit(1))
    out, _ = run_ops(blk.split_by_rows(9_000), params, filt, types)
    assert not out.columns[len(aggs)].valid_mask().all()  # the NULL key group
    if part == 0:
        assert not out.columns[2].valid_mask().any()  # sum over a NULL literal: NULL in every group
    else:
        assert out.columns[0].valid_mask().any()
    check_against_oracle(out, blk, types, params, filt)


@pytest.mark.parametrize("skew", [False, True])
def test_straight_line_kernel(jit, skew):
    """8-byte device columns and one CMP: the straight-line kernel evaluates, with x * y in the slot of
    the predicate-only column and two computed columns in slots of their own; skewed keys hit the
    hot-group cache."""
    n = 100_003  # whole tiles on the straight-line kernel, the remainder on the generic one
    rng = np.random.default_rng(12)
    k = (np.where(rng.random(n) < 0.9, 0, rng.integers(0, 5000, n)) if skew else rng.integers(0, 5000, n)).astype(np.int64)
    x = rng.integers(-1000, 1000, n).astype(np.float64)
    y = rng.integers(-1000, 1000, n).astype(np.float64)
    v = rng.integers(0, 1 << 20, n).astype(np.int64)
    blk = DataBlock([Column.from_data(c) for c in (k, x, y, v)])
    dev = DataBlock([to_device(c) for c in blk.columns], n)
    types = [abi.I64, abi.F64, abi.F64, abi.I64]
    params = AggregatorParams([0], [("sum", S.col(1) * S.col(2)), ("avg", S.col(1) + S.col(2)), ("min", S.col(1) - S.col(2)), ("count", None)])
    filt = E.eq(E.col(3) % E.lit(3), E.lit(0))
    out, variant = run_ops([dev], params, filt, types)
    assert "straight-line launches 1, generic launches 1" in variant, variant
    if skew:
        absorbed = int(variant.rsplit("hot-group cache ", 1)[1].split()[0].rstrip(";"))
        assert absorbed > 0, variant
    check_against_oracle(out, blk, types, params, filt)


def test_error_on_hand_off_without_finish(jit):
    n = 50_000
    k, a, b, v = _data(n, 9)
    b = np.where(np.arange(n) == 1234, 0, b).astype(np.int32)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b), Column.from_data(v)])
    types = [abi.I64, abi.I64, abi.I32, abi.I64]
    params = AggregatorParams([0], [("sum", S.col(1) // S.col(2))])
    with pytest.raises(OracleEvalError) as oe:
        composed(blk, types, params)
    assert oe.value.row == 1234 and oe.value.msg == "divided by zero"
    part = TransformPartialAggregate(params, types)
    part.transform(blk)
    fin = TransformFinalAggregate(params, types)
    with pytest.raises(DbxError) as e1:
        fin.transform(part)  # merge without finish: the failure still surfaces
    assert e1.value.status == abi.ERR_BAD_ARGUMENTS and "first failing row 1234" in e1.value.message
    with pytest.raises(DbxError) as e2:
        part.serialize()
    assert e2.value.status == abi.ERR_STATE
    part.close()
    fin.close()
