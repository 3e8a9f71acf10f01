"""Conditionals (IF / ASSUME_NOT_NULL) in computed columns of the fused filter / aggregate kernels, on both
builds (DBX_AGG_JIT 0 / 1), against the composed Filter -> EvalScalar -> Aggregate reference of
tests/conditional_oracle.py (which evaluates `if` lazily row by row) or exact numpy restatements."""
import numpy as np
import pytest

from conditional_oracle import composed
from float_agg_ref import exact_reference, sum_violations
from helpers import assert_group_results_equal, sorted_group_result_from_block, sorted_group_result_from_oracle
from databend_b200 import abi, expr as E, scalar_expr as S
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import AggregatorParams, TransformFilter, TransformFinalAggregate, TransformPartialAggregate, to_device

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["0", "1"], ids=["precompiled", "specialised"])
def jit(request, monkeypatch):
    monkeypatch.setenv("DBX_AGG_JIT", request.param)
    return request.param


def run_ops(blocks, params, filt, types):
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


def check(out, blk, types, params, filt):
    n_aggs, n_keys = len(params.aggregate_functions), len(params.group_columns)
    res, _ = composed(blk, types, params, filt)
    key_dtypes = [out.columns[n_aggs + j].dtype for j in range(n_keys)]
    assert_group_results_equal(sorted_group_result_from_block(out, n_aggs, n_keys), sorted_group_result_from_oracle(res, key_dtypes))


def _data(n, seed):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 50, n).astype(np.int64)
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    y = rng.integers(-100, 100, n).astype(np.int32)
    yv = rng.random(n) > 0.2
    v = rng.integers(0, 1 << 20, n).astype(np.int64)
    blk = DataBlock([Column.from_data(k), Column.from_data(x), Column.from_data(y, validity=yv), Column.from_data(v)])
    return blk, [abi.I64, abi.I64, abi.I32 | abi.NULLABLE, abi.I64]


def _aggs():
    c = S.call("gt", S.col(1), S.lit(0, abi.I64))
    return [("sum", S.if_(c, S.col(1), S.lit(0, abi.I64))),                                        # sum(if(c, x, 0))
            ("sum", S.if_(c, S.lit(1, abi.U8), S.lit(0, abi.U8))),                                 # sum(if(c, 1, 0))
            ("avg", S.case_([(c, S.cast(S.col(2), abi.I64))], dtype=abi.I64)),                     # CASE without ELSE: NULL rows skipped
            ("max", S.coalesce(S.col(2), S.lit(-7, abi.I32), dtype=abi.I32))]                      # coalesce over a nullable column


@pytest.mark.parametrize("blocks", ["one", "split65536", "device"])
def test_conditional_aggregates(jit, blocks):
    n = 150_000
    blk, types = _data(n, 1)
    params = AggregatorParams([0], _aggs())
    filt = E.ne(E.col(3) % E.lit(3), E.lit(0))
    bl = [blk] if blocks == "one" else blk.split_by_rows(65536) if blocks == "split65536" else [DataBlock([to_device(c) for c in blk.columns], n)]
    out, _ = run_ops(bl, params, filt, types)
    check(out, blk, types, params, filt)
    # min of a CASE without ELSE too (the one-expression operator limit keeps it in a second operator)
    p2 = AggregatorParams([0], [("min", S.case_([(S.call("lt", S.col(1), S.lit(0, abi.I64)), S.col(1))], dtype=abi.I64)), ("count", None)])
    out, _ = run_ops(bl, p2, filt, types)
    check(out, blk, types, p2, filt)


@pytest.mark.parametrize("path", ["partitioned", "growth", "no-group-by"])
def test_paths(jit, path, monkeypatch):
    n = 200_000
    blk, types = _data(n, 2)
    expected = 0
    if path == "partitioned":
        monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "4096")
        monkeypatch.setenv("DBX_AGG_PARTITION_ALWAYS", "1")
    if path == "growth":
        expected = 1
    keys = [] if path == "no-group-by" else [0]
    aggs = [("sum", S.if_(S.call("gt", S.col(1), S.lit(0, abi.I64)), S.col(1), S.lit(0, abi.I64))),
            ("sum", S.if_(S.call("lt", S.col(1), S.lit(-500, abi.I64)), S.lit(1, abi.U8), S.lit(0, abi.U8)))]
    params = AggregatorParams(keys, aggs, expected_groups=expected)
    filt = E.gt(E.col(3), E.lit(1000))
    out, variant = run_ops([blk], params, filt, types)
    if path == "partitioned":
        assert "two-pass (partitioned by table slice)" in variant, variant
    check(out, blk, types, params, filt)


def test_case_bucket_key_and_predicates(jit):
    """GROUP BY a CASE bucket; a CASE in the predicate as a BOOLCOL and as a CMP operand."""
    n = 120_000
    blk, types = _data(n, 3)
    x = S.col(1)
    bucket = S.case_([(S.call("lt", x, S.lit(-300, abi.I64)), S.lit(0, abi.U8)), (S.call("lt", x, S.lit(300, abi.I64)), S.lit(1, abi.U8))],
                     else_=S.lit(2, abi.U8))
    params = AggregatorParams([bucket], [("sum", S.col(3)), ("count", None)])
    boolcol = E.bool_column(S.if_(S.call("is_not_null", S.col(2)), S.call("gt", S.col(2), S.lit(0, abi.I32)), S.lit(False, abi.BOOL)))
    filt = E.and_(boolcol, E.gt(S.if_(S.call("gt", S.col(0), S.lit(25, abi.I64)), S.col(1), S.col(0)), E.lit(-200)))
    out, _ = run_ops(blk.split_by_rows(50_000), params, filt, types)
    check(out, blk, types, params, filt)
    # DBX_OP_FILTER with the same predicate
    f = TransformFilter(filt, types)
    got = f.transform(blk)
    f.close()
    k, xv, y = (blk.columns[i].values() for i in range(3))
    yv = blk.columns[2].valid_mask()
    keep = (yv & (y > 0)) & (np.where(k > 25, xv, k) > -200)
    np.testing.assert_array_equal(got.columns[3].values(), blk.columns[3].values()[keep])


def test_errors_only_on_kept_rows_and_taken_branches(jit):
    n = 60_000
    rng = np.random.default_rng(4)
    k = rng.integers(0, 10, n).astype(np.int64)
    x = rng.integers(1, 100, n).astype(np.int64)
    x[[5, 1005, 2005]] = 0
    v = rng.integers(0, 1 << 20, n).astype(np.int64)
    v[5] = 3  # row 5 dropped by the predicate
    v[1005] = 4
    v[2005] = 4
    c = np.ones(n, dtype=bool)
    c[1005] = False  # row 1005 kept but takes the else branch
    blk = DataBlock([Column.from_data(k), Column.from_data(x), Column.from_data(c, abi.BOOL), Column.from_data(v)])
    types = [abi.I64, abi.I64, abi.BOOL, abi.I64]
    params = AggregatorParams([0], [("sum", S.if_(S.col(2), S.lit(1000, abi.I64) // S.col(1), S.lit(0, abi.I64)))])
    filt = E.ne(E.col(3), E.lit(3))
    part = TransformPartialAggregate(params, types, filt)
    part.transform(blk)
    with pytest.raises(S.EvalError) as ei:
        part.on_finish()
    assert ei.value.row == 2005 and "divided by zero" in ei.value.message
    part.close()
    c[2005] = False
    blk = DataBlock([Column.from_data(k), Column.from_data(x), Column.from_data(c, abi.BOOL), Column.from_data(v)])
    out, _ = run_ops([blk], params, filt, types)
    check(out, blk, types, params, filt)


def test_q14_shape_float_sum(jit):
    """sum(if(ptype < 25, price * (1 - disc), 0.0)) without GROUP BY, held to float_agg_ref's bound."""
    n = 5_000_000
    rng = np.random.default_rng(14)
    price = rng.uniform(900.0, 105000.0, n)
    disc = rng.integers(0, 11, n) / 100.0
    ptype = rng.integers(0, 150, n).astype(np.int32)
    ship = rng.integers(0, 2500, n).astype(np.int32)
    blk = DataBlock([Column.from_data(c) for c in (price, disc, ptype, ship)])
    one = S.lit(1.0, abi.F64)
    rev = S.col(0) * (one - S.col(1))
    params = AggregatorParams([], [("sum", S.if_(S.call("lt", S.col(2), S.lit(25, abi.I32)), rev, S.lit(0.0, abi.F64)))])
    filt = E.and_(E.ge(E.col(3), E.lit(1000, abi.I32)), E.lt(E.col(3), E.lit(1030, abi.I32)))
    out, _ = run_ops([blk], params, filt, [abi.F64, abi.F64, abi.I32, abi.I32])
    keep = (ship >= 1000) & (ship < 1030)
    ref = exact_reference(np.zeros(n, dtype=np.int64), np.where(ptype < 25, price * (1 - disc), 0.0), keep)
    assert sum_violations(ref, {0: float(out.columns[0].values()[0])}) == []
