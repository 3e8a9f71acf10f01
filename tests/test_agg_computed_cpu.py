"""Computed columns without a GPU: the specialised build of a Q1-shaped plan compiles, and the Python
surface numbers expressions after the inputs and deduplicates them."""
import ctypes as C

from databend_b200 import abi, expr as E, lib, scalar_expr as S
from databend_b200.transforms import AggregatorParams


def test_expr_jit_selftest():
    buf = C.create_string_buffer(8192)
    assert lib.load().dbx_agg_expr_jit_selftest(buf, 8192) == abi.OK, buf.value.decode()
    assert buf.value == b"ok"


def test_flattening_numbers_and_dedups():
    prod = S.col(1) * S.col(2)
    params = AggregatorParams([S.col(0) % S.lit(10, abi.U8)], [("sum", prod), ("avg", S.col(1) * S.col(2)), ("count", 1)])
    filt = E.and_(E.gt(S.col(1) + S.col(2), E.lit(0)), E.bool_column(S.call("lt", S.col(0), S.col(3))))
    c = params.computed(4, filt)
    assert len(c.exprs) == 4  # key, product (once), sum, comparison
    cp = params.to_c(filt, c)
    assert cp.group_cols[0] == 4 and cp.aggs[0].arg_col == 5 and cp.aggs[1].arg_col == 5 and cp.aggs[2].arg_col == 1
    assert cp.filter.nodes[0].lhs.col == 6 and cp.filter.nodes[1].value == 7
    # a final built from the same params numbers the params' expressions alike
    assert [S.key(e) for e in params.computed(4).exprs] == [S.key(e) for e in c.exprs[:2]]
    # plain params keep working without a list
    p2 = AggregatorParams([0], [("sum", 1)]).to_c(E.eq(E.col(1) % E.lit(3), E.lit(0)))
    assert p2.aggs[0].arg_col == 1


def test_composed_oracle_q1_q6_by_hand():
    """The composed reference reproduces hand-computed Q1 / Q6 results on a tiny block."""
    import numpy as np
    from databend_b200.block import Column, DataBlock
    from computed_oracle import composed
    price = np.array([100.0, 200.0, 300.0, 400.0, 500.0])
    disc = np.array([0.5, 0.25, 0.0, 0.5, 0.75])
    tax = np.array([0.5, 0.0, 0.25, 0.0, 0.5])
    qty = np.array([10.0, 30.0, 20.0, 5.0, 40.0])
    flag = np.array([0, 1, 0, 1, 0], dtype=np.uint8)
    blk = DataBlock([Column.from_data(c) for c in (flag, price, disc, tax, qty)])
    types = [abi.U8, abi.F64, abi.F64, abi.F64, abi.F64]
    one = S.lit(1.0, abi.F64)
    dp = S.col(1) * (one - S.col(2))
    params = AggregatorParams([0], [("sum", dp), ("sum", dp * (one + S.col(3))), ("count", None)])
    (keys, kvalid, aggs, avalid, _), ctypes_ = composed(blk, types, params, E.lt(E.col(4), E.lit(35.0)), threads=1)
    got = {int(k): (a0, a1, int(c)) for k, a0, a1, c in zip(keys[0], aggs[0], aggs[1], aggs[2])}
    # kept rows 0..3: flag 0 -> rows 0, 2: dp 50 + 300, charge 75 + 375; flag 1 -> rows 1, 3: dp 150 + 200, charge 150 + 200
    assert got == {0: (350.0, 450.0, 2), 1: (350.0, 350.0, 2)}
    assert ctypes_ == [abi.F64, abi.F64]
    # Q6: sum(price * disc) WHERE qty < 24, no GROUP BY
    p6 = AggregatorParams([], [("sum", S.col(1) * S.col(2))])
    (_, _, aggs6, _, _), _ = composed(blk, types, p6, E.lt(E.col(4), E.lit(24.0)), threads=1)
    assert aggs6[0][0] == 100 * 0.5 + 300 * 0.0 + 400 * 0.5
