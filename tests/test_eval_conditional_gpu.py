"""dbx_eval_scalar on conditionals (IF / ASSUME_NOT_NULL) on both builds of the evaluator: the reference's
printed results (tests/golden/control.json), seeded random CASE / coalesce / nullif trees against the lazy
CPU oracle (tests/conditional_oracle.py) bit for bit, errors only on taken branches, type refusals, and one large block against np.where."""
import json
import os

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200 import scalar_expr as sx
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError
import conditional_oracle as eo
from test_eval_gpu import DT, NAME, NP, NUM, assert_matches, random_column, run_gpu, to_sexpr, to_tuple

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "control.json")


@pytest.fixture(params=["jit", "interp"])
def eval_mode(request, monkeypatch):
    if request.param == "interp":
        monkeypatch.setenv("DBX_EVAL_JIT", "0")
    return request.param


def load():
    with open(GOLD) as f:
        return json.load(f)


G = load()


def cols_of(case):
    cols = [(c["type"], [float(v) if c["type"][0] == "F" else v for v in c["values"]], c["valid"]) for c in case["columns"]]
    return cols or [("U8", [0] * case["rows"], None)]


@pytest.mark.parametrize("case", G["cases"] + G["sql_cases"], ids=lambda c: c["src"] + " " + c.get("sql", ""))
def test_reference_golden_outputs(gpu, eval_mode, case):
    t, vals, valid = run_gpu(cols_of(case), case["rows"], case["expr"])
    assert t == case["out_type"]
    exp_valid = case["out_valid"] or [1] * case["rows"]
    np.testing.assert_array_equal(valid.astype(int), np.asarray(exp_valid[:case["rows"]], dtype=int))
    skip = set(case.get("not_compared", {}).get("rows", []))
    for r in range(case["rows"]):
        if exp_valid[r] and r not in skip:
            assert float(vals[r]) == float(case["out_values"][r]), (r, vals[r], case["out_values"][r])


@pytest.mark.parametrize("case", G["errors"] + G["sql_errors"], ids=lambda c: c["src"])
def test_reference_error_cases(gpu, eval_mode, case):
    with pytest.raises(sx.EvalError, match=case["error"]) as ei:
        run_gpu(cols_of(case), case["rows"], case["expr"])
    assert ei.value.row == case["row"]


def _branch(rng, t, depth, k):
    """a random value expression of type t over columns 1..k (all of type t) of depth <= depth"""
    c = lambda: ["col", int(rng.integers(1, k + 1))]  # noqa: E731
    if depth == 0 or rng.random() < 0.3:
        return c() if rng.random() < 0.8 else ["lit", None, t]
    choice = rng.integers(0, 4)
    cond = ["call", ["lt", "gt", "eq", "noteq"][int(rng.integers(0, 4))], c(), c()] if rng.random() < 0.7 else ["col", 0]
    if choice == 0:  # CASE WHEN cond THEN x ELSE y
        return ["call", "if", cond, _branch(rng, t, depth - 1, k), _branch(rng, t, depth - 1, k)]
    if choice == 1:  # coalesce(x, y)
        x, y = c(), c()
        return ["call", "if", ["call", "is_not_null", x], ["call", "assume_not_null", x],
                ["call", "if", ["call", "is_not_null", y], ["call", "assume_not_null", y], ["lit", None, t]]]
    if choice == 2:  # nullif(x, y)
        x, y = c(), c()
        return ["call", "if", ["call", "eq", x, y], ["lit", None, t], x]
    return ["call", "if", ["call", "not", ["call", "is_not_null", c()]], c(), _branch(rng, t, depth - 1, k)]  # ifnull


def _stack_depth(e):
    """values on the evaluator's stack at the deepest point of the postfix program"""
    args = e[2:] if e[0] == "call" else [e[1]] if e[0] == "cast" else []
    return max([1] + [i + _stack_depth(a) for i, a in enumerate(args)])


def _nodes(e):
    args = e[2:] if e[0] == "call" else [e[1]] if e[0] == "cast" else []
    return 1 + sum(_nodes(a) for a in args)


@pytest.mark.parametrize("t", NUM + ["BOOL"])
def test_random_trees_against_oracle(gpu, eval_mode, t):
    """Nullable columns of every type (validity bit offsets != 0 through the slice, lengths not a multiple of 8)."""
    rng = np.random.default_rng(sum(map(ord, t)))
    rows = 1003
    for trial in range(4 if eval_mode == "jit" else 12):
        cols = [random_column(rng, "BOOL", rows, True)] + [random_column(rng, t, rows, True) for _ in range(3)]
        e = _branch(rng, t, 3, 3)
        while e[0] != "call" or _stack_depth(e) > 8 or _nodes(e) > 32:
            e = _branch(rng, t, 3, 3)
        et, _, evals, evalid = eo.evaluate(to_tuple(e), cols)
        blk = DataBlock([Column.from_data(np.asarray(v, dtype=bool if ct == "BOOL" else NP[ct]), DT[ct], validity=valid, validity_bit_offset=3 + i)
                         for i, (ct, v, valid) in enumerate(cols)], rows)
        col, odt = sx.eval_scalar(blk, to_sexpr(e))
        valid = col.valid_mask() if col.validity is not None else np.ones(rows, dtype=bool)
        assert_matches(NAME[odt & ~abi.NULLABLE], col.values(), valid, et, evals, evalid, (t, trial, e))


def test_untaken_division_by_zero_does_not_raise(gpu, eval_mode):
    a = ("I64", [1, 2, 0, 4, 0], None)
    c = ("BOOL", [1, 1, 0, 1, 0], None)
    # if(a <> 0, 100 / a, -1.0): the zero divisors sit on rows that take the else branch
    e = ["call", "if", ["call", "noteq", ["col", 1], ["lit", 0, "I64"]], ["call", "divide", ["lit", 100, "U8"], ["col", 1]], ["lit", -1.0, "F64"]]
    t, vals, valid = run_gpu([c, a], 5, e)
    assert t == "F64" and vals.tolist() == [100.0, 50.0, -1.0, 25.0, -1.0]
    # a NULL condition counts as false: the division on row 2 is not reached
    e = ["call", "if", ["col", 0], ["call", "modulo", ["lit", 7, "I64"], ["col", 1]], ["lit", 0, "I64"]]
    t, vals, valid = run_gpu([("BOOL", [1, 1, 1, 1, 0], [1, 1, 0, 1, 1]), a], 5, e)
    assert vals.tolist() == [0, 1, 0, 3, 0]


def test_taken_division_by_zero_raises_first_row(gpu, eval_mode):
    a = ("I64", [1, 2, 0, 4, 0, 0], None)
    c = ("BOOL", [1, 1, 0, 1, 1, 1], None)
    e = ["call", "if", ["col", 0], ["call", "div", ["lit", 100, "U8"], ["col", 1]], ["lit", 0, "I64"]]
    with pytest.raises(eo.EvalFailure) as oe:
        eo.evaluate(to_tuple(e), [c, a])
    assert oe.value.row == 4 and oe.value.msg == "divided by zero"
    with pytest.raises(sx.EvalError, match="divided by zero") as ei:
        run_gpu([c, a], 6, e)
    assert ei.value.row == 4
    # the condition's own error comes first on its row
    e = ["call", "if", ["call", "gt", ["call", "modulo", ["lit", 7, "I64"], ["col", 1]], ["lit", 0, "I64"]],
         ["call", "div", ["lit", 1, "U8"], ["col", 1]], ["lit", 0, "I64"]]
    with pytest.raises(sx.EvalError, match="Division by zero") as ei:
        run_gpu([c, a], 6, e)
    assert ei.value.row == 2


def test_refusals(gpu, eval_mode):
    blk = DataBlock([Column.from_data(np.array([1, 2], dtype=np.int64)), Column.from_data(np.array([1, 2], dtype=np.int32)),
                     Column.from_data(np.array([True, False]), abi.BOOL)])
    with pytest.raises(DbxError) as e:  # branches of two types
        sx.eval_scalar(blk, sx.if_(sx.col(2), sx.col(0), sx.col(1)))
    assert e.value.status == abi.ERR_INVALID and "one type" in e.value.message
    with pytest.raises(DbxError) as e:  # a non-Boolean condition
        sx.eval_scalar(blk, sx.if_(sx.col(0), sx.col(0), sx.col(0)))
    assert e.value.status == abi.ERR_INVALID and "Boolean" in e.value.message
    # a 3-arm CASE fits the 8-deep stack, a 4-arm one does not
    arms = lambda m: [x for i in range(m) for x in (sx.col(2), sx.lit(i, abi.I64))] + [sx.col(0)]  # noqa: E731
    col, dt = sx.eval_scalar(blk, sx.if_(*arms(3)))
    assert col.values().tolist() == [0, 2]
    with pytest.raises(DbxError) as e:
        sx.eval_scalar(blk, sx.if_(*arms(4)))
    assert e.value.status == abi.ERR_UNSUPPORTED


def test_large_block_against_np_where(gpu, eval_mode):
    n = (1 << 24) + 5
    rng = np.random.default_rng(3)
    x = rng.integers(-1000, 1000, n).astype(np.int32)
    y = rng.standard_normal(n)
    yv = rng.random(n) > 0.1
    blk = DataBlock([Column.from_data(x), Column.from_data(y, validity=yv)])
    # CASE WHEN x > 0 THEN coalesce(y, 0.0) ELSE cast(x as Float64) END
    e = sx.case_([(sx.call("gt", sx.col(0), sx.lit(0, abi.I32)), sx.coalesce(sx.col(1), sx.lit(0.0, abi.F64), dtype=abi.F64))],
                 else_=sx.cast(sx.col(0), abi.F64))
    col, dt = sx.eval_scalar(blk, e)
    want = np.where(x > 0, np.where(yv, y, 0.0), x.astype(np.float64))
    assert dt == abi.F64 | abi.NULLABLE
    assert col.valid_mask().all()
    np.testing.assert_array_equal(col.values().view(np.uint64), want.view(np.uint64))
