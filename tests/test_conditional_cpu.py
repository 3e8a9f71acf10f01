"""Conditionals without a GPU: the conditional oracle's lazy `if` / assume_not_null (tests/conditional_oracle.py) against the reference's
printed results (tests/golden/control.json, from make_control_golden.py), and the Python builders against
the binder's rewrites node for node."""
import json
import math
import os

import pytest

from databend_b200 import abi, scalar_expr as sx
import conditional_oracle as eo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "control.json")


def load():
    with open(GOLD) as f:
        return json.load(f)


def tree(e):
    if e[0] in ("col", "lit"):
        return tuple(e)
    if e[0] == "cast":
        return ("cast", tree(e[1]), e[2], e[3])
    return ("call", e[1]) + tuple(tree(a) for a in e[2:])


def columns_of(case):
    """the case's columns; a constant case runs on a one-column block of its row count"""
    cols = [(c["type"], [float(v) if c["type"][0] == "F" else v for v in c["values"]], c["valid"]) for c in case["columns"]]
    return cols or [("U8", [0] * case["rows"], None)]


def skipped_rows(case):
    return set(case.get("not_compared", {}).get("rows", []))


def same(t, got, exp):
    if t[0] == "F":
        exp = float(exp)
        return (math.isnan(got) and math.isnan(exp)) or got == exp
    return int(got) == int(exp)


GOLDEN = load()


@pytest.mark.parametrize("case", GOLDEN["cases"] + GOLDEN["sql_cases"], ids=lambda c: c["src"] + " " + c.get("sql", ""))
def test_oracle_matches_reference_output(case):
    t, _, vals, oks = eo.evaluate(tree(case["expr"]), columns_of(case))
    assert t == case["out_type"]
    exp_valid = case["out_valid"] or [1] * case["rows"]
    assert [int(o) for o in oks] == [int(v) for v in exp_valid[:case["rows"]]]
    for r in range(case["rows"]):
        if exp_valid[r] and r not in skipped_rows(case):
            assert same(t, vals[r], case["out_values"][r]), (r, vals[r], case["out_values"][r])


@pytest.mark.parametrize("case", GOLDEN["errors"] + GOLDEN["sql_errors"], ids=lambda c: c["src"])
def test_oracle_raises_reference_errors(case):
    with pytest.raises(eo.EvalFailure) as ei:
        eo.evaluate(tree(case["expr"]), columns_of(case))
    assert ei.value.msg == case["error"] and ei.value.row == case["row"]


def test_golden_counts():
    """control.txt:1-226 has 14 valued `if` cases and 2 error cases; other.txt:178 one assume_not_null case."""
    assert len([c for c in GOLDEN["cases"] if c["src"].startswith("control.txt")]) == 14
    assert len(GOLDEN["errors"]) == 2 and len(GOLDEN["sql_errors"]) == 1
    assert [c["src"] for c in GOLDEN["cases"] if "not_compared" in c] == ["other.txt:178"]


def program(e):
    """postfix program of an SExpr as (kind, func / col / dtype) pairs."""
    p = sx.flatten(e)
    out = []
    for i in range(p.n_nodes):
        n = p.nodes[i]
        if n.kind == abi.EXPR_CALL:
            out.append(("call", n.func))
        elif n.kind == abi.EXPR_COLUMN:
            out.append(("col", n.col))
        elif n.kind == abi.EXPR_CONST:
            out.append(("null", n.c.dtype) if n.c.is_null else ("lit", n.c.dtype, n.c.v.u64))
        else:
            out.append(("cast", n.cast_to))
    return out


C0, C1, C2 = ("col", 0), ("col", 1), ("col", 2)
IF, NOT, NN, ANN, EQ = ("call", abi.FN_IF), ("call", abi.FN_NOT), ("call", abi.FN_IS_NOT_NULL), ("call", abi.FN_ASSUME_NOT_NULL), ("call", abi.FN_EQ)


def test_if_emits_nested_ternary_nodes():
    e = sx.if_(sx.col(0), sx.col(1), sx.col(2), sx.lit(5, abi.I64), sx.lit(None, abi.I64))
    assert program(e) == [C0, C1, C2, ("lit", abi.I64, 5), ("null", abi.I64), IF, IF]
    with pytest.raises(AssertionError):
        sx.if_(sx.col(0), sx.col(1))


def test_case_rewrite():
    """scalar_rewrite.rs:117-142: with an operand each condition is eq(operand, c); no ELSE -> NULL."""
    e = sx.case_([(sx.lit(1, abi.I32), sx.col(1)), (sx.lit(2, abi.I32), sx.col(2))], operand=sx.col(0), dtype=abi.I64)
    assert program(e) == [C0, ("lit", abi.I32, 1), EQ, C1, C0, ("lit", abi.I32, 2), EQ, C2, ("null", abi.I64), IF, IF]
    e = sx.case_([(sx.col(0), sx.col(1))], else_=sx.col(2))
    assert program(e) == [C0, C1, C2, IF]


def test_coalesce_rewrite():
    """special_function.rs:559-606: NULL literals skipped, is_not_null / assume_not_null pairs, NULL else;
    only NULLs: if(NULL, NULL, NULL)."""
    e = sx.coalesce(sx.col(0), sx.lit(None, abi.I64), sx.col(1), dtype=abi.I64)
    assert program(e) == [C0, NN, C0, ANN, C1, NN, C1, ANN, ("null", abi.I64), IF, IF]
    assert program(sx.coalesce(sx.lit(None, abi.I64), dtype=abi.I64)) == [("null", abi.I64)] * 3 + [IF]


def test_nullif_iff_ifnull_nvl_nvl2():
    """rewrite_function.rs:40-86."""
    assert program(sx.nullif(sx.col(0), sx.col(1), abi.I32)) == [C0, C1, EQ, ("null", abi.I32), C0, IF]
    assert program(sx.iff(sx.col(0), sx.col(1), sx.col(2))) == [C0, C1, C2, IF]
    assert program(sx.ifnull(sx.col(0), sx.col(1))) == [C0, NN, NOT, C1, C0, IF]
    assert sx.nvl is sx.ifnull
    assert program(sx.nvl2(sx.col(0), sx.col(1), sx.col(2))) == [C0, NN, C1, C2, IF]


def test_is_distinct_from_rewrite():
    """scalar_rewrite.rs:59-89."""
    isnull = lambda c: [c, NN, NOT]  # noqa: E731
    both = isnull(C0) + isnull(C1) + [("call", abi.FN_AND)]
    either = isnull(C0) + isnull(C1) + [("call", abi.FN_OR)]
    for not_, cmp_ in ((False, abi.FN_NOTEQ), (True, abi.FN_EQ)):
        e = sx.is_distinct_from(sx.col(0), sx.col(1), not_=not_)
        assert program(e) == (both + [("lit", abi.BOOL, int(not_))] + either + [("lit", abi.BOOL, int(not not_))] + [C0, C1, ("call", cmp_)]
                              + [IF, IF, ANN])


def test_oracle_if_is_lazy_and_typed():
    cols = [("BOOL", [True, False, True], [1, 1, 0]), ("I64", [10, 0, 0], None)]
    e = ("call", "if", ("col", 0), ("call", "divide", ("lit", 1, "U8"), ("col", 1)), ("lit", -1.0, "F64"))
    t, nullable, vals, oks = eo.evaluate(e, cols)
    assert (t, nullable, vals, oks) == ("F64", False, [0.1, -1.0, -1.0], [True, True, True])
    with pytest.raises(ValueError):
        eo.infer(("call", "if", ("col", 1), ("col", 1), ("col", 1)), [("BOOL", False), ("I64", False)])
    t, nullable, vals, oks = eo.evaluate(("call", "assume_not_null", ("col", 1)), [("BOOL", [0], None), ("I64", [7], [0])])
    assert (t, nullable, vals, oks) == ("I64", False, [0], [True])
