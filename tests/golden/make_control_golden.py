"""Transcribes the reference's conditional-function cases into tests/golden/control.json.  Run in the build
container (reads /root/reference):

    python tests/golden/make_control_golden.py

Sources (paths under the reference source tree):
  * src/query/functions/tests/it/scalars/testdata/control.txt:1-226 — every `if` case: 14 with a printed
    output, parsed from their "checked expr" with make_arith_golden.py's parser, and the 2 error cases, which
    print only the SQL text and are transcribed by hand (columns from tests/it/scalars/control.rs:38-123).
  * src/query/functions/tests/it/scalars/testdata/other.txt:178-197 — assume_not_null; its row 2 lies under a
    NULL and is not compared (the reference returns the value under the NULL, which the Arrow layout leaves
    unspecified).
  * tests/sqllogictests/suites/query/functions/02_0010_function_if.test, 02_0057_function_nullif.test,
    02_0058_function_ifnull.test, 02_0070_function_nvl.test — the numeric cases, transcribed by hand with
    the binder's rewrites (sql/src/planner/semantic/type_check/rewrite_function.rs:40-86) and the type
    checker's casts written out; literal casts are folded into the literal's type as the checker does.
Transcription rules: CAST<T>(x AS T NULL) is the identity; CAST<NULL>(NULL AS T NULL) is a NULL literal of T;
a multi-arm `if` becomes nested ternary ifs: if(c1, r1, if(c2, r2, else))."""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_arith_golden as mg  # noqa: E402

mg.FUNCS = mg.FUNCS | {"if", "assume_not_null"}


def nest_if(args):
    if len(args) == 3:
        return ["call", "if"] + args
    return ["call", "if", args[0], args[1], nest_if(args[2:])]


class CP(mg.P):
    """make_arith_golden's parser plus the transcription rules above."""

    def expr(self):
        rest = self.s[self.i:]
        m = re.match(r"CAST<NULL>\(NULL AS ([A-Za-z0-9]+) NULL\)", rest)
        if m:
            self.i += len(m.group(0))
            return ["lit", None, mg.parse_type(m.group(1))[0]]
        m = re.match(r"CAST<([A-Za-z0-9]+)>\(", rest)
        if m:
            self.i += len(m.group(0))
            inner = self.expr()
            self.eat(" AS ")
            t = self.until_balanced(")")
            self.eat(")")
            if t == m.group(1) + " NULL":
                return inner
            return ["cast", inner, mg.parse_type(t)[0], 0]
        m = re.match(r"(if|assume_not_null)<", rest)
        if m:  # two generic groups: if<T0=...><Boolean NULL, T0, ...>(...)
            self.i += len(m.group(0))
            self.until_balanced(">")
            self.eat("><")
            self.until_balanced(">")
            self.eat(">(")
            args = [self.expr()]
            while self.peek(2) == ", ":
                self.eat(", ")
                args.append(self.expr())
            self.eat(")")
            return nest_if(args) if m.group(1) == "if" else ["call", "assume_not_null"] + args
        return super().expr()


# ---- builders for the hand transcriptions
def col(i): return ["col", i]
def lit(v, t): return ["lit", v, t]
def call(name, *a): return ["call", name] + list(a)
def cast(e, t): return ["cast", e, t, 0]
def if_(*a): return nest_if(list(a))
def is_null(e): return call("not", call("is_not_null", e))  # rewrite_function.rs:72-79 (ifnull / nvl)


def nullif(x, y, t): return if_(call("eq", x, y), lit(None, t), x)  # rewrite_function.rs:40-47
def ifnull(x, y): return if_(is_null(x), y, x)


def numbers(n): return [{"type": "U64", "values": list(range(n)), "valid": None}]


def ints(vals, t="I32"):
    return {"type": t, "values": [0 if v is None else v for v in vals], "valid": None if None not in vals else [int(v is not None) for v in vals]}


def case(src, sql, expr, columns, out_type, out):
    rows = len(out)
    return {"src": src, "sql": sql, "expr": expr, "columns": columns, "rows": rows, "out_type": out_type,
            "out_values": [0 if v is None else v for v in out], "out_valid": None if None not in out else [int(v is not None) for v in out]}


def sql_cases():
    N = col(0)
    IF = "02_0010_function_if.test"
    out = [
        case(IF + ":26", "select if(number>1, true, false) from numbers(3)", if_(call("gt", N, lit(1, "U64")), lit(True, "BOOL"), lit(False, "BOOL")),
             numbers(3), "BOOL", [0, 0, 1]),
        case(IF + ":34", "select if(number>1, number, 1) from numbers(3)", if_(call("gt", N, lit(1, "U64")), N, lit(1, "U64")), numbers(3), "U64", [1, 1, 2]),
        case(IF + ":41", "select if(number<1, 2, number) from numbers(3)", if_(call("lt", N, lit(1, "U64")), lit(2, "U64"), N), numbers(3), "U64", [2, 1, 2]),
        case(IF + ":55", "select if(number<1, true, null) from numbers(3)", if_(call("lt", N, lit(1, "U64")), lit(True, "BOOL"), lit(None, "BOOL")),
             numbers(3), "BOOL", [1, None, None]),
        case(IF + ":62", "select if(number<4, number, number / 0) from numbers(3)",
             if_(call("lt", N, lit(4, "U64")), cast(N, "F64"), call("divide", N, lit(0, "U8"))), numbers(3), "F64", [0.0, 1.0, 2.0]),
        case(IF + ":69", "select if(number>4, number / 0, number) from numbers(3)",
             if_(call("gt", N, lit(4, "U64")), call("divide", N, lit(0, "U8")), cast(N, "F64")), numbers(3), "F64", [0.0, 1.0, 2.0]),
        case(IF + ":79", "select if (number > 0, 1 / number, null) from numbers(2)",
             if_(call("gt", N, lit(0, "U64")), call("divide", lit(1, "U8"), N), lit(None, "F64")), numbers(2), "F64", [None, 1.0]),
        case(IF + ":96", "SELECT if (number % 3 = 1, null, number) as a FROM numbers(7)",
             if_(call("eq", call("modulo", N, lit(3, "U8")), lit(1, "U8")), lit(None, "U64"), N), numbers(7), "U64", [0, None, 2, 3, None, 5, 6]),
        case(IF + ":118", "select if(number = 1, number, number = 0, number, number / 0) from numbers(1)",
             if_(call("eq", N, lit(1, "U64")), cast(N, "F64"), call("eq", N, lit(0, "U64")), cast(N, "F64"), call("divide", N, lit(0, "U8"))),
             numbers(1), "F64", [0.0]),
        case(IF + ":156", "select if(true, null, number) from numbers(1)", if_(lit(True, "BOOL"), lit(None, "U64"), N), numbers(1), "U64", [None]),
        case(IF + ":156", "select if(false, null, number) from numbers(1)", if_(lit(False, "BOOL"), lit(None, "U64"), N), numbers(1), "U64", [0]),
        case(IF + ":161", "select if(true, number, null) from numbers(1)", if_(lit(True, "BOOL"), N, lit(None, "U64")), numbers(1), "U64", [0]),
        case(IF + ":161", "select if(false, number, null) from numbers(1)", if_(lit(False, "BOOL"), N, lit(None, "U64")), numbers(1), "U64", [None]),
        case(IF + ":176", "select if(a=1, a*2, a*3) from t (a INT NULL: 1, 2, NULL, 4)",
             if_(call("eq", col(0), lit(1, "I32")), call("multiply", col(0), lit(2, "U8")), call("multiply", col(0), lit(3, "U8"))),
             [ints([1, 2, None, 4])], "I64", [2, 6, None, 12]),
    ]
    NI = "02_0057_function_nullif.test"
    one = [{"type": "U8", "values": [0], "valid": None}]  # a one-row block for the constant cases
    out += [
        case(NI + ":5", "SELECT NULLIF(2, 1)", nullif(lit(2, "U8"), lit(1, "U8"), "U8"), one, "U8", [2]),
        case(NI + ":10", "SELECT NULLIF(1, 2)", nullif(lit(1, "U8"), lit(2, "U8"), "U8"), one, "U8", [1]),
        case(NI + ":15", "SELECT NULLIF(1, NULL)", nullif(lit(1, "U8"), lit(None, "U8"), "U8"), one, "U8", [1]),
        case(NI + ":20", "SELECT NULLIF(NULL, 1)", nullif(lit(None, "U8"), lit(1, "U8"), "U8"), one, "U8", [None]),
        case(NI + ":56", "SELECT a, b, NULLIF(a, b) FROM t (a, b INT)", nullif(col(0), col(1), "I32"),
             [ints([0, 0, 1, 1]), ints([0, 1, 0, 1])], "I32", [None, 0, 1, None]),
        case(NI + ":73", "SELECT a, b, NULLIF(a, b) FROM t (a, b INT NULL)", nullif(col(0), col(1), "I32"),
             [ints([0, 0, 0, 1, 1, 1, None, None, None]), ints([0, 1, None, 0, 1, None, 0, 1, None])], "I32", [None, 0, 0, 1, None, 1, None, None, None]),
        case(NI + ":95", "SELECT a, b, NULLIF(a, b) FROM t (a, b INT NULL)", nullif(col(0), col(1), "I32"),
             [ints([None] * 5), ints([0, 1, None, 0, 1])], "I32", [None] * 5),
        case(NI + ":113", "SELECT a, b, NULLIF(a, b) FROM t (a, b INT NULL)", nullif(col(0), col(1), "I32"),
             [ints([0, 1, 0, 1, None]), ints([None] * 5)], "I32", [0, 1, 0, 1, None]),
    ]
    for fname, fn in (("02_0058_function_ifnull.test", "IFNULL"), ("02_0070_function_nvl.test", "NVL")):
        scal = [((1, 1), 1), ((2, 1), 2), ((1, 2), 1), ((1, None), 1), ((None, 1), 1)]
        lines = [4, 9, 14, 19, 24] if fn == "IFNULL" else [15, 20, 25, 30, 35]
        for ln, ((x, y), r) in zip(lines, scal):
            out.append(case(f"{fname}:{ln}", f"SELECT {fn}({'NULL' if x is None else x}, {'NULL' if y is None else y})",
                            ifnull(lit(x, "U8"), lit(y, "U8")), one, "U8", [r]))
        t1, t2 = (65, 82) if fn == "IFNULL" else (76, 93)
        out.append(case(f"{fname}:{t1}", f"SELECT a, b, {fn}(a, b) FROM t (a, b INT)", ifnull(col(0), col(1)),
                        [ints([0, 0, 1, 1]), ints([0, 1, 0, 1])], "I32", [0, 0, 1, 1]))
        out.append(case(f"{fname}:{t2}", f"SELECT a, b, {fn}(a, b) FROM t (a, b INT NULL)", ifnull(col(0), col(1)),
                        [ints([0, 1, None, None, None]), ints([None, None, 0, 1, None])], "I32", [0, 1, 0, 1, None]))
    errors = [
        {"src": IF + ":76", "sql": "select if(number<4, number / 0, number) from numbers(3)",
         "expr": if_(call("lt", N, lit(4, "U64")), call("divide", N, lit(0, "U8")), cast(N, "F64")), "columns": numbers(3), "rows": 3,
         "error": "divided by zero", "row": 0},
    ]
    return out, errors


def main():
    mg.P = CP
    cases = [c for c in mg.cases_of("control.txt") if int(c["src"].split(":")[1]) < 226]
    assert len(cases) == 14, len(cases)
    (anm,) = [c for c in mg.cases_of("other.txt") if c["src"] == "other.txt:178"]
    anm["not_compared"] = {"rows": [2], "reason": "the value under a NULL: the reference returns it, the Arrow layout leaves it unspecified"}
    cases.append(anm)
    one = {"type": "U8", "values": [0], "valid": None}
    errors = [
        {"src": "control.txt:82", "sql": "if(false, 1, 1 / 0)",
         "expr": if_(lit(False, "BOOL"), cast(lit(1, "U8"), "F64"), call("divide", lit(1, "U8"), lit(0, "U8"))), "columns": [one], "rows": 1,
         "error": "divided by zero", "row": 0},
        {"src": "control.txt:220", "sql": "if(cond_a, 1 / expr_a, expr_else)",  # columns: control.rs:113-122
         "expr": if_(col(0), call("divide", lit(1, "U8"), col(1)), cast(col(2), "F64")),
         "columns": [{"type": "BOOL", "values": [1, 1, 1, 0], "valid": None}, {"type": "I64", "values": [1, 2, 0, 4], "valid": None},
                     {"type": "I64", "values": [9, 10, 11, 12], "valid": None}], "rows": 4, "error": "divided by zero", "row": 2},
    ]
    sql, sql_errors = sql_cases()
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "control.json"), "w") as f:
        json.dump({"generated_by": "tests/golden/make_control_golden.py", "cases": cases, "errors": errors, "sql_cases": sql, "sql_errors": sql_errors},
                  f, indent=0)
    print(len(cases), "cases;", len(errors), "error cases;", len(sql), "SQL cases;", len(sql_errors), "SQL error cases", file=sys.stderr)
    for c in cases:
        print(c["src"], c["checked"], "->", c["out_type"], c["out_values"], c["out_valid"])


if __name__ == "__main__":
    main()
