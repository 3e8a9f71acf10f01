"""Regenerates tests/golden/window.json from the reference's window-function sqllogictests.

Run from the repository root with the reference source tree at REFERENCE (default ../reference).
Takes the numeric cases of tests/sqllogictests/suites/query/window_function/{window_bound,window_basic,
window_ntile}.test: the tables are read from their CREATE TABLE / INSERT statements, and each case's
expected rows from the block under its query.  Strings and dates become integer codes that keep their
order and equality (the sorted distinct values of the column, numbered from 0), per column.

Each case names its window (partition keys, order keys, functions and frames, as the binder would
give them: an ORDER BY without a frame is RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW), the
query's select list (table columns and `$i` for function i) and its final ORDER BY (`-name`:
descending).  The test compares
the reference's rows with the oracle's without depending on the order of rows the final ORDER BY
leaves tied: rows are compared as multisets inside each run of equal final-order keys (as one
multiset when the query has no ORDER BY)."""
import json
import os
import re
import sys

REF = os.environ.get("REFERENCE", os.path.join(os.path.dirname(__file__), "..", "..", "..", "reference"))
SUITE = os.path.join(REF, "tests", "sqllogictests", "suites", "query", "window_function")

DEFAULT_FRAME = ["range", "unbounded_preceding", "current_row"]


def _value(v):
    if v.startswith("'"):
        return v[1:-1]
    if v.upper() == "NULL":
        return None
    return int(v) if re.fullmatch(r"-?\d+", v) else float(v)


def parse_tables(text):
    tables = {}
    for name, body in re.findall(r"CREATE TABLE `?(\w+)`?\s*\((.*?)\)\s*;?\s*\n", text, re.S | re.I):
        cols = [c.strip().split()[0].strip("`") for c in body.split(",")]
        tables[name.lower()] = {"cols": cols, "rows": []}
    for name, body in re.findall(r"insert into (\w+) values\s*(.*?)\n", text, re.I):
        rows = re.findall(r"\(([^()]*)\)", body)
        for r in rows:
            vals = [v.strip() for v in r.split(",")]
            tables.setdefault(name.lower(), {"cols": [], "rows": []})["rows"].append([_value(v) for v in vals])
    return tables


def encode(table):
    """column -> list of ints; string columns as order-preserving codes (and the code maps)."""
    cols, codes = {}, {}
    for j, c in enumerate(table["cols"]):
        vals = [r[j] for r in table["rows"]]
        if any(isinstance(v, str) for v in vals):
            m = {s: i for i, s in enumerate(sorted(set(vals)))}
            codes[c] = m
            vals = [m[v] for v in vals]
        cols[c] = vals
    return cols, codes


def expected_rows(text, marker, select, codes):
    at = text.index(marker)
    assert text.find(marker, at + 1) < 0, f"query marker not unique: {marker!r}"
    body = text[text.index("\n----\n", at) + 6:]
    rows = []
    for line in body.split("\n"):
        if not line.strip():
            break
        fields = line.split()
        assert len(fields) == len(select), (marker, line)
        row = []
        for name, f in zip(select, fields):
            if f == "NULL":
                row.append(None)
            elif name in codes:
                row.append(codes[name][f])
            elif re.fullmatch(r"-?\d+", f):
                row.append(int(f))
            else:
                row.append(float(f))
        rows.append(row)
    return rows


def fn(name, arg=None, n=0, default=None, frame=None):
    return {"name": name, "arg": arg, "n": n, "default": default, "frame": frame}


def rows_frame(start, end):
    return ["rows", start, end]


# (file, table, unique marker in the query, partition_by, order_by [(col, asc, nulls_first)], functions, select, final order)
CASES = [
    ("window_bound", "tenk1", "rows between 2 preceding and 2 following) su", [], [["unique1", True, False]],
     [fn("sum", "unique1", frame=rows_frame(["preceding", 2], ["following", 2]))], ["$0"], ["unique1"]),
    ("window_bound", "tenk1", "rows between 2 preceding and 1 preceding) su", [], [["unique1", True, False]],
     [fn("sum", "unique1", frame=rows_frame(["preceding", 2], ["preceding", 1]))], ["$0"], ["unique1"]),
    ("window_bound", "tenk1", "rows between 1 following and 3 following) su", [], [["unique1", True, False]],
     [fn("sum", "unique1", frame=rows_frame(["following", 1], ["following", 3]))], ["$0"], ["unique1"]),
    ("window_bound", "tenk1", "rows between unbounded preceding and 1 following) su", [], [["unique1", True, False]],
     [fn("sum", "unique1", frame=rows_frame("unbounded_preceding", ["following", 1]))], ["$0"], ["unique1"]),
    ("window_bound", "tenk1", "first_value(unique1) over (order by unique1 rows between 1 preceding", [], [["unique1", True, False]],
     [fn("nth_value", "unique1", n=1, frame=rows_frame(["preceding", 1], "unbounded_following"))], ["unique1", "$0"], ["unique1"]),
    ("window_bound", "tenk1", "first_value(ten) OVER (PARTITION BY four ORDER BY ten rows between 1 preceding", ["four"], [["ten", True, False]],
     [fn("nth_value", "ten", n=1, frame=rows_frame(["preceding", 1], ["following", 1]))], ["four", "ten", "$0"], ["four", "ten"]),
    ("window_bound", "tenk1", "first_value(unique1) OVER (PARTITION BY two, four ORDER BY ten, twenty rows between 1 following",
     ["two", "four"], [["ten", True, False], ["twenty", True, False]],
     [fn("nth_value", "unique1", n=1, frame=rows_frame(["following", 1], "unbounded_following"))], ["two", "four", "unique1", "$0"],
     ["two", "four", "unique1", "$0"]),
    ("window_bound", "tenk1", "last_value(unique1) over (order by unique1 rows between current row", [], [["unique1", True, False]],
     [fn("nth_value", "unique1", n=0, frame=rows_frame("current_row", "unbounded_following"))], ["unique1", "$0"], ["unique1"]),
    ("window_bound", "tenk1", "last_value(ten) OVER (PARTITION BY four ORDER BY ten rows between current row", ["four"], [["ten", True, False]],
     [fn("nth_value", "ten", n=0, frame=rows_frame("current_row", ["following", 1]))], ["four", "ten", "$0"], ["four", "ten"]),
    ("window_bound", "tenk1", "(PARTITION BY two, four ORDER BY ten, twenty rows between unbounded preceding and 1 preceding) lv",
     ["two", "four"], [["ten", True, False], ["twenty", True, False]],
     [fn("nth_value", "unique1", n=0, frame=rows_frame("unbounded_preceding", ["preceding", 1]))], ["two", "four", "unique1", "$0"],
     ["two", "four", "unique1", "$0"]),
    ("window_basic", "empsalary", "sum(salary) OVER (PARTITION BY depname ORDER BY empno) FROM empsalary ORDER BY depname, empno",
     ["depname"], [["empno", True, False]], [fn("sum", "salary", frame=DEFAULT_FRAME)], ["depname", "empno", "salary", "$0"],
     ["depname", "empno"]),
    ("window_basic", "empsalary", "sum(salary) OVER (PARTITION BY depname ORDER BY salary) ss", ["depname"], [["salary", True, False]],
     [fn("sum", "salary", frame=DEFAULT_FRAME)], ["$0"], ["depname", "$0"]),
    ("window_basic", "empsalary", "SELECT row_number() OVER (PARTITION BY depname ORDER BY salary) rn FROM empsalary ORDER BY depname, rn\n", ["depname"], [["salary", True, False]],
     [fn("row_number")], ["$0"], ["depname", "$0"]),
    ("window_basic", "empsalary", "dense_rank() OVER (PARTITION BY depname ORDER BY salary) FROM", ["depname"], [["salary", True, False]],
     [fn("dense_rank")], ["depname", "salary", "$0"], ["depname", "salary"]),
    ("window_basic", "empsalary", "salary, rank() OVER (PARTITION BY depname ORDER BY salary) FROM", ["depname"], [["salary", True, False]],
     [fn("rank")], ["depname", "salary", "$0"], ["depname", "salary"]),
    ("window_basic", "empsalary", "percent_rank() OVER (PARTITION BY depname ORDER BY salary) FROM", ["depname"], [["salary", True, False]],
     [fn("percent_rank")], ["depname", "salary", "$0"], ["depname", "salary"]),
    ("window_basic", "empsalary", "lag(salary, 2) OVER (ORDER BY enroll_date) FROM", [], [["enroll_date", True, False]],
     [fn("lag", "salary", n=2)], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lag(salary, -2) OVER (ORDER BY enroll_date) FROM", [], [["enroll_date", True, False]],
     [fn("lag", "salary", n=-2)], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lag(salary, 2, 888) OVER (ORDER BY enroll_date) FROM", [], [["enroll_date", True, False]],
     [fn("lag", "salary", n=2, default=["const", 888])], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lag(salary, 2, salary) OVER (ORDER BY enroll_date) FROM", [], [["enroll_date", True, False]],
     [fn("lag", "salary", n=2, default="salary")], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lead(salary, 2) OVER (ORDER BY enroll_date) FROM empsalary\n", [], [["enroll_date", True, False]],
     [fn("lead", "salary", n=2)], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lead(salary, -2) OVER (ORDER BY enroll_date) FROM", [], [["enroll_date", True, False]],
     [fn("lead", "salary", n=-2)], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lead(salary, 2, 888) OVER (ORDER BY enroll_date) FROM", [], [["enroll_date", True, False]],
     [fn("lead", "salary", n=2, default=["const", 888])], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lead(salary, 2, salary) OVER (ORDER BY enroll_date) FROM", [], [["enroll_date", True, False]],
     [fn("lead", "salary", n=2, default="salary")], ["salary", "$0"], None),
    ("window_basic", "empsalary", "lead(salary, 2) OVER (ORDER BY enroll_date) c FROM empsalary2 ORDER BY salary desc", [],
     [["enroll_date", True, False]], [fn("lead", "salary", n=2)], ["salary", "$0"], ["-salary"]),
    ("window_basic", "empsalary", "ntile(3) OVER (PARTITION BY depname ORDER BY salary) AS rank_group FROM empsalary order by 1,2,3;",
     ["depname"], [["salary", True, False]], [fn("ntile", n=3)], ["depname", "salary", "$0"], ["depname", "salary", "$0"]),
    ("window_basic", "empsalary", "SELECT depname, min(salary) OVER (PARTITION BY depname ORDER BY salary, empno) m1,", ["depname"],
     [["salary", True, False], ["empno", True, False]],
     [fn("min", "salary", frame=DEFAULT_FRAME), fn("max", "salary", frame=DEFAULT_FRAME), fn("avg", "salary", frame=DEFAULT_FRAME)],
     ["depname", "$0", "$1", "$2"], ["depname", "empno"]),
]
NTILE_CASES = [("NTILE(2) OVER (PARTITION BY TeamName ORDER BY Score ASC)", ["TeamName"], 2, ["TeamName", "Score"]),
               ("NTILE(2) OVER (ORDER BY Score ASC)", [], 2, ["Score"]),
               ("NTILE(1000) OVER (PARTITION BY TeamName ORDER BY Score ASC)", ["TeamName"], 1000, ["TeamName", "Score"]),
               ("NTILE(1) OVER (PARTITION BY TeamName ORDER BY Score ASC)", ["TeamName"], 1, ["TeamName", "Score"])]


def main():
    texts = {f: open(os.path.join(SUITE, f + ".test")).read() for f in ("window_bound", "window_basic", "window_ntile")}
    tables = {}
    for f, t in texts.items():
        for name, tab in parse_tables(t).items():
            if tab["rows"]:
                tables[(f, name)] = tab
    out = []

    def add(file, tname, marker, pb, ob, funcs, select, final):
        cols, codes = encode(tables[(file, tname)])
        out.append({"name": f"{file}: {marker.strip()}", "table": cols, "partition_by": pb, "order_by": ob, "funcs": funcs,
                    "select": select, "final_order": final, "expected": expected_rows(texts[file], marker, select, codes)})

    for case in CASES:
        add(*case)
    for marker, pb, n, final in NTILE_CASES:
        add("window_ntile", "scoreboard", marker, pb, [["Score", True, False]], [fn("ntile", n=n)],
            ["TeamName", "Player", "Score", "$0"], final)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "window.json")
    with open(path, "w") as f:
        json.dump({"source": "tests/sqllogictests/suites/query/window_function/{window_bound,window_basic,window_ntile}.test",
                   "cases": out}, f, indent=1)
    print(f"{len(out)} cases -> {path}", file=sys.stderr)


if __name__ == "__main__":
    main()
