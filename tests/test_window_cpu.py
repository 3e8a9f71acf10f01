"""Window operator, no GPU needed: the ctypes mirror of dbx_window_* against include/dbx.h, and the
window oracle against the reference's own test cases and hand-checked ones."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np

from databend_b200 import abi
from databend_b200.transforms import WindowFunc

from window_oracle import Col, golden_inputs, golden_mismatch, window

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_window_structs_match_the_header(tmp_path):
    structs = {
        "dbx_window_frame": (abi.WindowFrame, ["units", "start", "end", "start_offset", "end_offset"]),
        "dbx_window_func": (abi.WindowFunc, ["kind", "agg_kind", "arg_col", "default_col", "n", "ignore_nulls", "distinct", "frame"]),
        "dbx_window_params": (abi.WindowParams, ["n_partition_cols", "partition_cols", "n_order_cols", "order_cols", "order_asc",
                                                 "order_nulls_first", "n_funcs", "funcs"]),
    }
    enums = {"DBX_OP_WINDOW": abi.OP_WINDOW, "DBX_WIN_ROW_NUMBER": abi.WIN_ROW_NUMBER, "DBX_WIN_NTILE": abi.WIN_NTILE,
             "DBX_WIN_LAG": abi.WIN_LAG, "DBX_WIN_NTH_VALUE": abi.WIN_NTH_VALUE, "DBX_WIN_AGGREGATE": abi.WIN_AGGREGATE,
             "DBX_FRAME_RANGE": abi.FRAME_RANGE, "DBX_BOUND_UNBOUNDED_PRECEDING": abi.BOUND_UNBOUNDED_PRECEDING,
             "DBX_BOUND_CURRENT_ROW": abi.BOUND_CURRENT_ROW, "DBX_BOUND_UNBOUNDED_FOLLOWING": abi.BOUND_UNBOUNDED_FOLLOWING,
             "DBX_MAX_WINDOW_FUNCS": abi.MAX_WINDOW_FUNCS}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "dbx.h")}"', "int main(void) {"]
    for cname, (_, fields) in structs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for f in fields:
            lines.append(f'  printf("{cname}.{f} %zu\\n", offsetof({cname}, {f}));')
    for name in enums:
        lines.append(f'  printf("{name} %d\\n", (int){name});')
    lines += ["  return 0;", "}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-std=c11", "-o", str(exe), str(src)])
    out = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, (ctype, fields) in structs.items():
        assert int(out[cname]) == C.sizeof(ctype), cname
        for f in fields:
            assert int(out[f"{cname}.{f}"]) == getattr(ctype, f).offset, f"{cname}.{f}"
    for name, v in enums.items():
        assert int(out[name]) == v, name


def test_oracle_matches_the_reference_cases():
    """Every numeric case of the reference's window_bound, window_basic and window_ntile suites."""
    with open(os.path.join(ROOT, "tests", "golden", "window.json")) as f:
        cases = json.load(f)["cases"]
    assert len(cases) >= 31
    for case in cases:
        names, cols, pb, ob, funcs = golden_inputs(case)
        perm, res = window(cols, pb, ob, funcs)
        msg = golden_mismatch(case, names, cols, perm, res)
        assert msg is None, msg


def test_golden_comparison_rejects_a_wrong_row():
    with open(os.path.join(ROOT, "tests", "golden", "window.json")) as f:
        cases = json.load(f)["cases"]
    for case in cases:
        names, cols, pb, ob, funcs = golden_inputs(case)
        perm, res = window(cols, pb, ob, funcs)
        v, ok = res[-1]
        v = v.copy()
        v[int(np.flatnonzero(ok)[len(np.flatnonzero(ok)) // 2])] += 1
        assert golden_mismatch(case, names, cols, perm, res[:-1] + [(v, ok)]) is not None, case["name"]


def _col(vals, dtype=abi.I64, valid=None):
    return Col(np.asarray(vals, np.int64 if dtype == abi.I64 else np.float64), None if valid is None else np.asarray(valid, bool), dtype,
               valid is not None)


def test_oracle_ranking_and_frames_by_hand():
    part = _col([1, 1, 1, 2, 2, 1])
    t = _col([10, 20, 20, 5, 6, 30])
    v = _col([1, 2, 3, 4, 5, 6], valid=[1, 1, 0, 1, 1, 1])
    cols = [part, t, v]
    funcs = [WindowFunc("row_number"), WindowFunc("rank"), WindowFunc("dense_rank"), WindowFunc("percent_rank"),
             WindowFunc("cume_dist"), WindowFunc("ntile", n=3), WindowFunc("lag", arg=2, n=1), WindowFunc("lead", arg=2, n=1, default=0),
             WindowFunc("sum", arg=2, frame=("range", "unbounded_preceding", "current_row")),
             WindowFunc("count", arg=2, frame=("rows", ("preceding", 1), ("following", 1))),
             WindowFunc("sum", arg=2, frame=("rows", ("following", 1), ("preceding", 1))),
             WindowFunc("nth_value", arg=2, n=2, frame=("rows", "unbounded_preceding", "unbounded_following")),
             WindowFunc("max", arg=1, frame=("rows", ("preceding", 2), ("preceding", 1)))]
    perm, res = window(cols, [0], [(1, True, False)], funcs)
    assert list(perm) == [0, 1, 2, 5, 3, 4]
    got = [list(zip(r[0].tolist(), r[1].tolist())) for r in res]
    ok = lambda xs: [(x, True) for x in xs]
    assert got[0] == ok([1, 2, 3, 4, 1, 2])
    assert got[1] == ok([1, 2, 2, 4, 1, 2])
    assert got[2] == ok([1, 2, 2, 3, 1, 2])
    assert got[3] == ok([0.0, 1 / 3, 1 / 3, 1.0, 0.0, 1.0])
    assert got[4] == ok([0.25, 0.75, 0.75, 1.0, 0.5, 1.0])
    assert got[5] == ok([1, 1, 2, 3, 1, 2])
    assert got[6] == [(0, False), (1, True), (2, True), (0, False), (0, False), (4, True)]  # row 2's arg is NULL
    assert got[7] == [(2, True), (0, False), (6, True), (1, True), (5, True), (2, True)]  # default = partition column
    assert got[8] == ok([1, 3, 3, 9, 4, 9])  # RANGE: peers (t = 20) share the frame end
    assert got[9] == ok([2, 2, 2, 1, 2, 2])
    assert got[10] == [(0, False)] * 6  # start bound after end bound: empty on every row
    assert got[11] == [(2, True), (2, True), (2, True), (2, True), (5, True), (5, True)]
    assert got[12] == [(0, False), (10, True), (20, True), (20, True), (0, False), (5, True)]


def test_oracle_float_sums_follow_row_order_and_empty_frames():
    x = _col([1e16, 1.0, -1e16, 1.0], dtype=abi.F64)
    cols = [x]
    perm, res = window(cols, [], [], [WindowFunc("sum", arg=0, frame=("rows", "unbounded_preceding", "current_row")),
                                      WindowFunc("avg", arg=0, frame=("rows", ("preceding", 1), "current_row")),
                                      WindowFunc("min", arg=0, frame=("rows", "current_row", "unbounded_following"))])
    assert list(perm) == [0, 1, 2, 3]
    assert res[0][0].tolist() == [1e16, 1e16 + 1.0, (1e16 + 1.0) - 1e16, (1e16 + 1.0) - 1e16 + 1.0]
    assert res[1][0].tolist() == [1e16, (1e16 + 1.0) / 2, (1.0 - 1e16) / 2, (-1e16 + 1.0) / 2]
    assert res[2][0].tolist() == [-1e16, -1e16, -1e16, 1.0]
    nan = _col([float("nan"), -0.0, 0.0], dtype=abi.F64)
    _, res = window([nan], [], [], [WindowFunc("max", arg=0, frame=("rows", "unbounded_preceding", "current_row")),
                                   WindowFunc("min", arg=0, frame=("rows", "current_row", "unbounded_following"))])
    assert math.isnan(res[0][0][0]) and math.isnan(res[0][0][2])
    assert math.copysign(1.0, res[1][0][1]) == -1.0 and math.copysign(1.0, res[1][0][2]) == 1.0
