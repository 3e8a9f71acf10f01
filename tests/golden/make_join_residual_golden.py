"""Writes tests/golden/join_residual.json: equi joins with a residual (non-equi) ON condition and their
answers, transcribed by hand from the reference's sqllogictests (paths relative to the databend source
tree, tests/sqllogictests/suites/query/join/).  Each case names its probe ("left") and build ("right")
tables, the key pair, the residual as a small tree over ["probe", col] / ["build", col] / literals, an
optional WHERE applied after the join (same form), the SELECT list and the expected rows (None = NULL).
Run:  python tests/golden/make_join_residual_golden.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LEFT_OUTER = "tests/sqllogictests/suites/query/join/left_outer.test"
JOIN = "tests/sqllogictests/suites/query/join/join.test"

T1_A = {"types": ["Int32", "Int32"], "rows": [[1, 2], [3, 4], [7, 8]]}            # t1(a, b)
T2_A = {"types": ["Int32", "Int32"], "rows": [[1, 4], [2, 3], [6, 8]]}            # t2(c, d)
T1_B = {"types": ["Int32", "Int32"], "rows": [[1, 2], [2, 4], [3, 6], [4, 8], [5, 10]]}  # t1(a, b)
T2_B = {"types": ["Int32", "Int32"], "rows": [[1, 2], [1, 4], [1, 6], [1, 8], [1, 10]]}  # t2(a, b)
T1_C = {"types": ["Int32", "UInt64"], "rows": [[1, 1696549154011], [2, 1696549154013]]}  # t1(id, val)
T2_C = {"types": ["Int32", "UInt64"], "rows": [[1, 1697650260000], [3, 1696549154009], [2, 1696549154010], [2, 1696549154013]]}

ALL = [["probe", 0], ["probe", 1], ["build", 0], ["build", 1]]
NULL_EXT = [[1, 2, None, None], [3, 4, None, None], [7, 8, None, None]]

golden = {"cases": [
    {"name": "left_on_key_and_probe_gt", "kind": "LEFT", "probe": T1_A, "build": T2_A, "probe_key": 0, "build_key": 0,
     # select * from t1 left outer join t2 on t1.a = t2.c and t1.a > 3
     "residual": [">", ["probe", 0], 3], "where": None, "select": ALL, "expect": NULL_EXT, "src": f"{LEFT_OUTER}:44-50"},
    {"name": "left_on_key_and_build_gt", "kind": "LEFT", "probe": T1_A, "build": T2_A, "probe_key": 0, "build_key": 0,
     # select * from t1 left outer join t2 on t1.a = t2.c and t2.c > 4
     "residual": [">", ["build", 0], 4], "where": None, "select": ALL, "expect": NULL_EXT, "src": f"{LEFT_OUTER}:51-57"},
    {"name": "left_conjunct_duplicate_build", "kind": "LEFT", "probe": T1_B, "build": T2_B, "probe_key": 0, "build_key": 0,
     # select * from t1 left join t2 on t1.a = t2.a and t1.b > t2.b
     "residual": [">", ["probe", 1], ["build", 1]], "where": None, "select": ALL,
     "expect": [[1, 2, None, None], [2, 4, None, None], [3, 6, None, None], [4, 8, None, None], [5, 10, None, None]],
     "src": f"{LEFT_OUTER}:237-246"},
    {"name": "left_eq_residual_then_where", "kind": "LEFT", "probe": T1_C, "build": T2_C, "probe_key": 0, "build_key": 0,
     # select t1.id, t1.val from t1 left join t2 on t1.id = t2.id and t1.val = t2.val where t1.val >= t2.val
     "residual": ["=", ["probe", 1], ["build", 1]], "where": [">=", ["probe", 1], ["build", 1]],
     "select": [["probe", 0], ["probe", 1]], "expect": [[2, 1696549154013]], "src": f"{JOIN}:168-171"},
]}

with open(os.path.join(HERE, "join_residual.json"), "w") as f:
    json.dump(golden, f, indent=1)
print("wrote join_residual.json")
