"""Writes tests/golden/*.json: known-answer vectors transcribed from the reference's OWN test
data (the reference is Rust and cannot be run here, so values are copied by hand from its
golden files; each case carries the file:line it comes from, relative to the databend source tree).
Run:  python tests/golden/make_golden.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
AGG = "src/query/functions/tests/it/aggregates/testdata"

aggregates = {
    "columns": {  # aggregates/sum.rs:19-100, avg.rs:16-64, count.rs
        "a": {"dtype": "I64", "values": [4, 3, 2, 1]},
        "b": {"dtype": "U64", "values": [1, 2, 1, 3]},
        "f": {"dtype": "F64", "values": [1.25, -2.5, 3.75, 4.5]},
        "i32_col": {"dtype": "I32", "values": [-10, 20, -30, 40]},
        "x_null": {"dtype": "U64", "values": [1, 2, 3, 4], "validity": [True, True, False, False]},
        "all_null": {"dtype": "U64", "values": [1, 2, 3, 4], "validity": [False, False, False, False]},
        "const_int": {"dtype": "I32", "const": 5, "rows": 4},
        "const_int_null": {"dtype": "I32", "const": None, "rows": 4},
    },
    # group-by simulator: rows alternate between two groups, row i -> group i % 2
    # (aggregate_simulation_support.rs:256-258)
    "cases": [
        {"fn": "sum", "arg": "a", "single": [10], "single_valid": [True], "grouped": [6, 4], "grouped_valid": [True, True], "dtype": "I64", "src": f"{AGG}/sum.txt:21-28, sum_group_by.txt:21-28"},
        {"fn": "sum", "arg": "const_int", "single": [20], "single_valid": [True], "grouped": [10, 10], "grouped_valid": [True, True], "dtype": "I64", "src": f"{AGG}/sum.txt:31-38, sum_group_by.txt:31-38"},
        {"fn": "sum", "arg": "const_int_null", "single": [0], "single_valid": [False], "grouped": [0, 0], "grouped_valid": [False, False], "dtype": "I64", "src": f"{AGG}/sum.txt:41-48, sum_group_by.txt:41-48"},
        {"fn": "sum", "arg": "f", "single": [7.0], "single_valid": [True], "grouped": [5.0, 2.0], "grouped_valid": [True, True], "dtype": "F64", "src": f"{AGG}/sum.txt:51-58, sum_group_by.txt:51-58"},
        {"fn": "sum", "arg": "x_null", "single": [3], "single_valid": [True], "grouped": [1, 2], "grouped_valid": [True, True], "dtype": "U64", "src": f"{AGG}/sum.txt:91-98, sum_group_by.txt:91-98"},
        {"fn": "sum", "arg": "all_null", "single": [0], "single_valid": [False], "grouped": [0, 0], "grouped_valid": [False, False], "dtype": "U64", "src": f"{AGG}/sum.txt:101-108, sum_group_by.txt:101-108"},
        {"fn": "avg", "arg": "a", "single": [2.5], "single_valid": [True], "grouped": [3.0, 2.0], "grouped_valid": [True, True], "dtype": "F64", "src": f"{AGG}/avg.txt:21-28, avg_group_by.txt:21-28"},
        {"fn": "avg", "arg": "i32_col", "single": [5.0], "single_valid": [True], "grouped": [-20.0, 30.0], "grouped_valid": [True, True], "dtype": "F64", "src": f"{AGG}/avg.txt:31-38, avg_group_by.txt:31-38"},
        {"fn": "avg", "arg": "f", "single": [1.75], "single_valid": [True], "grouped": [2.5, 1.0], "grouped_valid": [True, True], "dtype": "F64", "src": f"{AGG}/avg.txt:41-48, avg_group_by.txt:41-48"},
        {"fn": "avg", "arg": "x_null", "single": [1.5], "single_valid": [True], "grouped": [1.0, 2.0], "grouped_valid": [True, True], "dtype": "F64", "src": f"{AGG}/avg.txt:71-78, avg_group_by.txt:71-78"},
        {"fn": "avg", "arg": "all_null", "single": [0.0], "single_valid": [False], "grouped": [0.0, 0.0], "grouped_valid": [False, False], "dtype": "F64", "src": f"{AGG}/avg.txt:81-88, avg_group_by.txt:81-88"},
        {"fn": "count", "arg": "a", "single": [4], "single_valid": [True], "grouped": [2, 2], "grouped_valid": [True, True], "dtype": "U64", "src": f"{AGG}/count.txt:41-48, count_group_by.txt:41-48"},
        {"fn": "count", "arg": None, "single": [4], "single_valid": [True], "grouped": [2, 2], "grouped_valid": [True, True], "dtype": "U64", "src": f"{AGG}/count.txt:31-38, count_group_by.txt:31-38"},
        {"fn": "count", "arg": "const_int", "single": [4], "single_valid": [True], "grouped": [2, 2], "grouped_valid": [True, True], "dtype": "U64", "src": f"{AGG}/count.txt:11-18, count_group_by.txt:11-18"},
        {"fn": "count", "arg": "const_int_null", "single": [0], "single_valid": [True], "grouped": [0, 0], "grouped_valid": [True, True], "dtype": "U64", "src": f"{AGG}/count.txt:21-28, count_group_by.txt:21-28"},
        {"fn": "count", "arg": "x_null", "single": [2], "single_valid": [True], "grouped": [1, 1], "grouped_valid": [True, True], "dtype": "U64", "src": f"{AGG}/count.txt:51-58, count_group_by.txt:51-58"},
        {"fn": "count", "arg": "all_null", "single": [0], "single_valid": [True], "grouped": [0, 0], "grouped_valid": [True, True], "dtype": "U64", "src": f"{AGG}/count.txt:91-98, count_group_by.txt:91-98"},
    ],
}

VEC = "src/query/functions/tests/it/scalars/testdata/vector.txt"
SLT = "tests/sqllogictests/suites/query/functions/02_0063_function_vector.test"
vector_distance = {
    "cosine": [
        {"a": [1, 0, 0], "b": [1, 0, 0], "out": "0", "src": f"{VEC}:1-7"},
        {"a": [1, 0, 0], "b": [-1, 0, 0], "out": "2", "src": f"{VEC}:10-16"},
        {"a": [1, 2, 3], "b": [4, 5, 6], "out": "0.02536821", "src": f"{VEC}:19-25"},
        {"a": [0, 0, 0], "b": [1, 2, 3], "out": "NaN", "src": f"{VEC}:28-34"},
        {"a": [1, -2, 3], "b": [-4, 5, -6], "out": "1.974632", "src": f"{VEC}:37-43"},
        {"a": [0.1, 0.2, 0.3], "b": [0.4, 0.5, 0.6], "out": "0.02536827", "src": f"{VEC}:46-52"},
        {"a": [1, 0], "b": [0, 1], "out": "1", "src": f"{VEC}:55-61"},
        {"a": [1, 2], "b": [3, 4], "out": "0.01613009", "src": f"{VEC}:64-73"},
        {"a": [5.1, 6.2], "b": [7.3, 8.4], "out": "0.0003668666", "src": f"{VEC}:74"},
        {"a": [9.4, 10.6], "b": [11.1, 12.3], "out": "0.0000377297", "src": f"{VEC}:75"},
        {"a": [1.1, 2.2, 3], "b": [1, 1, 1], "out": "0.06241274", "src": f"{SLT}:16-19,100-106"},
        {"a": [1, 2.2, 3], "b": [4, 6, 8], "out": "0.0069953203", "src": f"{SLT}:16-19,100-106"},
        {"a": [1, 2, 3], "b": [3, 5, 7], "out": "0.0025851727", "src": f"{SLT}:100-107"},
        {"a": [0.1, 0.2, 0.3], "b": [0.4, 0.5, 0.6], "out": "0.025368273", "src": f"{SLT}:73-79"},
        {"a": [1, 2, 3, 4, 5, 6, 7, 8], "b": [100, 101, 102, 103, 104, 105, 106, 107], "out": "0.099043",
         "approx": 1e-6, "src": "src/common/vector/tests/it/distance.rs:20-25 (1.0 - 0.900_957, assert_relative_eq)"},
        {"a": [3, 45, 7, 2, 5, 20, 13, 12], "b": [2, 54, 13, 15, 22, 34, 50, 1], "out": "0.1264194",
         "approx": 1e-6, "src": "src/common/vector/tests/it/distance.rs:28-33 (1.0 - 0.873_580_6)"},
    ],
    "l2": [
        {"a": [1, 2, 3], "b": [1, 2, 3], "out": "0", "src": f"{VEC}:368-374"},
        {"a": [1, 2, 3], "b": [4, 5, 6], "out": "5.196152", "src": f"{VEC}:377-383"},
        {"a": [0, 0, 0], "b": [1, 2, 3], "out": "3.741658", "src": f"{VEC}:386-392"},
        {"a": [1, -2, 3], "b": [-4, 5, -6], "out": "12.4499", "src": f"{VEC}:395-401"},
        {"a": [0.1, 0.2, 0.3], "b": [0.4, 0.5, 0.6], "out": "0.5196152", "src": f"{VEC}:404-410"},
        {"a": [1, 2], "b": [3, 4], "out": "2.828427", "src": f"{VEC}:413-419"},
        {"a": [1.1, 2.2, 3], "b": [1, 1, 1], "out": "2.3345234", "src": f"{SLT}:41-44"},
        {"a": [1, 2.2, 3], "b": [4, 6, 8], "out": "6.959885", "src": f"{SLT}:41-44"},
        {"a": [1, 2, 3], "b": [3, 5, 7], "out": "5.3851647", "src": f"{SLT}:100-107"},
    ],
}

sort = {  # src/query/expression/tests/it/sort.rs:29-100 (row ids instead of the string column)
    "cases": [
        {"values": [6, 4, 3, 2, 1, 1, 7], "dtype": "I64", "asc": True, "nulls_first": False, "limit": None,
         "sorted": [1, 1, 2, 3, 4, 6, 7], "rows": [4, 5, 3, 2, 1, 0, 6], "src": "sort.rs:41-52"},
        {"values": [6, 4, 3, 2, 1, 1, 7], "dtype": "I64", "asc": True, "nulls_first": False, "limit": 4,
         "sorted": [1, 1, 2, 3], "rows": [4, 5, 3, 2], "src": "sort.rs:53-64"},
    ],
}

kernel = {  # src/query/expression/tests/it/kernel.rs:54-68 + testdata/kernel-pass.txt:1-18
    "filter": {
        "bitmap": [True, False, False, False, True],
        "columns": [
            {"dtype": "I32", "values": [0, 1, 2, 3, -4]},
            {"dtype": "U8", "values": [10, 11, 12, 13, 14], "validity": [False, True, False, False, False]},
        ],
        "result": [{"values": [0, -4], "validity": [True, True]}, {"values": [10, 14], "validity": [False, False]}],
        "src": "kernel.rs:54-68, kernel-pass.txt:1-18",
    },
    "take": {  # kernel.rs:94-108
        "indices": [0, 3, 1],
        "columns": [
            {"dtype": "I32", "values": [0, 1, 2, 3, -4]},
            {"dtype": "U8", "values": [10, 11, 12, 13, 14], "validity": [False, True, False, False, False]},
        ],
        "result": [{"values": [0, 3, 1], "validity": [True, True, True]}, {"values": [10, 13, 11], "validity": [False, False, True]}],
        "src": "kernel.rs:94-108",
    },
    "concat": [{  # kernel.rs:70-92 (numeric columns 0 and 1), kernel-pass.txt:21-52
        "blocks": [
            [{"dtype": "I32", "values": [0, 1, 2, 3, -4]},
             {"dtype": "U8", "values": [10, 11, 12, 13, 14], "validity": [False, True, False, False, False]}],
            [{"dtype": "I32", "values": [5, 6]}, {"dtype": "U8", "values": [15, 16], "validity": [False, True]}],
        ],
        "result": [{"values": [0, 1, 2, 3, -4, 5, 6], "validity": [True] * 7},
                   {"values": [10, 11, 12, 13, 14, 15, 16], "validity": [False, True, False, False, False, False, True]}],
        "src": "kernel.rs:70-92, kernel-pass.txt:21-52",
    }],
    "scatter": [{  # kernel.rs:181-196, kernel-pass.txt:211-247
        "indices": [0, 0, 1, 2, 1],
        "scatter_size": 3,
        "columns": [
            {"dtype": "I32", "values": [0, 1, 2, 3, -4]},
            {"dtype": "U8", "values": [10, 11, 12, 13, 14], "validity": [False, True, False, False, False]},
        ],
        "results": [
            [{"values": [0, 1], "validity": [True, True]}, {"values": [10, 11], "validity": [False, True]}],
            [{"values": [2, -4], "validity": [True, True]}, {"values": [12, 14], "validity": [False, False]}],
            [{"values": [3], "validity": [True]}, {"values": [13], "validity": [False]}],
        ],
        "src": "kernel.rs:181-196, kernel-pass.txt:211-247",
    }],
}

misc = {
    "config1": {"sql": "SELECT sum(number) FROM numbers(10000000) WHERE number%3=0", "answer": 16666668333333,
                "src": "BASELINE.json configs[0]; closed form 3*(3333333*3333334/2)"},
    "agg_hashtable": {"ns": [100, 1000, 10000, 100000], "m": 4,
                      "src": "src/query/functions/tests/it/aggregates/agg_hashtable.rs:52-199"},
    "agg_hash": {  # group_hash.rs:555-570 evaluated by hand with Python big ints in tests
        "src": "src/query/expression/src/aggregate/group_hash.rs:555-570"},
}

for name, obj in [("aggregates", aggregates), ("vector_distance", vector_distance), ("sort", sort), ("kernel", kernel),
                  ("misc", misc)]:
    with open(os.path.join(HERE, name + ".json"), "w") as f:
        json.dump(obj, f, indent=1)
print("wrote golden fixtures")
