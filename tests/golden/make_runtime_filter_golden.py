"""Writes tests/golden/runtime_filter.json: known answers for the join runtime filters, transcribed by
hand from the reference's own unit tests (paths relative to the databend source tree, src/query).
Run:  python tests/golden/make_runtime_filter_golden.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SBBF = "catalog/src/sbbf.rs"
CONVERT = "service/src/pipelines/processors/transforms/hash_join/runtime_filter/convert.rs"

golden = {
    "salt": {"values": [0x47b6137b, 0x44974d91, 0x8824ad5b, 0xa2b7289d, 0x705495c7, 0x2df1424b, 0x9efc4947, 0x5c6bfb31],
             "src": f"{SBBF}:97-106"},
    "optimal_num_of_bytes": {  # (input, expected)
        "cases": [[0, 32], [9, 32], [31, 32], [32, 32], [33, 64], [99, 128], [1024, 1024], [999_000_000, 128 * 1024 * 1024]],
        "src": f"{SBBF}:602-615"},
    "num_of_bits_from_ndv_fpp": {  # (fpp, ndv, num_bits)
        "cases": [
            [0.1, 10, 57], [0.01, 10, 96], [0.001, 10, 146],
            [0.1, 100, 577], [0.01, 100, 968], [0.001, 100, 1460],
            [0.1, 1000, 5772], [0.01, 1000, 9681], [0.001, 1000, 14607],
            [0.1, 10000, 57725], [0.01, 10000, 96815], [0.001, 10000, 146076],
            [0.1, 100000, 577254], [0.01, 100000, 968152], [0.001, 100000, 1460769],
            [0.1, 1000000, 5772541], [0.01, 1000000, 9681526], [0.001, 1000000, 14607697],
            [1e-50, 1_000_000_000_000, 14226231280773240832],
        ],
        "src": f"{SBBF}:617-642"},
    "selectivity_only_disables_bloom": {
        # packet: 2 build rows of an Int32 key {1, 10}, build_table_rows = 10, selectivity threshold 1 %
        "build_rows": 2, "build_table_rows": 10, "selectivity_threshold": 1, "keys": [1, 10],
        "expect": {"bloom": False, "inlist": True, "inlist_value_count": 2, "min_max": True, "enabled": True},
        "src": f"{CONVERT}:306-362"},
}

with open(os.path.join(HERE, "runtime_filter.json"), "w") as f:
    json.dump(golden, f, indent=1)
print("wrote runtime_filter.json")
