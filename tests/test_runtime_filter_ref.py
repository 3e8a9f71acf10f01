"""The CPU restatement of the join runtime filters (tests/runtime_filter_ref.py): the reference's own
known answers, no false negatives, the false-positive rate, the threshold edges, and the ABI layout of
the new structs."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

import runtime_filter_ref as rf
from databend_b200 import abi
from databend_b200.block import Column

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
with open(os.path.join(ROOT, "tests", "golden", "runtime_filter.json")) as f:
    GOLDEN = json.load(f)


def test_salt_matches_the_reference():
    assert [int(x) for x in rf.SALT] == GOLDEN["salt"]["values"]


@pytest.mark.parametrize("case", GOLDEN["optimal_num_of_bytes"]["cases"])
def test_optimal_num_of_bytes(case):
    assert rf.optimal_num_of_bytes(case[0]) == case[1]


@pytest.mark.parametrize("case", GOLDEN["num_of_bits_from_ndv_fpp"]["cases"])
def test_num_of_bits_from_ndv_fpp(case):
    fpp, ndv, bits = case
    assert rf.num_of_bits_from_ndv_fpp(ndv, fpp) == bits


def test_selectivity_rule_disables_only_the_bloom():
    g = GOLDEN["selectivity_only_disables_bloom"]
    col = Column.from_data(np.array(g["keys"], dtype=np.int32))
    (part,) = rf.build([col], [abi.I32], build_table_rows=g["build_table_rows"], selectivity_threshold=g["selectivity_threshold"])
    e = g["expect"]
    assert (part["bloom"] is not None) == e["bloom"]
    assert (part["inlist"] is not None) == e["inlist"] and len(part["inlist"]) == e["inlist_value_count"]
    assert part["has_min_max"] == e["min_max"] and (part["min"], part["max"]) == (1, 10)


def _random_build(n, seed=7):
    rng = np.random.default_rng(seed)
    return rng.choice(np.arange(10 * n, dtype=np.int64), size=n, replace=False), rng


def test_bloom_has_no_false_negatives_and_about_one_percent_false_positives():
    keys, rng = _random_build(100_000)
    (part,) = rf.build([Column.from_data(keys)], [abi.I64], build_table_rows=10**8)
    assert part["bloom"] is not None and part["bloom"].nbytes == rf.bloom_bytes(100_000)
    assert rf.apply([part], [Column.from_data(keys)]).all()
    probe = rng.integers(10**7, 2 * 10**7, size=1_000_000, dtype=np.int64)  # outside the build keys
    only_bloom = dict(part, has_min_max=False, inlist=None)
    fpr = rf.apply([only_bloom], [Column.from_data(probe)]).mean()
    assert 0 < fpr <= 0.015, fpr


def test_fmix64_and_block_index_by_hand():
    h = int(rf.fmix64(np.array([1], dtype=np.uint64))[0])
    x = 1
    for m in (0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53):
        x ^= x >> 33
        x = (x * m) % 2**64
    x ^= x >> 33
    assert h == x
    assert int(rf.block_index(np.array([h], dtype=np.uint64), 1000)[0]) == ((h >> 32) * 1000) >> 32


@pytest.mark.parametrize("rows,inlist", [(1024, True), (1025, False)])
def test_inlist_threshold_edge(rows, inlist):
    (part,) = rf.build([Column.from_data(np.arange(rows, dtype=np.int64) % 700)], [abi.I64])
    assert (part["inlist"] is not None) == inlist
    if inlist:
        assert len(part["inlist"]) == 700  # de-duplicated


@pytest.mark.parametrize("rows,bloom", [(3_000_000, True), (3_000_001, False)])
def test_bloom_threshold_edge(rows, bloom):
    assert (rows <= rf.DEFAULTS["bloom_threshold"] and rf.should_enable_bloom(rows, 10**9, 10)) == bloom


def test_selectivity_of_exactly_ten_percent_means_no_bloom():
    assert not rf.should_enable_bloom(10, 100, 10)
    assert rf.should_enable_bloom(9, 100, 10)
    assert not rf.should_enable_bloom(10, 0, 10)  # build_table_rows unknown


def test_empty_build_side_has_no_filters():
    (part,) = rf.build([Column.from_data(np.zeros(0, dtype=np.int64))], [abi.I64], build_table_rows=100)
    assert part["inlist"] is None and part["bloom"] is None and not part["has_min_max"]


def test_null_build_keys_are_left_out_and_null_probe_keys_rejected():
    b = Column.from_data(np.array([5, 1000, 7], dtype=np.int32), validity=[True, False, True])
    (part,) = rf.build([b], [abi.I64], build_table_rows=100)
    assert (part["min"], part["max"]) == (5, 7) and list(part["inlist"]) == [5, 7]
    p = Column.from_data(np.array([5, 7, 1000, 5], dtype=np.int64), validity=[True, True, True, False])
    assert list(rf.apply([part], [p])) == [True, True, False, False]


def test_common_type_of_mixed_pairs():
    assert rf.common_type(abi.U8, abi.I8)[:2] == (abi.I16, True)
    assert rf.common_type(abi.I32, abi.I64)[:2] == (abi.I64, True)
    assert rf.common_type(abi.U16, abi.U32)[:2] == (abi.U32, False)
    # UInt8 200 and Int8 -56 differ by value although their low bytes agree
    b = Column.from_data(np.array([200], dtype=np.uint8))
    (part,) = rf.build([b], [abi.I8], build_table_rows=100)
    p = Column.from_data(np.array([-56, 100], dtype=np.int8))
    assert list(rf.apply([part], [p])) == [False, False]


def test_runtime_filter_structs_match_the_header(tmp_path):
    structs = {
        "dbx_runtime_filter_params": (abi.RuntimeFilterParams, [f for f, _ in abi.RuntimeFilterParams._fields_]),
        "dbx_rf_part_info": (abi.RfPartInfo, [f for f, _ in abi.RfPartInfo._fields_]),
        "dbx_rf_info": (abi.RfInfo, [f for f, _ in abi.RfInfo._fields_]),
    }
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "dbx.h")}"', "int main(void) {"]
    for cname, (_, fields) in structs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fld in fields:
            lines.append(f'  printf("{cname}.{fld} %zu\\n", offsetof({cname}, {fld}));')
    lines.append('  printf("DBX_RF_MAX_INLIST %d\\n", DBX_RF_MAX_INLIST);')
    lines += ["  return 0;", "}"]
    src = tmp_path / "probe.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-std=c11", "-o", str(exe), str(src)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, (ctype, fields) in structs.items():
        assert int(out[cname]) == C.sizeof(ctype), cname
        for fld in fields:
            assert int(out[f"{cname}.{fld}"]) == getattr(ctype, fld).offset, f"{cname}.{fld}"
    assert int(out["DBX_RF_MAX_INLIST"]) == abi.RF_MAX_INLIST
