"""Hash joins on composite keys without a GPU: the reduction to single-key joins
(tests/join_multi_key_ref.py) against a nested loop over all pairs, goldens from the reference's SQL
tests, the C-ABI of the extra key columns and the key packing rule."""
import json
import os
import subprocess

import ctypes as C
import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column
from databend_b200.lib import DbxError
from databend_b200.transforms import join_key_layout
from join_multi_key_ref import composite_ids, golden_result, golden_table, hash_join_multi_key, sort_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = [abi.JOIN_INNER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI, abi.JOIN_LEFT,
         abi.JOIN_RIGHT, abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL]


def brute_force(kind, build_keys, probe_keys):
    """Every (probe, build) pair compared as tuples of Python ints; a NULL component never matches."""
    def tuples(cols):
        vals = [[int(x) for x in c.values()] for c in cols]
        valid = [c.valid_mask() for c in cols]
        return [tuple(v[i] for v in vals) if all(m[i] for m in valid) else None for i in range(cols[0].length)]
    bt, pt = tuples(build_keys), tuples(probe_keys)
    pairs = [(p, b) for p, x in enumerate(pt) for b, y in enumerate(bt) if x is not None and x == y]
    pm, bm = {p for p, _ in pairs}, {b for _, b in pairs}
    un_p = [(p, -1) for p in range(len(pt)) if p not in pm]
    un_b = [(-1, b) for b in range(len(bt)) if b not in bm]
    return {
        abi.JOIN_INNER: pairs, abi.JOIN_LEFT_SEMI: [(p, -1) for p in sorted(pm)], abi.JOIN_LEFT_ANTI: un_p,
        abi.JOIN_LEFT: pairs + un_p, abi.JOIN_RIGHT: pairs + un_b, abi.JOIN_RIGHT_SEMI: [(-1, b) for b in sorted(bm)],
        abi.JOIN_RIGHT_ANTI: un_b, abi.JOIN_FULL: pairs + un_p + un_b,
    }[kind]


def _random_keys(rng, n, dtypes, pool):
    """Key tuples drawn from `pool` (shared by both sides), some with one component perturbed (equal on
    the other columns only), every component nullable."""
    rows = pool[rng.integers(0, len(pool), n)].copy()
    near = rng.random(n) < 0.2
    comp = rng.integers(0, len(dtypes), n)
    rows[near, comp[near]] += 1
    cols = []
    for j, dt in enumerate(dtypes):
        info = np.iinfo({abi.I8: np.int8, abi.I16: np.int16, abi.I32: np.int32, abi.I64: np.int64,
                         abi.U8: np.uint8, abi.U16: np.uint16, abi.U32: np.uint32, abi.U64: np.uint64}[dt])
        v = np.clip(rows[:, j], max(info.min, -2**62), min(info.max, 2**62))
        cols.append(Column.from_data(v.astype(np.dtype(info.dtype)), dt, validity=rng.random(n) > 0.1))
    return cols


LAYOUTS = [
    ([abi.I32, abi.I32], [abi.I32, abi.I32]),
    ([abi.I16, abi.I32, abi.I8], [abi.I16, abi.I32, abi.I8]),
    ([abi.I32, abi.U16], [abi.I64, abi.I32]),
    ([abi.I64, abi.I64], [abi.I64, abi.I64]),
    ([abi.I32, abi.U64], [abi.I32, abi.U64]),
    ([abi.I32] * 4, [abi.I32] * 4),
]


@pytest.mark.parametrize("layout", range(len(LAYOUTS)))
def test_reduction_agrees_with_brute_force(layout):
    bt, pt = LAYOUTS[layout]
    rng = np.random.default_rng(100 + layout)
    pool = rng.integers(-3, 4, (12, len(bt)))
    unsigned = [j for j, (b, p) in enumerate(zip(bt, pt)) if b in (abi.U8, abi.U16, abi.U32, abi.U64) or p in (abi.U8, abi.U16, abi.U32, abi.U64)]
    pool[:, unsigned] = np.abs(pool[:, unsigned])
    build, probe = _random_keys(rng, 90, bt, pool), _random_keys(rng, 140, pt, pool)
    for kind in KINDS:
        pi, bi = hash_join_multi_key(kind, build, probe)
        assert sorted(zip(pi.tolist(), bi.tolist())) == sorted(brute_force(kind, build, probe)), (layout, kind)


def test_ids_compare_by_value_across_widths_and_signedness():
    # Int16 -1 == Int64 -1 (sign extension); UInt16 65535 != Int32 -1 (distinct fields); 2^63 (UInt64)
    # differs from every signed value
    b = [Column.from_data(np.array([-1, 7, -1], np.int16)), Column.from_data(np.array([65535, 1, 5], np.uint16))]
    p = [Column.from_data(np.array([-1, 7, -1], np.int64)), Column.from_data(np.array([-1, 1, 5], np.int32))]
    bid, pid = composite_ids(b, p)
    assert bid.values()[0] != pid.values()[0]
    assert bid.values()[1] == pid.values()[1] and bid.values()[2] == pid.values()[2]
    u = Column.from_data(np.array([2**63, 1], np.uint64))
    s = Column.from_data(np.array([-2**63, 1], np.int64))
    bid, pid = composite_ids([u], [s])
    assert bid.values()[0] != pid.values()[0] and bid.values()[1] == pid.values()[1]
    # any NULL component makes the id NULL
    b = [Column.from_data(np.array([1, 2], np.int32)), Column.from_data(np.array([3, 4], np.int32), validity=[True, False])]
    bid, _ = composite_ids(b, b)
    assert bid.valid_mask().tolist() == [True, False]


def _golden_cases():
    with open(os.path.join(ROOT, "tests", "golden", "join_multi_key.json")) as f:
        return json.load(f)["cases"]


GOLDEN_KINDS = {"inner": abi.JOIN_INNER, "left": abi.JOIN_LEFT, "right": abi.JOIN_RIGHT}


def test_goldens_from_the_reference_sql_tests():
    n = 0
    for case in _golden_cases():
        probe, build = golden_table(case["tables"][case["probe"]]), golden_table(case["tables"][case["build"]])
        pk, bk = [k[0] for k in case["keys"]], [k[1] for k in case["keys"]]
        for q in case["queries"]:
            pi, bi = hash_join_multi_key(GOLDEN_KINDS[q["kind"]], [build[c] for c in bk], [probe[c] for c in pk])

            def row(cols, i):
                return tuple(int(c.values()[i]) if i >= 0 and c.valid_mask()[i] else None for c in cols)
            rows = [(row(probe, x), row(build, y)) for x, y in zip(pi.tolist(), bi.tolist())]
            assert golden_result(q, rows) == sort_rows(q["expected"]), (case["source"], q["sql"])
            n += 1
    assert n == 4


def test_golden_key_layouts():
    """The crdb goldens take the 64-bit key (two Int32), join.test's Int32 + UInt64 the 128-bit one."""
    fields, bits = join_key_layout([abi.I32, abi.I32], [abi.I32, abi.I32])
    assert (fields, bits) == ([(0, 32), (32, 32)], 64)
    fields, bits = join_key_layout([abi.I32, abi.U64], [abi.I32, abi.U64])
    assert (fields, bits) == ([(0, 32), (64, 64)], 128)


def test_packing_rule():
    L = join_key_layout
    assert L([abi.I64], [abi.I64]) == ([(0, 64)], 64)
    assert L([abi.I16, abi.I32, abi.I8], [abi.I16, abi.I32, abi.I8]) == ([(0, 16), (16, 32), (48, 8)], 56)
    # mixed widths: the larger size; signed S with unsigned U: max(S, 2U)
    assert L([abi.I32, abi.U16], [abi.I64, abi.I32]) == ([(0, 64), (64, 32)], 96)
    assert L([abi.U16], [abi.I16]) == ([(0, 32)], 32)
    assert L([abi.U32], [abi.I8]) == ([(0, 64)], 64)
    assert L([abi.U8, abi.U64], [abi.U32, abi.U64]) == ([(0, 32), (64, 64)], 128)
    assert L([abi.I32] * 4, [abi.I32] * 4) == ([(0, 32), (32, 32), (64, 32), (96, 32)], 128)
    # a field never straddles bit 64
    assert L([abi.I32, abi.I8, abi.I32], [abi.I32, abi.I8, abi.I32]) == ([(0, 32), (32, 8), (64, 32)], 96)
    # wider than 128 bits, float keys, signed with UInt64: refused
    assert L([abi.I64, abi.I64, abi.I8], [abi.I64, abi.I64, abi.I8])[1] > 128
    for bt, pt in (([abi.F64], [abi.F64]), ([abi.I32], [abi.U64]), ([abi.BOOL], [abi.BOOL])):
        with pytest.raises(DbxError) as ei:
            L(bt, pt)
        assert ei.value.status == abi.ERR_UNSUPPORTED


def test_abi_pins_the_extra_key_columns(tmp_path):
    with open(os.path.join(ROOT, "include", "dbx.h")) as f:
        header = f.read()
    assert "#define DBX_MAX_JOIN_KEYS 4" in header and abi.MAX_JOIN_KEYS == 4
    fields = ["kind", "build_key_col", "probe_key_col", "n_build_cols", "expected_build_rows", "n_extra_keys",
              "extra_build_key_cols", "extra_probe_key_cols"]
    lines = ["#include <stdio.h>", "#include <stddef.h>", f'#include "{os.path.join(ROOT, "include", "dbx.h")}"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(dbx_join_params));']
    lines += [f'  printf("{f} %zu\\n", offsetof(dbx_join_params, {f}));' for f in fields]
    lines += ['  printf("extra %zu\\n", sizeof(((dbx_join_params*)0)->extra_build_key_cols));', "  return 0;", "}"]
    (tmp_path / "probe.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c11", "-o", str(tmp_path / "probe"), str(tmp_path / "probe.c")])
    out = {k: int(v) for k, v in (l.split() for l in subprocess.check_output([str(tmp_path / "probe")], text=True).splitlines())}
    assert out["size"] == C.sizeof(abi.JoinParams) == 56
    for f in fields:
        assert out[f] == getattr(abi.JoinParams, f).offset, f
    assert out["n_extra_keys"] == 24 and out["extra"] == 12
    # a zeroed tail is the single-key join
    p = abi.JoinParams()
    assert p.n_extra_keys == 0 and list(p.extra_build_key_cols) == [0, 0, 0]
