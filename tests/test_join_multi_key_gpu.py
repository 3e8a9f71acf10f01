"""Hash joins on composite keys on the device against the reduction to single-key joins
(tests/join_multi_key_ref.py), for every join kind and the key layouts of both table-key widths:
64-bit packed keys (the single-key entry) and 128-bit ones ({k0, k1, row1, p0} entries).  Results
are compared as multisets of (value, validity) rows."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError, check, load
from databend_b200.transforms import HashJoin, _Op, join_key_layout, schema_types, to_device
from join_multi_key_ref import golden_result, golden_table, hash_join_multi_key, sort_rows

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

KINDS = {"inner": abi.JOIN_INNER, "left_semi": abi.JOIN_LEFT_SEMI, "left_anti": abi.JOIN_LEFT_ANTI, "left": abi.JOIN_LEFT,
         "right": abi.JOIN_RIGHT, "right_semi": abi.JOIN_RIGHT_SEMI, "right_anti": abi.JOIN_RIGHT_ANTI, "full": abi.JOIN_FULL}
PROBE_ONLY, BUILD_ONLY = ("left_semi", "left_anti"), ("right_semi", "right_anti")
NP = {abi.I8: np.int8, abi.I16: np.int16, abi.I32: np.int32, abi.I64: np.int64,
      abi.U8: np.uint8, abi.U16: np.uint16, abi.U32: np.uint32, abi.U64: np.uint64}
# (build key dtypes, probe key dtypes)
LAYOUTS = {
    "2xI32": ([abi.I32, abi.I32], [abi.I32, abi.I32]),
    "I16+I32+I8": ([abi.I16, abi.I32, abi.I8], [abi.I16, abi.I32, abi.I8]),
    "mixed": ([abi.I32, abi.U16], [abi.I64, abi.I32]),
    "2xI64": ([abi.I64, abi.I64], [abi.I64, abi.I64]),
    "I32+U64": ([abi.I32, abi.U64], [abi.I32, abi.U64]),
    "4xI32": ([abi.I32] * 4, [abi.I32] * 4),
}


def rows_sorted(cols):
    """[(values, validity)] per column -> lexicographically sorted 2-D array of (value, validity) pairs"""
    arr = []
    for v, m in cols:
        v = v.astype(np.float64) if v.dtype.kind == "f" else v.view(np.int64) if v.dtype == np.uint64 else v.astype(np.int64)
        arr += [np.where(m, v, 0), m.astype(np.int64)]
    a = np.stack(arr, axis=1)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def take(col, idx):
    v, m = col.values(), col.valid_mask()
    if len(v) == 0:
        return np.zeros(len(idx), dtype=v.dtype), np.zeros(len(idx), dtype=bool)
    return v[np.maximum(idx, 0)], m[np.maximum(idx, 0)] & (idx >= 0)


def key_values(rng, pool, rows, dt):
    info = np.iinfo(NP[dt])
    return np.clip(pool[rows], max(int(info.min), -2**62), min(int(info.max), 2**62)).astype(NP[dt])


def tables(layout, seed, nb=6000, npr=20_000, unique=False, nullable=True):
    """Build side: the key columns interleaved with three payload columns (more than the entries
    inline, so some are gathered by build row), duplicate tuples unless `unique`.  Probe side: key
    tuples from the build side, near misses (one component changed), negative values and misses."""
    bt, pt = LAYOUTS[layout]
    rng = np.random.default_rng(seed)
    nk = len(bt)
    unsigned = [j for j in range(nk) if bt[j] not in (abi.I8, abi.I16, abi.I32, abi.I64) or pt[j] not in (abi.I8, abi.I16, abi.I32, abi.I64)]
    small = any(NP[t] in (np.int8, np.int16) for t in bt)
    lo, hi = (-60, 60) if small else (-4000, 4000)
    pool = rng.integers(lo, hi, (nb if unique else nb // 3, nk))
    pool[:, unsigned] = np.abs(pool[:, unsigned])
    if unique:
        pool = np.unique(pool, axis=0)
        nb = len(pool)
        b_rows = rng.permutation(nb)
    else:
        b_rows = rng.integers(0, len(pool), nb)
    p_rows = rng.integers(0, len(pool), npr)
    bkeys = [key_values(rng, pool[:, j], b_rows, bt[j]) for j in range(nk)]
    pkeys = [key_values(rng, pool[:, j], p_rows, pt[j]) for j in range(nk)]
    near = rng.random(npr) < 0.15
    comp = rng.integers(0, nk, npr)
    for j in range(nk):
        sel = near & (comp == j)
        pkeys[j][sel] = (pkeys[j][sel].astype(np.int64) + 1).astype(NP[pt[j]])
    def valid(n):
        return (rng.random(n) > 0.05) if nullable else None
    payload = [Column.from_data(rng.integers(-2**40, 2**40, nb).astype(np.int64), validity=valid(nb)),
               Column.from_data(rng.normal(size=nb).astype(np.float32)),
               Column.from_data(rng.integers(-100, 100, nb).astype(np.int8), validity=valid(nb))]
    bcols, bk = [], []
    for j in range(nk):
        if j < len(payload):
            bcols.append(payload[j])
        bk.append(len(bcols))
        bcols.append(Column.from_data(bkeys[j], bt[j], validity=valid(nb)))
    bcols += payload[nk:]
    pcols = [Column.from_data(pkeys[j], pt[j], validity=valid(npr)) for j in range(nk)]
    pcols.append(Column.from_data(np.arange(npr, dtype=np.int64)))
    return DataBlock(bcols, nb), DataBlock(pcols, npr), bk, list(range(nk))


def expected(kind, build, probe, bk, pk):
    pi, bi = hash_join_multi_key(KINDS[kind], [build.columns[c] for c in bk], [probe.columns[c] for c in pk])
    cols = [] if kind in BUILD_ONLY else [take(c, pi) for c in probe.columns]
    if kind not in PROBE_ONLY:
        cols += [take(c, bi) for c in build.columns]
    return cols, len(pi)


def got_columns(blocks, n_cols):
    return [(np.concatenate([b.columns[i].values() for b in blocks]), np.concatenate([b.columns[i].valid_mask() for b in blocks]))
            for i in range(n_cols)]


def is_nullable(col):
    return col.validity is not None or (col.is_const and col.const_value is None)


def check_nullability(kind, build, probe, probe_blocks, final_blocks):
    """As for single keys (dbx.h): LEFT makes the build columns Nullable, RIGHT the probe columns,
    FULL both; the other columns keep their type's nullability."""
    bn = [is_nullable(c) for c in build.columns]
    pn = [is_nullable(c) for c in probe.columns]
    if kind in PROBE_ONLY:
        want = pn
    elif kind in BUILD_ONLY:
        want = bn
    else:
        want = [n or kind in ("right", "full") for n in pn] + [n or kind in ("left", "full") for n in bn]
    for blk in probe_blocks:
        assert [is_nullable(c) for c in blk.columns] == want, kind
    for blk in final_blocks:
        if kind in BUILD_ONLY:
            assert [is_nullable(c) for c in blk.columns] == want, kind
        else:
            assert all(c.is_const and c.const_value is None for c in blk.columns[:len(pn)])
            assert [is_nullable(c) for c in blk.columns[len(pn):]] == want[len(pn):], kind


def run(kind, build, probe, bk, pk, build_split=None, probe_split=None, device_resident=False):
    j = HashJoin(schema_types(build), schema_types(probe), bk, pk, kind=KINDS[kind])
    for b in (build.split_by_rows(build_split) if build_split else [build]):
        j.add_block(b)
    j.final_build()
    probe_blocks = []
    for p in (probe.split_by_rows(probe_split) if probe_split else [probe]):
        if device_resident:
            p = DataBlock([to_device(c) for c in p.columns], p.num_rows)
        probe_blocks.extend(j.probe_block(p))
    final_blocks = j.final_probe()
    j.close()
    return probe_blocks, final_blocks


def run_and_compare(kind, build, probe, bk, pk, **kw):
    probe_blocks, final_blocks = run(kind, build, probe, bk, pk, **kw)
    check_nullability(kind, build, probe, probe_blocks, final_blocks)
    exp, n = expected(kind, build, probe, bk, pk)
    outs = probe_blocks + final_blocks
    assert sum(o.num_rows for o in outs) == n, kind
    if n:
        np.testing.assert_array_equal(rows_sorted(got_columns(outs, len(exp))), rows_sorted(exp), err_msg=kind)
    return probe_blocks, final_blocks


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_layouts_every_kind(gpu, layout, kind, monkeypatch):
    """Nullable components on both sides, duplicate build tuples, near misses, negative values;
    multi-block build and probe sides, device-resident probe blocks, and a unique build side (the
    early-stop probe); the build key columns of the output are decoded from the table entries."""
    build, probe, bk, pk = tables(layout, 11)
    run_and_compare(kind, build, probe, bk, pk)
    run_and_compare(kind, build, probe, bk, pk, build_split=1700, probe_split=4500)
    run_and_compare(kind, build, probe, bk, pk, probe_split=7000, device_resident=True)
    ub, up, bk, pk = tables(layout, 12, nb=5000, npr=30_000, unique=True)
    run_and_compare(kind, ub, up, bk, pk, probe_split=9000)
    run_and_compare(kind, ub, up, bk, pk, device_resident=True)
    monkeypatch.setenv("DBX_JOIN_NO_UNIQUE", "1")
    run_and_compare(kind, build, probe, bk, pk, probe_split=7000)
    run_and_compare(kind, ub, up, bk, pk)


def test_sign_extension_and_distinct_fields(gpu):
    """Build Int16 -1 matches probe Int64 -1; build UInt16 65535 does not match probe Int32 -1."""
    build = DataBlock([Column.from_data(np.array([-1, -1, 5, -32768], np.int16)), Column.from_data(np.array([65535, 7, 65535, 0], np.uint16)),
                       Column.from_data(np.array([10, 20, 30, 40], np.int64))])
    probe = DataBlock([Column.from_data(np.array([-1, -1, 5, 5, -32768, 65535 - 65536], np.int64)),
                       Column.from_data(np.array([-1, 7, 65535, -1, 0, 7], np.int32))])
    j = HashJoin(schema_types(build), schema_types(probe), [0, 1], [0, 1])
    j.add_block(build)
    j.final_build()
    (out,) = j.probe_block(probe)
    got = sorted(zip(out.columns[0].values().tolist(), out.columns[1].values().tolist(), out.columns[2].values().tolist(),
                     out.columns[3].values().tolist(), out.columns[4].values().tolist()))
    # probe (-1, 7) meets build (-1, 7); (5, 65535) meets (5, 65535); (-32768, 0) meets (-32768, 0);
    # (-1, -1) and (5, -1) meet nothing (65535 as UInt16 is not -1 as Int32)
    assert got == [(-32768, 0, -32768, 0, 40), (-1, 7, -1, 7, 20), (-1, 7, -1, 7, 20), (5, 65535, 5, 65535, 30)]
    j.close()


def _create(build_types, probe_types, bk, pk, n_extra=None):
    p = abi.JoinParams()
    p.kind, p.build_key_col, p.probe_key_col, p.n_build_cols = abi.JOIN_INNER, bk[0], pk[0], len(build_types)
    p.n_extra_keys = len(bk) - 1 if n_extra is None else n_extra
    for i in range(1, min(len(bk), abi.MAX_JOIN_KEYS)):
        p.extra_build_key_cols[i - 1], p.extra_probe_key_cols[i - 1] = bk[i], pk[i]
    return _Op(abi.OP_JOIN, p, list(build_types) + list(probe_types), 0)


def test_refusals(gpu):
    I32, I64 = abi.I32, abi.I64
    cases = [
        ([I32] * 5, [I32] * 5, [0, 1, 2, 3], [0, 1, 2, 3], 4, abi.ERR_INVALID, "n_extra_keys"),
        ([I32] * 2, [I32] * 2, [0, 1], [0, 1], -1, abi.ERR_INVALID, "n_extra_keys"),
        ([I32] * 2, [I32] * 2, [0, 2], [0, 1], None, abi.ERR_INVALID, "outside the schema"),
        ([I32] * 2, [I32] * 2, [0, 1], [0, 5], None, abi.ERR_INVALID, "outside the schema"),
        ([I32, abi.F64], [I32, abi.F64], [0, 1], [0, 1], None, abi.ERR_UNSUPPORTED, "integer"),
        ([I32, abi.BOOL], [I32, abi.BOOL], [0, 1], [0, 1], None, abi.ERR_UNSUPPORTED, "integer"),
        ([I32, I32], [I32, abi.U64], [0, 1], [0, 1], None, abi.ERR_UNSUPPORTED, "UInt64"),
        ([I64, I64, abi.I8], [I64, I64, abi.I8], [0, 1, 2], [0, 1, 2], None, abi.ERR_UNSUPPORTED, "256-bit"),
    ]
    for bt, pt, bk, pk, n_extra, status, msg in cases:
        with pytest.raises(DbxError) as ei:
            _create(bt, pt, bk, pk, n_extra)
        assert ei.value.status == status, (bt, pt, bk, pk)
        assert msg in str(ei.value), str(ei.value)
    # the Python side refuses unequal or too long key lists before the library sees them
    for bk, pk in (([0, 1], [0]), ([0, 1, 2, 3, 4], [0, 1, 2, 3, 4])):
        with pytest.raises(DbxError) as ei:
            HashJoin([I32] * 5, [I32] * 5, bk, pk)
        assert ei.value.status == abi.ERR_INVALID
    # exactly 128 bits is accepted
    assert join_key_layout([I32] * 4, [I32] * 4)[1] == 128
    _create([I32] * 4, [I32] * 4, [0, 1, 2, 3], [0, 1, 2, 3]).close()


@pytest.mark.parametrize("layout", ["2xI32", "2xI64"])
def test_larger_unique_build_side_over_a_split_probe(gpu, layout):
    """The packed kernels at 60 000 x 200 000 rows with the probe side in 70 000-row blocks."""
    build, probe, bk, pk = tables(layout, 31, nb=60_000, npr=200_000, unique=True)
    for kind in ("inner", "left", "right", "full"):
        run_and_compare(kind, build, probe, bk, pk, probe_split=70_000)


def test_goldens_on_the_device(gpu):
    with open(os.path.join(ROOT, "tests", "golden", "join_multi_key.json")) as f:
        cases = json.load(f)["cases"]
    for case in cases:
        probe = golden_table(case["tables"][case["probe"]])
        build = golden_table(case["tables"][case["build"]])
        pk, bk = [k[0] for k in case["keys"]], [k[1] for k in case["keys"]]
        pb, bb = DataBlock(probe, probe[0].length), DataBlock(build, build[0].length)
        for q in case["queries"]:
            j = HashJoin(schema_types(bb), schema_types(pb), bk, pk, kind=KINDS[q["kind"]])
            j.add_block(bb)
            j.final_build()
            outs = j.probe_block(pb) + j.final_probe()
            j.close()
            rows = []
            for o in outs:
                vals = [(c.values(), c.valid_mask()) for c in o.columns]
                for i in range(o.num_rows):
                    t = tuple(int(v[i]) if m[i] else None for v, m in vals)
                    rows.append((t[:len(probe)], t[len(probe):]))
            assert golden_result(q, rows) == sort_rows(q["expected"]), (case["source"], q["sql"])


def test_device_pull_nullability(gpu):
    build = DataBlock([Column.from_data(np.arange(10, dtype=np.int32)), Column.from_data(np.arange(10, dtype=np.int64) * 3),
                       Column.from_data(np.arange(10, dtype=np.int64) + 100)])
    probe = DataBlock([Column.from_data(np.array([1, 2, 3, 42], np.int32)), Column.from_data(np.array([3, 6, 10, 0], np.int64))])
    L = load()
    for kind in KINDS:
        j = HashJoin(schema_types(build), schema_types(probe), [0, 1], [0, 1], kind=KINDS[kind])
        j.add_block(build)
        j.final_build()
        outs = j.probe_block(probe, abi.MEM_DEVICE) + j.final_probe(abi.MEM_DEVICE)
        n = 0
        for b in outs:
            n += b.num_rows
            cols = [b.cols[i] for i in range(b.num_cols)]
            assert all(c.mem == abi.MEM_DEVICE for c in cols if not c.is_const)
            if kind in ("left", "full") and b.num_cols == 5 and not cols[0].is_const:
                assert all(c.validity for c in cols[2:])
            if kind == "inner":
                assert not any(c.validity for c in cols)
                got = np.empty(b.num_rows, dtype=np.int64)
                check(L.dbx_memcpy_d2h(0, got.ctypes.data, cols[3].data, got.nbytes))  # build key decoded from the entry
                assert sorted(got.tolist()) == [3, 6]
            check(L.dbx_block_release(C.byref(b)))
        # matches: (1, 3) and (2, 6); (3, 10) is a near miss
        assert n == {"inner": 2, "left_semi": 2, "left_anti": 2, "left": 4, "right": 10, "right_semi": 2, "right_anti": 8, "full": 12}[kind], kind
        j.close()


def test_lifecycle_and_empty_sides(gpu):
    build, probe, bk, pk = tables("2xI64", 41, nb=2000, npr=5000)
    for kind in KINDS:
        j = HashJoin(schema_types(build), schema_types(probe), bk, pk, kind=KINDS[kind])
        results = []
        for _ in range(2):
            j.reset()
            j.add_block(build)
            j.final_build()
            outs = []
            for p in probe.split_by_rows(1500):
                outs.extend(j.probe_block(p))
            outs.extend(j.final_probe())
            assert j.final_probe() == []  # a second call queues nothing
            exp, n = expected(kind, build, probe, bk, pk)
            results.append(rows_sorted(got_columns(outs, len(exp))))
        np.testing.assert_array_equal(results[0], rows_sorted(exp))
        np.testing.assert_array_equal(results[1], results[0])
        j.close()
        # empty build side, empty probe side
        run_and_compare(kind, build.slice(0, 0), probe, bk, pk)
        run_and_compare(kind, build, probe.slice(0, 0), bk, pk)


@pytest.mark.parametrize("layout", ["2xI32", "2xI64"])
def test_ten_million_probe_rows(gpu, layout):
    """1e7 probe rows into 2^20 unique build tuples (the config-3 shape at a tenth of the dims)."""
    rng = np.random.default_rng(53)
    nb, npr = 1 << 20, 10_000_000
    k = rng.permutation(nb).astype(np.int64) * 5 - 2_000_000
    if layout == "2xI32":
        parts = [(k & 0xFFFF).astype(np.int32), (k >> 16).astype(np.int32)]
    else:
        parts = [k, -k * 3]
    pick = rng.integers(0, nb, npr)
    pparts = [p[pick].copy() for p in parts]
    pparts[1][::97] += 1  # near misses
    build = DataBlock([Column.from_data(p) for p in parts] + [Column.from_data(rng.integers(0, 2**40, nb).astype(np.int64))], nb)
    probe = DataBlock([Column.from_data(p) for p in pparts] + [Column.from_data(rng.integers(0, 2**31, npr).astype(np.int32))], npr)
    run_and_compare("inner", build, probe, [0, 1], [0, 1], probe_split=4_000_000)
