"""Build-side ("right") hash joins on the device against their CPU restatement: RIGHT, RIGHT SEMI,
RIGHT ANTI and FULL (right_join.rs, right_join_semi.rs, right_join_anti.rs,
hash_join_probe_state.rs:455-567).  Probe blocks mark the build rows they match, final_probe emits
the build rows each kind keeps; results are compared as multisets of (value, validity) rows."""
import ctypes as C

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError, check, load
from databend_b200.transforms import HashJoin, schema_types, to_device
from join_build_side_ref import hash_join_build_side

pytestmark = pytest.mark.gpu

KINDS = {"right": abi.JOIN_RIGHT, "right_semi": abi.JOIN_RIGHT_SEMI, "right_anti": abi.JOIN_RIGHT_ANTI, "full": abi.JOIN_FULL}
BUILD_ONLY = ("right_semi", "right_anti")


def oracle():
    from oracle import oracle as orc
    return orc


def rows_sorted(vals_valid):
    """[(values, validity)] per column -> lexicographically sorted 2-D array of (value, validity) pairs"""
    arr = []
    for v, m in vals_valid:
        v = v.astype(np.float64) if v.dtype.kind == "f" else v.view(np.int64) if v.dtype == np.uint64 else v.astype(np.int64)
        arr.append(np.where(m, v, 0))
        arr.append(m.astype(np.int64))
    a = np.stack(arr, axis=1)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def take(col, idx):
    """(values, validity) of col at idx; -1 = the row carries NULL on this side"""
    v, m = col.values(), col.valid_mask()
    if len(v) == 0:
        return np.zeros(len(idx), dtype=v.dtype), np.zeros(len(idx), dtype=bool)
    return v[np.maximum(idx, 0)], m[np.maximum(idx, 0)] & (idx >= 0)


def expected(kind, build, probe, bk, pk):
    pi, bi = hash_join_build_side(KINDS[kind], build.columns[bk], probe.columns[pk])
    cols = [] if kind in BUILD_ONLY else [take(c, pi) for c in probe.columns]
    cols += [take(c, bi) for c in build.columns]
    return cols, len(pi)


def got_columns(blocks, n_cols):
    return [(np.concatenate([b.columns[i].values() for b in blocks]), np.concatenate([b.columns[i].valid_mask() for b in blocks]))
            for i in range(n_cols)]


def is_nullable(col):
    return col.validity is not None or (col.is_const and col.const_value is None)


def check_nullability(kind, build, probe, probe_blocks, final_blocks):
    """Output nullability as in dbx.h: RIGHT probe columns Nullable everywhere, FULL every column
    Nullable, build columns otherwise as typed; the final blocks' probe side is Const NULL."""
    nb, npc = build.num_columns(), probe.num_columns()
    build_nul = [is_nullable(c) for c in build.columns]
    if kind in BUILD_ONLY:
        assert probe_blocks == []
        for blk in final_blocks:
            assert blk.num_columns() == nb
            assert [is_nullable(c) for c in blk.columns] == build_nul
        return
    for blk in probe_blocks + final_blocks:
        assert blk.num_columns() == npc + nb
        assert all(is_nullable(c) for c in blk.columns[:npc])
        want_build = [True] * nb if kind == "full" else build_nul
        assert [is_nullable(c) for c in blk.columns[npc:]] == want_build
    for blk in final_blocks:
        assert all(c.is_const and c.const_value is None for c in blk.columns[:npc])
    assert all(not c.is_const for blk in probe_blocks for c in blk.columns)


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
    assert sum(o.num_rows for o in outs) == n
    if n:
        np.testing.assert_array_equal(rows_sorted(got_columns(outs, len(exp))), rows_sorted(exp))
    return probe_blocks, final_blocks


def random_tables(seed, nb=6000, npr=20_000, key_range=3000):
    """Nullable keys on both sides, duplicate build keys, misses on both sides."""
    rng = np.random.default_rng(seed)
    build = DataBlock([Column.from_data(rng.integers(0, key_range, nb).astype(np.int64), validity=rng.random(nb) > 0.08),
                       Column.from_data(rng.integers(-99, 99, nb).astype(np.int32)),
                       Column.from_data(rng.normal(size=nb), validity=rng.random(nb) > 0.3)])
    probe = DataBlock([Column.from_data(rng.integers(-200, key_range + 800, npr).astype(np.int64), validity=rng.random(npr) > 0.1),
                       Column.from_data(np.arange(npr, dtype=np.int64))])
    return build, probe


@pytest.mark.parametrize("kind", list(KINDS))
def test_random_nullable_duplicates_and_misses(gpu, kind, monkeypatch):
    build, probe = random_tables(5)
    run_and_compare(kind, build, probe, 0, 0)
    # build side in several blocks, probe side in several blocks: matches accumulate across blocks
    run_and_compare(kind, build, probe, 0, 0, build_split=1700, probe_split=4500)
    run_and_compare(kind, build, probe, 0, 0, probe_split=7000, device_resident=True)
    monkeypatch.setenv("DBX_JOIN_NO_UNIQUE", "1")
    run_and_compare(kind, build, probe, 0, 0, probe_split=7000)


@pytest.mark.parametrize("kind", list(KINDS))
def test_unique_and_duplicate_build_sides_over_split_probes(gpu, kind):
    """Unique build keys (the early-stop probe) at 60 000 x 200 000 rows, over a probe split into
    blocks and over a device-resident probe block; then a build side of the same size with
    duplicate and NULL keys."""
    rng = np.random.default_rng(19)
    nb, npr = 60_000, 200_000
    dk = rng.permutation(nb).astype(np.int64) * 7 - 1000
    build = DataBlock([Column.from_data(dk), Column.from_data(rng.integers(-9, 9, nb).astype(np.int64))])
    probe = DataBlock([Column.from_data(np.concatenate([dk[rng.integers(0, nb * 8 // 10, npr - 5000)], rng.integers(10**9, 2 * 10**9, 5000)])),
                       Column.from_data(rng.integers(0, 2**31, npr).astype(np.int32))])
    run_and_compare(kind, build, probe, 0, 0, probe_split=70_000)
    run_and_compare(kind, build, probe, 0, 0, device_resident=True)
    dup, p2 = random_tables(29, nb=60_000, npr=100_000, key_range=40_000)
    run_and_compare(kind, dup, p2, 0, 0, probe_split=60_000)


@pytest.mark.parametrize("kind", list(KINDS))
def test_wide_build_side_inline_and_gathered_columns(gpu, kind):
    """Key in the middle of five build columns: final blocks gather the two columns the table
    entries carry inline and the remaining ones alike (nullable and narrow ones included)."""
    rng = np.random.default_rng(23)
    nb, npr = 7000, 9000
    build = DataBlock([Column.from_data(rng.normal(size=nb).astype(np.float32), validity=rng.random(nb) > 0.2),
                       Column.from_data(rng.integers(-2**62, 2**62, nb).astype(np.int64)),
                       Column.from_data(rng.integers(0, 3000, nb).astype(np.uint32), validity=rng.random(nb) > 0.05),   # key
                       Column.from_data(rng.integers(0, 60000, nb).astype(np.uint16), validity=rng.random(nb) > 0.5),
                       Column.from_data(rng.integers(-100, 100, nb).astype(np.int8)),
                       Column.from_data(rng.normal(size=nb))])
    probe = DataBlock([Column.from_data(rng.integers(0, 3500, npr).astype(np.int64)),
                       Column.from_data(rng.integers(0, 100, npr).astype(np.int8))])
    run_and_compare(kind, build, probe, 2, 0, build_split=1500, probe_split=2500)


def test_null_key_build_rows(gpu):
    """A NULL-key build row is never inserted, so never matched: RIGHT, RIGHT ANTI and FULL emit
    it from final_probe, RIGHT SEMI never does (even when a probe row has the same raw value)."""
    build = DataBlock([Column.from_data(np.array([5, 7, 5, 9, 11], dtype=np.int64), validity=[True, True, True, True, False]),
                       Column.from_data(np.array([50, 70, 51, 90, 110], dtype=np.int64))])
    probe = DataBlock([Column.from_data(np.array([5, 6, 9, 5, 11, 7], dtype=np.int64), validity=[True, True, True, False, True, True]),
                       Column.from_data(np.array([1.5, 2.5, 3.5, 4.5, 5.5, 6.5]))])
    for kind in KINDS:
        _, final = run_and_compare(kind, build, probe, 0, 0)
        tags = sorted(np.concatenate([b.columns[-1].values() for b in final]).tolist()) if final else []
        assert (110 in tags) == (kind != "right_semi"), kind
    _, final = run("right_semi", build, probe, 0, 0)
    assert sorted(final[0].columns[1].values().tolist()) == [50, 51, 70, 90]  # duplicate key 5: both rows, each once


def test_device_pull_nullability_and_const_null_probe_side(gpu):
    build = DataBlock([Column.from_data(np.arange(10, dtype=np.int64)), Column.from_data(np.arange(10, dtype=np.int32))])
    probe = DataBlock([Column.from_data(np.array([1, 2, 3, 42], dtype=np.int64)), Column.from_data(np.arange(4, dtype=np.float64))])
    L = load()
    for kind in KINDS:
        j = HashJoin(schema_types(build), schema_types(probe), 0, 0, kind=KINDS[kind])
        j.add_block(build)
        j.final_build()
        probe_out = j.probe_block(probe, abi.MEM_DEVICE)
        final_out = j.final_probe(abi.MEM_DEVICE)
        assert len(final_out) == 1
        for b in probe_out + final_out:
            assert all(b.cols[i].mem == abi.MEM_DEVICE for i in range(b.num_cols) if not b.cols[i].is_const)
        if kind in BUILD_ONLY:
            assert probe_out == []
            (f,) = final_out
            assert f.num_cols == 2 and f.num_rows == (3 if kind == "right_semi" else 7)
            assert not f.cols[0].validity and not f.cols[1].validity
        else:
            for b in probe_out:
                assert b.num_cols == 4 and not b.cols[0].is_const
                assert b.cols[0].validity and b.cols[1].validity  # probe side Nullable in every block
                assert bool(b.cols[2].validity) == (kind == "full")
            (f,) = final_out
            assert f.num_rows == 7
            for i in (0, 1):
                assert f.cols[i].is_const == 1 and f.cols[i].konst.is_null == 1 and f.cols[i].len == 7
            for i in (2, 3):
                assert not f.cols[i].is_const and bool(f.cols[i].validity) == (kind == "full")
            got = np.empty(7, dtype=np.int64)
            check(L.dbx_memcpy_d2h(0, got.ctypes.data, f.cols[2].data, 56))
            assert sorted(got.tolist()) == [0, 4, 5, 6, 7, 8, 9]
        for b in probe_out + final_out:
            check(L.dbx_block_release(C.byref(b)))
        j.close()


def test_lifecycle(gpu):
    build, probe = random_tables(7, nb=2000, npr=5000)
    # final_probe on the probe-side kinds yields nothing
    for k in (abi.JOIN_INNER, abi.JOIN_LEFT, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI):
        j = HashJoin(schema_types(build), schema_types(probe), 0, 0, kind=k)
        j.add_block(build)
        j.final_build()
        assert j.probe_block(probe) or k == abi.JOIN_LEFT_ANTI
        assert j.final_probe() == []
        j.close()
    for kind in KINDS:
        j = HashJoin(schema_types(build), schema_types(probe), 0, 0, kind=KINDS[kind])
        with pytest.raises(DbxError) as ei:  # before final_build
            j.final_probe()
        assert ei.value.status == abi.ERR_STATE
        j.add_block(build)
        j.final_build()
        # final_probe with no probe block: every build row (RIGHT, ANTI, FULL) or none (SEMI)
        first = j.final_probe()
        assert sum(b.num_rows for b in first) == (0 if kind == "right_semi" else build.num_rows)
        with pytest.raises(DbxError) as ei:  # probe after final_probe
            j.probe_block(probe)
        assert ei.value.status == abi.ERR_STATE
        assert j.final_probe() == []  # a second call queues nothing
        # reset, then the same query: the same result, so the matched map was cleared
        results = []
        for _ in range(2):
            j.reset()
            j.add_block(build)
            j.final_build()
            outs = []
            for p in probe.split_by_rows(1500):
                outs.extend(j.probe_block(p))
            outs.extend(j.final_probe())
            n_cols = build.num_columns() + (0 if kind in BUILD_ONLY else probe.num_columns())
            results.append(rows_sorted(got_columns(outs, n_cols)))
        exp, n = expected(kind, build, probe, 0, 0)
        np.testing.assert_array_equal(results[0], rows_sorted(exp))
        np.testing.assert_array_equal(results[1], results[0])
        j.close()


def test_empty_sides(gpu):
    """join.test:7-25 and 89-102: an empty build side gives nothing for RIGHT / SEMI / ANTI and every
    probe row with a NULL build side for FULL; an empty probe side leaves final_probe's stream."""
    n100 = DataBlock([Column.from_data(np.arange(100, dtype=np.int64))])
    empty = DataBlock([Column.from_data(np.zeros(0, dtype=np.int32))])
    for kind in KINDS:
        probe_blocks, final_blocks = run_and_compare(kind, empty, n100, 0, 0)
        assert final_blocks == []
        if kind == "full":
            assert sum(b.num_rows for b in probe_blocks) == 100
            assert not probe_blocks[0].columns[1].valid_mask().any()
        else:
            assert probe_blocks == []
    build = DataBlock([Column.from_data(np.arange(10, dtype=np.int64)), Column.from_data(np.arange(10, dtype=np.int64))])
    for kind in KINDS:
        run_and_compare(kind, build, n100.slice(0, 0), 0, 0)


@pytest.mark.parametrize("kind", ["right_anti", "full"])
def test_config3_shape_with_unreferenced_dims(gpu, kind):
    """1e6 facts x 65 536 dims on an int64 key, 10 % of the dims referenced by no fact."""
    orc = oracle()
    n_dim, n_fact = 1 << 16, 1_000_000
    dk = orc.synth_fill(5, 99, 16, 0, n_dim)
    dv = orc.synth_fill(1, 100, 0, 0, n_dim)
    pick = orc.synth_fill(0, 101, n_dim * 9 // 10, 0, n_fact)  # facts reference the first 90 % of the dim rows
    fk = dk[pick]
    fv = orc.synth_fill(1, 102, 0, 0, n_fact)
    build = DataBlock([Column.from_data(dk), Column.from_data(dv)])
    probe = DataBlock([Column.from_data(fk), Column.from_data(fv)])
    probe_blocks, final_blocks = run_and_compare(kind, build, probe, 0, 0, build_split=20_000, probe_split=300_000)
    unref = n_dim - len(np.unique(pick))
    assert sum(b.num_rows for b in final_blocks) == unref
    run_and_compare(kind, build, probe, 0, 0, device_resident=True)
