"""Parity of the device inner hash join against the CPU oracle.

The reference pins join results only at SQL level (tests/sqllogictests/suites/query/join/*.test,
needing a server), so parity is against the restated oracle (hashjoin_hashtable.rs:95-190,
fixed_keys.rs:47-166) as multisets of joined rows, plus hand-written cases."""
import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import HashJoin, schema_types, to_device

pytestmark = pytest.mark.gpu


def oracle():
    from oracle import oracle as orc
    return orc


def joined_rows_sorted(cols):
    """rows as a lexicographically sorted 2-D array of (value, validity) pairs"""
    arr = []
    for c in cols:
        v = c.values().astype(np.float64) if c.values().dtype.kind == "f" else c.values().astype(np.int64) if c.dtype != abi.U64 else c.values().view(np.int64)
        m = c.valid_mask()
        arr.append(np.where(m, v, 0))
        arr.append(m.astype(np.int64))
    a = np.stack(arr, axis=1) if arr else np.zeros((0, 0))
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def run_join(build: DataBlock, probe: DataBlock, bk: int, pk: int, build_split=None, probe_split=None, device_resident=False):
    j = HashJoin(schema_types(build), schema_types(probe), bk, pk)
    for b in (build.split_by_rows(build_split) if build_split else [build]):
        j.add_block(b)
    j.final_build()
    outs = []
    for p in (probe.split_by_rows(probe_split) if probe_split else [probe]):
        if device_resident:
            p = DataBlock([to_device(c) for c in p.columns], p.num_rows)
        outs.extend(j.probe_block(p))
    j.close()
    pi, bi = oracle().hash_join_inner(build.columns[bk], probe.columns[pk])
    n_cols = probe.num_columns() + build.num_columns()
    # expected rows from the oracle's (probe_idx, build_idx) pairs
    exp_cols = []
    for c in probe.columns:
        exp_cols.append(Column.from_data(c.values()[pi], c.dtype, validity=c.valid_mask()[pi]))
    for c in build.columns:
        exp_cols.append(Column.from_data(c.values()[bi], c.dtype, validity=c.valid_mask()[bi]))
    got_rows = sum(o.num_rows for o in outs)
    assert got_rows == len(pi)
    if got_rows == 0:
        return
    got_cols = []
    for ci in range(n_cols):
        vals = np.concatenate([o.columns[ci].values() for o in outs])
        valid = np.concatenate([o.columns[ci].valid_mask() for o in outs])
        got_cols.append(Column.from_data(vals, outs[0].columns[ci].dtype, validity=valid))
    np.testing.assert_array_equal(joined_rows_sorted(got_cols), joined_rows_sorted(exp_cols))


def test_small_handwritten(gpu):
    build = DataBlock([Column.from_data(np.array([5, 7, 5, 9, 11], dtype=np.int64), validity=[True, True, True, True, False]),
                       Column.from_data(np.array([50, 70, 51, 90, 110], dtype=np.int64))])
    probe = DataBlock([Column.from_data(np.array([5, 6, 9, 5, 11, 7], dtype=np.int64), validity=[True, True, True, False, True, True]),
                       Column.from_data(np.array([1.5, 2.5, 3.5, 4.5, 5.5, 6.5]))])
    run_join(build, probe, 0, 0)


def test_config3_shape_unique_dim(gpu):
    """fact x dim on int64 key, every fact row matches exactly once (SURVEY 8d row 3)."""
    orc = oracle()
    n_dim, n_fact = 1 << 16, 1_000_000
    dk = orc.synth_fill(5, 99, 16, 0, n_dim)          # unique keys: bijection on [0, 2^16)
    dv = orc.synth_fill(1, 100, 0, 0, n_dim)
    pick = orc.synth_fill(0, 101, n_dim, 0, n_fact)   # uniform dim row per fact row
    fk = dk[pick]
    fv = orc.synth_fill(1, 102, 0, 0, n_fact)
    build = DataBlock([Column.from_data(dk), Column.from_data(dv)])
    probe = DataBlock([Column.from_data(fk), Column.from_data(fv)])
    run_join(build, probe, 0, 0, build_split=20_000, probe_split=300_000)
    run_join(build, probe, 0, 0, device_resident=True)


def test_many_to_many_and_misses(gpu):
    rng = np.random.default_rng(17)
    build = DataBlock([Column.from_data(rng.integers(0, 500, 5000).astype(np.int32)), Column.from_data(rng.normal(size=5000)),
                       Column.from_data(rng.integers(0, 255, 5000).astype(np.uint8), validity=rng.random(5000) > 0.3)])
    probe = DataBlock([Column.from_data(rng.integers(-5, 5, 4000).astype(np.int16)),
                       Column.from_data(rng.integers(-100, 700, 4000).astype(np.int64), validity=rng.random(4000) > 0.1)])
    run_join(build, probe, 0, 1, build_split=1234, probe_split=999)  # ~10 matches per probe row: retry path


def test_empty_sides(gpu):
    build = DataBlock([Column.from_data(np.arange(10, dtype=np.int64)), Column.from_data(np.arange(10, dtype=np.int64))])
    probe = DataBlock([Column.from_data(np.arange(100, 110, dtype=np.int64))])
    run_join(build, probe, 0, 0)                       # no matches
    run_join(build.slice(0, 0), probe, 0, 0)           # empty build side
    run_join(build, probe.slice(0, 0), 0, 0)           # empty probe block


def test_wide_build_side_inline_and_gather(gpu):
    """Key in the middle of five build columns: two payload columns ride in the table entries
    (one of them nullable), the remaining ones are gathered by build row (one nullable, narrow)."""
    rng = np.random.default_rng(23)
    nb, npb = 7000, 9000
    build = DataBlock([Column.from_data(rng.normal(size=nb).astype(np.float32), validity=rng.random(nb) > 0.2),
                       Column.from_data(rng.integers(-2**62, 2**62, nb).astype(np.int64)),
                       Column.from_data(rng.integers(0, 3000, nb).astype(np.uint32)),            # key
                       Column.from_data(rng.integers(0, 60000, nb).astype(np.uint16), validity=rng.random(nb) > 0.5),
                       Column.from_data(rng.normal(size=nb))])
    probe = DataBlock([Column.from_data(rng.integers(0, 3500, npb).astype(np.int64)),
                       Column.from_data(rng.integers(0, 100, npb).astype(np.int8))])
    run_join(build, probe, 2, 0, build_split=1500, probe_split=2500)


def test_duplicate_build_keys_misses_and_one_long_chain(gpu):
    """Duplicate build keys with misses on both sides, over a probe split into blocks and over a
    device-resident probe block; then a build side whose keys are all equal, so that one probe
    sequence is as long as the build side and every matching probe row emits all of it."""
    rng = np.random.default_rng(31)
    nb, npb = 60_000, 200_000
    build = DataBlock([Column.from_data(rng.integers(0, 50_000, nb).astype(np.int64)), Column.from_data(rng.integers(-9, 9, nb).astype(np.int64)),
                       Column.from_data(rng.normal(size=nb))])
    probe = DataBlock([Column.from_data(rng.integers(-1000, 60_000, npb).astype(np.int64)), Column.from_data(rng.integers(0, 2**31, npb).astype(np.int32))])
    run_join(build, probe, 0, 0, probe_split=70_000)
    run_join(build, probe, 0, 0, device_resident=True)
    skew = DataBlock([Column.from_data(np.full(nb, 7, dtype=np.int64)), Column.from_data(np.arange(nb, dtype=np.int64))])
    few = DataBlock([Column.from_data(np.array([7, 8, 7], dtype=np.int64))])
    run_join(skew, few, 0, 0)


@pytest.mark.parametrize("kind_name", ["semi", "anti"])
def test_left_semi_and_anti(gpu, kind_name):
    """LEFT SEMI / LEFT ANTI (left_join_semi.rs, left_join_anti.rs): probe rows with at least one /
    with no match, probe columns only, each row at most once; a NULL probe key never matches."""
    rng = np.random.default_rng(41)
    nb, npb = 20_000, 50_000
    build = DataBlock([Column.from_data(rng.integers(0, 9000, nb).astype(np.int64), validity=rng.random(nb) > 0.05),
                       Column.from_data(rng.normal(size=nb))])
    probe = DataBlock([Column.from_data(rng.integers(-500, 12_000, npb).astype(np.int64), validity=rng.random(npb) > 0.1),
                       Column.from_data(np.arange(npb, dtype=np.int64))])  # unique row tag
    pi, _ = oracle().hash_join_inner(build.columns[0], probe.columns[0])
    matched = np.zeros(npb, dtype=bool)
    matched[pi] = True
    expect = np.nonzero(matched if kind_name == "semi" else ~matched)[0]
    kind = abi.JOIN_LEFT_SEMI if kind_name == "semi" else abi.JOIN_LEFT_ANTI
    j = HashJoin(schema_types(build), schema_types(probe), 0, 0, kind=kind)
    j.add_block(build)
    j.final_build()
    outs = []
    for p in probe.split_by_rows(17_000):
        outs.extend(j.probe_block(p))
    j.close()
    assert all(o.num_columns() == 2 for o in outs)
    tags = np.sort(np.concatenate([o.columns[1].values() for o in outs])) if outs else np.empty(0, np.int64)
    np.testing.assert_array_equal(tags, expect)
    keys = np.concatenate([o.columns[0].values() for o in outs])
    kval = np.concatenate([o.columns[0].valid_mask() for o in outs])
    order = np.argsort(np.concatenate([o.columns[1].values() for o in outs]))
    np.testing.assert_array_equal(kval[order], probe.columns[0].valid_mask()[expect])
    m = kval[order]
    np.testing.assert_array_equal(keys[order][m], probe.columns[0].values()[expect][m])


def test_left_outer(gpu):
    """LEFT join (left_join.rs): every probe row; rows without a match carry NULL in all build
    columns (which come back Nullable).  Compared as a multiset with rows derived from the oracle's
    inner pairs plus the unmatched probe rows."""
    rng = np.random.default_rng(43)
    nb, npb = 8_000, 30_000
    build = DataBlock([Column.from_data(rng.integers(0, 6000, nb).astype(np.int32)),
                       Column.from_data(rng.integers(-99, 99, nb).astype(np.int64)),
                       Column.from_data(rng.normal(size=nb), validity=rng.random(nb) > 0.3),
                       Column.from_data(rng.integers(0, 200, nb).astype(np.uint8))])
    probe = DataBlock([Column.from_data(rng.integers(-100, 8000, npb).astype(np.int64), validity=rng.random(npb) > 0.1),
                       Column.from_data(np.arange(npb, dtype=np.int64))])
    pi, bi = oracle().hash_join_inner(build.columns[0], probe.columns[0])
    matched = np.zeros(npb, dtype=bool)
    matched[pi] = True
    un = np.nonzero(~matched)[0]
    exp_cols = []
    for c in probe.columns:
        idx = np.concatenate([pi, un])
        exp_cols.append(Column.from_data(c.values()[idx], c.dtype, validity=c.valid_mask()[idx]))
    for c in build.columns:
        vals = np.concatenate([c.values()[bi], np.zeros(len(un), dtype=c.values().dtype)])
        valid = np.concatenate([c.valid_mask()[bi], np.zeros(len(un), dtype=bool)])
        exp_cols.append(Column.from_data(vals, c.dtype, validity=valid))
    j = HashJoin(schema_types(build), schema_types(probe), 0, 0, kind=abi.JOIN_LEFT)
    j.add_block(build)
    j.final_build()
    outs = []
    for p in probe.split_by_rows(11_000):
        outs.extend(j.probe_block(p))
    j.close()
    assert sum(o.num_rows for o in outs) == len(pi) + len(un)
    got_cols = []
    for ci in range(6):
        vals = np.concatenate([o.columns[ci].values() for o in outs])
        valid = np.concatenate([o.columns[ci].valid_mask() for o in outs])
        got_cols.append(Column.from_data(vals, outs[0].columns[ci].dtype, validity=valid))
    np.testing.assert_array_equal(joined_rows_sorted(got_cols), joined_rows_sorted(exp_cols))


def test_mixed_width_keys_and_signed_vs_uint64_refused(gpu):
    """Keys of different widths / signedness compare by VALUE (both widened to 64 bits): Int8 -1
    matches Int32 -1 and never UInt16 65535; the one pair without a 64-bit super type, signed vs
    UInt64, is refused (the widened images of -1 and 2^64-1 coincide)."""
    from databend_b200.lib import DbxError
    build = DataBlock([Column.from_data(np.array([-1, 5, 127, -128], dtype=np.int8)), Column.from_data(np.arange(4, dtype=np.int64))])
    probe = DataBlock([Column.from_data(np.array([-1, 5, 255, 127, -128, 65535], dtype=np.int32)), Column.from_data(np.arange(6, dtype=np.float64))])
    run_join(build, probe, 0, 0)
    probe_u = DataBlock([Column.from_data(np.array([65535, 5, 255, 127], dtype=np.uint16)), Column.from_data(np.arange(4, dtype=np.float64))])
    run_join(build, probe_u, 0, 0)
    b64 = DataBlock([Column.from_data(np.array([-1, 5], dtype=np.int64))])
    p64 = DataBlock([Column.from_data(np.array([2**64 - 1, 5], dtype=np.uint64))])
    for a, b in ((b64, p64), (p64, b64)):
        with pytest.raises(DbxError, match="signed key cannot be compared with a UInt64"):
            HashJoin(schema_types(a), schema_types(b), 0, 0)
