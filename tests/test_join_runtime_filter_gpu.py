"""Join runtime filters on the device against the CPU restatement (tests/runtime_filter_ref.py): the
built min-max, IN-list and bloom words bit for bit, the apply bitmaps bit for bit, and join results
that do not change when the filter drops probe rows, in the probe kernel or through apply -> FILTER."""
import numpy as np
import pytest

import runtime_filter_ref as rf
from databend_b200 import abi, expr as E
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError
from databend_b200.transforms import HashJoin, TransformFilter, schema_types, to_device
from test_join_multi_key_gpu import expected, got_columns, rows_sorted, tables

pytestmark = pytest.mark.gpu

NP = {abi.I8: np.int8, abi.I16: np.int16, abi.I32: np.int32, abi.I64: np.int64,
      abi.U8: np.uint8, abi.U16: np.uint16, abi.U32: np.uint32, abi.U64: np.uint64}
INT_TYPES = list(NP)
FILTERED_KINDS = {"inner": abi.JOIN_INNER, "left_semi": abi.JOIN_LEFT_SEMI, "right": abi.JOIN_RIGHT,
                  "right_semi": abi.JOIN_RIGHT_SEMI, "right_anti": abi.JOIN_RIGHT_ANTI}


def rand_keys(rng, dt, n, span=None):
    info = np.iinfo(NP[dt])
    lo, hi = int(info.min), int(info.max)
    if span is not None:
        lo, hi = max(lo, -span), min(hi, span)
    return rng.integers(lo, hi, n, endpoint=True, dtype=np.int64 if dt != abi.U64 else np.uint64).astype(NP[dt])


def build_join(build_cols, probe_types, bk, pk, kind=abi.JOIN_INNER):
    j = HashJoin(schema_types(DataBlock(build_cols)), probe_types, bk, pk, kind=kind)
    j.add_block(DataBlock(build_cols))
    j.final_build()
    return j


def check_filter(f, parts, build_rows):
    """Device filter == restatement: presence of each part, bounds, IN-list and bloom words."""
    info = f.info()
    assert info.build_rows == build_rows and len(info.parts) == len(parts)
    for i, (pi, ref) in enumerate(zip(info.parts, parts)):
        assert pi.key_dtype == ref["dtype"]
        assert pi.has_min_max == ref["has_min_max"]
        assert (pi.min, pi.max) == (ref["min"], ref["max"])
        assert pi.has_inlist == (ref["inlist"] is not None)
        if ref["inlist"] is not None:
            np.testing.assert_array_equal(f.inlist(i).astype(ref["inlist"].dtype), ref["inlist"])
        assert pi.has_bloom == (ref["bloom"] is not None)
        if ref["bloom"] is not None:
            assert pi.bloom_bytes == ref["bloom"].nbytes
            np.testing.assert_array_equal(f.bloom_words(i), ref["bloom"])


@pytest.mark.parametrize("bt", INT_TYPES, ids=lambda t: f"b{t}")
@pytest.mark.parametrize("pt", [abi.I64, abi.I16, abi.U32], ids=lambda t: f"p{t}")
def test_build_is_bit_identical_for_every_key_type(gpu, bt, pt):
    if (bt == abi.U64 and pt in (abi.I64, abi.I16)) or (pt == abi.U64 and bt in (abi.I8, abi.I16, abi.I32, abi.I64)):
        pytest.skip("signed with UInt64 has no common type: the join refuses it")
    rng = np.random.default_rng(bt * 16 + pt)
    n = 900  # IN-list, min-max and bloom all built
    vals = rand_keys(rng, bt, n, span=5000)
    vals[rng.integers(0, n, 200)] = vals[0]  # duplicates
    b = Column.from_data(vals, bt, validity=rng.random(n) > 0.1)
    pay = Column.from_data(np.arange(n, dtype=np.int64))
    j = build_join([b, pay], [pt, abi.I64], 0, 0)
    f = j.runtime_filter(build_table_rows=100 * n)
    parts = rf.build([b], [pt], build_table_rows=100 * n)
    check_filter(f, parts, n)
    # apply on a nullable probe block, sliced so the key's data and validity start at a bit offset
    npr = 5000
    pv = np.concatenate([vals[rng.integers(0, n, npr // 2)].astype(NP[pt], casting="unsafe") if bt == pt else
                         rand_keys(rng, pt, npr // 2, span=5000), rand_keys(rng, pt, npr - npr // 2, span=6000)])
    pc = Column.from_data(pv, pt, validity=rng.random(npr) > 0.2)
    blk = DataBlock([Column.from_data(np.arange(npr, dtype=np.int64)), pc]).slice(13, npr - 7)
    got = f.apply(blk, [1])
    assert got.dtype == abi.BOOL and got.data_bit_offset == 0 and got.validity is None
    want = rf.apply(parts, [blk.columns[1]])
    np.testing.assert_array_equal(got.values(), want)
    packed = np.packbits(want, bitorder="little")
    np.testing.assert_array_equal(got.data[:len(packed)], packed)
    info = f.info()
    assert info.apply_rows_checked == blk.num_rows and info.apply_rows_rejected == blk.num_rows - int(want.sum())
    assert info.apply_rows_rejected > 0
    f.close()
    j.close()


@pytest.mark.parametrize("n,inlist,bloom", [(1024, True, True), (1025, False, True), (3_000_000, False, True), (3_000_001, False, False)])
def test_threshold_edges(gpu, n, inlist, bloom):
    rng = np.random.default_rng(n)
    vals = rng.integers(-10**9, 10**9, n, dtype=np.int64)
    b = Column.from_data(vals, validity=rng.random(n) > 0.01)
    j = build_join([b], [abi.I64], 0, 0)
    f = j.runtime_filter(build_table_rows=10**9)
    parts = rf.build([b], [abi.I64], build_table_rows=10**9)
    assert (parts[0]["inlist"] is not None) == inlist and (parts[0]["bloom"] is not None) == bloom
    check_filter(f, parts, n)
    f.close()
    j.close()


@pytest.mark.parametrize("ndv", [1, 26, 27, 2000, 14_000_000 // 100])
def test_bloom_size_clamp_and_steps(gpu, ndv):
    """32-byte minimum, and the steps of the power-of-two size."""
    b = Column.from_data(np.arange(ndv, dtype=np.int32) * 7)
    j = build_join([b], [abi.I32], 0, 0)
    f = j.runtime_filter(build_table_rows=10**9)
    parts = rf.build([b], [abi.I32], build_table_rows=10**9)
    assert f.info().parts[0].bloom_bytes == rf.bloom_bytes(ndv)
    check_filter(f, parts, ndv)
    f.close()
    j.close()


def test_selectivity_disables_only_the_bloom_and_empty_build_has_none(gpu):
    b = Column.from_data(np.array([1, 10], dtype=np.int32))
    j = build_join([b], [abi.I32], 0, 0)
    f = j.runtime_filter(build_table_rows=10, selectivity_threshold=1)
    p = f.info().parts[0]
    assert (p.has_bloom, p.has_inlist, p.inlist_len, p.has_min_max) == (False, True, 2, True)
    f.close()
    f = j.runtime_filter(build_table_rows=20)  # exactly 10 %: no bloom
    assert not f.info().parts[0].has_bloom
    f.close()
    j.close()
    j = HashJoin([abi.I64], [abi.I64], 0, 0)
    j.final_build()
    f = j.runtime_filter(build_table_rows=100)
    p = f.info().parts[0]
    assert not (p.has_bloom or p.has_inlist or p.has_min_max)
    f.close()
    j.close()


def test_all_null_build_keys_reject_every_row(gpu):
    b = Column.from_data(np.array([3, 4], dtype=np.int64), validity=[False, False])
    j = build_join([b], [abi.I64], 0, 0)
    f = j.runtime_filter(build_table_rows=100)
    p = f.info().parts[0]
    assert p.min is None and p.max is None and p.inlist_len == 0
    got = f.apply(DataBlock([Column.from_data(np.array([3, 4, 5], dtype=np.int64))]), [0])
    assert not got.values().any()
    f.close()
    j.close()


def test_composite_key_parts_are_anded(gpu):
    build, probe, bk, pk = tables("mixed", 5, nb=3000, npr=8000)
    j = HashJoin(schema_types(build), schema_types(probe), bk, pk)
    j.add_block(build)
    j.final_build()
    f = j.runtime_filter(build_table_rows=10**6)
    parts = rf.build([build.columns[c] for c in bk], [probe.columns[c].dtype for c in pk], build_table_rows=10**6)
    check_filter(f, parts, build.num_rows)
    blk = probe.slice(5, probe.num_rows)
    np.testing.assert_array_equal(f.apply(blk, pk).values(), rf.apply(parts, [blk.columns[c] for c in pk]))
    f.close()
    j.close()


def filtered(f, block, pk, types):
    """apply -> DBX_OP_FILTER on the appended Boolean column -> the probe block without it"""
    mask = f.apply(block, pk)
    op = TransformFilter(E.bool_column(len(block.columns)), list(types) + [abi.BOOL])
    out = op.transform(DataBlock(block.columns + [mask], block.num_rows))
    op.close()
    return DataBlock(out.columns[:-1], out.num_rows)


def run_mode(kind, build, probe, bk, pk, mode, split=4096, device_resident=False):
    ptypes = schema_types(probe)
    j = HashJoin(schema_types(build), ptypes, bk, pk, kind=FILTERED_KINDS[kind])
    j.add_block(build)
    j.final_build()
    f = None
    if mode != "none":
        f = j.runtime_filter(in_probe=mode == "in_probe", build_table_rows=100 * build.num_rows)
    if mode == "in_probe":
        assert "runtime filter in the probe" in j.kernel_variant()
    outs = []
    for p in probe.split_by_rows(split):
        if mode == "apply":
            p = filtered(f, p, pk, ptypes)
            if p.num_rows == 0:
                continue
        if device_resident:
            p = DataBlock([to_device(c) for c in p.columns], p.num_rows)
        outs += j.probe_block(p)
    outs += j.final_probe()
    info = f.info() if f else None
    if f:
        f.close()
    j.close()
    return outs, info


def check_modes(kind, build, probe, bk, pk, modes, **kw):
    exp, n = expected(kind, build, probe, bk, pk)
    results = {}
    for mode in modes:
        outs, info = run_mode(kind, build, probe, bk, pk, mode, **kw)
        assert sum(o.num_rows for o in outs) == n, (kind, mode)
        if n:
            np.testing.assert_array_equal(rows_sorted(got_columns(outs, len(exp))), rows_sorted(exp), err_msg=f"{kind} {mode}")
        results[mode] = info
    return results


@pytest.mark.parametrize("kind", list(FILTERED_KINDS))
@pytest.mark.parametrize("unique", [False, True], ids=["dup", "unique"])
def test_single_key_join_output_is_unchanged_in_every_mode(gpu, kind, unique):
    rng = np.random.default_rng(11 + unique)
    nb, npr = 5000, 60_000
    keys = rng.choice(np.arange(200_000, dtype=np.int64), nb, replace=not unique)
    build = DataBlock([Column.from_data(keys, validity=rng.random(nb) > 0.05), Column.from_data(rng.integers(0, 99, nb)),
                       Column.from_data(rng.integers(0, 9, nb).astype(np.int32))])
    pk_vals = np.where(rng.random(npr) < 0.3, keys[rng.integers(0, nb, npr)], rng.integers(-1000, 220_000, npr))
    probe = DataBlock([Column.from_data(np.arange(npr, dtype=np.int64)), Column.from_data(pk_vals.astype(np.int64), validity=rng.random(npr) > 0.05)])
    res = check_modes(kind, build, probe, [0], [1], ["none", "in_probe", "apply"])
    ip, ap = res["in_probe"], res["apply"]
    assert ip.in_probe and ip.probe_rows_checked == npr and ip.probe_rows_rejected > 0
    assert ap.apply_rows_checked == npr and ap.apply_rows_rejected > ip.probe_rows_rejected  # apply also rejects NULL keys
    assert ap.parts[0].has_bloom and ap.parts[0].has_min_max


def test_in_probe_on_device_blocks_with_mixed_key_types(gpu):
    rng = np.random.default_rng(3)
    nb, npr = 3000, 40_000
    build = DataBlock([Column.from_data(rng.integers(-30000, 30000, nb).astype(np.int16), validity=rng.random(nb) > 0.1),
                       Column.from_data(np.arange(nb, dtype=np.int64))])
    probe = DataBlock([Column.from_data(rng.integers(-40000, 40000, npr).astype(np.int32), validity=rng.random(npr) > 0.1)])
    check_modes("inner", build, probe, [0], [0], ["none", "in_probe", "apply"], device_resident=True)


@pytest.mark.parametrize("kind", list(FILTERED_KINDS))
def test_composite_key_join_output_is_unchanged_with_apply(gpu, kind):
    build, probe, bk, pk = tables("I16+I32+I8", 21, nb=4000, npr=30_000)
    res = check_modes(kind, build, probe, bk, pk, ["none", "apply"])
    assert res["apply"].apply_rows_rejected > 0


def test_refusals(gpu):
    b = Column.from_data(np.arange(10, dtype=np.int64))
    for kind in (abi.JOIN_LEFT, abi.JOIN_LEFT_ANTI, abi.JOIN_FULL):
        j = build_join([b], [abi.I64], 0, 0, kind=kind)
        with pytest.raises(DbxError) as ei:
            j.runtime_filter()
        assert ei.value.status == abi.ERR_UNSUPPORTED
        j.close()
    j = HashJoin([abi.I64], [abi.I64], 0, 0)
    j.add_block(DataBlock([b]))
    with pytest.raises(DbxError) as ei:
        j.runtime_filter()
    assert ei.value.status == abi.ERR_STATE
    j.close()
    build, probe, bk, pk = tables("2xI32", 1, nb=100, npr=100)
    j = HashJoin(schema_types(build), schema_types(probe), bk, pk)
    j.add_block(build)
    j.final_build()
    with pytest.raises(DbxError) as ei:
        j.runtime_filter(in_probe=True)
    assert ei.value.status == abi.ERR_UNSUPPORTED
    with pytest.raises(DbxError) as ei:
        j.runtime_filter(inlist_threshold=abi.RF_MAX_INLIST + 1)
    assert ei.value.status == abi.ERR_INVALID
    j.close()


def test_reset_and_destroy_orders(gpu):
    rng = np.random.default_rng(9)
    keys = rng.integers(0, 10**6, 2000, dtype=np.int64)
    probe = DataBlock([Column.from_data(rng.integers(0, 10**6, 50_000, dtype=np.int64))])
    j = build_join([Column.from_data(keys)], [abi.I64], 0, 0)
    base = sum(o.num_rows for o in j.probe_block(probe))
    # destroy the handle while the join still probes with the filter
    f = j.runtime_filter(in_probe=True, build_table_rows=10**8)
    f.close()
    assert "runtime filter in the probe" in j.kernel_variant()
    assert sum(o.num_rows for o in j.probe_block(probe)) == base
    # reset drops the in-probe filter; the handle outlives the join's filter and the join itself
    f = j.runtime_filter(in_probe=True, build_table_rows=10**8)
    j.probe_block(probe)
    rej = f.info().probe_rows_rejected
    assert rej > 0
    j.reset()
    assert not f.info().in_probe and "runtime filter" not in j.kernel_variant()
    with pytest.raises(DbxError):
        j.runtime_filter()
    j.add_block(DataBlock([Column.from_data(keys)]))
    j.final_build()
    assert sum(o.num_rows for o in j.probe_block(probe)) == base
    assert f.info().probe_rows_rejected == rej
    j.close()
    assert f.apply(probe, [0]).values().sum() == f.last_passed
    f.close()
