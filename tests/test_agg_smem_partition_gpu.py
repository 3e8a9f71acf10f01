"""Two-pass aggregation with pass 2 in shared memory: pass 1 scatters the surviving rows by table
slice, then one CTA per slice aggregates its partition in shared memory and defers the rows whose
probe would leave the slice (or reach the probe limit, or whose key is the EMPTY pattern, or that
would add a group to a slice at its fill limit) to the fused kernel.  Tables with more slices than
pass 1 partitions into, or whose groups would overfill them, run pass 2 per L2 region instead.  The
paths are forced on small tables here; the operator's variant text says which pass 2 ran, every
result is compared with the oracle and the group keys are checked to be unique."""
import numpy as np
import pytest

from databend_b200 import expr as E
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import AggregatorParams, TransformFinalAggregate, TransformPartialAggregate, schema_types, to_device

pytestmark = pytest.mark.gpu

CONFIG2 = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2)])
V_MOD3 = E.eq(E.col(1) % E.lit(3), E.lit(0))


@pytest.fixture(autouse=True)
def force_two_pass(monkeypatch):
    monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "1")
    monkeypatch.setenv("DBX_AGG_PARTITION_ALWAYS", "1")


def oracle():
    from oracle import oracle as orc
    return orc


def device_blocks(blk, bounds):
    """blk's rows cut at `bounds`, each piece a device-resident block (one push each)"""
    out, lo = [], 0
    for hi in list(bounds) + [blk.num_rows]:
        cols = [to_device(Column.from_data(c.values()[lo:hi].copy())) for c in blk.columns]
        out.append(DataBlock(cols, hi - lo))
        lo = hi
    return out


def aggregate(blocks, params, filt, types):
    part = TransformPartialAggregate(params, types, filt)
    fin = TransformFinalAggregate(params, types)
    try:
        for b in blocks:
            part.transform(b)
        variant = part.kernel_variant()
        fin.transform(part.on_finish())
        return fin.on_finish()[0], variant
    finally:
        part.close()
        fin.close()


def group_dict(key_vals, key_valid, agg_vals, agg_valid):
    """{key tuple: aggregate tuple}; fails when a key appears twice"""
    out = {}
    for i in range(len(key_vals[0])):
        k = tuple((int(v[i]) if ok[i] else None) for v, ok in zip(key_vals, key_valid))
        assert k not in out, f"group {k} appears twice"
        out[k] = tuple((a[i].item() if ok[i] else None) for a, ok in zip(agg_vals, agg_valid))
    return out


def key_image(values):
    return values.view(np.int64) if values.dtype.itemsize == 8 else values.astype(np.int64)


def pass2_text(chunks, regions=0):
    return f"chunks: {chunks} (pass 2 in shared memory: {chunks - regions}, in L2 regions: {regions})"


def check(blk, params, filt, bounds=(), chunks=None, regions=0):
    """aggregates blk pushed in pieces through the forced two-pass path and compares with the oracle;
    `chunks` chunks took the two-pass path, `regions` of them with pass 2 in L2 regions"""
    out, variant = aggregate(device_blocks(blk, bounds), params, filt, schema_types(blk))
    assert "two-pass" in variant, variant
    if chunks is not None:
        assert pass2_text(chunks, regions) in variant, variant
    compare_with_oracle(out, blk, params, filt)
    return variant


def compare_with_oracle(out, blk, params, filt):
    n_aggs, n_keys = len(params.aggregate_functions), len(params.group_columns)
    keys = [out.columns[n_aggs + j] for j in range(n_keys)]
    got = group_dict([key_image(k.values()) for k in keys], [k.valid_mask() for k in keys],
                     [out.columns[i].values() for i in range(n_aggs)], [out.columns[i].valid_mask() for i in range(n_aggs)])
    rk, rkv, ra, rav, _ = oracle().filter_group_agg(blk, params.to_c(filt), threads=4)
    exp = group_dict([k.view(np.int64) for k in rk], rkv, ra, rav)
    assert got.keys() == exp.keys()
    for k in exp:
        assert got[k] == exp[k], (k, got[k], exp[k])


def config2_block(n, n_keys, seed=42):
    orc = oracle()
    return DataBlock([Column.from_data(orc.synth_fill(0, seed, n_keys, 0, n)), Column.from_data(orc.synth_fill(1, seed + 1, 0, 0, n)),
                      Column.from_data(orc.synth_fill(2, seed + 2, 20, 0, n))])


def test_config2_plan():
    blk = config2_block(2_000_003, 400_000)
    check(blk, CONFIG2, V_MOD3, chunks=1)  # default 64 MB table: 512 slices
    check(blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=200_000), V_MOD3, chunks=1)


def test_every_update_kind_narrow_and_float_arguments():
    rng = np.random.default_rng(3)
    n = 600_000
    blk = DataBlock([Column.from_data(rng.integers(-50_000, 50_000, n).astype(np.int64)),
                     Column.from_data(rng.integers(-30_000, 30_000, n).astype(np.int16)),
                     Column.from_data(rng.integers(-2**31, 2**31, n).astype(np.int32)),
                     Column.from_data(rng.integers(0, 256, n).astype(np.uint8)),
                     Column.from_data(rng.integers(0, 2**64, n, dtype=np.uint64)),
                     Column.from_data((rng.integers(-4000, 4000, n) * 0.25).astype(np.float32)),
                     Column.from_data(rng.integers(-2**40, 2**40, n).astype(np.float64))])
    params = AggregatorParams([0], [("sum", 1), ("min", 2), ("count", None), ("avg", 3), ("max", 4), ("sum", 5), ("min", 5), ("max", 6)],
                              expected_groups=60_000)
    check(blk, params, E.gt(E.col(2), E.lit(-2**30)), chunks=1)
    params = AggregatorParams([0], [("max", 1), ("max", 2), ("min", 3), ("min", 4), ("max", 5), ("count", 6), ("avg", 6), ("min", 6)],
                              expected_groups=60_000)
    check(blk, params, E.gt(E.col(2), E.lit(-2**30)), chunks=1)


def test_packed_multi_column_keys():
    rng = np.random.default_rng(5)
    n = 700_000
    blk = DataBlock([Column.from_data(rng.integers(0, 3000, n).astype(np.int32)), Column.from_data(rng.integers(0, 50, n).astype(np.uint16)),
                     Column.from_data(rng.integers(-1000, 1000, n).astype(np.int16)), Column.from_data((rng.integers(0, 4000, n) * 0.25).astype(np.float32))])
    params = AggregatorParams([0, 1], [("sum", 2), ("min", 2), ("max", 3), ("count", None), ("avg", 3)], expected_groups=150_000)
    check(blk, params, E.gt(E.col(2), E.lit(-900)), chunks=1)


def test_float_keys_nan_and_signed_zero(monkeypatch):
    # one NaN group, separate +0.0 and -0.0 groups: compared bit for bit with the one-pass path
    rng = np.random.default_rng(7)
    n = 500_000
    k = rng.integers(0, 20_000, n) * 0.5
    r = rng.random(n)
    k = np.where(r < 0.01, np.nan, np.where(r < 0.02, -np.nan, np.where(r < 0.03, 0.0, np.where(r < 0.04, -0.0, k))))
    blk = DataBlock([Column.from_data(k), Column.from_data(rng.integers(0, 1000, n).astype(np.int64))])
    params = AggregatorParams([0], [("sum", 1), ("count", None), ("max", 1)], expected_groups=30_000)
    outs = []
    for forced in (True, False):
        if not forced:
            monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "0")
        out, variant = aggregate(device_blocks(blk, ()), params, None, schema_types(blk))
        assert (pass2_text(1) in variant) == forced, variant
        bits = out.columns[3].values().view(np.uint64)
        assert len(np.unique(bits)) == out.num_rows
        order = np.argsort(bits, kind="stable")
        outs.append([out.columns[i].values()[order].view(np.uint64) for i in range(4)])
    assert len(outs[0][3]) == 20_002  # 20 000 values + NaN + -0.0
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)


def test_key_equal_to_the_empty_pattern():
    blk = config2_block(400_000, 50_000)
    k = blk.columns[0].values().copy()
    k[::7] = np.iinfo(np.int64).min  # the EMPTY pattern: deferred to the fused kernel's special slot
    blk = DataBlock([Column.from_data(k), blk.columns[1], blk.columns[2]])
    check(blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=60_000), V_MOD3, chunks=1)


def test_nearly_full_table_probes_cross_slices_and_wrap():
    # 30 000 groups for 8 slices of 4096 slots: the slices fill to their limit (3/4), probe chains run over
    # slice ends and from the last bucket to bucket 0, and the table grows before the deferred rows run
    blk = config2_block(900_000, 30_000)
    check(blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=15_000), None, chunks=1)


def test_growth_triggered_by_deferred_rows():
    # a fresh operator with more groups than slots: the slices stop at their fill limit, the table grows,
    # and the deferred rows (most of them) run through the fused kernel, overflowing and replaying once more
    blk = config2_block(900_000, 50_000)
    check(blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=15_000), None, chunks=1)


def test_table_populated_by_an_earlier_one_pass_push():
    # the first push is too small for the two-pass path; the second one finds its groups in the table
    blk = config2_block(1_000_000, 100_000)
    check(blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=100_000), V_MOD3, bounds=[40_000], chunks=1)


def test_several_pushes():
    blk = config2_block(1_200_000, 200_000)
    check(blk, CONFIG2, V_MOD3, bounds=[300_000, 600_000, 900_000], chunks=4)


def test_skew_falls_back_to_one_pass():
    rng = np.random.default_rng(17)
    n = 700_000
    ks = np.where(rng.random(n) < 0.5, np.int64(7), rng.integers(0, 100_000, n).astype(np.int64))
    blk = DataBlock([Column.from_data(ks), Column.from_data(rng.integers(0, 1000, n).astype(np.int64)),
                     Column.from_data(rng.integers(0, 100, n).astype(np.float64))])
    variant = check(blk, CONFIG2, None, chunks=0)
    assert "fallbacks (skew): 1" in variant, variant


def test_tables_with_more_slices_than_partitions_use_l2_regions():
    # 2^23 slots = 2048 slices of 4096: more than pass 1 partitions into, so pass 2 runs per L2 region
    blk = config2_block(600_000, 100_000)
    check(blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=2_100_000), V_MOD3, chunks=1, regions=1)


def test_group_count_of_the_previous_query_selects_l2_regions():
    # query 1 on a fresh operator: 50 000 groups for 32 768 slots, the slices reach their fill limit and the
    # table grows; after the reset the table starts at 32 768 slots again, and the previous query's group
    # count sends pass 2 to L2 regions
    blk = config2_block(900_000, 50_000)
    params = AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=15_000)
    types = schema_types(blk)
    part = TransformPartialAggregate(params, types, V_MOD3)
    fin = TransformFinalAggregate(params, types)
    try:
        for query, regions in ((1, 0), (2, 1)):
            part.reset()
            fin.reset()
            part.transform(device_blocks(blk, ())[0])
            assert pass2_text(query, regions) in part.kernel_variant(), part.kernel_variant()
            fin.transform(part.on_finish())
            compare_with_oracle(fin.on_finish()[0], blk, params, V_MOD3)
    finally:
        part.close()
        fin.close()
