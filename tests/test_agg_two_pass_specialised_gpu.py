"""Both passes of the partitioned aggregation compiled for the operator's plan (NVRTC): for plans forced
onto the two-pass path with pass 2 in shared memory, the specialised kernels and the precompiled ones
(DBX_AGG_JIT=0) give bit-identical results, the operator's variant text says which passes ran
specialised, and the results match the oracle."""
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


def aggregate(blk, params, filt):
    part = TransformPartialAggregate(params, schema_types(blk), filt)
    fin = TransformFinalAggregate(params, schema_types(blk))
    try:
        part.transform(DataBlock([to_device(Column.from_data(c.values().copy())) for c in blk.columns], blk.num_rows))
        variant = part.kernel_variant()
        fin.transform(part.on_finish())
        return fin.on_finish()[0], variant
    finally:
        part.close()
        fin.close()


def bit_images(out, params):
    """every result column as 64-bit images, rows ordered by the group key columns"""
    n_aggs, n_keys = len(params.aggregate_functions), len(params.group_columns)
    cols = []
    for c in out.columns:
        v = c.values()
        v = v.view(np.uint64) if v.dtype.itemsize == 8 else v.astype(np.int64).view(np.uint64)
        cols.append(np.where(c.valid_mask(), v, np.uint64(0xDEAD)))
    order = np.lexsort([cols[n_aggs + j] for j in reversed(range(n_keys))])
    return [c[order] for c in cols]


def compare_with_oracle(out, blk, params, filt):
    from oracle import oracle as orc
    n_aggs, n_keys = len(params.aggregate_functions), len(params.group_columns)
    key_img = [out.columns[n_aggs + j].values() for j in range(n_keys)]
    key_img = [k.view(np.int64) if k.dtype.itemsize == 8 else k.astype(np.int64) for k in key_img]
    got = {tuple(int(k[i]) for k in key_img): tuple(out.columns[a].values()[i].item() for a in range(n_aggs)) for i in range(out.num_rows)}
    assert len(got) == out.num_rows, "a group appears twice"
    rk, _, ra, _, _ = orc.filter_group_agg(blk, params.to_c(filt), threads=4)
    exp = {tuple(int(k.view(np.int64)[i]) for k in rk): tuple(a[i].item() for a in ra) for i in range(len(rk[0]))}
    assert got.keys() == exp.keys()
    for k in exp:
        assert got[k] == exp[k], (k, got[k], exp[k])


def check(monkeypatch, blk, params, filt):
    results = {}
    for jit in ("1", "0"):
        monkeypatch.setenv("DBX_AGG_JIT", jit)
        out, variant = aggregate(blk, params, filt)
        assert "(pass 2 in shared memory: 1, in L2 regions: 0)" in variant, variant
        if jit == "1":
            assert variant.startswith("specialised"), variant
            assert "specialised launches: pass 1 1 of 1, pass 2 1 of 1" in variant, variant
        else:
            assert "specialised launches: pass 1 0 of 1, pass 2 0 of 1" in variant, variant
        results[jit] = bit_images(out, params)
        if jit == "1":
            compare_with_oracle(out, blk, params, filt)
    assert len(results["1"][0]) == len(results["0"][0])
    for a, b in zip(results["1"], results["0"]):
        np.testing.assert_array_equal(a, b)


def config2_block(n, n_keys, seed=42):
    from oracle import oracle as orc
    return DataBlock([Column.from_data(orc.synth_fill(0, seed, n_keys, 0, n)), Column.from_data(orc.synth_fill(1, seed + 1, 0, 0, n)),
                      Column.from_data(orc.synth_fill(2, seed + 2, 20, 0, n))])


def test_config2_plan(monkeypatch):
    check(monkeypatch, config2_block(2_000_003, 400_000), CONFIG2, V_MOD3)


def test_packed_multi_column_keys(monkeypatch):
    rng = np.random.default_rng(11)
    n = 700_000
    blk = DataBlock([Column.from_data(rng.integers(0, 3000, n).astype(np.int32)), Column.from_data(rng.integers(0, 50, n).astype(np.uint16)),
                     Column.from_data(rng.integers(-1000, 1000, n).astype(np.int64))])
    check(monkeypatch, blk, AggregatorParams([0, 1], [("sum", 2), ("count", None)], expected_groups=150_000), E.gt(E.col(2), E.lit(-900)))


def test_float_keys(monkeypatch):
    rng = np.random.default_rng(13)
    n = 500_000
    k = rng.integers(0, 20_000, n) * 0.5
    r = rng.random(n)
    k = np.where(r < 0.01, np.nan, np.where(r < 0.02, 0.0, np.where(r < 0.03, -0.0, k)))
    blk = DataBlock([Column.from_data(k), Column.from_data(rng.integers(0, 1000, n).astype(np.int64))])
    params = AggregatorParams([0], [("sum", 1), ("count", None)], expected_groups=30_000)
    results = {}
    for jit in ("1", "0"):  # NaN keys: compared bit for bit between the builds (the dict-based oracle check cannot hold NaN)
        monkeypatch.setenv("DBX_AGG_JIT", jit)
        out, variant = aggregate(blk, params, None)
        assert f"specialised launches: pass 1 {jit} of 1, pass 2 {jit} of 1" in variant, variant
        results[jit] = bit_images(out, params)
    assert len(results["1"][2]) == 20_002  # 20 000 values + NaN + -0.0
    for a, b in zip(results["1"], results["0"]):
        np.testing.assert_array_equal(a, b)


def test_min_max(monkeypatch):
    rng = np.random.default_rng(17)
    n = 600_000
    blk = DataBlock([Column.from_data(rng.integers(-50_000, 50_000, n).astype(np.int64)),
                     Column.from_data(rng.integers(-2**62, 2**62, n).astype(np.int64)),
                     Column.from_data(rng.integers(0, 2**64, n, dtype=np.uint64)),
                     Column.from_data(rng.integers(-2**40, 2**40, n).astype(np.float64))])
    params = AggregatorParams([0], [("min", 1), ("max", 1), ("min", 2), ("max", 2), ("min", 3), ("max", 3)], expected_groups=60_000)
    check(monkeypatch, blk, params, None)


def test_narrow_arguments(monkeypatch):
    rng = np.random.default_rng(19)
    n = 600_000
    blk = DataBlock([Column.from_data(rng.integers(-50_000, 50_000, n).astype(np.int64)),
                     Column.from_data(rng.integers(-30_000, 30_000, n).astype(np.int16)),
                     Column.from_data(rng.integers(0, 256, n).astype(np.uint8)),
                     Column.from_data(rng.integers(-2**31, 2**31, n).astype(np.int32)),
                     Column.from_data((rng.integers(-4000, 4000, n) * 0.25).astype(np.float32))])
    params = AggregatorParams([0], [("sum", 1), ("avg", 2), ("sum", 3), ("min", 3), ("sum", 4), ("max", 4)], expected_groups=60_000)
    check(monkeypatch, blk, params, E.gt(E.col(3), E.lit(-2**30)))


def test_several_predicate_nodes(monkeypatch):
    blk = config2_block(1_500_000, 200_000, seed=7)
    filt = E.or_(E.and_(V_MOD3, E.gt(E.col(2), E.lit(1000.0))), E.lt(E.col(0), E.lit(5000)))
    check(monkeypatch, blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=200_000), filt)
