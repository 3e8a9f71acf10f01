"""Pass 1 of the two-pass aggregation on the bulk-copy ring (filter_partition_ring_body): whole tiles of every
column slot reach the filtering threads through a ring of shared-memory stages filled by the bulk-copy unit,
a partial last tile is loaded directly, and a column that does not start 16-byte aligned sends the push to
the plain pass-1 kernel.  The two-pass path is forced on small tables; every result is compared with the
oracle (floating-point sums with the exact per-group reference), and the operator's variant text says
whether the ring ran."""
import numpy as np
import pytest

import float_agg_ref as R
from databend_b200 import abi, expr as E, scalar_expr as S
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import AggregatorParams, TransformFinalAggregate, TransformPartialAggregate, schema_types, to_device

pytestmark = pytest.mark.gpu

CONFIG2 = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2)])
V_MOD3 = E.eq(E.col(1) % E.lit(3), E.lit(0))


@pytest.fixture(autouse=True)
def force_two_pass(monkeypatch):
    monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "1")
    monkeypatch.setenv("DBX_AGG_PARTITION_ALWAYS", "1")


@pytest.fixture(params=["1", "0"], ids=["specialised", "precompiled"])
def jit(request, monkeypatch):
    monkeypatch.setenv("DBX_AGG_JIT", request.param)
    return request.param


def oracle():
    from oracle import oracle as orc
    return orc


def ring_text(ring, launches):
    return f"pass 1 on the bulk-copy ring: {ring} of {launches}"


def device_blocks(blk, bounds=()):
    """blk's rows cut at `bounds`, each piece a device-resident block (one push each)"""
    out, lo = [], 0
    for hi in list(bounds) + [blk.num_rows]:
        out.append(DataBlock([to_device(Column.from_data(c.values()[lo:hi].copy())) for c in blk.columns], hi - lo))
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


def key_image(values):
    return values.view(np.int64) if values.dtype.itemsize == 8 else values.astype(np.int64)


def group_dict(key_vals, agg_vals, agg_valid):
    out = {}
    for i in range(len(key_vals[0])):
        k = tuple(int(v[i]) for v in key_vals)
        assert k not in out, f"group {k} appears twice"
        out[k] = tuple((a[i].item() if ok[i] else None) for a, ok in zip(agg_vals, agg_valid))
    return out


def compare_with_oracle(out, blk, params, filt):
    n_aggs, n_keys = len(params.aggregate_functions), len(params.group_columns)
    got = group_dict([key_image(out.columns[n_aggs + j].values()) for j in range(n_keys)],
                     [out.columns[i].values() for i in range(n_aggs)], [out.columns[i].valid_mask() for i in range(n_aggs)])
    rk, _, ra, rav, _ = oracle().filter_group_agg(blk, params.to_c(filt), threads=4)
    exp = group_dict([k.view(np.int64) for k in rk], ra, rav)
    assert got.keys() == exp.keys()
    for k in exp:
        assert got[k] == exp[k], (k, got[k], exp[k])


def check(blocks, blk, params, filt, ring, launches=1, fallbacks=0):
    out, variant = aggregate(blocks, params, filt, schema_types(blk))
    assert ring_text(ring, launches) in variant, variant
    assert f"one-pass fallbacks (skew): {fallbacks}" in variant, variant
    compare_with_oracle(out, blk, params, filt)
    return out, variant


def config2_block(n, n_keys, seed=42):
    orc = oracle()
    return DataBlock([Column.from_data(orc.synth_fill(0, seed, n_keys, 0, n)), Column.from_data(orc.synth_fill(1, seed + 1, 0, 0, n)),
                      Column.from_data(orc.synth_fill(2, seed + 2, 20, 0, n))])


@pytest.mark.parametrize("n", [65_536, 65_537, 2**20 + 17, 2**20 + 1023])
def test_whole_and_partial_last_tiles(jit, n):
    blk = config2_block(n, 30_000)
    _, variant = check(device_blocks(blk), blk, CONFIG2, V_MOD3, ring=1)
    assert f"specialised launches: pass 1 {jit} of 1" in variant, variant


@pytest.mark.parametrize("n", [2**20 + 5, 2**20 + 4096])
def test_narrow_integer_keys_and_arguments(jit, n):
    # 1- and 2-byte tile tails are not multiples of 16 bytes; every width is widened as the direct loads widen it
    rng = np.random.default_rng(11)
    blk = DataBlock([Column.from_data(rng.integers(-30_000, 30_000, n).astype(np.int16)),
                     Column.from_data(rng.integers(-128, 128, n).astype(np.int8)),
                     Column.from_data(rng.integers(0, 256, n).astype(np.uint8)),
                     Column.from_data(rng.integers(-2**31, 2**31, n).astype(np.int32)),
                     Column.from_data(rng.integers(0, 2**16, n).astype(np.uint16)),
                     Column.from_data(rng.integers(0, 2**32, n).astype(np.uint32))])
    params = AggregatorParams([0], [("sum", 1), ("min", 1), ("max", 2), ("sum", 3), ("min", 3), ("max", 4), ("sum", 5), ("count", None)],
                              expected_groups=60_000)
    check(device_blocks(blk), blk, params, E.gt(E.col(1), E.lit(-100)), ring=1)
    int8_key = DataBlock([Column.from_data(rng.integers(-128, 128, n).astype(np.int8)), Column.from_data(rng.integers(-1000, 1000, n).astype(np.int32))])
    check(device_blocks(int8_key), int8_key, AggregatorParams([0], [("sum", 1), ("count", None)], expected_groups=4096), None, ring=1)


def test_column_at_an_odd_row_offset_takes_the_plain_kernel(jit):
    n = 300_001
    blk = config2_block(n + 1, 40_000)
    dev = device_blocks(blk)[0]
    # every column one row into its allocation: 8 bytes past a 16-byte boundary
    shifted = DataBlock([c.slice(1, n + 1) for c in dev.columns], n)
    host = DataBlock([Column.from_data(c.values()[1:].copy()) for c in blk.columns])
    check([shifted], host, CONFIG2, V_MOD3, ring=0)
    # one misaligned column is enough
    mixed = DataBlock([dev.columns[0].slice(0, n), dev.columns[1].slice(1, n + 1), dev.columns[2].slice(0, n)], n)
    host = DataBlock([Column.from_data(blk.columns[0].values()[:n].copy()), Column.from_data(blk.columns[1].values()[1:].copy()),
                      Column.from_data(blk.columns[2].values()[:n].copy())])
    check([mixed], host, CONFIG2, V_MOD3, ring=0)
    del dev


def test_ring_off_switch(monkeypatch):
    monkeypatch.setenv("DBX_AGG_PART_RING", "0")
    blk = config2_block(400_000, 30_000)
    check(device_blocks(blk), blk, CONFIG2, V_MOD3, ring=0)


def test_computed_columns(jit):
    n = 2**20 + 333
    rng = np.random.default_rng(5)
    k = rng.integers(0, 200_000, n).astype(np.int64)
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    b = rng.integers(-1000, 1000, n).astype(np.int32)
    blk = DataBlock([Column.from_data(k), Column.from_data(a), Column.from_data(b)])
    params = AggregatorParams([S.col(0) % S.lit(50_000, abi.I64)], [("sum", S.col(1) * S.col(2)), ("max", S.col(1) - S.col(2)), ("count", None)],
                              expected_groups=60_000)
    out, variant = aggregate(device_blocks(blk), params, E.gt(E.col(1), E.lit(-500)), [abi.I64, abi.I64, abi.I32])
    assert ring_text(1, 1) in variant and "fallbacks (skew): 0" in variant, variant
    keep = a > -500
    kk, prod, diff = k[keep] % 50_000, a[keep] * b[keep].astype(np.int64), a[keep] - b[keep]
    order = np.argsort(out.columns[3].values())
    got_k = out.columns[3].values()[order]
    uk, start = np.unique(np.sort(kk, kind="stable"), return_index=True)
    by_key = np.argsort(kk, kind="stable")
    np.testing.assert_array_equal(got_k, uk)
    np.testing.assert_array_equal(out.columns[0].values()[order], np.add.reduceat(prod[by_key], start))
    np.testing.assert_array_equal(out.columns[1].values()[order], np.maximum.reduceat(diff[by_key], start))
    np.testing.assert_array_equal(out.columns[2].values()[order], np.diff(np.append(start, len(kk))))


def test_packed_keys(jit):
    rng = np.random.default_rng(9)
    n = 900_000
    blk = DataBlock([Column.from_data(rng.integers(0, 3000, n).astype(np.int32)), Column.from_data(rng.integers(0, 50, n).astype(np.uint16)),
                     Column.from_data(rng.integers(-1000, 1000, n).astype(np.int16)), Column.from_data((rng.integers(0, 4000, n) * 0.25).astype(np.float32))])
    params = AggregatorParams([0, 1], [("sum", 2), ("min", 2), ("max", 3), ("count", None), ("avg", 3)], expected_groups=150_000)
    check(device_blocks(blk), blk, params, E.gt(E.col(2), E.lit(-900)), ring=1)


def test_float_keys_and_float_sums():
    rng = np.random.default_rng(13)
    n = 2**20 + 100
    k = rng.integers(0, 40_000, n) * 0.5
    r = rng.random(n)
    k = np.where(r < 0.01, np.nan, np.where(r < 0.02, -0.0, k))
    x = rng.standard_normal(n) * np.exp2(rng.integers(-30, 30, n))
    blk = DataBlock([Column.from_data(k), Column.from_data(rng.integers(0, 1000, n).astype(np.int64)), Column.from_data(x)])
    params = AggregatorParams([0], [("count", None), ("max", 1), ("sum", 2), ("avg", 2)], expected_groups=50_000)
    out, variant = aggregate(device_blocks(blk), params, None, schema_types(blk))
    assert ring_text(1, 1) in variant, variant
    nan_key = np.int64(0x7FF8000000000000)  # every NaN is one group
    got_k = out.columns[4].values()
    keys = np.where(np.isnan(got_k), nan_key, key_image(got_k))
    assert len(np.unique(keys)) == out.num_rows
    row_keys = np.where(np.isnan(k), nan_key, key_image(k))
    ref = R.exact_reference(row_keys, x, np.ones(n, dtype=bool))
    sums = {int(kk): float(v) for kk, v in zip(keys, out.columns[2].values())}
    avgs = {int(kk): float(v) for kk, v in zip(keys, out.columns[3].values())}
    assert R.sum_violations(ref, sums) == []
    assert R.avg_violations(ref, avgs) == []
    counts = {int(kk): int(v) for kk, v in zip(keys, out.columns[0].values())}
    uk, cnt = np.unique(row_keys, return_counts=True)
    assert counts == {int(a): int(b) for a, b in zip(uk, cnt)}


def test_skew_overflows_a_partition_and_falls_back(jit):
    rng = np.random.default_rng(17)
    n = 700_000
    ks = np.where(rng.random(n) < 0.5, np.int64(7), rng.integers(0, 100_000, n).astype(np.int64))
    blk = DataBlock([Column.from_data(ks), Column.from_data(rng.integers(0, 1000, n).astype(np.int64)),
                     Column.from_data(rng.integers(0, 100, n).astype(np.float64))])
    check(device_blocks(blk), blk, CONFIG2, None, ring=1, fallbacks=1)


def test_several_pushes(jit):
    blk = config2_block(1_500_000, 200_000)
    check(device_blocks(blk, [300_000, 700_001, 1_100_000]), blk, CONFIG2, V_MOD3, ring=4, launches=4)
