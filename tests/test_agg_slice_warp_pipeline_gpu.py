"""Pass 2 of the partitioned aggregation with every warp streaming its own rows: a partition is cut into
blocks of slice_warp_rows(NS) rows (64 for up to 3 slots, 32 for 4 to 6, 24 for 7 and 8), block b goes
to warp b mod 32, and each warp copies its blocks into its own double buffer in whole 16-byte pairs of
rows.  Each slice of the table gets a partition of a chosen size here (empty, one row, around one block,
around a full round over the 32 warps, odd sizes for the pair rule), one slice takes a hot key hit by
every warp at once, and every plan runs with the kernels specialised for it and precompiled
(DBX_AGG_JIT=0).  Integer results must equal the oracle's; float sums and averages must lie within
float_agg_ref's bound of the exact per-group value."""
import numpy as np
import pytest

from databend_b200.block import Column, DataBlock
from databend_b200.transforms import AggregatorParams, TransformFinalAggregate, TransformPartialAggregate, schema_types, to_device
from float_agg_ref import avg_violations, exact_reference, sum_violations

pytestmark = pytest.mark.gpu

N_SLICES = 32
CHOSEN = 16                  # slices 0..15 get the partition sizes under test, the rest filler rows
MIN_ROWS = 70_000            # a push of fewer than 65 536 rows never takes the two-pass path
SLICE_BYTES = 128 << 10      # shared memory for one slice's keys and state words
STAGE_BYTES = 96 << 10       # every warp's two row buffers
WARPS = 32


@pytest.fixture(autouse=True)
def force_two_pass(monkeypatch):
    monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "1")
    monkeypatch.setenv("DBX_AGG_PARTITION_ALWAYS", "1")


def warp_rows(ns):
    r = 64
    while r > 8 and WARPS * 2 * ns * 8 * r > STAGE_BYTES:
        r -= 32 if r > 32 else 8
    return r


def agg_hash(k):
    """agg_hash_u64 over a uint64 array"""
    with np.errstate(over="ignore"):
        x = k.astype(np.uint64)
        m = np.uint64(0xd6e8feb86659fd93)
        x ^= x >> np.uint64(32)
        x *= m
        x ^= x >> np.uint64(32)
        x *= m
        x ^= x >> np.uint64(32)
    return x


def slice_keys(n_words):
    """per slice, candidate int64 keys whose bucket lies in it, for a table of N_SLICES slices; and the
    expected_groups that sizes the table so"""
    s = 4
    while 2 * s * 8 * (1 + n_words) <= SLICE_BYTES:
        s *= 2
    cap = N_SLICES * s
    nb = cap // 4
    shift = (nb.bit_length() - 1) - (N_SLICES.bit_length() - 1)
    cand = np.arange(1, 64 * cap, dtype=np.int64) * 7919
    part = (agg_hash(cand) & np.uint64(nb - 1)) >> np.uint64(shift)
    return [cand[part == i] for i in range(N_SLICES)], cap // 2


def sizes_for(ns):
    """one partition size per slice: empty, one row, around one and two blocks, a few warps' worth,
    around a full round over all warps, and one block past it; odd sizes leave half a copy pair"""
    w = warp_rows(ns)
    full = WARPS * w
    return with_filler([0, 1, w - 1, w, w + 1, 2 * w - 1, 2 * w + 1, 5 * w + 3, full - w, full - 1, full, full + 1,
                        full + w, full + w + 1, 2 * full + 7, 3 * w])


def with_filler(sizes):
    """sizes of the CHOSEN slices, then the other slices' share of the rows the push needs at least"""
    assert len(sizes) == CHOSEN
    fill = max(0, MIN_ROWS - sum(sizes)) // (N_SLICES - CHOSEN) + 1
    return sizes + [fill] * (N_SLICES - CHOSEN)


def build_keys(pools, sizes, rng, groups_per_slice=40, hot=None):
    """keys of sum(sizes) rows, sizes[i] of them from slice i's pool (a few groups per slice, so warps
    meet on the same groups); slice `hot` takes a single key"""
    parts = []
    for i, c in enumerate(sizes):
        g = 1 if i == hot else min(max(c, 1), groups_per_slice)
        parts.append(pools[i][rng.integers(0, g, c)])
    k = np.concatenate(parts)
    return k[rng.permutation(len(k))]


def aggregate(blk, params, monkeypatch, jit):
    monkeypatch.setenv("DBX_AGG_JIT", jit)
    part = TransformPartialAggregate(params, schema_types(blk), None)
    fin = TransformFinalAggregate(params, schema_types(blk))
    try:
        part.transform(DataBlock([to_device(Column.from_data(c.values().copy())) for c in blk.columns], blk.num_rows))
        variant = part.kernel_variant()
        fin.transform(part.on_finish())
        out = fin.on_finish()[0]
    finally:
        part.close()
        fin.close()
    assert "(pass 2 in shared memory: 1, in L2 regions: 0)" in variant, variant
    assert f"pass 2 {1 if jit == '1' else 0} of 1" in variant, variant
    return out


def check(monkeypatch, blk, params, float_aggs):
    """runs both builds; integer aggregates equal the oracle's, float_aggs ({aggregate index: (kind, column)})
    within float_agg_ref's bound"""
    from oracle import oracle as orc
    n_aggs = len(params.aggregate_functions)
    rk, _, ra, _, _ = orc.filter_group_agg(blk, params.to_c(None), threads=4)
    exp = {int(k): tuple(a[i].item() for a in ra) for i, k in enumerate(rk[0].view(np.int64))}
    keys = blk.columns[0].values()
    refs = {a: exact_reference(keys, blk.columns[col].values(), np.ones(blk.num_rows, bool)) for a, (_, col) in float_aggs.items()}
    for jit in ("1", "0"):
        out = aggregate(blk, params, monkeypatch, jit)
        got_keys = [int(k) for k in out.columns[n_aggs].values().view(np.int64)]
        assert len(set(got_keys)) == len(got_keys), "a group appears twice"
        assert set(got_keys) == exp.keys()
        for a in range(n_aggs):
            vals = out.columns[a].values()
            got = {k: vals[i].item() for i, k in enumerate(got_keys)}
            if a in float_aggs:
                kind = float_aggs[a][0]
                errors = (sum_violations if kind == "sum" else avg_violations)(refs[a], got)
                assert not errors, (jit, errors[:5])
            else:
                for k in got_keys:
                    assert got[k] == exp[k][a], (jit, a, k, got[k], exp[k][a])


def test_three_slots_block_boundaries(monkeypatch):
    # config 2's shape (key, Int64 sum and count, f64 avg): 64-row blocks, two rows per lane
    rng = np.random.default_rng(23)
    pools, eg = slice_keys(3)  # state words: count(*), sum(v), sum(x)
    k = build_keys(pools, sizes_for(3), rng)
    n = len(k)
    blk = DataBlock([Column.from_data(k), Column.from_data(rng.integers(-2**31, 2**31, n).astype(np.int64)),
                     Column.from_data(rng.standard_normal(n) * 1e3)])
    params = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2), ("sum", 2)], expected_groups=eg)
    check(monkeypatch, blk, params, {2: ("avg", 2), 3: ("sum", 2)})


def test_hot_key_hit_by_every_warp(monkeypatch):
    # slice 3 holds one key for 6 000 rows, so all 32 warps update it at once: compare-and-swap retries on
    # the f64 sum, and Int64 values next to +-2^31 carry into and borrow from the high 32-bit half
    rng = np.random.default_rng(29)
    pools, eg = slice_keys(6)
    sizes = [300] * CHOSEN
    sizes[3] = 6000
    sizes = with_filler(sizes)
    k = build_keys(pools, sizes, rng, hot=3)
    n = len(k)
    edge = np.array([2**31 - 1, 2**31, -2**31, -2**31 - 1, 2**32 - 1, -(2**32) + 1], dtype=np.int64)
    v = edge[rng.integers(0, len(edge), n)] + rng.integers(-3, 4, n)
    blk = DataBlock([Column.from_data(k), Column.from_data(v), Column.from_data(rng.standard_normal(n) * 1e6),
                     Column.from_data(rng.integers(0, 2**62, n).astype(np.int64))])
    params = AggregatorParams([0], [("sum", 1), ("count", None), ("sum", 2), ("avg", 1), ("sum", 3), ("min", 1), ("max", 3)],
                              expected_groups=eg)
    check(monkeypatch, blk, params, {2: ("sum", 2)})


def test_five_slots(monkeypatch):
    # 32-row blocks, one row per lane
    rng = np.random.default_rng(31)
    pools, eg = slice_keys(5)
    k = build_keys(pools, sizes_for(5), rng)
    n = len(k)
    blk = DataBlock([Column.from_data(k), Column.from_data(rng.integers(-2**40, 2**40, n).astype(np.int64)),
                     Column.from_data(rng.integers(-2**31, 2**31, n).astype(np.int32)),
                     Column.from_data(rng.random(n) - 0.5), Column.from_data(rng.integers(0, 2**63, n, dtype=np.uint64))])
    params = AggregatorParams([0], [("sum", 1), ("min", 2), ("sum", 3), ("max", 4)], expected_groups=eg)
    check(monkeypatch, blk, params, {2: ("sum", 3)})


@pytest.mark.parametrize("ns", [7, 8])
def test_seven_and_eight_slots(monkeypatch, ns):
    # 24-row blocks: the two buffers of 32 rows each would not fit for every warp
    assert warp_rows(ns) == 24
    rng = np.random.default_rng(37 + ns)
    pools, eg = slice_keys(ns)  # count(*) and one sum per value column
    k = build_keys(pools, sizes_for(ns), rng)
    n = len(k)
    cols = [Column.from_data(k)]
    for j in range(1, ns - 1):
        cols.append(Column.from_data(rng.integers(-2**31 - 5, 2**31 + 5, n).astype(np.int64) * j))
    cols.append(Column.from_data(rng.standard_normal(n)))
    blk = DataBlock(cols)
    aggs = [("sum", j) for j in range(1, ns - 1)] + [("sum", ns - 1)]
    params = AggregatorParams([0], aggs, expected_groups=eg)
    check(monkeypatch, blk, params, {len(aggs) - 1: ("sum", ns - 1)})
