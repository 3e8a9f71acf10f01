"""Floating-point sum / avg / min / max on every aggregation path, checked against the exact per-group
reference of tests/float_agg_ref.py instead of the oracle's row-order sum.

Data (float_agg_ref.py): heavy cancellation, f32 arguments with full mantissas and f32 subnormals,
dedicated groups for NaN (sign bit, payload), infinities, all -0.0, both zeros, f64 subnormals, overflow
pairs, NULL-only arguments and a small contribution next to a large one, and a group-size spread from
one group with half of the rows down to groups of one row.  Every plan is sum, avg, min, max and
count of one Float64 or Float32 argument plus count(*), behind the filter `v % 5 <> 0`.

Per result: group keys, count columns and validity equal the C oracle exactly; sum and avg lie within
the proven rounding bound of the exact sum; min and max equal the device rule bit for bit (-0.0 orders
below +0.0, a NaN result is the canonical quiet NaN), so every path gives the same min / max columns.
The two-pass, ring and pinned-gather paths read columns without validity bitmaps only; they run the
datasets with every argument non-NULL, where the NULL-only group's NaN values count.  Where the operator
reports its path (`kernel_variant()`), the test asserts it."""
import ctypes as C

import numpy as np
import pytest

import float_agg_ref as R
from databend_b200 import abi, expr as E
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import (AggregatorParams, TransformFinalAggregate, TransformPartialAggregate, schema_types,
                                      to_device)

pytestmark = pytest.mark.gpu

FILT = E.ne(E.col(1) % E.lit(R.FILTER_MOD), E.lit(0))
ARG_COL = {"x": 2, "y": 3}
DATASETS = {"cancellation": R.cancellation_dataset, "spread": R.spread_dataset, "specials": R.specials_dataset}
_datasets, _refs = {}, {}


@pytest.fixture(autouse=True)
def _device(gpu):
    """the library is built and a device is present"""


def dataset(name):
    if name not in _datasets:
        _datasets[name] = DATASETS[name]()
    return _datasets[name]


def plan(col, expected_groups=0, group=True):
    c = ARG_COL[col] if isinstance(col, str) else col
    return AggregatorParams([0] if group else [], [("sum", c), ("avg", c), ("min", c), ("max", c), ("count", c), ("count", None)],
                            expected_groups=expected_groups)


def block(ds, nullable=True):
    return DataBlock([Column.from_data(ds["k"]), Column.from_data(ds["v"]),
                      Column.from_data(ds["x"], validity=ds["xv"] if nullable else None),
                      Column.from_data(ds["y"], validity=ds["yv"] if nullable else None)])


def on_device(blocks):
    return [DataBlock([to_device(c) for c in b.columns], b.num_rows) for b in blocks]


def key_image(values):
    """integer image of a group key column: integers as Int64, floats as their bits with one NaN"""
    if values.dtype == np.float64:
        return np.where(np.isnan(values), np.int64(0x7FF8000000000000), values.view(np.int64))
    if values.dtype == np.float32:
        return np.where(np.isnan(values), 0x7FC00000, values.view(np.uint32).astype(np.int64))
    return values.astype(np.int64)


def aggregate(blocks, params, filt, types, n_partials=1):
    """Filter -> n_partials partials (blocks dealt round robin) -> final; also the partials' variant texts"""
    parts = [TransformPartialAggregate(params, types, filt) for _ in range(n_partials)]
    fin = TransformFinalAggregate(params, types)
    try:
        for i, b in enumerate(blocks):
            parts[i % n_partials].transform(b)
        variants = [p.kernel_variant() for p in parts]
        for p in parts:
            fin.transform(p.on_finish())
        return fin.on_finish()[0], variants
    finally:
        for op in parts + [fin]:
            op.close()


def verify(out, blk, params, filt, label):
    """`out` against the oracle (keys, counts, validity) and the exact reference (sum, avg, min, max).
    `label` names blk's contents: the exact reference is cached under it.  Returns the min / max bits."""
    from oracle import oracle as orc
    n_aggs, grouped = len(params.aggregate_functions), bool(params.group_columns)
    got_keys = key_image(out.columns[n_aggs].values()) if grouped else np.zeros(out.num_rows, dtype=np.int64)
    assert len(np.unique(got_keys)) == out.num_rows, "a group appears twice"
    rk, _, ra, rav, _ = orc.filter_group_agg(blk, params.to_c(filt), threads=8)
    if not grouped:
        exp_keys = np.zeros(len(ra[0]), dtype=np.int64)
    elif blk.columns[0].dtype == abi.F32:  # the oracle keeps an f32 key's bits in the low half of its word
        exp_keys = key_image(rk[0].astype(np.uint32).view(np.float32))
    else:
        exp_keys = key_image(rk[0].view(np.float64) if blk.columns[0].dtype == abi.F64 else rk[0].view(np.int64))
    pos = {int(k): i for i, k in enumerate(exp_keys)}
    assert sorted(pos) == sorted(got_keys.tolist())
    order = np.array([pos[int(k)] for k in got_keys], dtype=np.int64)
    filt_rows = blk.columns[1].values() % R.FILTER_MOD != 0 if filt is not None else np.ones(blk.num_rows, dtype=bool)
    row_keys = key_image(blk.columns[0].values()) if grouped else np.zeros(blk.num_rows, dtype=np.int64)
    images = []
    for a, (kind, c) in enumerate(params.aggregate_functions):
        col = out.columns[a]
        valid = col.valid_mask()
        np.testing.assert_array_equal(valid, rav[a][order], err_msg=f"validity of {kind}({c})")
        if kind == "count":
            np.testing.assert_array_equal(col.values(), ra[a][order], err_msg=f"count({c})")
            continue
        arg = blk.columns[c]
        if (label, c) not in _refs:
            _refs[(label, c)] = R.exact_reference(row_keys, arg.values(), filt_rows & arg.valid_mask())
        ref = _refs[(label, c)]
        got = {int(k): (v if ok else None) for k, v, ok in zip(got_keys, col.values(), valid)}
        if kind == "sum":
            errors = R.sum_violations(ref, got)
        elif kind == "avg":
            errors = R.avg_violations(ref, got)
        else:
            errors = R.minmax_violations(ref, got, kind, zeros="device", got_dtype=col.values().dtype)
            bits = col.values().view(np.uint64 if col.values().dtype.itemsize == 8 else np.uint32)
            images.append({int(k): int(b) for k, b, ok in zip(got_keys, bits, valid) if ok})
        assert errors == [], f"{kind}({c}) on {label}:\n" + "\n".join(errors)
    return images


def run(label, blocks, blk, params, filt=FILT, n_partials=1):
    out, variants = aggregate(blocks, params, filt, schema_types(blk), n_partials)
    return verify(out, blk, params, filt, label), variants


# ---------------------------------------------------------------- 1. one-pass fused kernel
@pytest.mark.parametrize("name", list(DATASETS))
@pytest.mark.parametrize("resident", ["host", "device"])
@pytest.mark.parametrize("jit", ["1", "0"])
def test_one_pass_fused(monkeypatch, name, resident, jit):
    monkeypatch.setenv("DBX_AGG_JIT", jit)
    ds = dataset(name)
    blk = block(ds)
    blocks = blk.split_by_rows(65536)
    if resident == "device":
        blocks = on_device(blocks)
    for col in ("x", "y"):
        _, variants = run(name, blocks, blk, plan(col))
        v = variants[0]
        assert v.startswith("specialised") if jit == "1" else v.startswith("off (DBX_AGG_JIT=0)"), v
        assert "two-pass" not in v, v


def test_constant_float_arguments():
    """sum(const) adds the constant once per row (aggregate_sum.rs:121-125): 0.1 is inexact, -0.0 sums to +0.0"""
    ds = dataset("cancellation")
    n = len(ds["k"])
    blk = DataBlock([Column.from_data(ds["k"]), Column.from_data(ds["v"]), Column.new_const(abi.F64, 0.1, n),
                     Column.new_const(abi.F64, -0.0, n)])
    for c in (2, 3):
        for blocks in (blk.split_by_rows(65536), [blk]):
            run("const", blocks, blk, plan(c))


# ---------------------------------------------------------------- 2. hot-group cache
@pytest.mark.parametrize("hot", ["1", "0"])
def test_hot_group_cache_on_skewed_keys(monkeypatch, hot):
    monkeypatch.setenv("DBX_AGG_HOT", hot)
    blk = block(dataset("spread"))
    for col in ("x", "y"):
        run("spread", on_device([blk]), blk, plan(col))
        run("spread", blk.split_by_rows(100_000), blk, plan(col))


# ---------------------------------------------------------------- 3. / 4. two-pass path
def _force_two_pass(monkeypatch, jit="1"):
    monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "1")
    monkeypatch.setenv("DBX_AGG_PARTITION_ALWAYS", "1")
    monkeypatch.setenv("DBX_AGG_JIT", jit)


@pytest.mark.parametrize("name", ["cancellation", "specials"])
@pytest.mark.parametrize("jit", ["1", "0"])
def test_two_pass_shared_memory_slices(monkeypatch, name, jit):
    _force_two_pass(monkeypatch, jit)
    blk = block(dataset(name), nullable=False)
    for col in ("x", "y"):
        _, (v,) = run(name + "/non-null", on_device([blk]), blk, plan(col, expected_groups=8000))
        assert "(pass 2 in shared memory: 1, in L2 regions: 0)" in v, v
        assert f"specialised launches: pass 1 {jit} of 1, pass 2 {jit} of 1" in v, v


def test_two_pass_fill_limit_deferred_rows_and_growth(monkeypatch):
    """4 000 groups for a 2 048-slot table: the slice stops at its fill limit, the table grows and the
    deferred rows run through the fused kernel"""
    _force_two_pass(monkeypatch)
    blk = block(dataset("cancellation"), nullable=False)
    for col in ("x", "y"):
        _, (v,) = run("cancellation/non-null", on_device([blk]), blk, plan(col, expected_groups=1000))
        assert "(pass 2 in shared memory: 1, in L2 regions: 0)" in v, v


@pytest.mark.parametrize("name", ["cancellation", "specials"])
def test_two_pass_l2_regions(monkeypatch, name):
    _force_two_pass(monkeypatch)
    monkeypatch.setenv("DBX_AGG_REGION_BYTES", "65536")
    blk = block(dataset(name), nullable=False)
    for col in ("x", "y"):
        # 2^23 slots: more slices than pass 1 partitions into
        _, (v,) = run(name + "/non-null", on_device([blk]), blk, plan(col, expected_groups=2_100_000))
        assert "(pass 2 in shared memory: 0, in L2 regions: 1)" in v, v


# ---------------------------------------------------------------- 5. overflow and replay
@pytest.mark.parametrize("name", ["spread", "specials"])
def test_one_pass_overflow_and_replay(name):
    blk = block(dataset(name))
    for col in ("x", "y"):
        run(name, on_device([blk]), blk, plan(col, expected_groups=16))
        run(name, blk.split_by_rows(100_000), blk, plan(col, expected_groups=16))


# ---------------------------------------------------------------- 6. two f64 columns in one plan
@pytest.mark.parametrize("name", ["cancellation", "specials"])
def test_two_f64_columns_straight_line(monkeypatch, name):
    """sum, avg, min and max of two f64 columns next to count(*) in one specialised plan; device-resident 8-byte columns"""
    monkeypatch.setenv("DBX_AGG_JIT", "1")
    ds = dataset(name)
    blk = DataBlock([Column.from_data(ds["k"]), Column.from_data(ds["v"]), Column.from_data(ds["x"]),
                     Column.from_data(ds["y"].astype(np.float64))])
    params = AggregatorParams([0], [("sum", 2), ("avg", 2), ("min", 2), ("max", 2), ("count", None), ("sum", 3), ("avg", 3), ("min", 3)])
    _, (v,) = run(name + "/two-f64", on_device([blk]), blk, params)
    assert v.startswith("specialised"), v


# ---------------------------------------------------------------- 7. no GROUP BY
def test_no_group_by_ten_million_rows():
    """filter_single_agg_kernel: per-thread partials, warp shuffles, one atomic per warp"""
    ds = R.cancellation_dataset(n=10_000_000, groups=1, seed=7)
    blk = block(ds)
    for col in ("x", "y"):
        _, (v,) = run("1e7", on_device([blk]), blk, plan(col, group=False))
        assert v == "off (plan shape not specialised)", v
    blk = block(dataset("specials"))
    for col in ("x", "y"):  # NaN and both infinities in the one group: sum NaN, max the canonical NaN
        images, _ = run("specials/no-group", on_device([blk]), blk, plan(col, group=False))
        assert images[1][0] == R.NAN_BITS[np.dtype(np.float64 if col == "x" else np.float32)]


# ---------------------------------------------------------------- 8. merging partial results
@pytest.mark.parametrize("name", list(DATASETS))
def test_three_partials_merged(name):
    blk = block(dataset(name))
    for col in ("x", "y"):
        run(name, blk.split_by_rows(50_000), blk, plan(col), n_partials=3)
        run(name, on_device(blk.split_by_rows(70_000)), blk, plan(col), n_partials=3)


def _concat_results(outs, n_cols):
    return DataBlock([Column.from_data(np.concatenate([o.columns[i].values() for o in outs]), outs[0].columns[i].dtype,
                                       validity=np.concatenate([o.columns[i].valid_mask() for o in outs])) for i in range(n_cols)])


@pytest.mark.parametrize("name", ["cancellation", "specials"])
def test_partition_exchange_simulated_ranks(name):
    from databend_b200.lib import check, load
    L = load()
    world = 4
    blk = block(dataset(name))
    types = schema_types(blk)
    for col in ("x", "y"):
        params = plan(col)
        parts, runs = [], []
        for r in range(world):
            lo, hi = blk.num_rows * r // world, blk.num_rows * (r + 1) // world
            p = TransformPartialAggregate(params, types, FILT)
            p.transform(blk.slice(lo, hi))
            p.on_finish()
            rows_ptr, offs, rb = C.c_void_p(), (C.c_int64 * (world + 1))(), C.c_int32(0)
            check(L.dbx_agg_partial_partition(p.handle, world, C.byref(rows_ptr), offs, C.byref(rb)), p.handle)
            parts.append(p)
            runs.append((rows_ptr, list(offs), rb.value))
        outs = []
        for q in range(world):
            fin = TransformFinalAggregate(params, types)
            for rows_ptr, offs, rb in runs:
                fin.merge_rows(rows_ptr.value + offs[q] * rb, offs[q + 1] - offs[q])
            outs.append(fin.on_finish()[0])
            fin.close()
        for rows_ptr, _, _ in runs:
            check(L.dbx_device_free(0, rows_ptr))
        for p in parts:
            p.close()
        verify(_concat_results(outs, 7), blk, params, FILT, name)


@pytest.mark.parametrize("name", ["cancellation", "specials"])
def test_peer_exchange_simulated_ranks(name):
    from databend_b200.exchange import PeerExchange
    world = 4
    blk = block(dataset(name))
    types = schema_types(blk)
    for col in ("x", "y"):
        params = plan(col)
        parts = [TransformPartialAggregate(params, types, FILT) for _ in range(world)]
        fins = [TransformFinalAggregate(params, types) for _ in range(world)]
        xs = [PeerExchange(parts[r], r, world) for r in range(world)]
        for x in xs:
            x.connect_local(xs)
        for r in range(world):
            parts[r].transform(blk.slice(blk.num_rows * r // world, blk.num_rows * (r + 1) // world))
            parts[r].on_finish()
        for r in range(world):
            xs[r].scatter(parts[r])
        for r in range(world):
            parts[r].synchronize()  # one GPU: every scatter has run before a merge may spin
        for r in range(world):
            xs[r].merge(fins[r])
        outs = [f.on_finish()[0] for f in fins]
        for op in xs + parts + fins:
            op.close()
        verify(_concat_results(outs, 7), blk, params, FILT, name)


@pytest.mark.parametrize("name", ["cancellation", "specials"])
def test_spill_serialize_and_merge(name):
    """partial(A) -> serialize -> merge_serialized, partial(B) adopted directly"""
    blk = block(dataset(name))
    types = schema_types(blk)
    half = blk.num_rows // 2
    for col in ("x", "y"):
        params = plan(col)
        pa, pb = TransformPartialAggregate(params, types, FILT), TransformPartialAggregate(params, types, FILT)
        pa.transform(blk.slice(0, half))
        pb.transform(blk.slice(half, blk.num_rows))
        pa.on_finish()
        pb.on_finish()
        spill, _ = pa.serialize()
        fin = TransformFinalAggregate(params, types)
        fin.transform(pb)
        fin.merge_serialized(spill)
        out = fin.on_finish()[0]
        for op in (pa, pb, fin):
            op.close()
        verify(out, blk, params, FILT, name)


# ---------------------------------------------------------------- 9. pinned host blocks through the device gather
def test_small_pinned_host_blocks_gathered_by_the_device():
    from databend_b200 import lib
    L = lib.load()
    ds = dataset("specials")
    src = block(ds, nullable=False)
    n = src.num_rows
    ptrs, cols = [], []
    try:
        for c in src.columns:
            vals = c.values()
            p = C.c_void_p()
            lib.check(L.dbx_host_alloc(vals.nbytes, C.byref(p)))
            ptrs.append(p)
            arr = np.frombuffer((C.c_char * vals.nbytes).from_address(p.value), dtype=vals.dtype)
            arr[:] = vals
            cols.append(Column.from_data(arr))
        pinned = DataBlock(cols, n)
        for split in (65536, 9999):
            for col in ("x", "y"):
                run("specials/non-null", pinned.split_by_rows(split), src, plan(col))
    finally:
        for p in ptrs:
            L.dbx_host_free(p)


# ---------------------------------------------------------------- 10. float group keys
@pytest.mark.parametrize("key_dtype", [np.float64, np.float32])
def test_float_group_keys_with_real_valued_sums(key_dtype):
    """keys group by bit pattern except that every NaN is one group; -0.0 and +0.0 are two groups"""
    ds = dataset("spread")
    rng = np.random.default_rng(5)
    n = len(ds["k"])
    k = (ds["k"] * 0.25).astype(key_dtype)
    r = rng.random(n)
    k[r < 0.02] = np.nan
    k[(r >= 0.02) & (r < 0.03)] = -0.0
    k[(r >= 0.03) & (r < 0.035)] = np.inf
    k[(r >= 0.035) & (r < 0.04)] = -np.inf
    k[::997] = np.array([0x7FF8000000000123], dtype=np.uint64).view(np.float64)[0] if key_dtype == np.float64 else \
        np.array([0xFFC00123], dtype=np.uint32).view(np.float32)[0]
    blk = DataBlock([Column.from_data(k), Column.from_data(ds["v"]), Column.from_data(ds["x"], validity=ds["xv"]),
                     Column.from_data(ds["y"], validity=ds["yv"])])
    for col in ("x", "y"):
        run(f"float keys {np.dtype(key_dtype)}", blk.split_by_rows(100_000), blk, plan(col), n_partials=2)
        run(f"float keys {np.dtype(key_dtype)}", on_device([blk]), blk, plan(col))
