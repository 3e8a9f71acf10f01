"""Parity of the fused filter -> hash-aggregate CUDA path against the CPU oracle.

Modelled on the reference's differential tests
(src/query/service/tests/it/pipelines/filter/filter_executor.rs:18-70: random blocks + random
predicates, operator == evaluator) and on functions/tests/it/aggregates/agg_hashtable.rs:52-199.
Integer results are bit-exact; f64 sums are bit-exact on integer-valued data (< 2^53) and
within rtol 1e-12 otherwise (atomic accumulation order differs from the CPU's).
"""
import numpy as np
import pytest

from databend_b200 import abi, expr as E
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError
from databend_b200.transforms import (AggregatorParams, TransformFinalAggregate, TransformPartialAggregate,
                                      filter_group_aggregate, schema_types, to_device)
from helpers import assert_group_results_equal, sorted_group_result_from_block, sorted_group_result_from_oracle

pytestmark = pytest.mark.gpu


def oracle():
    from oracle import oracle as orc
    return orc


def run_both(block, params, filt, n_partials=1, split=None, device_resident=False, float_exact=True, rtol=0.0,
             input_types=None):
    orc = oracle()
    types = input_types or schema_types(block)
    blocks = [block] if not split else block.split_by_rows(split)
    if device_resident:
        blocks = [DataBlock([to_device(c) for c in b.columns], b.num_rows) for b in blocks]
    out = filter_group_aggregate(blocks, params, filt, input_types=types, n_partials=n_partials)
    ref = orc.filter_group_agg(block, params.to_c(filt), threads=4)
    n_aggs, n_keys = len(params.aggregate_functions), len(params.group_columns)
    g = sorted_group_result_from_block(out, n_aggs, n_keys)
    o = sorted_group_result_from_oracle(ref, [block.columns[c].dtype for c in params.group_columns])
    assert out.num_rows == (len(ref[2][0]) if ref[2] else len(ref[0][0]))
    assert_group_results_equal(g, o, float_exact=float_exact, rtol=rtol)
    return out


def config2_block(n, seed=42, n_keys=1000):
    orc = oracle()
    k = orc.synth_fill(0, seed, n_keys, 0, n)
    v = orc.synth_fill(1, seed + 1, 0, 0, n)
    x = orc.synth_fill(2, seed + 2, 20, 0, n)
    return DataBlock([Column.from_data(k), Column.from_data(v), Column.from_data(x)])


CONFIG2 = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2)])
V_MOD3 = E.eq(E.col(1) % E.lit(3), E.lit(0))


def test_config1_sum_numbers_mod3(gpu):
    """SELECT sum(number) FROM numbers(10000000) WHERE number % 3 = 0  ->  16666668333333"""
    n = 10_000_000
    blk = DataBlock([Column.from_data(np.arange(n, dtype=np.uint64))])
    params = AggregatorParams([], [("sum", 0)])
    out = run_both(blk, params, E.eq(E.col(0) % E.lit(3), E.lit(0)), split=65536 * 16)
    assert out.num_rows == 1
    assert int(out.columns[0].values()[0]) == 16666668333333
    assert out.columns[0].dtype == abi.U64 and out.columns[0].valid_mask()[0]


@pytest.mark.parametrize("n,n_keys", [(1, 1), (1000, 7), (65536, 1000), (300_001, 100_000), (2_000_000, 1_000_000)])
def test_config2_shape_host_blocks(gpu, n, n_keys):
    run_both(config2_block(n, n_keys=n_keys), CONFIG2, V_MOD3, split=65536)


def test_config2_device_resident_single_push(gpu):
    run_both(config2_block(3_000_000, n_keys=1_000_000), CONFIG2, V_MOD3, device_resident=True)


def test_config2_multiple_partials_merge(gpu):
    """max_threads copies of TransformPartialAggregate feeding one final (combine_payload)."""
    run_both(config2_block(500_000, n_keys=50_000), CONFIG2, V_MOD3, n_partials=3, split=65536)


def test_agg_hashtable_golden(gpu):
    """functions/tests/it/aggregates/agg_hashtable.rs:52-199: keys x % 4, two tables combined:
    min [0,1,2,3], max [0,1,2,3], sum [0, n/2, n, 3n/2], count n/2."""
    for n in [100, 1000, 10_000, 100_000]:
        vals = (np.arange(n) % 4).astype(np.int64)
        blk = DataBlock([Column.from_data(vals)])
        params = AggregatorParams([0], [("min", 0), ("max", 0), ("sum", 0), ("count", 0)])
        types = schema_types(blk)
        p1 = TransformPartialAggregate(params, types)
        p2 = TransformPartialAggregate(params, types)
        p1.transform(blk)
        p2.transform(blk)
        fin = TransformFinalAggregate(params, types)
        fin.transform(p1.on_finish())
        fin.transform(p2.on_finish())
        out = fin.on_finish()[0]
        g = sorted_group_result_from_block(out, 4, 1)
        np.testing.assert_array_equal(g["keys"][0], [0, 1, 2, 3])
        np.testing.assert_array_equal(g["aggs"][0], [0, 1, 2, 3])
        np.testing.assert_array_equal(g["aggs"][1], [0, 1, 2, 3])
        np.testing.assert_array_equal(g["aggs"][2], [0, n // 2, n, n // 2 * 3])
        np.testing.assert_array_equal(g["aggs"][3], [n // 2] * 4)
        assert g["aggs"][3].dtype == np.uint64 and g["aggs"][2].dtype == np.int64


def test_empty_input(gpu):
    blk = config2_block(1000)
    types = schema_types(blk)
    out = filter_group_aggregate([blk.slice(0, 0)], CONFIG2, V_MOD3, input_types=types)
    assert out.num_rows == 0
    # no GROUP BY over nothing: one row, sum NULL, count 0 (transform_single_key.rs)
    params = AggregatorParams([], [("sum", 1), ("count", 1)])
    out = filter_group_aggregate([blk.slice(0, 0)], params, None, input_types=types)
    assert out.num_rows == 1
    assert not out.columns[0].valid_mask()[0]
    assert int(out.columns[1].values()[0]) == 0


def test_all_rows_filtered_out(gpu):
    blk = config2_block(10_000)
    out = run_both(blk, CONFIG2, E.gt(E.col(1), E.lit(2**40)))
    assert out.num_rows == 0


def test_nullable_args_and_keys(gpu):
    rng = np.random.default_rng(7)
    n = 200_000
    k = rng.integers(-50, 50, n).astype(np.int64)
    kv = rng.random(n) > 0.1
    v = rng.integers(-2**62, 2**62, n).astype(np.int64)
    vv = rng.random(n) > 0.3
    x = rng.integers(0, 2**20, n).astype(np.float64)
    xv = rng.random(n) > 0.5
    blk = DataBlock([Column.from_data(k, validity=kv), Column.from_data(v, validity=vv, validity_bit_offset=3),
                     Column.from_data(x, validity=xv)])
    params = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2), ("min", 1), ("max", 2), ("count", None)])
    run_both(blk, params, None, split=50_000)
    run_both(blk, params, E.and_(E.ne(E.col(1) % E.lit(7), E.lit(0)), E.lt(E.col(2), E.lit(600000.0))), split=77_777)


def test_all_null_group_gives_null_sum(gpu):
    """sum(all_null) -> NULL, count -> 0 (testdata/sum.txt, count.txt `all_null`)."""
    blk = DataBlock([Column.from_data(np.array([0, 1, 0, 1], dtype=np.int64)),
                     Column.from_data(np.array([1, 2, 3, 4], dtype=np.uint64), validity=[False] * 4)])
    params = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 1)])
    out = run_both(blk, params, None)
    assert not out.columns[0].valid_mask().any()
    np.testing.assert_array_equal(out.columns[1].values(), [0, 0])


def test_wrapping_integer_sum(gpu):
    """Release builds wrap on i64/u64 overflow (Cargo.toml:577)."""
    v = np.array([2**63 - 1, 2**63 - 1, 5, -(2**63)], dtype=np.int64)
    u = np.array([2**64 - 1, 2**64 - 1, 7, 1], dtype=np.uint64)
    blk = DataBlock([Column.from_data(np.zeros(4, dtype=np.int64)), Column.from_data(v), Column.from_data(u)])
    params = AggregatorParams([0], [("sum", 1), ("sum", 2), ("avg", 1)])
    run_both(blk, params, None)


@pytest.mark.parametrize("dtype", [abi.I8, abi.I16, abi.I32, abi.U8, abi.U16, abi.U32, abi.U64, abi.F32, abi.F64])
def test_argument_dtypes(gpu, dtype):
    from databend_b200.block import np_dtype
    rng = np.random.default_rng(dtype)
    n = 100_003
    nd = np_dtype(dtype)
    if nd.kind == "f":
        vals = rng.integers(-1000, 1000, n).astype(nd)  # integer-valued: sums exact in any order
    else:
        info = np.iinfo(nd)
        vals = rng.integers(info.min, info.max, n, dtype=nd, endpoint=True)
    k = rng.integers(0, 1000, n).astype(np.int32)
    blk = DataBlock([Column.from_data(k), Column.from_data(vals)])
    params = AggregatorParams([0], [("sum", 1), ("avg", 1), ("min", 1), ("max", 1), ("count", 1)])
    run_both(blk, params, None, split=30_000)


def test_key_dtypes_and_sentinel_key(gpu):
    """i64::MIN is the table's EMPTY sentinel: it must still be a legal group key."""
    k = np.array([-(2**63), 5, -(2**63), 2**63 - 1, 5, 0], dtype=np.int64)
    v = np.arange(6, dtype=np.int64)
    run_both(DataBlock([Column.from_data(k), Column.from_data(v)]), AggregatorParams([0], [("sum", 1), ("count", None)]), None)
    ku = np.array([2**63, 5, 2**63, 2**64 - 1], dtype=np.uint64)
    run_both(DataBlock([Column.from_data(ku), Column.from_data(v[:4])]), AggregatorParams([0], [("sum", 1)]), None)


def test_const_columns(gpu):
    """BlockEntry::Const arguments are not materialised (sum(const_int) -> 20, testdata/sum.txt)."""
    blk = DataBlock([Column.from_data(np.array([4, 3, 2, 1], dtype=np.int64)), Column.new_const(abi.I32, 5, 4),
                     Column.new_const(abi.I32, None, 4)])
    types = [abi.I64, abi.I32, abi.I32 | abi.NULLABLE]
    params = AggregatorParams([], [("sum", 1), ("sum", 2), ("count", 2), ("count", 1)])
    out = run_both(blk, params, None, input_types=types)
    assert int(out.columns[0].values()[0]) == 20
    assert not out.columns[1].valid_mask()[0]
    assert int(out.columns[2].values()[0]) == 0 and int(out.columns[3].values()[0]) == 4


def test_predicate_shapes(gpu):
    rng = np.random.default_rng(3)
    n = 150_000
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    b = rng.integers(-1000, 1000, n).astype(np.int64)
    f = rng.normal(size=n)
    f[rng.random(n) < 0.01] = np.nan
    u = rng.integers(0, 2**64 - 1, n, dtype=np.uint64)
    flag = rng.random(n) < 0.5
    blk = DataBlock([Column.from_data(a), Column.from_data(b, validity=rng.random(n) > 0.2), Column.from_data(f),
                     Column.from_data(u), Column.from_data(flag, abi.BOOL)])
    params = AggregatorParams([0], [("sum", 1), ("count", None), ("max", 3)])
    preds = [
        E.eq(E.col(0) % E.lit(3), E.lit(0)),
        E.eq(E.col(0) % E.lit(-7), E.lit(-2, abi.I64)),
        E.lt(E.col(0), E.col(1)),
        E.ge(E.col(2), E.lit(0.25)),
        E.gt(E.col(2), E.lit(float("nan"))),  # NaN is the greatest value: nothing is greater
        E.eq(E.col(2), E.lit(float("nan"))),  # all NaNs are equal
        E.and_(E.ne(E.col(0), E.lit(5)), E.le(E.col(1), E.lit(100)), E.gt(E.col(3) % E.lit(10), E.lit(4))),
        E.or_(E.lt(E.col(0), E.lit(-900, abi.I64)), E.and_(E.bool_column(4), E.gt(E.col(1), E.lit(990)))),
        E.or_(E.bool_scalar(False), E.eq(E.lit(3), E.col(0))),
        E.lt(E.col(0), E.lit(2**63 + 5)),
        E.ge(E.col(3), E.lit(-1, abi.I64)),
    ]
    for p in preds:
        run_both(blk, params, p, split=40_000)


def test_division_by_zero_is_an_error(gpu):
    """arithmetic_modulo.rs:137-140: literal divisor 0 -> 'Division by zero' (BadArguments)."""
    blk = config2_block(100)
    with pytest.raises(DbxError) as ei:
        filter_group_aggregate([blk], CONFIG2, E.eq(E.col(1) % E.lit(0), E.lit(0)))
    assert ei.value.status == abi.ERR_BAD_ARGUMENTS and "Division by zero" in ei.value.message


def test_modulo_edge_values(gpu):
    """MIN % -1 = 0; sign follows the dividend."""
    a = np.array([-(2**63), -(2**63) + 1, -7, -1, 0, 1, 7, 2**63 - 1], dtype=np.int64)
    blk = DataBlock([Column.from_data(a)])
    params = AggregatorParams([0], [("count", None)])
    for d in [1, -1, 2, -2, 3, 7, -7, 2**31, 2**62, -(2**63), 2**63 - 1, 10**18, 6700417]:
        for rhs in [0, 1, -1, 2, -3]:
            run_both(blk, params, E.eq(E.col(0) % E.lit(d, abi.I64), E.lit(rhs, abi.I64)))


def test_table_growth_from_small_hint(gpu):
    """expected_groups far too small: the table must grow (resize) without losing rows."""
    blk = config2_block(400_000, n_keys=300_000)
    params = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2)], expected_groups=16)
    run_both(blk, params, V_MOD3, split=100_000)
    run_both(blk, params, None, device_resident=True)


def test_float_sum_tolerance(gpu):
    rng = np.random.default_rng(11)
    n = 200_000
    blk = DataBlock([Column.from_data(rng.integers(0, 100, n).astype(np.int64)), Column.from_data(rng.random(n))])
    params = AggregatorParams([0], [("sum", 1), ("avg", 1)])
    run_both(blk, params, None, float_exact=False, rtol=1e-12)


def test_operator_reset_reuse(gpu):
    blk = config2_block(100_000, n_keys=5_000)
    types = schema_types(blk)
    part = TransformPartialAggregate(CONFIG2, types, V_MOD3)
    fin = TransformFinalAggregate(CONFIG2, types)
    ref = None
    for _ in range(3):
        part.reset()
        fin.reset()
        part.transform(blk)
        fin.transform(part.on_finish())
        out = fin.on_finish()[0]
        g = sorted_group_result_from_block(out, 3, 1)
        if ref is None:
            ref = g
        else:
            assert_group_results_equal(g, ref)
    o = sorted_group_result_from_oracle(oracle().filter_group_agg(blk, CONFIG2.to_c(V_MOD3), 2), [abi.I64])
    assert_group_results_equal(ref, o)


def test_schema_mismatch_is_rejected(gpu):
    blk = config2_block(10)
    part = TransformPartialAggregate(CONFIG2, schema_types(blk), V_MOD3)
    with pytest.raises(DbxError):
        part.transform(DataBlock([blk.columns[0]]))
    with pytest.raises(DbxError):
        TransformPartialAggregate(AggregatorParams([0], [("median", 1)]), schema_types(blk))


def test_partition_exchange_merge_simulated_ranks(gpu):
    """The N>1 path on ONE GPU: N row-range partials -> hash-partition each into N owner runs ->
    final r merges run r of every partial (what the NCCL all-to-all delivers) -> the union of the
    finals equals the oracle.  Also checks the device owner rule against the host restatement."""
    import ctypes as C
    from databend_b200.exchange import owner_of
    from databend_b200.lib import check, load
    from databend_b200.transforms import DeviceBuffer
    L = load()
    world = 4
    blk = config2_block(600_000, n_keys=40_000)
    blk.columns[0].data[:7] = -(2**63)  # the sentinel-valued key travels through the exchange too
    types = schema_types(blk)
    parts, runs = [], []
    for r in range(world):
        lo, hi = blk.num_rows * r // world, blk.num_rows * (r + 1) // world
        p = TransformPartialAggregate(CONFIG2, types, V_MOD3)
        p.transform(blk.slice(lo, hi))
        p.on_finish()
        rows_ptr, offs, rb = C.c_void_p(), (C.c_int64 * (world + 1))(), C.c_int32(0)
        check(L.dbx_agg_partial_partition(p.handle, world, C.byref(rows_ptr), offs, C.byref(rb)), p.handle)
        total = offs[world]
        host = np.empty(total * rb.value // 8, dtype=np.uint64)
        check(L.dbx_memcpy_d2h(0, host.ctypes.data, rows_ptr, total * rb.value))
        host = host.reshape(total, rb.value // 8)
        for q in range(world):
            seg = host[offs[q]:offs[q + 1]]
            assert (owner_of(seg[:, 0], seg[:, 1], world) == q).all()
        parts.append(p)
        runs.append((rows_ptr, list(offs), rb.value))
    outs = []
    for q in range(world):
        fin = TransformFinalAggregate(CONFIG2, types)
        for (rows_ptr, offs, rb) in runs:
            n = offs[q + 1] - offs[q]
            fin.merge_rows(rows_ptr.value + offs[q] * rb, n)
        outs.append(fin.on_finish()[0])
        fin.close()
    for (rows_ptr, _, _) in runs:
        check(L.dbx_device_free(0, rows_ptr))
    merged = DataBlock([Column.from_data(np.concatenate([o.columns[i].values() for o in outs]), outs[0].columns[i].dtype,
                                         validity=np.concatenate([o.columns[i].valid_mask() for o in outs]))
                        for i in range(4)])
    g = sorted_group_result_from_block(merged, 3, 1)
    o = sorted_group_result_from_oracle(oracle().filter_group_agg(blk, CONFIG2.to_c(V_MOD3), 4), [abi.I64])
    assert_group_results_equal(g, o)


def test_peer_memory_exchange_simulated_ranks(gpu):
    """The peer-memory exchange (scatter straight into the owners' receive regions + flag-gated
    merge) with N ranks simulated on ONE GPU: three consecutive queries (epochs alternate the
    region parity), each checked against the oracle; every group lands on exactly its owner."""
    from databend_b200.exchange import PeerExchange, owner_of
    world = 4
    types = None
    parts, fins, xs = [], [], []
    blk0 = config2_block(10, n_keys=5)
    types = schema_types(blk0)
    for r in range(world):
        parts.append(TransformPartialAggregate(CONFIG2, types, V_MOD3))
        fins.append(TransformFinalAggregate(CONFIG2, types))
    for r in range(world):
        xs.append(PeerExchange(parts[r], r, world))
    for r in range(world):
        xs[r].connect_local(xs)
    for epoch, (rows, keys) in enumerate([(400_000, 30_000), (250_000, 90_000), (123_457, 1_000)]):
        blk = config2_block(rows, n_keys=keys, seed=100 + epoch)
        blk.columns[0].data[:3] = -(2**63)  # sentinel-valued key
        for r in range(world):
            parts[r].reset()
            fins[r].reset()
            lo, hi = rows * r // world, rows * (r + 1) // world
            parts[r].transform(blk.slice(lo, hi))
            parts[r].on_finish()
        for r in range(world):
            xs[r].scatter(parts[r])
        for r in range(world):
            parts[r].synchronize()  # one GPU: all scatters must have run before a merge may spin
        for r in range(world):
            xs[r].merge(fins[r])
        outs = [fins[r].on_finish()[0] for r in range(world)]
        for r, o in enumerate(outs):
            k = o.columns[3].values()
            kind = np.where(k == -(2**63), 1, 0)
            assert (owner_of(k.view(np.uint64), kind, world) == r).all()
        merged = DataBlock([Column.from_data(np.concatenate([o.columns[i].values() for o in outs]), outs[0].columns[i].dtype,
                                             validity=np.concatenate([o.columns[i].valid_mask() for o in outs]))
                            for i in range(4)])
        g = sorted_group_result_from_block(merged, 3, 1)
        o = sorted_group_result_from_oracle(oracle().filter_group_agg(blk, CONFIG2.to_c(V_MOD3), 4), [abi.I64])
        assert_group_results_equal(g, o)
    for x in xs:
        x.close()
    for p in parts + fins:
        p.close()


def test_peer_memory_exchange_region_overflow_is_loud(gpu):
    """A receive region that is too small must fail the query, never drop groups silently."""
    from databend_b200.exchange import PeerExchange
    from databend_b200.lib import DbxError
    blk = config2_block(100_000, n_keys=20_000)
    types = schema_types(blk)
    p = TransformPartialAggregate(CONFIG2, types, V_MOD3)
    f = TransformFinalAggregate(CONFIG2, types)
    x = PeerExchange(p, 0, 1, region_rows=64)
    x.connect_local([x])
    p.transform(blk)
    p.on_finish()
    x.scatter(p)
    x.merge(f)
    with pytest.raises(DbxError, match="receive region"):
        f.on_finish()
    x.close()
    p.close()
    f.close()


def _group_dict(key_vals, key_valid, agg_vals, agg_valid):
    out = {}
    n = len(agg_vals[0]) if agg_vals else len(key_vals[0])
    for i in range(n):
        k = tuple((int(v[i]) if ok[i] else None) for v, ok in zip(key_vals, key_valid))
        assert k not in out, f"group {k} appears twice"
        out[k] = tuple((a[i].item() if ok[i] else None) for a, ok in zip(agg_vals, agg_valid))
    return out


@pytest.mark.parametrize("device_resident", [False, True])
def test_multi_column_group_keys(gpu, device_resident):
    """GROUP BY (a Int32, b Nullable(Int16), c UInt8): the key columns are packed into one 64-bit
    word (HashMethodKeysU64, kernels/group_by.rs:66-79); NULL is a group value of its own
    (payload_row.rs NULL rules) and (NULL, x) differs from (0, x).  Parity with the oracle on
    keys, validity and every aggregate; also through two partials + final merge."""
    rng = np.random.default_rng(77)
    n = 300_000
    a = rng.integers(-40, 40, n).astype(np.int32)
    b = rng.integers(-3, 3, n).astype(np.int16)
    c = rng.integers(0, 5, n).astype(np.uint8)
    v = rng.integers(-2**40, 2**40, n).astype(np.int64)
    x = rng.integers(0, 1 << 20, n).astype(np.float64)
    bvalid = rng.random(n) > 0.15
    blk = DataBlock([Column.from_data(a), Column.from_data(b, validity=bvalid), Column.from_data(c), Column.from_data(v),
                     Column.from_data(x, validity=rng.random(n) > 0.1)])
    params = AggregatorParams([0, 1, 2], [("sum", 3), ("count", None), ("avg", 4), ("min", 3), ("max", 4)])
    filt = E.ne(E.col(3) % E.lit(5), E.lit(0))
    blocks = blk.split_by_rows(70_001)
    if device_resident:
        blocks = [DataBlock([to_device(col) for col in bb.columns], bb.num_rows) for bb in blocks]
    out = filter_group_aggregate(blocks, params, filt, input_types=schema_types(blk), n_partials=2)
    keys, kvalid, aggs, avalid, _ = oracle().filter_group_agg(blk, params.to_c(filt), threads=4)
    exp = _group_dict([keys[0].view(np.int64), keys[1].view(np.int64), keys[2].view(np.int64)], kvalid, aggs, avalid)
    assert out.num_columns() == 5 + 3
    gk = [out.columns[5 + j] for j in range(3)]
    assert [k.dtype for k in gk] == [abi.I32, abi.I16, abi.U8]
    got = _group_dict([k.values().astype(np.int64) for k in gk], [k.valid_mask() for k in gk],
                      [out.columns[i].values() for i in range(5)], [out.columns[i].valid_mask() for i in range(5)])
    assert got.keys() == exp.keys()
    for k in exp:
        assert got[k] == exp[k], (k, got[k], exp[k])
    assert any(k[1] is None for k in exp) and any(k[1] == 0 for k in exp)


def test_multi_column_keys_too_wide_is_loud(gpu):
    from databend_b200.lib import DbxError
    cols = [Column.from_data(np.arange(4, dtype=np.int64)) for _ in range(3)]
    blk = DataBlock(cols)
    with pytest.raises(DbxError, match="wider than 128 bits"):
        TransformPartialAggregate(AggregatorParams([0, 1, 2], [("count", None)]), schema_types(blk))
    # 128 value bits + one NULL flag do not fit either
    blk2 = DataBlock([cols[0], Column.from_data(np.arange(4, dtype=np.int64), validity=[True, False, True, True])])
    with pytest.raises(DbxError, match="wider than 128 bits"):
        TransformPartialAggregate(AggregatorParams([0, 1], [("count", None)]), schema_types(blk2))


def _check_multi_key(blk, key_cols, params, filt, key_dtypes, n_partials=1, split=None, device_resident=False, expected_groups=None):
    blocks = blk.split_by_rows(split) if split else [blk]
    if device_resident:
        blocks = [DataBlock([to_device(col) for col in bb.columns], bb.num_rows) for bb in blocks]
    out = filter_group_aggregate(blocks, params, filt, input_types=schema_types(blk), n_partials=n_partials)
    keys, kvalid, aggs, avalid, _ = oracle().filter_group_agg(blk, params.to_c(filt), threads=4)
    exp = _group_dict([k.view(np.int64) for k in keys], kvalid, aggs, avalid)
    na, nk = len(params.aggregate_functions), len(key_cols)
    gk = [out.columns[na + j] for j in range(nk)]
    assert [k.dtype for k in gk] == key_dtypes
    got = _group_dict([k.values().astype(np.int64) if k.dtype != abi.U64 else k.values().view(np.int64) for k in gk], [k.valid_mask() for k in gk],
                      [out.columns[i].values() for i in range(na)], [out.columns[i].valid_mask() for i in range(na)])
    assert got.keys() == exp.keys()
    for k in exp:
        assert got[k] == exp[k], (k, got[k], exp[k])
    if expected_groups is not None:
        assert len(exp) == expected_groups
    return exp


@pytest.mark.parametrize("device_resident", [False, True])
def test_wide_128_bit_group_keys(gpu, device_resident):
    """GROUP BY keys that need 65..128 bits are packed into TWO key words (HashMethodKeysU128,
    kernels/group_by.rs:66-79): buckets of two 16-byte keys, one 128-bit compare-and-swap per new
    group.  (Int64, Nullable(Int32), Int16) = 113 bits, with a filter, several partials and host /
    device blocks; then (Int64, UInt64) = exactly 128 bits including the key whose two words both
    equal the EMPTY pattern, and a table that has to grow from a tiny size hint."""
    rng = np.random.default_rng(123)
    n = 400_000
    a = rng.integers(-2**62, 2**62, 300).astype(np.int64)[rng.integers(0, 300, n)]
    b = rng.integers(-4, 4, n).astype(np.int32)
    c = rng.integers(0, 3, n).astype(np.int16)
    v = rng.integers(-2**40, 2**40, n).astype(np.int64)
    x = rng.integers(0, 1 << 20, n).astype(np.float64)
    blk = DataBlock([Column.from_data(a), Column.from_data(b, validity=rng.random(n) > 0.1), Column.from_data(c), Column.from_data(v),
                     Column.from_data(x, validity=rng.random(n) > 0.2)])
    params = AggregatorParams([0, 1, 2], [("sum", 3), ("count", None), ("avg", 4), ("min", 3), ("max", 4)])
    exp = _check_multi_key(blk, [0, 1, 2], params, E.ne(E.col(3) % E.lit(5), E.lit(0)), [abi.I64, abi.I32, abi.I16],
                           n_partials=2, split=90_001, device_resident=device_resident)
    assert any(k[1] is None for k in exp) and any(k[1] == 0 for k in exp)
    # exactly 128 bits, 200k distinct groups: growth from the default size, the EMPTY-pattern key
    m = 500_000
    k0 = rng.integers(0, 200_000, m).astype(np.int64) * 1_000_003
    k1 = (k0.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) ^ np.uint64(12345)
    k0[:7] = np.int64(-2**63)
    k1[:7] = np.uint64(2**63)
    k0[7:9] = np.int64(-2**63)   # same first word, different second word: a different group
    k1[7:9] = np.uint64(5)
    blk2 = DataBlock([Column.from_data(k0), Column.from_data(k1), Column.from_data(rng.integers(-100, 100, m).astype(np.int64))])
    params2 = AggregatorParams([0, 1], [("sum", 2), ("count", None)], expected_groups=64)
    exp2 = _check_multi_key(blk2, [0, 1], params2, None, [abi.I64, abi.U64], split=65536, device_resident=device_resident)
    assert exp2[(-2**63, -2**63)][1] == 7 and exp2[(-2**63, 5)][1] == 2


def test_wide_keys_do_not_cross_the_row_exchange(gpu):
    """The exchange / spill rows carry 64-bit keys: asking for them with 128-bit keys is an error, not a wrong answer."""
    from databend_b200.lib import DbxError
    blk = DataBlock([Column.from_data(np.arange(10, dtype=np.int64)), Column.from_data(np.arange(10, dtype=np.int64))])
    part = TransformPartialAggregate(AggregatorParams([0, 1], [("count", None)]), schema_types(blk))
    part.transform(blk)
    part.on_finish()
    with pytest.raises(DbxError, match="128-bit packed group keys"):
        part.serialize()
    part.close()


def test_device_resident_sums_count_avg_minmax(gpu):
    """sum(v), count(*), sum(x), avg(x2), min(v), max(x) over device columns through the straight-line
    kernel: integer and f64 sums next to min / max words in one row-major entry."""
    rng = np.random.default_rng(3)
    n = 1_500_000
    k = rng.integers(0, 20_000, n).astype(np.int64)
    v = rng.integers(-2**40, 2**40, n).astype(np.int64)
    x = rng.integers(0, 1 << 20, n).astype(np.float64)
    x2 = rng.integers(0, 1 << 18, n).astype(np.float64)
    blk = DataBlock([Column.from_data(k), Column.from_data(v), Column.from_data(x), Column.from_data(x2)])
    params = AggregatorParams([0], [("sum", 1), ("count", None), ("sum", 2), ("avg", 3), ("min", 1), ("max", 2)])
    run_both(blk, params, E.ne(E.col(1) % E.lit(7), E.lit(0)), device_resident=True)
    run_both(blk, params, None, device_resident=True, split=400_000, n_partials=2)


def test_default_red_layout_device_resident(gpu):
    run_both(config2_block(1_200_000, n_keys=30_000), CONFIG2, V_MOD3, device_resident=True)
    # the sentinel-valued key in the first rows, and a ragged tail that the generic kernel finishes
    blk = config2_block(3_000_017, n_keys=70_000)
    blk.columns[0].data[:5] = -(2**63)
    run_both(blk, CONFIG2, V_MOD3, device_resident=True)


def test_full_size_query_verified(gpu):
    """BASELINE.json configs[1] at its full size (1e9 rows, 1e6 keys; a quarter of it if HBM is
    short): EVERY group of the result against an independent recomputation of the query (torch
    bincount / index_add_ over all rows) and the CPU oracle on every row of a key subsample —
    the check bench.py runs outside its timed region."""
    import ctypes as C
    import sys
    import torch
    import torch.distributed as dist
    sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
    import bench
    from databend_b200 import lib
    from databend_b200.transforms import DeviceBuffer
    L = lib.load()
    free, _total = torch.cuda.mem_get_info(0)
    n = 1_000_000_000 if free > 60e9 else 250_000_000
    n_keys = 1_000_000
    bufs = [DeviceBuffer(n * 8, 0) for _ in range(3)]
    lib.check(L.dbx_synth_fill(0, 0, bench.SEEDS[0], n_keys, 0, n, bufs[0].ptr))
    lib.check(L.dbx_synth_fill(0, 1, bench.SEEDS[1], 0, 0, n, bufs[1].ptr))
    lib.check(L.dbx_synth_fill(0, 2, bench.SEEDS[2], 20, 0, n, bufs[2].ptr))
    blk = DataBlock([Column.device(abi.I64, n, bufs[0].ptr), Column.device(abi.I64, n, bufs[1].ptr),
                     Column.device(abi.F64, n, bufs[2].ptr)], n)
    types = [abi.I64, abi.I64, abi.F64]
    part = TransformPartialAggregate(CONFIG2, types, V_MOD3)
    fin = TransformFinalAggregate(CONFIG2, types)
    part.transform(blk)
    fin.transform(part.on_finish())
    out = fin.on_finish()[0]
    v = bench.verify_result(out, 0, 0, 1, [b.ptr for b in bufs], n, n_keys, torch, dist)
    part.close(); fin.close()
    for b in bufs:
        b.free()
    assert v["ok"], v
    assert v["groups"] == v["expected_groups"] == n_keys
    assert v["oracle_subsample"]["bit_exact"]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("device_resident", [False, True])
def test_float_group_keys(gpu, dtype, device_resident):
    """GROUP BY a float column (group_hash.rs:599-619, payload_row.rs match on OrderedFloat): rows
    group by bit pattern, every NaN is ONE group (canonical NaN), -0.0 and +0.0 are separate groups
    (they hash differently in the reference), +-inf are ordinary keys.  Parity with the oracle."""
    rng = np.random.default_rng(11)
    n = 400_000
    k = (rng.integers(-200, 200, n) / 8.0).astype(dtype)
    k[rng.random(n) < 0.02] = np.nan
    k[rng.random(n) < 0.01] = -0.0
    k[rng.random(n) < 0.005] = np.inf
    k[rng.random(n) < 0.005] = -np.inf
    nan2 = np.array([0x7FF8000000000123], dtype=np.uint64).view(np.float64)[0] if dtype == np.float64 else np.array([0x7FC00123], dtype=np.uint32).view(np.float32)[0]
    k[::1000] = nan2  # a NaN with another payload: same group
    v = rng.integers(-2**40, 2**40, n).astype(np.int64)
    x = rng.integers(0, 1 << 20, n).astype(np.float64)
    blk = DataBlock([Column.from_data(k), Column.from_data(v), Column.from_data(x)])
    params = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2), ("min", 1)])
    filt = E.ne(E.col(1) % E.lit(5), E.lit(0))
    blocks = blk.split_by_rows(150_000)
    if device_resident:
        blocks = [DataBlock([to_device(c) for c in b.columns], b.num_rows) for b in blocks]
    out = filter_group_aggregate(blocks, params, filt, input_types=schema_types(blk), n_partials=2)
    keys, kvalid, aggs, avalid, _ = oracle().filter_group_agg(blk, params.to_c(filt), threads=4)
    w = np.uint64 if dtype == np.float64 else np.uint32
    exp = {int(kb): tuple(a[i].item() for a in aggs) for i, kb in enumerate(keys[0].astype(np.uint64))}
    gk = out.columns[4].values()
    assert gk.dtype == dtype
    got = {int(kb): tuple(out.columns[a].values()[i].item() for a in range(4)) for i, kb in enumerate(gk.view(w).astype(np.uint64))}
    assert len(got) == out.num_rows, "a group appears twice"
    assert got.keys() == exp.keys()
    for kb in exp:
        assert got[kb] == exp[kb], (hex(kb), got[kb], exp[kb])
    nan_bits = [kb for kb in got if np.isnan(np.array([kb], dtype=np.uint64).astype(w).view(dtype)[0])]
    assert len(nan_bits) == 1
    zero_bits = {int(np.array([z], dtype=dtype).view(w)[0]) for z in (0.0, -0.0)}
    assert zero_bits <= got.keys()


def test_specialised_kernels_serve_grouped_plans(gpu, monkeypatch):
    """Grouped operators run kernels compiled for their plan (NVRTC at create time); the answer is the
    oracle's with them and with the plan-interpreting precompiled kernels (DBX_AGG_JIT=0) alike, for
    the benchmark plan, a nullable / min-max / packed-key plan, host blocks and device blocks."""
    types = [abi.I64, abi.I64, abi.F64]
    op = TransformPartialAggregate(CONFIG2, types, V_MOD3)
    assert op.kernel_variant().startswith("specialised"), op.kernel_variant()
    op.close()
    blk = config2_block(1_500_000, n_keys=300_000)
    for jit in ("1", "0"):
        monkeypatch.setenv("DBX_AGG_JIT", jit)
        op = TransformPartialAggregate(CONFIG2, types, V_MOD3)
        assert op.kernel_variant().startswith("specialised") == (jit == "1"), op.kernel_variant()
        op.close()
        run_both(blk, CONFIG2, V_MOD3, device_resident=True)
        run_both(blk, CONFIG2, V_MOD3, split=100_000)
        run_both(blk, CONFIG2, E.and_(E.gt(E.col(1), E.lit(5)), E.ne(E.col(1) % E.lit(7), E.lit(0))), device_resident=True)
        test_multi_column_group_keys(gpu, True)   # packed keys, nullable key / argument, min / max / avg
        test_multi_column_group_keys(gpu, False)
        test_nullable_args_and_keys(gpu)


@pytest.mark.parametrize("gather", ["1", "0"])
def test_small_pinned_host_blocks_gathered_by_the_device(gpu, monkeypatch, gather):
    """65 536-row blocks in PINNED host memory (the reference's max_block_size): the coalescing
    stage records the blocks and one gather kernel per batch reads them over PCIe (no per-block
    copy call); DBX_STAGE_NO_GATHER=1 is the DMA path.  Odd block sizes exercise the 16-byte tail."""
    import ctypes as C
    from databend_b200 import lib
    if gather == "0":
        monkeypatch.setenv("DBX_STAGE_NO_GATHER", "1")
    L = lib.load()
    n = 1_000_003
    src = config2_block(n, seed=9, n_keys=50_000)
    ptrs, cols = [], []
    for c in src.columns:
        p = C.c_void_p()
        lib.check(L.dbx_host_alloc(n * 8, C.byref(p)))
        ptrs.append(p)
        arr = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int64 if c.dtype != abi.F64 else C.c_double)), shape=(n,))
        arr[:] = c.values()
        cols.append(Column.from_data(arr))
    pinned = DataBlock(cols, n)
    try:
        for split in (65536, 65537, 9999):
            blocks = pinned.split_by_rows(split)
            out = filter_group_aggregate(blocks, CONFIG2, V_MOD3, input_types=schema_types(src))
            ref = oracle().filter_group_agg(src, CONFIG2.to_c(V_MOD3), threads=4)
            g = sorted_group_result_from_block(out, 3, 1)
            o = sorted_group_result_from_oracle(ref, [abi.I64])
            assert_group_results_equal(g, o)
    finally:
        for p in ptrs:
            L.dbx_host_free(p)


@pytest.mark.parametrize("hot", ["1", "0"])
def test_skewed_keys_hot_group_cache(gpu, monkeypatch, hot):
    """Heavily skewed keys (P(k) ~ 1/k, one key on half of the rows, and only 3 distinct keys): groups
    that repeat inside a warp's 32 rows are accumulated in a per-CTA shared-memory cache and merged
    into the table at the end of the kernel.  Same answer as the oracle with the cache (default) and
    without it (DBX_AGG_HOT=0), for every update kind (sum / count / avg / min / max, nullable
    arguments, nullable and sentinel-valued keys), device and host blocks."""
    if hot == "0":
        monkeypatch.setenv("DBX_AGG_HOT", "0")
    rng = np.random.default_rng(11)
    n = 2_000_000
    for variant in ("log_uniform", "half_one_key", "three_keys"):
        if variant == "log_uniform":
            k = np.minimum((np.exp(rng.random(n) * np.log(1e6)) - 1).astype(np.int64), 999_999)
        elif variant == "half_one_key":
            k = np.where(rng.random(n) < 0.5, np.int64(-2**63), rng.integers(0, 100_000, n).astype(np.int64))
        else:
            k = rng.integers(0, 3, n).astype(np.int64)
        kcol = Column.from_data(k, validity=rng.random(n) > 0.02)
        v = Column.from_data(rng.integers(-2**40, 2**40, n).astype(np.int64), validity=rng.random(n) > 0.25)
        x = Column.from_data(rng.integers(0, 1 << 20, n).astype(np.float64))
        f = Column.from_data((rng.integers(-500, 500, n) * 0.25).astype(np.float32), validity=rng.random(n) > 0.5)
        blk = DataBlock([kcol, v, x, f])
        params = AggregatorParams([0], [("sum", 1), ("count", None), ("count", 1), ("avg", 2), ("min", 1), ("max", 3), ("min", 3), ("max", 1)])
        filt = E.ne(E.col(2) % E.lit(7), E.lit(0))
        run_both(blk, params, filt, device_resident=True)
        run_both(blk, params, filt, split=300_000, n_partials=2)
        # a table far too small for the groups: rows overflow and are replayed, cached groups that find
        # the table full come back as rows and are merged after it has grown
        tiny = AggregatorParams(params.group_columns, params.aggregate_functions, expected_groups=16)
        run_both(blk, tiny, filt, device_resident=True)
        run_both(blk, tiny, filt, split=700_000)


def test_two_pass_aggregation_for_tables_beyond_l2(gpu, monkeypatch):
    """Tables that do not fit L2 are aggregated in two passes: filter + scatter of the surviving rows by
    table region, then one fused-kernel launch per region.  Forced here on small tables (thresholds via
    the environment): same answer as the oracle for the benchmark plan, narrow argument types, packed
    and float keys, a table that grows in the middle of the second pass, and skewed keys that overflow a
    partition (that chunk then takes the one-pass path)."""
    monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "1")
    monkeypatch.setenv("DBX_AGG_REGION_BYTES", "65536")
    monkeypatch.setenv("DBX_AGG_PARTITION_ALWAYS", "1")
    types = [abi.I64, abi.I64, abi.F64]
    blk = config2_block(2_000_003, n_keys=400_000)
    dev = DataBlock([to_device(c) for c in blk.columns], blk.num_rows)
    part = TransformPartialAggregate(CONFIG2, types, V_MOD3)
    fin = TransformFinalAggregate(CONFIG2, types)
    part.transform(dev)
    assert "two-pass" in part.kernel_variant() and "chunks: 1" in part.kernel_variant(), part.kernel_variant()
    fin.transform(part.on_finish())
    out = fin.on_finish()[0]
    ref = oracle().filter_group_agg(blk, CONFIG2.to_c(V_MOD3), threads=4)
    assert_group_results_equal(sorted_group_result_from_block(out, 3, 1), sorted_group_result_from_oracle(ref, [abi.I64]))
    part.close(); fin.close()
    run_both(blk, CONFIG2, V_MOD3, device_resident=True)
    run_both(blk, AggregatorParams([0], CONFIG2.aggregate_functions, expected_groups=64), V_MOD3, device_resident=True)  # grows while partitions are processed
    rng = np.random.default_rng(17)
    n = 700_000
    k1 = Column.from_data(rng.integers(0, 3000, n).astype(np.int32))
    k2 = Column.from_data(rng.integers(0, 50, n).astype(np.uint16))
    v = Column.from_data(rng.integers(-1000, 1000, n).astype(np.int16))
    x = Column.from_data((rng.integers(0, 4000, n) * 0.25).astype(np.float32))
    fk = Column.from_data(np.where(rng.random(n) < 0.01, np.nan, rng.integers(0, 5000, n) * 0.5))
    wide = DataBlock([k1, k2, v, x, fk])
    test_params = AggregatorParams([0, 1], [("sum", 2), ("min", 2), ("max", 3), ("count", None), ("avg", 3)])
    _check_multi_key(wide, [0, 1], test_params, E.gt(E.col(2), E.lit(-900)), [abi.I32, abi.U16], device_resident=True)
    # float key: compare through the no-partition path on the same data
    fparams = AggregatorParams([4], [("sum", 2), ("count", None)])
    outs = []
    for force in (True, False):
        if not force:
            monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "0")
        o = filter_group_aggregate([DataBlock([to_device(c) for c in wide.columns], n)], fparams, None, input_types=schema_types(wide))
        order = np.argsort(o.columns[2].values().view(np.uint64), kind="stable")
        outs.append([o.columns[i].values()[order] for i in range(3)])
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a.view(np.uint64) if a.dtype.kind == "f" else a, b.view(np.uint64) if b.dtype.kind == "f" else b)
    monkeypatch.setenv("DBX_AGG_PARTITION_BYTES", "1")
    # skew: half of the rows on one key overflow their partition -> one-pass fallback, still exact
    ks = np.where(rng.random(n) < 0.5, np.int64(7), rng.integers(0, 100_000, n).astype(np.int64))
    skew = DataBlock([Column.from_data(ks), Column.from_data(rng.integers(0, 1000, n).astype(np.int64)), Column.from_data(rng.integers(0, 100, n).astype(np.float64))])
    part = TransformPartialAggregate(CONFIG2, types)
    part.transform(DataBlock([to_device(c) for c in skew.columns], n))
    assert "fallbacks (skew): 1" in part.kernel_variant(), part.kernel_variant()
    part.close()
    run_both(skew, CONFIG2, None, device_resident=True)
