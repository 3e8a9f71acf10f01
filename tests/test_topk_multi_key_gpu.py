"""ORDER BY a, b [, c, d] LIMIT k: the streaming top-k over the composite order image.

Every case compares the row ids with the CPU oracle (oracle/sort_oracle.py: each key with its own
direction and NULL placement, OrderedFloat for floats, remaining ties by ascending row id), the
first key's values and validity bit for bit with the input, and, where the input fits, the same
operator without a LIMIT (the full sort) cut to k."""
import os
import subprocess
import sys

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import TransformTopN, schema_types, to_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sort_oracle():
    from oracle import sort_oracle as so
    return so


def _bits(v):
    v = np.ascontiguousarray(v)
    return v.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[v.dtype.itemsize])


def run_op(data, keys, limit, split=None, device_resident=False):
    """data: [(values, valid or None)]; keys: [(column, asc, nulls_first)], most significant first."""
    blk = DataBlock([Column.from_data(v, validity=m) for v, m in data])
    (c0, a0, n0), extra = keys[0], list(keys[1:])
    op = TransformTopN(c0, a0, n0, limit, schema_types(blk), extra_keys=extra)
    blocks = blk.split_by_rows(split) if split else [blk]
    for b in blocks:
        if device_resident:
            b = DataBlock([to_device(c) for c in b.columns], b.num_rows)
        op.transform(b)
    out = op.on_finish()
    op.close()
    return out


def check(data, keys, limit, split=None, device_resident=False, full_sort=True):
    out = run_op(data, keys, limit, split, device_resident)
    exp = sort_oracle().sort_permutation([(data[c][0], data[c][1], a, nf) for c, a, nf in keys], limit)
    rows = out.columns[1].values()
    np.testing.assert_array_equal(rows, exp)
    v0, m0 = data[keys[0][0]]
    valid = np.ones(len(v0), bool) if m0 is None else m0
    got_valid = out.columns[0].valid_mask()
    np.testing.assert_array_equal(got_valid, valid[exp])
    got = out.columns[0].values()
    assert got.dtype == v0.dtype
    np.testing.assert_array_equal(_bits(got)[got_valid], _bits(v0[exp])[got_valid])
    if m0 is not None:
        assert out.columns[0].validity is not None
    if full_sort:
        ref = run_op(data, keys, 0, split, device_resident)
        np.testing.assert_array_equal(rows, ref.columns[1].values()[:limit])
        np.testing.assert_array_equal(got_valid, ref.columns[0].valid_mask()[:limit])
        np.testing.assert_array_equal(_bits(got), _bits(ref.columns[0].values()[:limit]))
    return out


# ---------------------------------------------------------------- image widths
def test_w1_two_int32_keys():
    rng = np.random.default_rng(1)
    n = 200_003
    a = rng.integers(-50, 50, n).astype(np.int32)
    b = rng.integers(-2**31, 2**31, n, dtype=np.int64).astype(np.int32)
    for asc0, asc1 in [(True, True), (True, False), (False, True), (False, False)]:
        check([(a, None), (b, None)], [(0, asc0, False), (1, asc1, False)], 777, split=50_000)


def test_w1_int8_int16_pair():
    rng = np.random.default_rng(2)
    n = 100_000
    a = rng.integers(-128, 128, n).astype(np.int8)
    b = rng.integers(0, 2**16, n).astype(np.uint16)
    check([(a, None), (b, None)], [(0, False, False), (1, True, False)], 500)
    c = rng.integers(-2**15, 2**15, n).astype(np.int16)
    check([(a, None), (c, None)], [(0, True, False), (1, False, False)], 333, device_resident=True)


def test_w2_two_int64_keys():
    rng = np.random.default_rng(3)
    n = 300_000
    a = rng.integers(-1000, 1000, n).astype(np.int64)
    b = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    for dev in (False, True):
        check([(a, None), (b, None)], [(0, True, False), (1, False, False)], 1000, split=70_000, device_resident=dev)


def test_w3_two_nullable_int64_keys():
    rng = np.random.default_rng(4)
    n = 250_000
    a = rng.integers(-20, 20, n).astype(np.int64)
    am = rng.random(n) > 0.2
    b = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
    bm = rng.random(n) > 0.3
    for nf0, nf1 in [(True, True), (True, False), (False, True), (False, False)]:
        check([(a, am), (b, bm)], [(0, True, nf0), (1, False, nf1)], 900, split=60_000)


def test_w5_four_nullable_64bit_keys():
    rng = np.random.default_rng(5)
    n = 200_000
    a = rng.integers(0, 4, n).astype(np.uint64)
    b = rng.choice([np.nan, -0.0, 0.0, 1.5, -np.inf, np.inf], n)
    c = rng.integers(-3, 3, n).astype(np.int64)
    d = rng.standard_normal(n)
    ms = [rng.random(n) > p for p in (0.1, 0.2, 0.3, 0.1)]
    data = [(a, ms[0]), (b, ms[1]), (c, ms[2]), (d, ms[3])]
    check(data, [(0, True, True), (1, False, False), (2, True, False), (3, False, True)], 1500, split=45_000)
    check(data, [(0, False, False), (1, True, True), (2, False, True), (3, True, False)], 77, device_resident=True)


# ---------------------------------------------------------------- dtypes, extremes, directions, NULLs
def test_extremes_next_to_placement_bit_and_desc():
    rng = np.random.default_rng(6)
    n = 60_000
    u = rng.choice(np.array([0, 2**64 - 1, 1, 2**63], dtype=np.uint64), n)
    i = rng.choice(np.array([-2**63, 2**63 - 1, 0, -1], dtype=np.int64), n)
    f32 = rng.choice(np.array([np.nan, -0.0, 0.0, np.inf, -np.inf, 1.0], dtype=np.float32), n)
    f32[rng.random(n) < 0.01] = np.frombuffer(np.uint32(0x7FC01234).tobytes(), np.float32)[0]  # NaN payload
    f64 = rng.choice([np.nan, -0.0, 0.0, np.inf, -np.inf, -2.5], n)
    ms = [rng.random(n) > 0.15 for _ in range(4)]
    for order in ([0, 1, 2, 3], [2, 3, 0, 1], [3, 2, 1, 0], [1, 0, 3, 2]):
        for dirs in [(True, True, False, False), (False, False, True, True), (False, True, False, True)]:
            nfs = (dirs[1], not dirs[2], dirs[0], dirs[3])
            data = [(u, ms[0]), (i, ms[1]), (f32, ms[2]), (f64, ms[3])]
            check(data, [(order[j], dirs[j], nfs[j]) for j in range(4)], 600, split=25_000)
            check([(u, None), (i, None), (f32, None), (f64, None)], [(order[j], dirs[j], False) for j in range(4)], 300)


def test_every_direction_and_null_placement():
    rng = np.random.default_rng(7)
    n = 80_000
    a = rng.integers(-5, 5, n).astype(np.int16)
    am = rng.random(n) > 0.3
    b = rng.integers(-100, 100, n).astype(np.float32)
    bm = rng.random(n) > 0.3
    for asc0 in (True, False):
        for nf0 in (True, False):
            for asc1 in (True, False):
                for nf1 in (True, False):
                    check([(a, am), (b, bm)], [(0, asc0, nf0), (1, asc1, nf1)], 250, split=30_000)


def test_more_nulls_than_k_on_first_key():
    rng = np.random.default_rng(8)
    n = 50_000
    a = rng.integers(0, 100, n).astype(np.int32)
    am = rng.random(n) > 0.5  # ~25000 NULLs, k = 1000: with NULLS FIRST only the later key decides
    b = rng.integers(-10**9, 10**9, n).astype(np.int64)
    for nf in (True, False):
        check([(a, am), (b, None)], [(0, True, nf), (1, False, False)], 1000, split=12_000)


def test_fewer_rows_than_k_and_empty_blocks():
    rng = np.random.default_rng(9)
    n = 300
    a = rng.integers(0, 3, n).astype(np.int64)
    am = rng.random(n) > 0.3
    b = rng.standard_normal(n)
    check([(a, am), (b, None)], [(0, False, True), (1, True, False)], 5000, split=64)
    # empty pushes in between and an empty input
    blk = DataBlock([Column.from_data(a, validity=am), Column.from_data(b)])
    op = TransformTopN(0, True, False, 10, schema_types(blk), extra_keys=[(1, True, False)])
    empty = DataBlock([Column.from_data(a[:0], validity=am[:0]), Column.from_data(b[:0])], 0)
    op.transform(empty)
    op.transform(blk)
    op.transform(empty)
    out = op.on_finish()
    op.close()
    exp = sort_oracle().sort_permutation([(a, am, True, False), (b, None, True, False)], 10)
    np.testing.assert_array_equal(out.columns[1].values(), exp)
    op = TransformTopN(0, True, False, 10, schema_types(blk), extra_keys=[(1, True, False)])
    op.transform(empty)
    out = op.on_finish()
    op.close()
    assert out.num_rows == 0


# ---------------------------------------------------------------- ties, adversarial order, replay, large k
def test_heavy_ties_and_all_keys_equal():
    rng = np.random.default_rng(10)
    n = 400_000
    a = rng.integers(0, 3, n).astype(np.int8)  # low-cardinality first key: the later key is read densely
    b = rng.integers(0, 50, n).astype(np.float64)
    check([(a, None), (b, None)], [(0, True, False), (1, False, False)], 2000, split=100_000)
    z = np.zeros(n, np.int32)
    check([(z, None), (z.astype(np.int64), None)], [(0, True, False), (1, False, False)], 1234, split=90_000)


def test_sorted_adversarial_input():
    n = 500_000
    a = np.arange(n, dtype=np.float64)[::-1].copy()  # every row beats the boundary
    b = np.arange(n, dtype=np.int64)
    for dev in (False, True):
        check([(a, None), (b, None)], [(0, True, False), (1, True, False)], 1000, split=100_000, device_resident=dev)
        check([(b.astype(np.float64), None), (a, None)], [(0, False, False), (1, True, False)], 1000, device_resident=dev)


def test_large_k_takes_radix_order():
    rng = np.random.default_rng(11)
    n = 600_000
    a = rng.integers(0, 1000, n).astype(np.float64)
    b = rng.integers(-5, 5, n).astype(np.int32)
    bm = rng.random(n) > 0.1
    check([(a, None), (b, bm)], [(0, False, False), (1, True, True)], 20_000, split=150_000)
    check([(a, None), (b, bm)], [(0, True, True), (1, False, False)], 5000, device_resident=True)


_REPLAY = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_topk_multi_key_gpu as t
rng = np.random.default_rng(12)
n = 300_000
a = rng.standard_normal(n)
b = rng.integers(0, 7, n).astype(np.int64)
bm = rng.random(n) > 0.2
t.check([(a, None), (b, bm)], [(0, True, False), (1, False, True)], 100, split=100_000)
t.check([(b, bm), (a, None)], [(0, True, True), (1, False, False)], 100, device_resident=True)
a.sort()
t.check([(a[::-1].copy(), None), (b, None)], [(0, True, False), (1, True, False)], 100, device_resident=True)
print("ok")
"""


def test_forced_replay_with_small_candidate_list():
    """DBX_TOPK_CAP shrinks the candidate list, so the optimistic scans overflow and are replayed
    from the snapshot in pieces that fit (the cap is read once per process: run in a child)."""
    env = dict(os.environ, DBX_TOPK_CAP="1")
    r = subprocess.run([sys.executable, "-c", _REPLAY, ROOT, os.path.dirname(os.path.abspath(__file__))], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ok")


# ---------------------------------------------------------------- beyond 2^30 rows
def test_beyond_2_pow_30_rows():
    """One device-resident block of 2^28 rows pushed five times (1.34e9 rows, more than the full
    sort takes).  a = i % 1024 (Int16) ASC, b = i // 1024 (Int32) DESC: the winners are a = 0 with
    the largest b, and each (a, b) occurs once per push, so the global row id orders the pushes."""
    m = 1 << 28
    i = np.arange(m, dtype=np.int32)
    blk = DataBlock([to_device(Column.from_data((i % 1024).astype(np.int16))), to_device(Column.from_data(i // 1024))], m)
    del i
    k = 1000
    op = TransformTopN(0, True, False, k, [abi.I16, abi.I32], extra_keys=[(1, False, False)])
    for _ in range(5):
        op.transform(blk)
    out = op.on_finish()
    op.close()
    top_b = (m - 1) // 1024 - np.arange(k // 5)
    exp = (np.arange(5)[None, :] * m + top_b[:, None] * 1024).reshape(-1)
    np.testing.assert_array_equal(out.columns[1].values(), exp)
    assert not out.columns[0].values().any()


# ---------------------------------------------------------------- multi-GPU merge
def test_topk_merge_with_later_keys_equals_global_topk():
    """Row-range shards -> local multi-key top-k -> topk_merge with the later keys == the global result."""
    from databend_b200.distributed import topk_merge
    rng = np.random.default_rng(13)
    n, k, world = 200_000, 300, 4
    a = rng.integers(0, 50, n).astype(np.float64)
    a[rng.random(n) < 0.01] = np.nan
    am = rng.random(n) > 0.05
    b = rng.integers(-3, 3, n).astype(np.int32)
    bm = rng.random(n) > 0.1
    c = rng.integers(0, 2, n).astype(np.uint8)
    keys = [(True, False), (False, True), (True, False)]
    ref = sort_oracle().sort_permutation([(a, am, *keys[0]), (b, bm, *keys[1]), (c, None, *keys[2])], k)
    parts = []
    for r in range(world):
        lo, hi = n * r // world, n * (r + 1) // world
        blk = DataBlock([Column.from_data(a[lo:hi], validity=am[lo:hi]), Column.from_data(b[lo:hi], validity=bm[lo:hi]), Column.from_data(c[lo:hi])])
        op = TransformTopN(0, *keys[0], k, schema_types(blk), extra_keys=[(1, *keys[1]), (2, *keys[2])])
        op.transform(blk)
        out = op.on_finish()
        op.close()
        parts.append((out, lo))
    key0 = Column.from_data(np.concatenate([p.columns[0].values() for p, _ in parts]),
                            validity=np.concatenate([p.columns[0].valid_mask() for p, _ in parts]))
    rows = np.concatenate([p.columns[1].values() + lo for p, lo in parts])
    xb = Column.from_data(b[rows], validity=bm[rows])
    xc = Column.from_data(c[rows])
    merged = topk_merge(DataBlock([key0, Column.from_data(rows)], len(rows)), 0, k, *keys[0],
                        extra_keys=[(xb, *keys[1]), (xc, *keys[2])])
    np.testing.assert_array_equal(merged.columns[1].values(), ref)
    np.testing.assert_array_equal(merged.columns[0].valid_mask(), am[ref])
