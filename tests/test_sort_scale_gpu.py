"""ORDER BY and top-k where they can be wrong: sorts of many waves of radix-sort tiles, the 2^30 - 1
row limit, LIMIT around 4 Mi (the streaming top-k's largest k, above which everything is sorted
and cut), and float keys whose bits a sort can lose.

Row ids must equal the reference exactly, validity too, and every returned key must be the input
row's value bit for bit.  The reference is tests/sort_scale_ref.py on the device (held against the
CPU oracles in tests/test_sort_scale_ref_cpu.py, and against the C oracle at 2e7 rows here).

Tile arithmetic: `onesweep_kernel` sorts 4 096-key tiles with __launch_bounds__(256, 3) and 61 440 B
of dynamic shared memory, so at most 3 x 132 = 396 tiles are co-resident on an H100 (from the launch
bounds, not measured).  Inputs of more tiles than that make later tiles look back on tiles that
started late or retired long ago."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import sort_scale_ref as R
from databend_b200 import abi
from databend_b200.block import Column, DataBlock
from databend_b200.distributed import _dev_tensor
from databend_b200.lib import DbxError, check as dbx_check, load
from databend_b200.transforms import TransformTopN, _block_from_c, schema_types, to_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
TILE = 4096                # keys per radix-sort tile (rs::kTile)
ONE_WAVE = 3 * 132         # co-resident tiles on 132 SMs, from the launch bounds (not measured)
STREAMING_MAX_K = 1 << 22  # largest LIMIT the streaming top-k takes
ODD_PUSHES = [1_000_003, 65_537, 2_999_999]  # host pushes whose sizes are not multiples of 4 096
DTYPES = [np.float64, np.float32, np.int64, np.uint64, np.int32, np.int8]
SHAPES = ["few_distinct", "all_equal", "sorted", "reverse", "top_byte", "low_byte"]


# ---------------------------------------------------------------- data
def make_key(shape, nd, n, rng):
    nd = np.dtype(nd)
    w = 8 * nd.itemsize
    ut = np.dtype(f"u{nd.itemsize}")
    if shape == "random":
        if nd.kind == "f":
            return rng.standard_normal(n).astype(nd)
        info = np.iinfo(nd)
        return rng.integers(info.min, info.max, n, dtype=nd, endpoint=True)
    if shape == "few_distinct":  # each value's run of a digit spans thousands of tiles
        vals = {"f": [-1.5, 0.0, 2.5], "i": [3, -1, 0], "u": [3, 1, 0]}[nd.kind]
        return np.array(vals, nd)[rng.integers(0, 3, n)]
    if shape == "all_equal":
        return np.full(n, -2 if nd.kind in "fi" else 2, nd)
    if shape in ("sorted", "reverse"):
        x = np.sort(make_key("random", nd, n, rng))
        return x if shape == "sorted" else x[::-1].copy()
    r8 = rng.integers(0, 256, n, dtype=np.uint64)
    if shape == "top_byte":  # only the most significant byte varies (floats stay finite: exponent < all ones)
        low = {8: 0x0001_2345_6789_ABCD, 4: 0x0012_3456, 2: 0x5A, 1: 0}[nd.itemsize]
        bits = (r8 << np.uint64(w - 8)) | np.uint64(low)
    else:  # "low_byte": only the least significant byte varies
        if nd.kind == "f":
            high = 0x3FF0_0000_0000_0000 if w == 64 else 0x3F80_0000
        else:
            high = 0x1234_5678_9ABC_DE00 & ((1 << w) - 1)
        bits = np.uint64(high) | r8
    return bits.astype(ut).view(nd)


def pieces(n, sizes):
    out, s, i = [], 0, 0
    while s < n:
        m = min(sizes[i % len(sizes)], n - s)
        out.append(m)
        s += m
        i += 1
    return out


def _bits_t(a):
    """numpy array -> its bits as a signed torch tensor of the same width on the device."""
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view({1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[a.itemsize])).to(DEV)


def _assert_equal_t(got, exp, what):
    if got.shape != exp.shape:
        raise AssertionError(f"{what}: {got.shape[0]} rows, expected {exp.shape[0]}")
    bad = (got != exp).nonzero().flatten()
    if bad.numel():
        p = bad[:5].tolist()
        raise AssertionError(f"{what}: {bad.numel()} of {got.shape[0]} positions differ; first at {p}: "
                             f"got {got[p].tolist()}, expected {exp[p].tolist()}")


# ---------------------------------------------------------------- run and check
def run(data, keys, limit, pushes=None, device_resident=False):
    """data: [(values, valid or None)]; keys: [(column, asc, nulls_first)], most significant first.
    Returns the result block and the key column's null_count as the library reports it."""
    blk = DataBlock([Column.from_data(v, validity=m) for v, m in data])
    (c0, a0, n0), extra = keys[0], list(keys[1:])
    op = TransformTopN(c0, a0, n0, limit, schema_types(blk), extra_keys=extra)
    s = 0
    for m in pushes or [blk.num_rows]:
        b = blk.slice(s, s + m)
        s += m
        if device_resident:
            b = DataBlock([to_device(c) for c in b.columns], b.num_rows)
        op.transform(b)
    assert s == blk.num_rows
    op.finish()
    cb = op.pull_c(abi.MEM_HOST)
    null_count = cb.cols[0].null_count
    out = _block_from_c(cb, 0)
    op.close()
    return out, null_count


def check(data, keys, limit=0, pushes=None, device_resident=False):
    n = len(data[0][0])
    out, null_count = run(data, keys, limit, pushes, device_resident)
    exp = R.sort_permutation([R.key_spec(data[c][0], data[c][1], a, nf, DEV) for c, a, nf in keys], limit)
    assert out.num_rows == (min(n, limit) if limit else n)
    _assert_equal_t(torch.from_numpy(out.columns[1].values()).to(DEV), exp, "row ids")
    v0, m0 = data[keys[0][0]]
    got_valid = torch.from_numpy(out.columns[0].valid_mask()).to(DEV)
    exp_valid = torch.ones_like(got_valid) if m0 is None else torch.from_numpy(m0).to(DEV)[exp]
    _assert_equal_t(got_valid, exp_valid, "validity")
    if m0 is not None:
        assert out.columns[0].validity is not None
        assert null_count == int((~exp_valid).sum()), f"null_count {null_count}"
    got = _bits_t(out.columns[0].values())
    src = _bits_t(v0)[exp]
    _assert_equal_t(got[exp_valid], src[exp_valid], "key bits")
    return out


# ---------------------------------------------------------------- full sort beyond one wave of tiles
@pytest.mark.parametrize("n", [ONE_WAVE * TILE - 1, ONE_WAVE * TILE + 1, 1600 * TILE + 1])
def test_full_sort_around_one_wave(gpu, n):
    """Every key type in both directions, every data shape, nullable keys with both placements;
    host pushes split at non-multiples of 4 096 and device-resident pushes."""
    rng = np.random.default_rng(n)
    i = 0
    for nd in DTYPES:
        check([(make_key("random", nd, n, rng), None)], [(0, True, False)], pushes=pieces(n, ODD_PUSHES))
        check([(make_key("random", nd, n, rng), None)], [(0, False, False)], device_resident=True)
        for shape in SHAPES:
            i += 1
            check([(make_key(shape, nd, n, rng), None)], [(0, i % 2 == 0, False)],
                  pushes=pieces(n, ODD_PUSHES) if i % 3 else None, device_resident=i % 3 == 0)
    for nd in (np.float64, np.int32):
        x = make_key("few_distinct", nd, n, rng)
        m = rng.random(n) > 0.1
        for nf in (True, False):
            for asc in (True, False):
                check([(x, m)], [(0, asc, nf)], pushes=pieces(n, ODD_PUSHES), device_resident=asc)


LARGE = [
    # n, dtype, shape, asc, nullable (nulls_first), pushes (None: one), device resident
    (30_000_000, np.float64, "random", True, None, None, True),
    (30_000_000, np.float32, "random", False, None, ODD_PUSHES + [9_999_991], False),
    (30_000_000, np.int64, "reverse", True, None, None, True),
    (30_000_000, np.uint64, "top_byte", False, None, [7_777_777], False),
    (30_000_000, np.int32, "few_distinct", True, True, [11_111_111], False),
    (30_000_000, np.int8, "low_byte", True, None, [12_345_679], True),
    (100_000_000, np.float64, "random", True, None, None, True),
    (100_000_000, np.int32, "few_distinct", False, False, [33_333_331], False),
    (100_000_000, np.float32, "sorted", False, None, [50_000_001], True),
]


@pytest.mark.parametrize("case", LARGE, ids=[f"{c[0]}-{np.dtype(c[1]).name}-{c[2]}" for c in LARGE])
def test_full_sort_many_waves(gpu, case):
    n, nd, shape, asc, nulls_first, push, dev = case
    assert (n + TILE - 1) // TILE >= 4 * ONE_WAVE  # 18 waves at 3e7 rows, 61 at 1e8
    rng = np.random.default_rng(n + len(shape))
    x = make_key(shape, nd, n, rng)
    m = None if nulls_first is None else rng.random(n) > 0.07
    check([(x, m)], [(0, asc, bool(nulls_first))], pushes=pieces(n, push) if push else None, device_resident=dev)


def test_device_reference_matches_c_oracle_at_2e7(gpu):
    """The device reference equals the C oracle at 2e7 rows (ties, NaN, -0.0, NULLs), and so does the sort."""
    from oracle import oracle as orc
    rng = np.random.default_rng(20)
    n = 20_000_000
    x = rng.integers(-40, 40, n).astype(np.float64) / 8
    x[rng.random(n) < 0.01] = np.nan
    x[rng.random(n) < 0.01] = -0.0
    m = rng.random(n) > 0.05
    ref = R.sort_permutation([R.key_spec(x, m, False, True, DEV)]).cpu().numpy()
    np.testing.assert_array_equal(ref, orc.topk(Column.from_data(x, validity=m), False, True, n))
    check([(x, m)], [(0, False, True)], pushes=pieces(n, ODD_PUSHES))


# ---------------------------------------------------------------- several keys at scale
def test_several_keys_without_limit_and_cut_at_5e6(gpu):
    """Four keys of mixed types, directions and NULL placements over 1e7 rows and several pushes: one
    stable radix sort per key plus sort_gather_kernel; LIMIT 5 000 000 takes the same path and is cut."""
    rng = np.random.default_rng(41)
    n = 10_000_003
    a = rng.integers(-3, 4, n).astype(np.int8)
    am = rng.random(n) > 0.1
    b = np.where(rng.random(n) < 0.05, np.nan, rng.integers(-2, 3, n) * 0.5)
    b[rng.random(n) < 0.05] = -0.0
    bm = rng.random(n) > 0.15
    c = rng.integers(0, 2**64, n, dtype=np.uint64) >> np.uint64(58)
    d = rng.standard_normal(n).astype(np.float32)
    dm = rng.random(n) > 0.02
    data = [(a, am), (b, bm), (c, None), (d, dm)]
    keys = [(0, True, False), (1, False, True), (2, True, False), (3, False, False)]
    check(data, keys, 0, pushes=[2_500_001, 3_333_333, 4_166_669])
    check(data, keys, 5_000_000, pushes=[2_500_001, 3_333_333, 4_166_669])
    check(data, [(3, True, True), (1, True, False), (0, False, True)], 0, pushes=[6_000_001, 4_000_002], device_resident=True)


# ---------------------------------------------------------------- the LIMIT boundary
def _limit_data(n, rng):
    x = rng.integers(-500, 500, n).astype(np.float64) / 4  # ties: row ids decide
    x[rng.random(n) < 0.01] = np.nan
    m = rng.random(n) > 0.05
    y = rng.integers(-2**31, 2**31, n, dtype=np.int64).astype(np.int32)
    return x, m, y


@pytest.mark.parametrize("n_keys", [1, 2])
@pytest.mark.parametrize("k", [STREAMING_MAX_K, STREAMING_MAX_K + 1])
def test_limit_around_4mi(gpu, k, n_keys):
    """k = 4 Mi runs the streaming top-k, k = 4 Mi + 1 sorts everything: both return min(n, k) rows."""
    rng = np.random.default_rng(k + n_keys)
    n = 12_000_000
    x, m, y = _limit_data(n, rng)
    if n_keys == 1:
        check([(x, m)], [(0, True, False)], k, pushes=[5_000_011, 6_999_989])
        check([(x, m)], [(0, False, True)], k, device_resident=True)
    else:
        check([(x, m), (y, None)], [(0, True, False), (1, False, False)], k, pushes=[5_000_011, 6_999_989])
        check([(x, m), (y, None)], [(0, False, True), (1, True, False)], k, device_resident=True)


@pytest.mark.parametrize("n,k", [(4_000_000, STREAMING_MAX_K), (5_000_000, 5_000_000), (5_000_000, 10**9)])
def test_limit_at_least_n(gpu, n, k):
    rng = np.random.default_rng(n + k % 1000)
    x, m, y = _limit_data(n, rng)
    check([(x, m)], [(0, True, True)], k, pushes=[1_234_567, n - 1_234_567])
    check([(x, m), (y, None)], [(0, False, False), (1, True, False)], k)


@pytest.mark.parametrize("k", [4097, 6000])
def test_more_nulls_than_k_just_above_4096(gpu, k):
    """k above the one-CTA rank sort with more NULL rows than k: the NULL list takes the radix order."""
    rng = np.random.default_rng(k)
    n = 1_000_000
    x = rng.standard_normal(n)
    m = rng.random(n) > 0.5
    y = rng.integers(0, 5, n).astype(np.int16)
    for nf in (True, False):
        for asc in (True, False):
            check([(x, m)], [(0, asc, nf)], k, pushes=[300_007, 700_000 - 7], device_resident=not asc)
            check([(x, m), (y, None)], [(0, asc, nf), (1, not asc, False)], k, pushes=[300_007, 700_000 - 7])


_REPLAY = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[2])
import test_sort_scale_gpu as t
n, k = 3_000_000, 100_000
x = np.arange(n, 0, -1).astype(np.float64)  # ASC over descending data: every row beats the boundary
y = np.random.default_rng(3).integers(0, 9, n).astype(np.int32)
m = np.random.default_rng(4).random(n) > 0.3
t.check([(x, None)], [(0, True, False)], k, device_resident=True)
t.check([(x, m)], [(0, True, True)], k, pushes=[1_000_003, 1_999_997])
t.check([(x, None), (y, None)], [(0, True, False), (1, False, False)], k, device_resident=True)
t.check([(y, m), (x, None)], [(0, True, True), (1, True, False)], k, device_resident=True)
print("ok")
"""


def test_large_k_replay_with_small_candidate_list(gpu):
    """DBX_TOPK_CAP shrinks the candidate list to its floor (4k + 4096), so the optimistic scans
    overflow at k = 100 000 and are replayed from the snapshot (the cap is read once per process)."""
    env = dict(os.environ, DBX_TOPK_CAP="1")
    r = subprocess.run([sys.executable, "-c", _REPLAY, ROOT, os.path.dirname(os.path.abspath(__file__))], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("ok")


# ---------------------------------------------------------------- float key bits on every path
def special_floats(nd, n, rng):
    sp = R.F32_SPECIAL_BITS.view(np.float32) if nd == np.float32 else R.F64_SPECIAL_BITS.view(np.float64)
    x = rng.choice(sp, n)
    ordinary = rng.random(n) < 0.3
    x[ordinary] = rng.integers(-3, 4, ordinary.sum()).astype(nd) / nd(2)
    return x


PATHS = {  # name: (limit, float key position, number of keys)
    "topk_rank_sort": (1000, 0, 1),    # k <= 4096: one-CTA rank sort of the candidates
    "topk_radix": (6000, 0, 1),        # k > 4096: radix order of the candidates
    "full_sort": (0, 0, 1),
    "multi_topk_float_first": (6000, 0, 2),
    "multi_topk_rank_float_first": (1000, 0, 2),
    "multi_topk_float_later": (6000, 1, 2),
    "multi_full_sort_float_first": (0, 0, 2),
    "multi_full_sort_float_later": (0, 1, 2),
}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("nd", [np.float32, np.float64], ids=["f32", "f64"])
def test_float_key_bits(gpu, nd, path):
    """+-0, canonical, negative, payload and signalling NaN, +-inf, the extreme subnormals and +-max:
    the row ids follow OrderedFloat with row-id ties, and the key is returned bit for bit."""
    limit, pos, n_keys = PATHS[path]
    rng = np.random.default_rng(7)
    n = 40_000
    x = special_floats(nd, n, rng)
    m = rng.random(n) > 0.1
    other = rng.integers(-2, 3, n).astype(np.int32)
    for valid in (None, m):
        for asc in (True, False):
            for nf in (True, False):
                if valid is None and nf:
                    continue
                if n_keys == 1:
                    data, keys = [(x, valid)], [(0, asc, nf)]
                elif pos == 0:
                    data, keys = [(x, valid), (other, None)], [(0, asc, nf), (1, not asc, False)]
                else:
                    data, keys = [(other, None), (x, valid)], [(0, asc, False), (1, asc, nf)]
                check(data, keys, limit, pushes=[13_001, n - 13_001], device_resident=not asc)


# ---------------------------------------------------------------- 2^30 - 1 rows
# Device memory of one sort of n = 2^30 - 1 rows of a one-byte key (from sort_reserve and finish_full_sort):
#   sort_reserve at a capacity of 2^30 rows: ordered key 8 B + row id 4 B + original bits 8 B = 20 GiB
#   finish_full_sort: the radix sort's second (key, row id) pair 12 GiB, look-back status 2^18 tiles x 1 KiB
#   the result: key 1 B (Int16: 2 B) + row id 8 B per row = 9 (10) GiB, kept by the allocator's pool
#   the pushed block 0.25 GiB (Int16: 0.5 GiB) and the test's chunks below 1 GiB
# About 42 GiB for the first sort and 44 GiB while the second one runs next to the pool's 9 GiB.
NEED_2POW30 = 46 << 30
CHUNK = 1 << 26


def _pull_device(op, n):
    op.finish()
    b = op.pull_c(abi.MEM_DEVICE)
    assert b.num_rows == n
    return b


def test_2pow30_minus_1_rows(gpu):
    free, _ = torch.cuda.mem_get_info(0)
    if free < NEED_2POW30:
        pytest.skip(f"needs about {NEED_2POW30 >> 30} GiB of free device memory, {free / 2**30:.1f} GiB free")
    m = 1 << 28
    n = (1 << 30) - 1
    mask = (1 << 20) - 1
    # all keys equal: one digit holds every row, the last tile's inclusive prefix is n; the identity comes out
    blk8 = torch.full((m,), -5, dtype=torch.int8, device=DEV)
    col = Column.device(abi.I8, m, blk8.data_ptr())
    torch.cuda.synchronize()
    for asc in (True, False):
        op = TransformTopN(0, asc, False, 0, [abi.I8])
        for i in range(4):
            op.transform(DataBlock([col if i < 3 else col.slice(0, m - 1)], m if i < 3 else m - 1))
        if asc:
            with pytest.raises(DbxError) as e:  # one more row is refused
                op.transform(DataBlock([col.slice(0, 1)], 1))
            assert e.value.status == abi.ERR_UNSUPPORTED and "more than 2^30 - 1 rows" in e.value.message
        b = _pull_device(op, n)
        rows = _dev_tensor(b.cols[1].data, n * 8, 0).view(torch.int64)
        keys = _dev_tensor(b.cols[0].data, n, 0).view(torch.int8)
        for s in range(0, n, CHUNK):
            e_ = min(n, s + CHUNK)
            _assert_equal_t(rows[s:e_], torch.arange(s, e_, dtype=torch.int64, device=DEV), f"row ids [{s}, {e_})")
            assert bool((keys[s:e_] == -5).all())
        del rows, keys
        dbx_check(load().dbx_block_release(C.byref(b)))
        op.close()
    del blk8
    torch.cuda.empty_cache()
    # key = global row >> 20 (Int16) DESC: groups 1023 .. 0, each in ascending row order; group 1023 is one row short
    op = TransformTopN(0, False, False, 0, [abi.I16])
    for i in range(4):
        s = i * m
        k16 = torch.arange(s >> 20, (s + m) >> 20, dtype=torch.int16, device=DEV).repeat_interleave(1 << 20)
        ln = m if i < 3 else m - 1
        op.transform(DataBlock([Column.device(abi.I16, ln, k16.data_ptr())], ln))
        op.inputs_consumed()
        del k16
    torch.cuda.empty_cache()
    b = _pull_device(op, n)
    rows = _dev_tensor(b.cols[1].data, n * 8, 0).view(torch.int64)
    keys = _dev_tensor(b.cols[0].data, 2 * n, 0).view(torch.int16)
    first = (1 << 20) - 1  # rows of group 1023
    for s in range(0, n, CHUNK):
        e_ = min(n, s + CHUNK)
        p = torch.arange(s, e_, dtype=torch.int64, device=DEV)
        q = p - first
        g = torch.where(p < first, torch.full_like(p, 1023), 1022 - (q >> 20))
        exp = torch.where(p < first, (1023 << 20) + p, (g << 20) + (q & mask))
        _assert_equal_t(rows[s:e_], exp, f"row ids [{s}, {e_})")
        _assert_equal_t(keys[s:e_].to(torch.int64), g, f"keys [{s}, {e_})")
        del p, q, g, exp
    del rows, keys
    dbx_check(load().dbx_block_release(C.byref(b)))
    op.close()
    torch.cuda.empty_cache()
