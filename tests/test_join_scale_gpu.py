"""Hash joins where they can be wrong: the full 1e9 x 1e7 shape, many-to-many tables beyond L2, probe
runs across the table's end, every integer key-type pair at its extremes, odd block shapes and the
build / reset lifecycle, and more than 2^32 output rows from one probe block.

Every result is checked against tests/join_scale_ref.py: an exact reference by sorting (no hash
table) and a verifier that proves each output block is exactly the set of matching pairs, block by
block on device tensors (outputs are pulled with DBX_MEM_DEVICE and released after the check).  Large
inputs are generated on the device, seeded per block; keys built for chosen table slots are computed on
the host.  Every input is pushed as device-resident blocks.

Which probe kernels the groups reach (join_probe2_kernel<KW, PACKED, UNIQUE, MARK, RF>):
  config 3       KW 1 single key: UNIQUE and non-unique (DBX_JOIN_NO_UNIQUE), MARK for RIGHT ANTI / FULL
  many-to-many   non-unique, MARK for the build-side kinds, RF for INNER / RIGHT SEMI
  runs           UNIQUE and non-unique, MARK, RF (single keys), PACKED KW 1 (2 x Int32), PACKED KW 2 (2 x Int64)
  key types      UNIQUE, MARK, RF, PACKED KW 1 (a second Int32 key; KW 2 for the 64-bit first keys)
  shapes         UNIQUE and non-unique, MARK, RF
  > 2^32 rows    non-unique, no MARK
The library does not report which instantiation a join ran: UNIQUE follows from the build side having no
duplicate key, and the forced non-unique config-3 case from final_build reading DBX_JOIN_NO_UNIQUE.

Not tested, on purpose: the per-CTA totals of the probe are `unsigned int`, and a CTA step covers
512 probe rows, so one step passes 2^32 output rows only if its rows average more than 8.4M matches
each.  The linear-probing build costs about D^2 / 2 slot visits for D equal keys, so such a build
side would run for hours; the > 2^32 test below instead shows that the 64-bit cursor and positions
carry more than 2^32 rows of one probe block."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import join_scale_ref as R
from databend_b200 import abi
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError, check as dbx_check, load
from databend_b200.transforms import HashJoin

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda:0"
MULT = -0x61C8864680B583EB  # 0x9E3779B97F4A7C15 as int64: odd, so i -> i * MULT + ADD is a bijection
ADD = 0x1234_5678_9ABC


def gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def spread(i):
    """Distinct int64 keys from distinct indices."""
    return i * MULT + ADD


def pack_bits(valid):
    """bool tensor -> LSB-first bitmap (uint8) on the device."""
    n = valid.shape[0]
    v = torch.zeros((n + 7) // 8 * 8 + 64, dtype=torch.uint8, device=valid.device)
    v[:n] = valid.to(torch.uint8)
    w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device=valid.device)
    return (v.view(-1, 8) * w).sum(1, dtype=torch.uint8)


def dev_column(c: R.Col) -> Column:
    col = Column.device(c.dtype, c.values.shape[0], c.values.data_ptr())
    col._keep.append(c.values)
    if c.valid is not None:
        bits = pack_bits(c.valid)
        col.dev_validity = bits.data_ptr()
        col._keep.append(bits)
    return col


def dev_columns(s: R.Side):
    """Device Columns of a whole side, each bitmap packed once from bit 0; Column.slice(a, b) of them keeps
    the bitmap and gives the slice validity_bit_offset = a."""
    return [dev_column(c) for c in s.cols]


def dev_block(s: R.Side) -> DataBlock:
    return DataBlock([dev_column(c) for c in s.cols], s.n)


def types_of(s: R.Side):
    return [c.dtype | (abi.NULLABLE if c.valid is not None else 0) for c in s.cols]


def slice_side(s: R.Side, a: int, b: int) -> R.Side:
    return R.Side([R.Col(c.values[a:b], c.dtype, None if c.valid is None else c.valid[a:b]) for c in s.cols], s.keys, s.tag, s.base + a)


def release(blocks):
    for b in blocks:
        dbx_check(load().dbx_block_release(C.byref(b)))


def out_dtypes(kind, probe: R.Side, build: R.Side, final=False):
    pd, bd = [c.dtype for c in probe.cols], [c.dtype for c in build.cols]
    if final:
        return (pd if kind in (abi.JOIN_RIGHT, abi.JOIN_FULL) else []) + bd
    if kind in (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI):
        return pd
    return pd + bd


class Run:
    """One join: the operator, the reference and the verification of every block it emits."""

    def __init__(self, kind, build: R.Side, probe_types, probe_keys, build_blocks=None, expected_build_rows=0, rf=False,
                 no_unique=False, build_img=None, build_types=None, pushed=None):
        self.kind, self.rf = kind, rf
        bkeys = build.keys if len(build.keys) > 1 else build.keys[0]
        pkeys = probe_keys if len(probe_keys) > 1 else probe_keys[0]
        self.j = HashJoin(build_types or types_of(build), probe_types, bkeys, pkeys, kind=kind, expected_build_rows=expected_build_rows)
        self.load(build, build_blocks, no_unique, build_img, pushed)

    def load(self, build: R.Side, build_blocks=None, no_unique=False, build_img=None, pushed=None):
        """Push the build side (blocks [a, b) of its rows, or the DataBlocks `pushed` that hold its rows in
        order), final_build, and start the reference."""
        self.build = build
        for blk in pushed or [dev_block(slice_side(build, a, b)) for a, b in build_blocks or [(0, build.n)]]:
            self.j.add_block(blk)
        torch.cuda.synchronize()
        if no_unique:
            os.environ["DBX_JOIN_NO_UNIQUE"] = "1"
        try:
            self.j.final_build()
        finally:
            os.environ.pop("DBX_JOIN_NO_UNIQUE", None)
        self.ref = R.JoinRef(build.key_images()[0] if build_img is None else build_img, build.key_valid())
        self.f = None
        if self.rf:
            self.f = self.j.runtime_filter(in_probe=True, build_table_rows=100 * build.n)
            assert "runtime filter in the probe" in self.j.kernel_variant()
        self.out_rows = []
        self.probe_dtypes = []

    def probe(self, p: R.Side, img=None, blk=None):
        """Probe one block (the rows of `p`, pushed as `blk` if given) and check its output; returns the
        number of output rows."""
        self.probe_dtypes = [c.dtype for c in p.cols]
        lo, cnt = self.ref.probe(p.key_images()[0] if img is None else img, p.key_valid())
        blk = blk or dev_block(p)
        torch.cuda.synchronize()
        outs = self.j.probe_block(blk, out_mem=abi.MEM_DEVICE)
        try:
            rows = sum(b.num_rows for b in outs)
            cols = [R.out_cols_of(b, out_dtypes(self.kind, p, self.build)) for b in outs]
            R.check_probe_output(self.kind, cols, p, self.build, cnt)
            del cols
        finally:
            release(outs)
        self.out_rows.append(rows)
        return rows

    def finish(self, close=True):
        """final_probe, checked against the reference's matched map."""
        outs = self.j.final_probe(out_mem=abi.MEM_DEVICE)
        pd = self.probe_dtypes if self.kind in (abi.JOIN_RIGHT, abi.JOIN_FULL) else []
        try:
            cols = [R.out_cols_of(b, pd + [c.dtype for c in self.build.cols]) for b in outs]
            R.check_final_output(self.kind, cols, self.build, len(pd), self.ref.matched())
            del cols
        finally:
            release(outs)
        if self.f is not None:
            assert self.f.info().probe_rows_checked > 0
            self.f.close()
            self.f = None
        if close:
            self.j.close()


# ================================================================ 1. config 3 at full size
N_DIM = 10_000_000
N_FACT = 1_000_000_000
FACT_BLOCK = 1 << 26


@pytest.fixture(scope="module")
def dims():
    """1e7 unique Int64 dims: key, btag, a nullable F64 and a nullable Int16 (the F64 rides in the entry
    next to btag; the Int16 is gathered by build row)."""
    g = gen(7)
    i = torch.arange(N_DIM, device=DEV)
    cols = [R.Col(spread(i), abi.I64), R.Col(i.clone(), abi.I64),
            R.Col(torch.randn(N_DIM, device=DEV, generator=g, dtype=torch.float64).view(torch.int64), abi.F64,
                  torch.rand(N_DIM, device=DEV, generator=g) > 0.1),
            R.Col(torch.randint(-30000, 30000, (N_DIM,), device=DEV, generator=g, dtype=torch.int16), abi.I16,
                  torch.rand(N_DIM, device=DEV, generator=g) > 0.2)]
    return R.Side(cols, [0], 1)


def fact_block(start, n, seed):
    """About 2 % of the facts miss (keys spread from indices >= N_DIM), 1 % have NULL keys."""
    g = gen(seed)
    idx = torch.randint(0, N_DIM, (n,), device=DEV, generator=g)
    miss = torch.rand(n, device=DEV, generator=g) < 0.02
    idx = torch.where(miss, N_DIM + torch.randint(0, 1 << 40, (n,), device=DEV, generator=g), idx)
    valid = torch.rand(n, device=DEV, generator=g) >= 0.01
    return R.Side([R.Col(spread(idx), abi.I64, valid), R.Col(torch.arange(start, start + n, device=DEV), abi.I64)], [0], 1, start)


FACT_TYPES = [abi.I64 | abi.NULLABLE, abi.I64]
DIM_BLOCKS = [(0, 3_000_001), (3_000_001, 3_000_002), (3_000_002, 7_777_777), (7_777_777, N_DIM)]


@pytest.mark.parametrize("no_unique", [False, True], ids=["unique", "non_unique"])
def test_config3_inner_full_size(gpu, dims, no_unique):
    r = Run(abi.JOIN_INNER, dims, FACT_TYPES, [0], build_blocks=DIM_BLOCKS, no_unique=no_unique)
    total = 0
    for b, s in enumerate(range(0, N_FACT, FACT_BLOCK)):
        n = min(FACT_BLOCK, N_FACT - s)
        total += r.probe(fact_block(s, n, 100 + b))
    r.finish()
    assert 0.96 * N_FACT < total < 0.98 * N_FACT


@pytest.mark.parametrize("kind", [abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL], ids=["right_anti", "full"])
def test_config3_build_side_kinds(gpu, dims, kind):
    """1e8 facts: about 99.5 % of the dims are matched, so final_probe's scan over 1e7 build rows selects
    a scattered few tens of thousands."""
    r = Run(kind, dims, FACT_TYPES, [0], build_blocks=DIM_BLOCKS)
    n_fact = 100_000_000
    for b, s in enumerate(range(0, n_fact, FACT_BLOCK)):
        r.probe(fact_block(s, min(FACT_BLOCK, n_fact - s), 100 + b))
    m = r.ref.matched()
    assert 0 < int((~m).sum()) < N_DIM // 50
    r.finish()


# ================================================================ 2. many-to-many beyond L2
MM_BUILD = 30_000_000
MM_VALUES = 15_000_000
MM_PROBE = 200_000_000
MM_BLOCK = 1 << 25


@pytest.fixture(scope="module")
def mm_build():
    """3e7 rows over 1.5e7 key values (about two per key), 5 % NULL keys: cap = 2^26 entries = 2 GiB."""
    g = gen(11)
    v = torch.randint(0, MM_VALUES, (MM_BUILD,), device=DEV, generator=g)
    cols = [R.Col(spread(v), abi.I64, torch.rand(MM_BUILD, device=DEV, generator=g) >= 0.05),
            R.Col(torch.arange(MM_BUILD, device=DEV, dtype=torch.int32), abi.I32),
            R.Col(torch.randint(-2**62, 2**62, (MM_BUILD,), device=DEV, generator=g), abi.I64)]
    return R.Side(cols, [0], 1)


def mm_probe(start, n, seed):
    """Keys over 1.6e7 values (1 in 16 misses), 3 % NULL."""
    g = gen(seed)
    v = torch.randint(0, MM_VALUES + MM_VALUES // 15, (n,), device=DEV, generator=g)
    return R.Side([R.Col(spread(v), abi.I64, torch.rand(n, device=DEV, generator=g) >= 0.03),
                   R.Col(torch.arange(start, start + n, device=DEV), abi.I64)], [0], 1, start)


@pytest.mark.parametrize("kind,rf", [(k, False) for k in R.ALL_KINDS] + [(abi.JOIN_INNER, True), (abi.JOIN_RIGHT_SEMI, True)],
                         ids=[R.KIND_NAMES[k] for k in R.ALL_KINDS] + ["inner_rf", "right_semi_rf"])
def test_many_to_many_beyond_l2(gpu, mm_build, kind, rf):
    r = Run(kind, mm_build, FACT_TYPES, [0], build_blocks=[(0, 9_999_999), (9_999_999, MM_BUILD)], rf=rf)
    for b, s in enumerate(range(0, MM_PROBE, MM_BLOCK)):
        n = min(MM_BLOCK, MM_PROBE - s)
        rows = r.probe(mm_probe(s, n, 500 + b))
        if kind in (abi.JOIN_INNER, abi.JOIN_LEFT, abi.JOIN_RIGHT, abi.JOIN_FULL):
            # more rows than the first attempt's capacity: every block takes the exact-size retry
            assert rows > n + n // 8 + 1024, (b, rows, n)
    r.finish()


# ================================================================ 3. runs across the table's end
KEY_LAYOUTS = {  # build key dtypes (as many as key columns), probe key dtypes
    "i64": ([abi.I64], [abi.I64]),
    "i32": ([abi.I32], [abi.I32]),
    "packed_2xi32": ([abi.I32, abi.I32], [abi.I32, abi.I32]),
    "wide_2xi64": ([abi.I64, abi.I64], [abi.I64, abi.I64]),
}
RUNS = {1024: (8, 300, 0), 1 << 21: (4096, 8192, 520_000), 1 << 25: (4096, 8192, 10_000_000)}  # cap: (width, cluster keys, others)


def key_columns(layout, slots, cap, rng):
    """Key column values (numpy, one array per key column) of keys homed at `slots`, by inverting the hash
    (the "i32" layout searches the 32-bit space instead: narrow_keys)."""
    if layout == "i64":
        return [R.words_homed_at(slots, cap, rng).view(np.int64)]
    if layout == "packed_2xi32":
        w = R.words_homed_at(slots, cap, rng)
        return [(w & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.int32), (w >> np.uint64(32)).astype(np.uint32).view(np.int32)]
    if layout == "wide_2xi64":
        k0, k1 = R.wide_words_homed_at(slots, cap, rng)
        return [k0.view(np.int64), k1.view(np.int64)]
    raise ValueError(layout)


def narrow_keys(lo, hi, cap, count, start, exclude):
    v = R.narrow_values_homed_in(lo, hi, cap, count + len(exclude), abi.I32, start)
    v = np.setdiff1d(v, exclude)
    assert len(v) >= count
    return v[:count]


def run_scenario(layout, cap, dup, rng):
    """Build and probe key columns (numpy) for a table of `cap` slots: a cluster of keys homed in the
    last `width` slots, keys homed in the wrapped part [0, 32), ordinary keys, and NULL-key rows.
    Returns (build key arrays, build valid, probe key arrays, probe valid)."""
    width, n_cluster, n_other = RUNS[cap]
    n_keys = n_cluster // 2 if dup else n_cluster
    copies = 2 if dup else 1
    if layout == "i32":
        top = narrow_keys(cap - width, cap, cap, n_keys, -2**31, np.array([], np.int32))
        wrap = narrow_keys(0, 32, cap, 16, -2**31, top)
        absent_top = narrow_keys(cap - width, cap, cap, min(width, 512), 0, np.concatenate([top, wrap]))
        absent_wrap = narrow_keys(0, min(2 * width, 512), cap, 256, 0, np.concatenate([top, wrap]))
        used = np.concatenate([top, wrap, absent_top, absent_wrap])
        other = np.setdiff1d(np.unique(rng.integers(-2**31, 2**31, int(n_other * 1.1) + 10).astype(np.int32)), used)
        other = rng.permutation(other)[:n_other]
        assert len(other) == n_other
        b_keys = [np.concatenate([np.repeat(top, copies), wrap, other])]
        absent = [np.concatenate([absent_top, absent_wrap])]
    else:
        top = key_columns(layout, rng.integers(cap - width, cap, n_keys), cap, rng)
        wrap = key_columns(layout, rng.integers(0, 32, 16), cap, rng)
        other = key_columns(layout, rng.integers(0, cap, n_other), cap, rng)
        absent_top = key_columns(layout, rng.integers(cap - width, cap, min(width, 512)), cap, rng)
        absent_wrap = key_columns(layout, rng.integers(0, min(2 * width, 512), 256), cap, rng)
        b_keys = [np.concatenate([np.repeat(t, copies), w, o]) for t, w, o in zip(top, wrap, other)]
        absent = [np.concatenate([a, b]) for a, b in zip(absent_top, absent_wrap)]
    nb = len(b_keys[0])
    b_keys = [np.concatenate([k, k[:8]]) for k in b_keys]  # 8 NULL-key rows
    b_valid = np.concatenate([np.ones(nb, bool), np.zeros(8, bool)])
    # probe: every cluster and wrapped key twice, a sample of ordinary keys, the absent keys, NULLs
    n_cw = n_keys * copies + 16
    sample = rng.choice(np.arange(n_cw, nb), min(nb - n_cw, 200_000), replace=False) if nb > n_cw else np.array([], np.int64)
    rows = np.concatenate([np.arange(n_cw), np.arange(n_cw), sample])
    p_keys = [np.concatenate([k[rows], a]) for k, a in zip(b_keys, absent)]
    npr = len(p_keys[0])
    p_valid = rng.random(npr) >= 0.05
    perm = rng.permutation(npr)
    return b_keys, b_valid, [k[perm] for k in p_keys], p_valid[perm]


def scenario_sides(b_keys, b_valid, p_keys, p_valid, rng):
    nk = len(b_keys)
    nb, npr = len(b_keys[0]), len(p_keys[0])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    dt = abi.I64 if b_keys[0].dtype == np.int64 else abi.I32
    bcols = [R.Col(t(k), dt, t(b_valid) if i == 0 else None) for i, k in enumerate(b_keys)]
    bcols += [R.Col(torch.arange(nb, device=DEV), abi.I64),
              R.Col(t(rng.integers(-2**31, 2**31, nb).astype(np.int32)), abi.I32, t(rng.random(nb) > 0.2))]
    pcols = [R.Col(t(k), dt, t(p_valid) if i == 0 else None) for i, k in enumerate(p_keys)]
    pcols += [R.Col(torch.arange(npr, device=DEV), abi.I64)]
    return R.Side(bcols, list(range(nk)), nk), R.Side(pcols, list(range(nk)), nk)


def run_all_kinds(build: R.Side, probe: R.Side, single_key, cuts=None, **kw):
    bimg, pimg = R.combined_images(build.key_images(), probe.key_images())
    cuts = cuts or [0, probe.n // 3, probe.n]
    modes = [(k, False) for k in R.ALL_KINDS]
    if single_key:
        modes += [(abi.JOIN_INNER, True), (abi.JOIN_RIGHT_SEMI, True)]
    for kind, rf in modes:
        r = Run(kind, build, types_of(probe), probe.keys, rf=rf, build_img=bimg, **kw)
        for a, b in zip(cuts[:-1], cuts[1:]):
            r.probe(slice_side(probe, a, b), pimg[a:b])
        r.finish()


# the Int32 keys are searched for on the host, so they stop at 2^21 slots
RUN_CASES = [(cap, layout) for cap in RUNS for layout in KEY_LAYOUTS if not (layout == "i32" and cap == 1 << 25)]


@pytest.mark.parametrize("dup", [False, True], ids=["unique", "dup"])
@pytest.mark.parametrize("cap,layout", RUN_CASES, ids=[f"cap{c}-{l}" for c, l in RUN_CASES])
def test_runs_across_the_table_end(gpu, cap, layout, dup):
    rng = np.random.default_rng(cap + 7 * dup + len(layout))
    b_keys, b_valid, p_keys, p_valid = run_scenario(layout, cap, dup, rng)
    build, probe = scenario_sides(b_keys, b_valid, p_keys, p_valid, rng)
    assert R.next_pow2_cap(build.n) == cap
    run_all_kinds(build, probe, single_key=len(b_keys) == 1)


@pytest.mark.parametrize("layout", list(KEY_LAYOUTS))
def test_duplicate_pair_straddles_the_end(gpu, layout):
    """A key with two entries homed at slot cap - 1 and nothing else homed there or at 0: the pair sits
    in slots 1023 and 0 of a 1024-slot table (tests/test_join_scale_ref_cpu.py simulates it)."""
    cap = 1024
    rng = np.random.default_rng(41 + len(layout))
    if layout == "i32":
        pair = narrow_keys(cap - 1, cap, cap, 1, -2**31, np.array([], np.int32))
        others = narrow_keys(2, cap // 2, cap, 200, 0, pair)
        b_keys = [np.concatenate([pair, pair, others])]
        p_keys = [np.concatenate([pair, pair, others, narrow_keys(cap - 1, cap, cap, 4, 0, np.concatenate([pair, others]))])]
    else:
        pair = key_columns(layout, np.array([cap - 1]), cap, rng)
        others = key_columns(layout, rng.integers(2, cap // 2, 200), cap, rng)
        absent = key_columns(layout, np.full(4, cap - 1), cap, rng)  # absent keys homed at cap - 1 walk past the pair
        b_keys = [np.concatenate([p, p, o]) for p, o in zip(pair, others)]
        p_keys = [np.concatenate([p, p, o, a]) for p, o, a in zip(pair, others, absent)]
    build, probe = scenario_sides(b_keys, np.ones(len(b_keys[0]), bool), p_keys, rng.random(len(p_keys[0])) > 0.02, rng)
    assert R.next_pow2_cap(build.n) == cap
    run_all_kinds(build, probe, single_key=len(b_keys) == 1, cuts=[0, probe.n])


# ================================================================ 4. every key-type pair
INFO = {dt: np.iinfo(R.NP_DTYPE[dt]) for dt in R.INT_TYPES}
SPECIALS = sorted({v for dt in R.INT_TYPES for v in (int(INFO[dt].min), int(INFO[dt].max), 0, 1, -1)} |
                  {255, 65535, 2**32 - 1, 127, -128, 2**63 - 1})


def values_of(dt):
    """Every special value representable in dt: each type's min, max, 0, +-1, and the values whose raw bits
    alias across types (UInt8 255 / Int8 -1, UInt16 65535 / Int16 -1, UInt32 2^32 - 1 / Int32 -1 / Int64 2^32 - 1)."""
    return [v for v in SPECIALS if INFO[dt].min <= v <= INFO[dt].max]


def refused(bt, pt):
    return (bt == abi.U64 and pt in R.SIGNED) or (pt == abi.U64 and bt in R.SIGNED)


def int_col(vals, dt, valid=None):
    a = np.array(vals, dtype=object).astype(R.NP_DTYPE[dt])
    return R.Col(torch.from_numpy(a.view(f"i{a.itemsize}")).to(DEV), dt, None if valid is None else torch.tensor(valid, device=DEV))


@pytest.mark.parametrize("bt", R.INT_TYPES, ids=[np.dtype(R.NP_DTYPE[d]).name for d in R.INT_TYPES])
def test_every_key_type_pair(gpu, bt):
    for pt in R.INT_TYPES:
        for two in (False, True):
            bkeys, pkeys = ([0, 2], [0, 2]) if two else (0, 0)
            btypes = [bt | abi.NULLABLE, abi.I64] + ([abi.I32] if two else [])
            ptypes = [pt | abi.NULLABLE, abi.I64] + ([abi.I32] if two else [])
            if refused(bt, pt):
                with pytest.raises(DbxError) as e:
                    HashJoin(btypes, ptypes, bkeys, pkeys)
                assert e.value.status == abi.ERR_UNSUPPORTED and "UInt64" in e.value.message
                continue
            bv, pv = values_of(bt), values_of(pt)
            second = [-2**31, -1, 0, 2**31 - 1]
            if two:  # every first value with every second value on the build side; the probe misses some seconds
                brows = [(v, s) for v in bv for s in second] + [(0, 0)]
                prows = [(v, s) for v in pv for s in second + [5]] * 2 + [(0, 0)]
            else:
                brows = [(v, 0) for v in bv] + [(0, 0)]
                prows = [(v, 0) for v in pv] * 3 + [(0, 0)]
            bvalid = [True] * (len(brows) - 1) + [False]  # one NULL key row on each side
            pvalid = [True] * (len(prows) - 1) + [False]
            bcols = [int_col([r[0] for r in brows], bt, bvalid), R.Col(torch.arange(len(brows), device=DEV), abi.I64)]
            pcols = [int_col([r[0] for r in prows], pt, pvalid), R.Col(torch.arange(len(prows), device=DEV), abi.I64)]
            if two:
                bcols.append(int_col([r[1] for r in brows], abi.I32))
                pcols.append(int_col([r[1] for r in prows], abi.I32))
            build = R.Side(bcols, [0, 2] if two else [0], 1)
            probe = R.Side(pcols, [0, 2] if two else [0], 1)
            # the expected counts by Python-integer equality, against the reference's
            exp = [sum(1 for b, bok in zip(brows, bvalid) if bok and pok and b == p) for p, pok in zip(prows, pvalid)]
            bimg, pimg = R.combined_images(build.key_images(), probe.key_images())
            ref = R.JoinRef(bimg, build.key_valid())
            _, cnt = ref.probe(pimg, probe.key_valid())
            assert cnt.tolist() == exp, (bt, pt, two)
            assert sum(exp) >= 4  # 0 and 1 match in every pair
            modes = [(abi.JOIN_INNER, False), (abi.JOIN_LEFT_ANTI, False), (abi.JOIN_RIGHT_SEMI, False)]
            if not two:
                modes.append((abi.JOIN_INNER, True))
            for kind, rf in modes:
                r = Run(kind, build, ptypes, probe.keys, rf=rf, build_img=bimg, build_types=btypes)
                r.probe(probe, pimg)
                r.finish()


# ================================================================ 5. block shapes and lifecycle
def small_build(n, n_values, seed, nullable=True):
    g = gen(seed)
    v = torch.randint(0, n_values, (n,), device=DEV, generator=g)
    cols = [R.Col(spread(v), abi.I64, (torch.rand(n, device=DEV, generator=g) > 0.05) if nullable else None),
            R.Col(torch.arange(n, device=DEV), abi.I64),
            R.Col(torch.randint(-100, 100, (n,), device=DEV, generator=g, dtype=torch.int16), abi.I16,
                  torch.rand(n, device=DEV, generator=g) > 0.3),
            R.Col(torch.randint(-2**31, 2**31, (n,), device=DEV, generator=g, dtype=torch.int32), abi.I32)]
    return R.Side(cols, [0], 1)


def small_probe(start, n, n_values, seed, pad=0):
    """Probe rows over 1.25 x n_values values; `pad` extra leading rows so a slice starts at an odd bit."""
    g = gen(seed)
    m = n + pad
    v = torch.randint(0, n_values + n_values // 4, (m,), device=DEV, generator=g)
    s = R.Side([R.Col(spread(v), abi.I64, torch.rand(m, device=DEV, generator=g) > 0.05),
                R.Col(torch.arange(start - pad, start + n, device=DEV), abi.I64),
                R.Col(torch.randint(-100, 100, (m,), device=DEV, generator=g, dtype=torch.int8), abi.I8,
                      torch.rand(m, device=DEV, generator=g) > 0.5)], [0], 1, start - pad)
    return slice_side(s, pad, m) if pad else s


PROBE_TYPES = [abi.I64 | abi.NULLABLE, abi.I64, abi.I8 | abi.NULLABLE]
SHAPES = [1, 255, 256, 257, 511, 512, 513, (1 << 20) + 1]


@pytest.mark.parametrize("dup", [False, True], ids=["unique", "dup"])
def test_probe_block_shapes(gpu, dup):
    """Blocks around the 512-row step of the two-rows-per-thread probe, one after the other."""
    nb = 100_000
    n_values = nb // 2 if dup else 10 * nb
    build = small_build(nb, n_values, 21 + dup)
    if not dup:  # distinct keys: spread() of distinct values
        build.cols[0] = R.Col(spread(torch.randperm(n_values, device=DEV, generator=gen(3))[:nb]), abi.I64, build.cols[0].valid)
        build._img = []
    for kind, rf in [(k, False) for k in R.ALL_KINDS] + [(abi.JOIN_INNER, True)]:
        r = Run(kind, build, PROBE_TYPES, [0], rf=rf)
        s = 0
        for i, n in enumerate(SHAPES):
            r.probe(small_probe(s, n, n_values, 50 + i))
            s += n
        r.finish()


ODD_STARTS = [1, 2, 3, 4, 5, 6, 7, 9, 4099]  # validity bit offsets 1 .. 7, and two above one byte


def test_odd_offset_device_slices(gpu):
    """Device-resident blocks that are Column.slice()s of whole device columns, starting at rows
    s + 4096 k for the starts s of ODD_STARTS: every nullable column reaches the join with the whole
    bitmap and validity_bit_offset = the block's first row (nonzero, 1 .. 7 mod 8, not reduced mod 8),
    on the build side (push: bits to bytes) and the probe side (key and carried columns)."""
    nb = 40_000
    full = small_build(nb, nb // 3, 31)
    # build blocks [a, b) with a = start + 4096 k (a % 8 = start % 8); the rows between them are never pushed
    cuts = [(a + 4096 * k, a + 4096 * k + 1500 + 37 * k) for k, a in enumerate(ODD_STARTS)]
    btag = torch.full((nb,), -1, dtype=torch.int64, device=DEV)  # btag = position among the pushed rows
    base = 0
    for a, b in cuts:
        btag[a:b] = torch.arange(base, base + b - a, device=DEV)
        base += b - a
    full.cols[1] = R.Col(btag, abi.I64)
    bcols = dev_columns(full)
    rows = torch.cat([torch.arange(a, b, device=DEV) for a, b in cuts])
    build = R.Side([R.Col(c.values[rows], c.dtype, None if c.valid is None else c.valid[rows]) for c in full.cols], [0], 1)
    # the probe: one whole side, ptag = row, probed as slices at the same kind of starts
    pfull = small_probe(0, 60_000, nb // 3, 70)
    pcols = dev_columns(pfull)
    pcuts = [(a + 4096 * k, a + 4096 * k + 3000 + 7 * k) for k, a in enumerate(ODD_STARTS)] + [(50_003, 60_000)]
    torch.cuda.synchronize()

    def sliced(cols, a, b):
        blk = DataBlock([c.slice(a, b) for c in cols], b - a)
        for c, full_c in zip(blk.columns, cols):  # the same bitmap, offset by a
            assert (c.dev_validity, c.validity_bit_offset) == ((full_c.dev_validity, a) if full_c.dev_validity else (0, 0))
        assert a % 8 != 0
        return blk
    for kind in (abi.JOIN_INNER, abi.JOIN_LEFT, abi.JOIN_FULL, abi.JOIN_RIGHT_SEMI):
        r = Run(kind, build, PROBE_TYPES, [0], pushed=[sliced(bcols, a, b) for a, b in cuts])
        for a, b in pcuts:
            r.probe(slice_side(pfull, a, b), blk=sliced(pcols, a, b))
        r.finish()


@pytest.mark.parametrize("hint", [0, 10, 50_000_000], ids=["no_hint", "too_small", "too_large"])
def test_build_block_sizes_and_growth(gpu, hint):
    """Build blocks of 1, 7, 4095 and 65 537 rows, repeated: the build columns grow by copies many times."""
    sizes = [1, 7, 4095, 65_537] * 3
    nb = sum(sizes)
    build = small_build(nb, nb // 3, 41)
    cuts, s = [], 0
    for n in sizes:
        cuts.append((s, s + n))
        s += n
    for kind in (abi.JOIN_INNER, abi.JOIN_RIGHT, abi.JOIN_LEFT_SEMI):
        r = Run(kind, build, PROBE_TYPES, [0], build_blocks=cuts, expected_build_rows=hint)
        r.probe(small_probe(0, 300_000, nb // 3, 90))
        r.finish()


@pytest.mark.parametrize("kind", [abi.JOIN_RIGHT, abi.JOIN_FULL], ids=["right", "full"])
def test_reset_large_small_large(gpu, kind):
    """reset() and rebuild at cap 2^25, then 1024, then 2^25 again on one operator: no stale table
    entries or matched bytes may leak into the next build's results.  The probe keys overlap every
    build's keys (the same spread values), so a stale entry would match."""
    r = None
    for step, (nb, seed) in enumerate([(9_000_000, 41), (300, 42), (8_500_000, 43)]):
        build = small_build(nb, nb // 2, seed)
        assert R.next_pow2_cap(nb) == (1024 if nb == 300 else 1 << 25)
        if r is None:
            r = Run(kind, build, PROBE_TYPES, [0])
        else:
            r.j.reset()
            r.load(build)
        r.probe(small_probe(0, 2_000_000, 4_000_000, 95 + step))
        r.finish(close=False)
    r.j.close()


# ================================================================ 6. more than 2^32 rows from one probe block
# Device memory: the output is 2^25 x 130 = 4 362 076 160 rows of Int8 pkey + Int32 ptag + Int8 bkey +
# UInt16 btag = 8 B per row, 32.5 GiB, allocated once the first attempt (1.125 x 2^25 rows, 0.3 GiB, kept
# by the library's pool) overflows.  The probe block is 160 MiB, the per-ptag accumulators 3 x 256 MiB,
# and one 2^26-row chunk of the check holds at most about 3 GiB of int64 temporaries (ptag, btag image,
# ones, btag^2, each 512 MiB, and a copy or two in flight).  About 37 GiB in all, with the CUDA context;
# measured on an H100 80GB HBM3: 32.8 GiB after the probe, 35.2 GiB at the check's peak.
NEED_2POW32 = 40 << 30
BIG_CHUNK = 1 << 26
BIG_KEYS, BIG_DUPS, BIG_PROBE = 256, 130, 1 << 25

_BIG = r"""
import sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import test_join_scale_gpu as t
t.more_than_2pow32_rows()
print("ok")
"""


def more_than_2pow32_rows():
    """The check, run in its own process so the 32 GiB the library's pool keeps afterwards go with it.

    A full pair sort does not fit next to the output, so the rows are checked in chunks: every row's
    build key equals its probe key (and the probe key is the probe row's), each ptag occurs exactly 130
    times, and per ptag the sums of btag and btag^2 equal those of the 130 build rows of its key.  A row
    lost, never written, or overwritten through a position truncated to 32 bits changes a ptag's count
    or its sums (an overwrite replaces one ptag's (ptag, btag) by another's)."""
    free0, _ = torch.cuda.mem_get_info(0)
    bk = torch.arange(BIG_KEYS, device=DEV).repeat_interleave(BIG_DUPS)  # 0..255 as Int8 bits -128..127
    nb = bk.shape[0]
    build = R.Side([R.Col(bk.to(torch.int8), abi.I8), R.Col(torch.arange(nb, device=DEV).to(torch.int16), abi.U16)], [0], 1)
    g = gen(77)
    pk = torch.randint(-128, 128, (BIG_PROBE,), device=DEV, generator=g, dtype=torch.int8)
    ptag = torch.arange(BIG_PROBE, device=DEV, dtype=torch.int32)
    j = HashJoin([abi.I8, abi.U16], [abi.I8, abi.I32], 0, 0)
    j.add_block(dev_block(build))
    j.final_build()
    blk = DataBlock([dev_column(R.Col(pk, abi.I8)), dev_column(R.Col(ptag, abi.I32))], BIG_PROBE)
    torch.cuda.synchronize()
    outs = j.probe_block(blk, out_mem=abi.MEM_DEVICE)
    free1, _ = torch.cuda.mem_get_info(0)
    total = sum(b.num_rows for b in outs)
    assert total == BIG_PROBE * BIG_DUPS > 2**32, total
    # expected per key (Int8 value v): sums of btag and btag^2 over its 130 build rows
    bt = torch.arange(nb, device=DEV)
    key_of = build.cols[0].values.to(torch.int64) + 128
    s1 = torch.zeros(256, dtype=torch.int64, device=DEV).index_add_(0, key_of, bt)
    s2 = torch.zeros(256, dtype=torch.int64, device=DEV).index_add_(0, key_of, bt * bt)
    cnt = torch.zeros(BIG_PROBE, dtype=torch.int64, device=DEV)
    g1 = torch.zeros(BIG_PROBE, dtype=torch.int64, device=DEV)
    g2 = torch.zeros(BIG_PROBE, dtype=torch.int64, device=DEV)
    chunk = BIG_CHUNK
    free_min = free1
    try:
        for b in outs:
            cols = R.out_cols_of(b, [abi.I8, abi.I32, abi.I8, abi.U16])
            n = b.num_rows
            for s in range(0, n, chunk):
                e = min(n, s + chunk)
                p = cols[1].values[s:e].to(torch.int64)
                assert bool(((p >= 0) & (p < BIG_PROBE)).all()), f"ptag out of range in rows [{s}, {e})"
                assert bool((cols[0].values[s:e] == pk[p]).all()), f"probe key is not the probe row's in [{s}, {e})"
                assert bool((cols[2].values[s:e] == cols[0].values[s:e]).all()), f"build key != probe key in [{s}, {e})"
                q = R.image(cols[3].values[s:e], abi.U16)
                cnt.index_add_(0, p, torch.ones_like(p))
                g1.index_add_(0, p, q)
                g2.index_add_(0, p, q * q)
                free_min = min(free_min, torch.cuda.mem_get_info(0)[0])
                del p, q
            del cols
    finally:
        release(outs)
    k = pk.to(torch.int64) + 128
    bad = cnt != BIG_DUPS
    assert not bool(bad.any()), f"{int(bad.sum())} ptags without exactly {BIG_DUPS} rows, first {R._first_bad(bad)}"
    bad = (g1 != s1[k]) | (g2 != s2[k])
    assert not bool(bad.any()), f"{int(bad.sum())} ptags with the wrong btag sums, first {R._first_bad(bad)}"
    j.close()
    print(f"{total} output rows; device memory in use: {(free0 - free1) / 2**30:.1f} GiB after the probe, "
          f"{(free0 - free_min) / 2**30:.1f} GiB at the check's peak (sampled after each chunk's temporaries; "
          f"torch's own peak reserved {torch.cuda.max_memory_reserved(0) / 2**30:.1f} GiB)")


def test_more_than_2pow32_rows_from_one_probe_block(gpu):
    free, _ = torch.cuda.mem_get_info(0)
    if free < NEED_2POW32:
        pytest.skip(f"needs about {NEED_2POW32 >> 30} GiB of free device memory, {free / 2**30:.1f} GiB free")
    r = subprocess.run([sys.executable, "-c", _BIG, ROOT, os.path.dirname(os.path.abspath(__file__))],
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().endswith("ok")
    print(r.stdout)
