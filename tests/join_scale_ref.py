"""Exact hash-join reference and output verifier in torch, for joins too large for the CPU oracles.

The reference uses no hash table.  The widened key images of the valid build rows are sorted once;
each probe row's matches are the range [lo, hi) that `searchsorted` gives for its key image, so its
expected match count is hi - lo (0 for a NULL key).  The ranges are difference-arrayed back onto the
sorted build rows and accumulated across probe blocks, which gives the matched map the build-side
kinds (RIGHT, RIGHT SEMI, RIGHT ANTI, FULL) select from, without holding every probe row at once.
Everything runs wherever its tensors live: the GPU tests keep it on the device,
tests/test_join_scale_ref_cpu.py holds it against `oracle.hash_join` and `join_build_side_ref` on the CPU.

The verifier needs a unique row tag on each side (a probe column `ptag`, a build column `btag`).  An
output block of a probe-phase kind is exactly right if and only if
  1. every pair is valid: both keys non-NULL, equal key images, and every output column equal to its
     source row (the probe row named by ptag, the build row named by btag) in value and validity;
  2. the number of output rows of each probe row equals its expected count;
  3. no (ptag, btag) pair occurs twice.
1 and 3 make the output a set of true pairs, 2 makes it all of them.  LEFT / FULL add the unmatched
probe rows once each with every build column NULL; LEFT SEMI / LEFT ANTI emit each selected probe row
once.  final_probe blocks must hold exactly the selected build rows, with a Const NULL probe side.

Also the slot construction of the table-geometry tests: the join's home slot is
agg_hash_u64(image) & (cap - 1), and agg_hash_u64 is a bijection of 64-bit words (xor-shift by 32 is
an involution, 0xd6e8feb86659fd93 has the inverse 0xcfee444d8b59a89b mod 2^64), so a key can be
computed for any chosen home slot."""
from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
import torch

from databend_b200 import abi
from databend_b200.exchange import agg_hash_np

# torch storage of every fixed-width dtype: a signed integer view of the same width (bit-exact)
TORCH_DTYPE = {abi.I8: torch.int8, abi.U8: torch.int8, abi.I16: torch.int16, abi.U16: torch.int16, abi.I32: torch.int32,
               abi.U32: torch.int32, abi.I64: torch.int64, abi.U64: torch.int64, abi.F32: torch.int32, abi.F64: torch.int64}
NP_DTYPE = {abi.I8: np.int8, abi.U8: np.uint8, abi.I16: np.int16, abi.U16: np.uint16, abi.I32: np.int32, abi.U32: np.uint32,
            abi.I64: np.int64, abi.U64: np.uint64, abi.F32: np.float32, abi.F64: np.float64}
SIGNED = (abi.I8, abi.I16, abi.I32, abi.I64)
UNSIGNED = (abi.U8, abi.U16, abi.U32, abi.U64)
INT_TYPES = SIGNED + UNSIGNED
PROBE_SIDE_KINDS = (abi.JOIN_INNER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI, abi.JOIN_LEFT)
BUILD_SIDE_KINDS = (abi.JOIN_RIGHT, abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL)
ALL_KINDS = PROBE_SIDE_KINDS + BUILD_SIDE_KINDS
KIND_NAMES = {abi.JOIN_INNER: "inner", abi.JOIN_LEFT_SEMI: "left_semi", abi.JOIN_LEFT_ANTI: "left_anti", abi.JOIN_LEFT: "left",
              abi.JOIN_RIGHT: "right", abi.JOIN_RIGHT_SEMI: "right_semi", abi.JOIN_RIGHT_ANTI: "right_anti", abi.JOIN_FULL: "full"}

MUL = 0xD6E8FEB86659FD93
INV_MUL = 0xCFEE444D8B59A89B
GOLDEN = 0x9E3779B97F4A7C15


def dtype_bits(dtype: int) -> int:
    return 8 * np.dtype(NP_DTYPE[dtype]).itemsize


def image(values: torch.Tensor, dtype: int) -> torch.Tensor:
    """The 64-bit key image as int64 bits: signed keys sign-extended, unsigned ones zero-extended."""
    v = values.to(torch.int64)
    bits = dtype_bits(dtype)
    if dtype in UNSIGNED and bits < 64:
        v = v & ((1 << bits) - 1)
    return v


# ---------------------------------------------------------------- the two sides
@dataclass
class Col:
    """A column in torch: `values` in TORCH_DTYPE[dtype], `valid` a bool tensor or None (all valid)."""
    values: torch.Tensor
    dtype: int
    valid: Optional[torch.Tensor] = None

    def valid_or_ones(self) -> torch.Tensor:
        return self.valid if self.valid is not None else torch.ones(self.values.shape[0], dtype=torch.bool, device=self.values.device)


@dataclass
class Side:
    """The rows of one side: its columns, the key columns and the tag column.  `base` is the tag of row 0
    (a probe block's first global row), so the tag of row i is base + i."""
    cols: List[Col]
    keys: List[int]
    tag: int
    base: int = 0
    _img: list = field(default_factory=list, repr=False)

    @property
    def n(self) -> int:
        return self.cols[0].values.shape[0]

    def key_images(self) -> List[torch.Tensor]:
        if not self._img:
            self._img = [image(self.cols[k].values, self.cols[k].dtype) for k in self.keys]
        return self._img

    def key_valid(self) -> torch.Tensor:
        v = torch.ones(self.n, dtype=torch.bool, device=self.cols[0].values.device)
        for k in self.keys:
            if self.cols[k].valid is not None:
                v &= self.cols[k].valid
        return v


def combined_images(build_imgs: List[torch.Tensor], probe_imgs: List[torch.Tensor]):
    """One int64 image per row for composite keys, equal exactly when every key pair is equal: each
    pair's images are replaced by their rank among the images of both sides, and the ranks are
    combined in mixed radix."""
    if len(build_imgs) == 1:
        return build_imgs[0], probe_imgs[0]
    nb = build_imgs[0].shape[0]
    bc = torch.zeros(nb, dtype=torch.int64, device=build_imgs[0].device)
    pc = torch.zeros(probe_imgs[0].shape[0], dtype=torch.int64, device=probe_imgs[0].device)
    scale = 1
    for b, p in zip(build_imgs, probe_imgs):
        u, inv = torch.unique(torch.cat([b, p]), return_inverse=True)
        bc += inv[:nb] * scale
        pc += inv[nb:] * scale
        scale *= u.shape[0]
        assert scale < 1 << 62, "composite key ranks overflow the combined image"
    return bc, pc


# ---------------------------------------------------------------- the reference
class JoinRef:
    """Expected match counts by sorting, and the matched map accumulated across probe blocks."""

    def __init__(self, build_img: torch.Tensor, build_valid: Optional[torch.Tensor]):
        dev = build_img.device
        self.n_build = build_img.shape[0]
        rows = torch.arange(self.n_build, device=dev) if build_valid is None else build_valid.nonzero().flatten()
        self.keys, order = torch.sort(build_img[rows], stable=True)
        self.rows = rows[order]
        self.diff = torch.zeros(self.rows.shape[0] + 1, dtype=torch.int64, device=dev)

    def probe(self, probe_img: torch.Tensor, probe_valid: Optional[torch.Tensor]):
        """(lo, count) per probe row: its matches are the sorted build rows self.rows[lo : lo + count].
        The block's matches are added to the matched map."""
        lo = torch.searchsorted(self.keys, probe_img, right=False)
        hi = torch.searchsorted(self.keys, probe_img, right=True)
        cnt = hi - lo
        if probe_valid is not None:
            cnt = torch.where(probe_valid, cnt, torch.zeros_like(cnt))
        hit = cnt > 0
        one = torch.ones(int(hit.sum()), dtype=torch.int64, device=lo.device)
        self.diff.index_add_(0, lo[hit], one)
        self.diff.index_add_(0, hi[hit], -one)
        return lo, cnt

    def matched(self) -> torch.Tensor:
        """Build rows matched by at least one probe row so far (NULL-key rows never are)."""
        m = torch.zeros(self.n_build, dtype=torch.bool, device=self.diff.device)
        m[self.rows] = torch.cumsum(self.diff, 0)[:-1] > 0
        return m

    def pairs(self, lo: torch.Tensor, cnt: torch.Tensor):
        """Every matching (probe row, build row) pair of a block, materialised (small inputs only)."""
        p = torch.repeat_interleave(torch.arange(cnt.shape[0], device=cnt.device), cnt)
        first = torch.cumsum(cnt, 0) - cnt
        off = torch.arange(p.shape[0], device=cnt.device) - first[p]
        return p, self.rows[lo[p] + off]


def expected_rows(kind: int, cnt: torch.Tensor) -> torch.Tensor:
    """Output rows of each probe row during the probe, per kind."""
    if kind in (abi.JOIN_LEFT_SEMI,):
        return (cnt > 0).to(torch.int64)
    if kind == abi.JOIN_LEFT_ANTI:
        return (cnt == 0).to(torch.int64)
    if kind in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI):
        return torch.zeros_like(cnt)
    if kind in (abi.JOIN_LEFT, abi.JOIN_FULL):
        return torch.clamp(cnt, min=1)
    return cnt


# ---------------------------------------------------------------- output blocks
@dataclass
class OutCol:
    """One output column: values (None for a Const entry), valid (None: all valid), const_null."""
    values: Optional[torch.Tensor]
    valid: Optional[torch.Tensor] = None
    const_null: bool = False


def unpack_bits(bits: torch.Tensor, n: int) -> torch.Tensor:
    """LSB-first bitmap (uint8 tensor) -> n bools."""
    shifts = torch.arange(8, dtype=torch.uint8, device=bits.device)
    return ((bits[: (n + 7) // 8].unsqueeze(1) >> shifts) & 1).flatten()[:n].bool()


def out_cols_of(block, dtypes: List[int], device: int = 0) -> List[OutCol]:
    """Views of a library-owned device block (dbx_op_pull with DBX_MEM_DEVICE): valid until it is released."""
    from databend_b200.distributed import _dev_tensor
    cols = []
    assert block.num_cols == len(dtypes), (block.num_cols, dtypes)
    for i, dt in enumerate(dtypes):
        c = block.cols[i]
        assert c.dtype == dt, (i, c.dtype, dt)
        if c.is_const:
            cols.append(OutCol(None, None, bool(c.konst.is_null)))
            continue
        assert c.mem == abi.MEM_DEVICE
        n = c.len
        size = np.dtype(NP_DTYPE[dt]).itemsize
        v = _dev_tensor(c.data, n * size, device).view(TORCH_DTYPE[dt]) if n else torch.empty(0, dtype=TORCH_DTYPE[dt], device=f"cuda:{device}")
        valid = unpack_bits(_dev_tensor(c.validity, (n + 7) // 8, device), n) if c.validity and n else None
        cols.append(OutCol(v, valid))
    return cols


def _first_bad(mask: torch.Tensor, n: int = 5):
    return mask.nonzero().flatten()[:n].tolist()


def _check_col(what: str, got: OutCol, src: Col, rows: torch.Tensor):
    """got[i] == src[rows[i]] in validity, and in value where valid."""
    assert got.values is not None, f"{what}: a Const column where values were expected"
    assert got.values.shape[0] == rows.shape[0], f"{what}: {got.values.shape[0]} rows, expected {rows.shape[0]}"
    exp_valid = src.valid[rows] if src.valid is not None else None
    gv = got.valid
    if exp_valid is not None or gv is not None:
        ev = exp_valid if exp_valid is not None else torch.ones_like(rows, dtype=torch.bool)
        gv = gv if gv is not None else torch.ones_like(rows, dtype=torch.bool)
        bad = ev != gv
        assert not bool(bad.any()), f"{what}: validity differs at {int(bad.sum())} rows, first {_first_bad(bad)}"
    else:
        ev = None
    bad = got.values != src.values[rows]
    if ev is not None:
        bad &= ev
    assert not bool(bad.any()), f"{what}: values differ at {int(bad.sum())} rows, first {_first_bad(bad)}"


def _tags(what: str, col: OutCol, src: Col, base: int, n: int) -> torch.Tensor:
    t = image(col.values, src.dtype) - base
    bad = (t < 0) | (t >= n)
    assert not bool(bad.any()), f"{what}: tag outside the side's rows at {_first_bad(bad)}"
    return t


def check_probe_output(kind: int, blocks: List[List[OutCol]], probe: Side, build: Side, cnt: torch.Tensor):
    """The output of one probe block (0 or more output blocks, concatenated) against the expected
    match count of each of its probe rows (JoinRef.probe)."""
    name = KIND_NAMES[kind]
    npc, nbc = len(probe.cols), len(build.cols)
    with_build = kind in (abi.JOIN_INNER, abi.JOIN_LEFT, abi.JOIN_RIGHT, abi.JOIN_FULL)
    want = expected_rows(kind, cnt)
    if kind in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI):
        assert not blocks, f"{name}: the probe emitted {len(blocks)} blocks; the build-side semi / anti kinds emit only in final_probe"
        return
    ncols = npc + (nbc if with_build else 0)
    for b in blocks:
        assert len(b) == ncols, f"{name}: {len(b)} output columns, expected {ncols}"
    if not blocks:
        total = int(want.sum())
        assert total == 0, f"{name}: no output, expected {total} rows"
        return
    if len(blocks) == 1:
        out = blocks[0]
    else:
        out = [OutCol(torch.cat([b[c].values for b in blocks]),
                      None if all(b[c].valid is None for b in blocks) else
                      torch.cat([b[c].valid if b[c].valid is not None else torch.ones_like(b[c].values, dtype=torch.bool) for b in blocks]))
               for c in range(ncols)]
    n = probe.n
    ptag = _tags(f"{name} ptag", out[probe.tag], probe.cols[probe.tag], probe.base, n)
    # 2. per-probe-row counts
    got = torch.bincount(ptag, minlength=n)
    bad = got != want
    assert not bool(bad.any()), (f"{name}: {int(bad.sum())} probe rows have the wrong number of output rows; first rows "
                                 f"{_first_bad(bad)}: got {got[bad][:5].tolist()}, expected {want[bad][:5].tolist()}")
    # 1. probe columns are the probe row's
    for c in range(npc):
        _check_col(f"{name} probe column {c}", out[c], probe.cols[c], ptag)
    if not with_build:
        return
    bout = out[npc:]
    bt = bout[build.tag]
    if kind in (abi.JOIN_LEFT, abi.JOIN_FULL):
        assert bt.valid is not None, f"{name}: the build tag column must be nullable"
        matched = bt.valid
        un = ~matched
        # unmatched rows: every build column NULL, and only probe rows without a match
        for c in range(nbc):
            v = bout[c].valid
            assert v is not None, f"{name}: build column {c} must be nullable"
            bad = un & v
            assert not bool(bad.any()), f"{name}: an unmatched row carries a non-NULL build column {c} at {_first_bad(bad)}"
        bad = un & (cnt[ptag] != 0)
        assert not bool(bad.any()), f"{name}: a probe row with matches was also emitted unmatched at {_first_bad(bad)}"
        sel = matched.nonzero().flatten()
        ptag_m = ptag[sel]
        bout = [OutCol(c.values[sel], None if c.valid is None else c.valid[sel]) for c in bout]
        bt = bout[build.tag]
    else:
        assert bt.valid is None or bool(bt.valid.all()), f"{name}: a NULL build tag"
        ptag_m = ptag
    btag = _tags(f"{name} btag", bt, build.cols[build.tag], build.base, build.n)
    # 1. keys: both valid and equal images
    pv, bv = probe.key_valid(), build.key_valid()
    bad = ~pv[ptag_m] | ~bv[btag]
    assert not bool(bad.any()), f"{name}: a pair with a NULL key at {_first_bad(bad)}"
    for i, (pi, bi) in enumerate(zip(probe.key_images(), build.key_images())):
        bad = pi[ptag_m] != bi[btag]
        assert not bool(bad.any()), f"{name}: key {i} differs between the paired rows at {_first_bad(bad)}"
    for c in range(nbc):
        _check_col(f"{name} build column {c}", bout[c], build.cols[c], btag)
    # 3. no pair twice
    pair, _ = torch.sort(ptag_m * build.n + btag)
    bad = pair[1:] == pair[:-1]
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} repeated (probe, build) pairs"


def check_final_output(kind: int, blocks: List[List[OutCol]], build: Side, n_probe_cols: int, matched: torch.Tensor):
    """final_probe's blocks: exactly the build rows the kind selects from the matched map, each once."""
    name = KIND_NAMES[kind]
    if kind not in BUILD_SIDE_KINDS:
        assert not blocks, f"{name}: final_probe emitted {len(blocks)} blocks"
        return
    sel = matched if kind == abi.JOIN_RIGHT_SEMI else ~matched
    exp = sel.nonzero().flatten()
    if not blocks:
        assert exp.shape[0] == 0, f"{name}: final_probe emitted nothing, expected {exp.shape[0]} build rows"
        return
    npc = n_probe_cols if kind in (abi.JOIN_RIGHT, abi.JOIN_FULL) else 0
    parts = []
    for b in blocks:
        assert len(b) == npc + len(build.cols), f"{name}: final block has {len(b)} columns"
        for c in range(npc):
            assert b[c].values is None and b[c].const_null, f"{name}: final block probe column {c} is not Const NULL"
        bo = b[npc:]
        btag = _tags(f"{name} final btag", bo[build.tag], build.cols[build.tag], build.base, build.n)
        for c in range(len(build.cols)):
            _check_col(f"{name} final build column {c}", bo[c], build.cols[c], btag)
        parts.append(btag)
    got, _ = torch.sort(torch.cat(parts))
    if got.shape[0] != exp.shape[0]:
        extra = got.shape[0] - exp.shape[0]
        raise AssertionError(f"{name}: final_probe emitted {got.shape[0]} build rows, expected {exp.shape[0]} ({extra:+d})")
    bad = got != exp
    assert not bool(bad.any()), f"{name}: final_probe build rows differ from the selected set at {_first_bad(bad)}"


# ---------------------------------------------------------------- slot construction (uint64 numpy arrays)
def agg_hash(x: np.ndarray) -> np.ndarray:
    return agg_hash_np(np.asarray(x, dtype=np.uint64))


def agg_hash_inv(h: np.ndarray) -> np.ndarray:
    """The inverse of agg_hash: the same xor-shifts with the inverse multiplier, in reverse order."""
    x = np.asarray(h, dtype=np.uint64).copy()
    c, s = np.uint64(INV_MUL), np.uint64(32)
    with np.errstate(over="ignore"):
        x ^= x >> s
        x *= c
        x ^= x >> s
        x *= c
        x ^= x >> s
    return x


def agg_hash_wide(k0: np.ndarray, k1: np.ndarray) -> np.ndarray:
    """The 128-bit key's hash (common.cuh agg_hash_wide)."""
    with np.errstate(over="ignore"):
        return agg_hash(np.asarray(k0, dtype=np.uint64) ^ (agg_hash(k1) + np.uint64(GOLDEN)))


def hashes_homed_at(slots: np.ndarray, cap: int, rng: np.random.Generator) -> np.ndarray:
    """Random 64-bit hashes whose low log2(cap) bits are the given slots."""
    hi = rng.integers(0, 2**64, len(slots), dtype=np.uint64, endpoint=False)
    return (hi & ~np.uint64(cap - 1)) | np.asarray(slots, dtype=np.uint64)


def words_homed_at(slots: np.ndarray, cap: int, rng: np.random.Generator) -> np.ndarray:
    """64-bit key images (uint64) whose home slot in a table of `cap` entries is the given slot."""
    return agg_hash_inv(hashes_homed_at(slots, cap, rng))


def wide_words_homed_at(slots: np.ndarray, cap: int, rng: np.random.Generator):
    """(k0, k1) 128-bit keys homed at the given slots: k1 is free, k0 = inv(h) ^ (agg_hash(k1) + golden)."""
    k1 = rng.integers(0, 2**64, len(slots), dtype=np.uint64, endpoint=False)
    with np.errstate(over="ignore"):
        k0 = agg_hash_inv(hashes_homed_at(slots, cap, rng)) ^ (agg_hash(k1) + np.uint64(GOLDEN))
    return k0, k1


def narrow_values_homed_in(lo: int, hi: int, cap: int, count: int, dtype: int, start: int = 0) -> np.ndarray:
    """`count` distinct values of a narrow integer dtype whose home slot lies in [lo, hi), found by
    scanning the type's values upward from `start` (the image is not a free 64-bit word)."""
    nd = np.dtype(NP_DTYPE[dtype])
    info = np.iinfo(nd)
    out = []
    got = 0
    chunk = 1 << 20
    v0 = max(start, int(info.min))
    while got < count:
        assert v0 <= info.max, "the type has too few values homed in the range"
        v = np.arange(v0, min(v0 + chunk, int(info.max) + 1), dtype=np.int64)
        home = agg_hash(v.astype(np.uint64)) & np.uint64(cap - 1)  # the image: v sign- or zero-extended
        sel = v[(home >= np.uint64(lo)) & (home < np.uint64(hi))]
        out.append(sel[: count - got])
        got += len(out[-1])
        v0 += chunk
    return np.concatenate(out).astype(nd)


def next_pow2_cap(build_rows: int) -> int:
    """The join table's slot count for a build side of `build_rows` rows: max(next_pow2(2 rows), 1024)."""
    return max(1 << (2 * max(build_rows, 1) - 1).bit_length(), 1024)


def home_slots(words: np.ndarray, cap: int) -> np.ndarray:
    return (agg_hash(words) & np.uint64(cap - 1)).astype(np.int64)


def linear_probe_insert(homes: np.ndarray, cap: int) -> np.ndarray:
    """Slot of each entry when the homes are inserted one after the other into an empty linear-probing
    table of `cap` slots (each takes the first free slot from its home on, wrapping at cap - 1 -> 0).
    The set of occupied slots does not depend on the insertion order; which entry sits where does."""
    parent = {}

    def find(s):
        path = []
        while s in parent:
            path.append(s)
            s = parent[s]
        for p in path:
            parent[p] = s
        return s
    slots = np.empty(len(homes), dtype=np.int64)
    assert len(homes) < cap
    for i, h in enumerate(homes.tolist()):
        s = find(h)
        slots[i] = s
        parent[s] = (s + 1) % cap
    return slots


def run_of(occupied: np.ndarray, slot: int):
    """(start, length) of the maximal circular run of occupied slots that holds `slot`."""
    cap = len(occupied)
    assert occupied[slot] and not occupied.all()
    s = slot
    while occupied[(s - 1) % cap]:
        s = (s - 1) % cap
    n = 0
    while occupied[(s + n) % cap]:
        n += 1
    return s, n
