"""Plain CPU restatement of the join runtime filters (numpy; paths relative to the databend source
tree, src/query).  The GPU tests compare the device's min-max, IN-list, bloom words and apply bitmaps
with it bit for bit; tests/golden/runtime_filter.json pins it to the reference's own test data.

  thresholds on the build rows (NULL keys included)     service/.../hash_join/runtime_filter/local_builder.rs:86-139
  IN-list de-duplicated                                 local_builder.rs:147-156,251-274
  bloom enabled: build_rows > 0, build_table_rows known, build_rows / build_table_rows * 100 < threshold
                                                        service/.../hash_join/runtime_filter/builder.rs:17-57
  a packet with no build rows carries no filters        local_builder.rs:231-233
  bloom hash: the key's bits as KeysU8/U16/U32/U64, zero-extended, murmur3 fmix64
                                                        expression/src/kernels/group_by.rs:72-75, common/hashtable/src/traits.rs:227-251
  SBBF size, block index, mask, insert, check           catalog/src/sbbf.rs:97-170,220-262

Two choices of this project (DESIGN §2): NULL build keys are left out of all three filters (ndv = the
non-NULL build keys), and each key pair works in its common type (the join's key rule), on both sides.
"""
import math

import numpy as np

from databend_b200 import abi

SALT = np.array([0x47b6137b, 0x44974d91, 0x8824ad5b, 0xa2b7289d, 0x705495c7, 0x2df1424b, 0x9efc4947, 0x5c6bfb31], dtype=np.uint32)
BITSET_MIN_LENGTH, BITSET_MAX_LENGTH = 32, 128 * 1024 * 1024
FPP = 0.01
DEFAULTS = dict(enable_inlist=True, enable_bloom=True, enable_min_max=True, inlist_threshold=1024, bloom_threshold=3_000_000,
                min_max_threshold=2**64 - 1, build_table_rows=0, selectivity_threshold=10)
_SIGNED = {abi.I8, abi.I16, abi.I32, abi.I64}
_BYTES = {abi.I8: 1, abi.U8: 1, abi.I16: 2, abi.U16: 2, abi.I32: 4, abi.U32: 4, abi.I64: 8, abi.U64: 8}
_BY_WIDTH = {(True, 1): abi.I8, (True, 2): abi.I16, (True, 4): abi.I32, (True, 8): abi.I64,
             (False, 1): abi.U8, (False, 2): abi.U16, (False, 4): abi.U32, (False, 8): abi.U64}


def optimal_num_of_bytes(n: int) -> int:
    """sbbf.rs:225-229: clamp to [32, 128 MiB], then the next power of two."""
    n = max(min(n, BITSET_MAX_LENGTH), BITSET_MIN_LENGTH)
    return 1 << (n - 1).bit_length()


def num_of_bits_from_ndv_fpp(ndv: int, fpp: float) -> int:
    """sbbf.rs:236-239 in f64, with Rust's saturating `as usize` (NaN and negatives give 0)."""
    bits = -8.0 * float(ndv) / math.log(1.0 - math.pow(fpp, 1.0 / 8.0))
    if not bits > 0:
        return 0
    return 2**64 - 1 if bits >= 2.0**64 else int(bits)


def bloom_bytes(ndv: int) -> int:
    """Sbbf::new_with_ndv_fpp(ndv, 0.01) (sbbf.rs:244-252, convert.rs:249-255)."""
    return optimal_num_of_bytes(num_of_bits_from_ndv_fpp(ndv, FPP) // 8)


def should_enable_bloom(build_rows: int, build_table_rows: int, selectivity_threshold: int) -> bool:
    """builder.rs:17-57; build_table_rows = 0 stands for None (no statistics)."""
    if build_rows == 0 or build_table_rows <= 0:
        return False
    return (float(build_rows) / float(build_table_rows)) * 100.0 < float(selectivity_threshold)


def fmix64(x: np.ndarray) -> np.ndarray:
    """BloomHash for the primitive keys (traits.rs:227-251), vectorised over uint64."""
    x = np.asarray(x, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xff51afd7ed558ccd)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xc4ceb9fe1a85ec53)
        x ^= x >> np.uint64(33)
    return x


def common_type(build_dtype: int, probe_dtype: int):
    """(dtype, signed, bytes) of a key pair: the join's rule (same signedness: the larger size; signed S
    with unsigned U: max(S, 2 U) bytes)."""
    bs, ps = build_dtype in _SIGNED, probe_dtype in _SIGNED
    bz, pz = _BYTES[build_dtype], _BYTES[probe_dtype]
    n = max(bz, pz) if bs == ps else (max(bz, 2 * pz) if bs else max(pz, 2 * bz))
    signed = bs or ps
    return _BY_WIDTH[(signed, n)], signed, n


def images(values: np.ndarray) -> np.ndarray:
    """Keys as the 64-bit images the join compares: sign- or zero-extended to 64 bits."""
    v = np.asarray(values)
    return (v.astype(np.int64).view(np.uint64) if v.dtype.kind == "i" else v.astype(np.uint64))


def _order_key(img: np.ndarray, signed: bool) -> np.ndarray:
    return img.view(np.int64) if signed else img


def block_index(h: np.ndarray, n_blocks: int) -> np.ndarray:
    """sbbf.rs:220-222 (n_blocks < 2^32)."""
    return (((h >> np.uint64(32)) * np.uint64(n_blocks)) & np.uint64(0xFFFFFFFFFFFFFFFF)) >> np.uint64(32)


def masks(h: np.ndarray) -> np.ndarray:
    """Block::mask (sbbf.rs:121-170): [n, 8] uint32, one bit per word."""
    x = (h & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    with np.errstate(over="ignore"):
        idx = (x[:, None] * SALT[None, :]) >> np.uint32(27)
    return (np.uint32(1) << idx).astype(np.uint32)


def sbbf_insert(words: np.ndarray, hashes: np.ndarray):
    """Sbbf::insert_hash_batch into words ([n_blocks * 8] uint32)."""
    blocks = words.reshape(-1, 8)
    bi = block_index(hashes, blocks.shape[0]).astype(np.int64)
    m = masks(hashes)
    for i in range(8):
        np.bitwise_or.at(blocks[:, i], bi, m[:, i])


def sbbf_check(words: np.ndarray, hashes: np.ndarray) -> np.ndarray:
    """Sbbf::check_hash per hash."""
    blocks = words.reshape(-1, 8)
    bi = block_index(hashes, blocks.shape[0]).astype(np.int64)
    m = masks(hashes)
    return np.all((blocks[bi] & m) == m, axis=1)


def build(build_keys, probe_dtypes, **params):
    """build_keys: one Column per key pair (build side); probe_dtypes: the probe key dtypes.
    Returns one dict per pair: dtype, signed, min / max (common type, None without a non-NULL key),
    has_min_max, inlist (sorted distinct keys, or None), bloom (uint32 words, or None)."""
    p = dict(DEFAULTS, **params)
    rows = build_keys[0].length
    bloom_on = p["enable_bloom"] and rows <= p["bloom_threshold"] and should_enable_bloom(rows, p["build_table_rows"], p["selectivity_threshold"])
    out = []
    for col, pd in zip(build_keys, probe_dtypes):
        dtype, signed, width = common_type(col.dtype, pd)
        part = dict(dtype=dtype, signed=signed, width=width, min=None, max=None, has_min_max=False, inlist=None, bloom=None)
        out.append(part)
        if rows == 0:
            continue
        img = images(col.values())[col.valid_mask()]
        conv = _order_key(img, signed).astype(np.dtype(np.int64 if signed else np.uint64))
        if len(img):
            part["min"], part["max"] = int(conv.min()), int(conv.max())
        part["has_min_max"] = bool(p["enable_min_max"] and rows <= p["min_max_threshold"])
        if p["enable_inlist"] and rows <= p["inlist_threshold"]:
            part["inlist"] = np.unique(conv)
        if bloom_on:
            words = np.zeros(bloom_bytes(len(img)) // 4, dtype=np.uint32)
            mask = np.uint64((1 << (8 * width)) - 1)
            sbbf_insert(words, fmix64(img & mask))
            part["bloom"] = words
    return out


def apply(parts, probe_keys) -> np.ndarray:
    """ExprBloomFilter::apply ANDed over the filters and key pairs: True where the probe row may match.
    A NULL probe key is rejected (it never matches)."""
    n = probe_keys[0].length
    keep = np.ones(n, dtype=bool)
    for part, col in zip(parts, probe_keys):
        keep &= col.valid_mask()
        img = images(col.values())
        conv = _order_key(img, part["signed"])
        if part["has_min_max"]:
            if part["min"] is None:
                keep[:] = False
            else:
                keep &= (conv >= part["min"]) & (conv <= part["max"])
        if part["inlist"] is not None:
            keep &= np.isin(conv, part["inlist"])
        if part["bloom"] is not None:
            mask = np.uint64((1 << (8 * part["width"])) - 1)
            keep &= sbbf_check(part["bloom"], fmix64(img & mask))
    return keep
