"""Device-side reference of the ORDER BY order, for inputs too large for the CPU oracles.

The C oracle (`oracle.topk`) and `oracle/sort_oracle.sort_permutation` are practical up to about
2e7 rows.  This module writes the same order in torch, so it runs wherever its tensors live (the
GPU tests run it on the device, tests/test_sort_scale_ref_cpu.py holds it against both oracles on
the CPU):

  * every key becomes an int64 order image whose signed order is the key's order: floats with every
    NaN (any sign, payload or signalling bit) mapped to one value above +inf and -0.0 to +0.0, then
    bits ^ ((bits >> 63) & 0x7FFF...) (OrderedFloat: NaN greatest and equal to itself, -0 == +0);
    signed integers widened; UInt64 with the sign bit flipped; DESC takes ~image;
  * one stable torch.sort per key, least significant key first, starting from the row ids, so the
    remaining ties keep ascending row id; a nullable key adds one more stable sort on its NULL flag
    (NULL rows tie on the value and are placed as one run before or after the valid rows).
"""
import numpy as np
import torch

_I64_MAX = 0x7FFF_FFFF_FFFF_FFFF

# Float keys whose bits a sort can lose: +-0, canonical / negative / payload / signalling NaN,
# +-inf, the smallest and largest subnormals of both signs, +-max.
F32_SPECIAL_BITS = np.array([0x00000000, 0x80000000, 0x7FC00000, 0xFFC00000, 0x7FC01234, 0x7F800001, 0xFF800001, 0x7F800000,
                             0xFF800000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x7F7FFFFF, 0xFF7FFFFF], dtype=np.uint32)
F64_SPECIAL_BITS = np.array([0x0000000000000000, 0x8000000000000000, 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000001234,
                             0x7FF0000000000001, 0xFFF0000000000001, 0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001,
                             0x8000000000000001, 0x000FFFFFFFFFFFFF, 0x800FFFFFFFFFFFFF, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF],
                            dtype=np.uint64)


def as_tensor(a, device=None) -> torch.Tensor:
    """numpy array -> torch tensor (unsigned types as their same-width signed view plus a dtype tag)."""
    a = np.ascontiguousarray(a)
    t = torch.from_numpy(a.view({1: np.int8, 2: np.int16, 4: np.int32, 8: np.int64}[a.itemsize]) if a.dtype.kind == "u" and a.itemsize > 1 else a)
    return t.to(device) if device is not None else t


def order_image(values: torch.Tensor, asc: bool, unsigned: bool = False) -> torch.Tensor:
    """int64 image of one key column; `unsigned`: the (signed-view) tensor holds unsigned integers."""
    v = values
    if v.dtype in (torch.float32, torch.float64):
        d = v.to(torch.float64)
        d = torch.where(d == 0, torch.zeros_like(d), d)  # -0.0 == +0.0
        b = d.view(torch.int64)
        img = b ^ ((b >> 63) & _I64_MAX)
        img = torch.where(torch.isnan(d), torch.full_like(img, _I64_MAX), img)  # every NaN: above +inf
    elif unsigned:
        w = v.element_size() * 8
        if w == 64:
            img = v.view(torch.int64) ^ torch.iinfo(torch.int64).min
        else:
            img = v.to(torch.int64) & ((1 << w) - 1)
    else:
        img = v.to(torch.int64)
    return img if asc else ~img


def sort_permutation(keys, limit: int = 0) -> torch.Tensor:
    """keys: [(values, valid or None, asc, nulls_first[, unsigned])] as tensors on one device, most
    significant first (values via as_tensor).  Returns the row ids in output order (int64)."""
    n = keys[0][0].shape[0]
    dev = keys[0][0].device
    perm = torch.arange(n, dtype=torch.int64, device=dev)
    for key in reversed(keys):
        values, valid, asc, nulls_first = key[:4]
        unsigned = key[4] if len(key) > 4 else False
        img = order_image(values, asc, unsigned)
        if valid is not None:
            img = torch.where(valid, img, torch.zeros_like(img))
        perm = perm[torch.sort(img[perm], stable=True).indices]
        del img
        if valid is not None:
            flag = (valid if nulls_first else ~valid).to(torch.int8)  # NULLS FIRST: NULL 0, valid 1
            perm = perm[torch.sort(flag[perm], stable=True).indices]
    return perm[:limit] if limit else perm


def key_spec(values: np.ndarray, valid, asc: bool, nulls_first: bool, device=None):
    """One sort_permutation key from numpy data."""
    return (as_tensor(values, device), None if valid is None else torch.from_numpy(np.asarray(valid, bool)).to(device or "cpu"),
            asc, nulls_first, values.dtype.kind == "u")
