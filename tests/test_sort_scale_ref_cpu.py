"""The device-side sort reference of tests/sort_scale_ref.py is the CPU oracles' order.

It is held against `oracle.topk` (the C oracle, one key) and `oracle/sort_oracle.sort_permutation`
(several keys) on small random inputs full of the float keys a sort can get wrong, and all three
against hand-written orders: every NaN bit pattern is one value, greater than +inf, and -0.0 ties
+0.0, with ties in ascending row id."""
import numpy as np
import pytest

import sort_scale_ref as R
from databend_b200.block import Column
from oracle import oracle as orc
from oracle import sort_oracle


def _f32(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def _f64(bits):
    return np.asarray(bits, np.uint64).view(np.float64)


def special_floats(nd, n, rng):
    """Random special values (heavy ties) mixed with a few ordinary ones."""
    sp = _f32(R.F32_SPECIAL_BITS) if nd == np.float32 else _f64(R.F64_SPECIAL_BITS)
    x = rng.choice(sp, n)
    ordinary = rng.random(n) < 0.3
    x[ordinary] = rng.integers(-3, 4, ordinary.sum()).astype(nd) / nd(2)
    return x


def random_keys(dtype, n, rng):
    nd = np.dtype(dtype)
    if nd.kind == "f":
        return special_floats(nd.type, n, rng)
    info = np.iinfo(nd)
    x = rng.integers(info.min, info.max, n, dtype=nd, endpoint=True)
    x[rng.random(n) < 0.5] = rng.choice(np.array([info.min, info.max, 0, 1], dtype=nd), 1)[0]  # ties and extremes
    return x


def ref_rows(keys, limit=0):
    return R.sort_permutation([R.key_spec(v, m, a, nf) for v, m, a, nf in keys], limit).numpy()


DTYPES = [np.float32, np.float64, np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64]


@pytest.mark.parametrize("dtype", DTYPES)
def test_one_key_equals_both_oracles(dtype):
    rng = np.random.default_rng(np.dtype(dtype).num)
    n = 3000
    x = random_keys(dtype, n, rng)
    m = rng.random(n) > 0.2
    for valid in (None, m):
        for asc in (True, False):
            for nf in (True, False):
                got = ref_rows([(x, valid, asc, nf)])
                col = Column.from_data(x, validity=valid)
                np.testing.assert_array_equal(got, orc.topk(col, asc, nf, n))
                np.testing.assert_array_equal(got, sort_oracle.sort_permutation([(x, valid, asc, nf)]))
                np.testing.assert_array_equal(ref_rows([(x, valid, asc, nf)], 777), orc.topk(col, asc, nf, 777))


def test_several_keys_equal_sort_oracle():
    rng = np.random.default_rng(3)
    n = 4000
    cols = [random_keys(d, n, rng) for d in (np.float32, np.int8, np.float64, np.uint64)]
    cols[1] = (cols[1] % 3).astype(np.int8)  # low cardinality: the later keys decide often
    masks = [rng.random(n) > p for p in (0.2, 0.1, 0.3, 0.0)]
    for t in range(8):
        dirs = [(t >> j) & 1 == 0 for j in range(4)]
        nfs = [(t + j) % 3 == 0 for j in range(4)]
        order = [(t + j) % 4 for j in range(4)]
        keys = [(cols[c], masks[c] if c != 3 else None, dirs[j], nfs[j]) for j, c in enumerate(order)]
        for limit in (0, 1000):
            np.testing.assert_array_equal(ref_rows(keys, limit), sort_oracle.sort_permutation(keys, limit))


@pytest.mark.parametrize("nd", [np.float32, np.float64])
def test_every_nan_is_one_value_above_inf(nd):
    """NaNs of any sign, payload or signalling bit are equal and greatest: ASC puts them last in
    row order, DESC first in row order.  A negative NaN is not below -inf."""
    sp_bits = R.F32_SPECIAL_BITS if nd == np.float32 else R.F64_SPECIAL_BITS
    sp = _f32(sp_bits) if nd == np.float32 else _f64(sp_bits)
    nans = sp[np.isnan(sp)]
    x = np.concatenate([nans, np.array([np.inf, -np.inf, 1.0], nd), nans[::-1]])
    nan_rows = np.flatnonzero(np.isnan(x))
    assert len(nans) == 5 and np.signbit(nans).any()
    i_inf, i_ninf, i_one = len(nans), len(nans) + 1, len(nans) + 2
    asc = np.concatenate([[i_ninf, i_one, i_inf], nan_rows])
    desc = np.concatenate([nan_rows, [i_inf, i_one, i_ninf]])
    col = Column.from_data(x)
    for is_asc, exp in ((True, asc), (False, desc)):
        np.testing.assert_array_equal(ref_rows([(x, None, is_asc, False)]), exp)
        np.testing.assert_array_equal(orc.topk(col, is_asc, False, len(x)), exp)
        np.testing.assert_array_equal(sort_oracle.sort_permutation([(x, None, is_asc, False)]), exp)


@pytest.mark.parametrize("nd", [np.float32, np.float64])
def test_negative_zero_ties_positive_zero_by_row_id(nd):
    x = np.array([0.0, -0.0, 1.0, -0.0, 0.0, -1.0, -0.0], nd)
    asc = np.array([5, 0, 1, 3, 4, 6, 2])
    desc = np.array([2, 0, 1, 3, 4, 6, 5])
    col = Column.from_data(x)
    for is_asc, exp in ((True, asc), (False, desc)):
        np.testing.assert_array_equal(ref_rows([(x, None, is_asc, False)]), exp)
        np.testing.assert_array_equal(orc.topk(col, is_asc, False, len(x)), exp)
        np.testing.assert_array_equal(sort_oracle.sort_permutation([(x, None, is_asc, False)]), exp)


def test_nulls_tie_and_later_keys_decide():
    """NULL rows of an earlier key tie whatever their value slot holds; the later key, then row id decide."""
    a = np.array([5, 1, 9, 1, 7], np.int32)
    am = np.array([False, True, False, True, False])
    b = np.array([2.0, 3.0, 2.0, 3.0, 1.0])
    for nf, exp in ((True, [4, 0, 2, 1, 3]), (False, [1, 3, 4, 0, 2])):
        keys = [(a, am, True, nf), (b, None, True, False)]
        np.testing.assert_array_equal(ref_rows(keys), exp)
        np.testing.assert_array_equal(sort_oracle.sort_permutation(keys), exp)
