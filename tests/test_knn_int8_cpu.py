"""Vector(Int8) on the host: the column type, its constructor, and the distance oracle for int8
arguments against an independent restatement.

The reference widens both Int8 sides element by element (`*v as f32`, scalars/vector.rs:515-524)
and calls the f32 cosine_distance / l2_distance (src/common/vector/src/distance.rs:19-35,65-80).
The oracle does the same: `distance_rows` converts its arguments to float32 (exact for int8) and
runs the f32 functions.  The restatement here computes the sums exactly in int64 and then only the
reference's final f32 operations, which is the same value wherever the f32 sums are exact: every
product of two widened values has magnitude <= 2^14 and every (a-b)^2 <= 65 025, so cosine's sums
(an 8-way fold) are exact for every input with dim <= 1024, L2's (a sequential fold of
non-negative terms) for every input with dim <= 258."""
import os
import re

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import DTYPE_NAMES, Column
from databend_b200.vector import const_vector

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle():
    from oracle import oracle as orc
    return orc


def restated_cosine(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    a64, b64 = a.astype(np.int64), b.astype(np.int64)
    ab = (a64 * b64).sum(-1).astype(np.float32)
    aa = (a64 * a64).sum(-1).astype(np.float32)
    bb = (b64 * b64).sum(-1).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.float32(1.0) - ab / (np.sqrt(aa) * np.sqrt(bb))


def restated_l2(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    d = a.astype(np.int64) - b.astype(np.int64)
    return np.sqrt((d * d).sum(-1).astype(np.float32))


def assert_bits(got, exp):
    got, exp = np.asarray(got, np.float32), np.asarray(exp, np.float32)
    nan = np.isnan(exp)
    np.testing.assert_array_equal(np.isnan(got), nan)
    np.testing.assert_array_equal(got[~nan].view(np.uint32), exp[~nan].view(np.uint32))


def int8_rows(rng, rows, dim):
    x = rng.integers(-128, 128, (rows, dim), dtype=np.int64).astype(np.int8)
    x[0] = 0             # zero row: NaN for cosine
    x[1] = -128          # extremes
    x[2] = 127
    x[3, ::2], x[3, 1::2] = 127, -128   # alternating signs
    return x


@pytest.mark.parametrize("dim", [1, 3, 7, 8, 9, 64, 100, 257, 258, 768, 1024])
def test_int8_oracle_matches_exact_restatement(dim):
    rng = np.random.default_rng(dim)
    a, b = int8_rows(rng, 500, dim), int8_rows(rng, 500, dim)[::-1].copy()
    orc = oracle()
    assert_bits(orc.distance_rows(abi.DIST_COSINE, a, b), restated_cosine(a, b))
    assert_bits(orc.distance_rows(abi.DIST_COSINE, a, b[7]), restated_cosine(a, b[7][None]))
    if dim <= 258:
        assert_bits(orc.distance_rows(abi.DIST_L2, a, b), restated_l2(a, b))
        assert_bits(orc.distance_rows(abi.DIST_L2, b[7], a), restated_l2(b[7][None], a))


def test_int8_oracle_l2_beyond_258_when_sum_fits():
    """dim > 258: still exact for every pair whose sum S is <= 2^24."""
    rng = np.random.default_rng(3)
    a = rng.integers(-20, 21, (300, 4096)).astype(np.int8)
    b = rng.integers(-20, 21, (300, 4096)).astype(np.int8)
    s = ((a.astype(np.int64) - b) ** 2).sum(-1)
    assert s.max() <= 2 ** 24
    assert_bits(oracle().distance_rows(abi.DIST_L2, a, b), restated_l2(a, b))


def test_dtype_code_matches_header():
    with open(os.path.join(ROOT, "include", "dbx.h")) as f:
        m = re.search(r"DBX_VEC_I8\s*=\s*(\d+)", f.read())
    assert m and int(m.group(1)) == abi.VEC_I8 == 12
    assert DTYPE_NAMES[abi.VEC_I8] == "Vector(Int8)"


def test_vector_int8_constructor():
    x = np.arange(-6, 6, dtype=np.int8).reshape(4, 3)
    c = Column.vector_int8(x)
    assert (c.dtype, c.length, c.vec_dim) == (abi.VEC_I8, 4, 3)
    assert c.values().dtype == np.int8
    np.testing.assert_array_equal(c.values(), x)
    np.testing.assert_array_equal(c.slice(1, 3).values(), x[1:3])
    with pytest.raises(TypeError):
        Column.vector_int8(x.astype(np.int16))
    with pytest.raises(TypeError):
        Column.vector_int8(x[0])
    # a device column slices by vec_dim bytes per row
    d = Column.device(abi.VEC_I8, 10, 4096, vec_dim=3)
    assert d.slice(2, 5).dev_ptr == 4096 + 6
    assert Column.device(abi.VEC_F32, 10, 4096, vec_dim=3).slice(2, 5).dev_ptr == 4096 + 24


def test_column_vector_still_float32():
    x = np.arange(-6, 6, dtype=np.int8).reshape(4, 3)
    c = Column.vector(x)
    assert (c.dtype, c.vec_dim) == (abi.VEC_F32, 3)
    assert c.values().dtype == np.float32
    np.testing.assert_array_equal(c.values(), x.astype(np.float32))


def test_const_vector_keeps_int8():
    q = np.array([1, -2, 3], dtype=np.int8)
    c = const_vector(q, 5)
    assert (c.dtype, c.vec_dim, c.length) == (abi.VEC_I8, 3, 5)
    assert c.const_value.dtype == np.int8
    assert const_vector(q.astype(np.float32), 5).dtype == abi.VEC_F32
    assert const_vector(None, 5, dim=3, dtype=abi.VEC_I8).dtype == abi.VEC_I8
    with pytest.raises(TypeError):
        const_vector([1.5, 2.0, 3.0], 5, dtype=abi.VEC_I8)
