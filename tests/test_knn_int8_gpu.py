"""Vector(Int8) on the device: row-wise cosine_distance / l2_distance, brute-force kNN on the int8
tensor cores, and the block kernels.

Row-wise distances are bit-exact with the oracle (the reference widens Int8 to f32 and runs the f32
functions, scalars/vector.rs:497-556).  kNN returns the oracle's ranking by (distance, row id) with
distances bit for bit (tolerance 0), and every query is either certified or answered exactly."""
import os

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column, DataBlock, pack_bitmap
from databend_b200.expr import col, lit, gt
from databend_b200.kernels import concat, scatter, take, take_ranges
from databend_b200.lib import DbxError
from databend_b200.transforms import (AggregatorParams, HashJoin, TransformFilter, TransformPartialAggregate, TransformTopN,
                                      schema_types, to_device)
from databend_b200.vector import VectorTopN, const_vector, eval_distance

pytestmark = pytest.mark.gpu
FN = {"cosine": "cosine_distance", "l2": "l2_distance"}
KIND = {"cosine": abi.DIST_COSINE, "l2": abi.DIST_L2}


def oracle():
    from oracle import oracle as orc
    return orc


def assert_bits(got, exp):
    got, exp = np.asarray(got, np.float32), np.asarray(exp, np.float32)
    nan = np.isnan(exp)
    np.testing.assert_array_equal(np.isnan(got), nan)
    np.testing.assert_array_equal(got[~nan].view(np.uint32), exp[~nan].view(np.uint32))


def rand_i8(rng, shape, lo=-128, hi=128):
    return rng.integers(lo, hi, shape, dtype=np.int8)


def special_rows(x):
    """Rows the accumulators and the exact kernels must survive: all -128, all 127, alternating
    signs, zero."""
    x = x.copy()
    x[0] = -128
    x[1] = 127
    x[2, ::2], x[2, 1::2] = 127, -128
    x[3] = 0
    return x


# ---------------------------------------------------------------- row-wise distance
@pytest.mark.parametrize("kind", ["cosine", "l2"])
@pytest.mark.parametrize("dim", [1, 3, 7, 8, 9, 64, 100, 257, 258, 259, 768, 1024, 1025, 1536, 4096])
def test_distance_rows_bit_exact(gpu, kind, dim):
    rng = np.random.default_rng(dim * 3 + (kind == "l2"))
    rows = 600
    a = special_rows(rand_i8(rng, (rows, dim)))
    b = special_rows(rand_i8(rng, (rows, dim)))[::-1].copy()
    orc = oracle()
    assert_bits(eval_distance(FN[kind], Column.vector_int8(a), Column.vector_int8(b)).values(),
                orc.distance_rows(KIND[kind], a, b, threads=8))
    # const rhs with device-resident lhs, const lhs
    q = b[5]
    assert_bits(eval_distance(FN[kind], to_device(Column.vector_int8(a)), const_vector(q, rows)).values(),
                orc.distance_rows(KIND[kind], a, q, threads=8))
    assert_bits(eval_distance(FN[kind], const_vector(q, rows), Column.vector_int8(a)).values(),
                orc.distance_rows(KIND[kind], q, a, threads=8))


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_distance_rows_nullable_with_bit_offsets(gpu, kind):
    rng = np.random.default_rng(11)
    rows, dim = 1001, 37
    a, b = rand_i8(rng, (rows, dim)), rand_i8(rng, (rows, dim))
    va, vb = rng.random(rows) > 0.3, rng.random(rows) > 0.2
    ca, cb = Column.vector_int8(a), Column.vector_int8(b)
    ca.validity, ca.validity_bit_offset = pack_bitmap(va, 3), 3
    cb.validity, cb.validity_bit_offset = pack_bitmap(vb, 6), 6
    exp = oracle().distance_rows(KIND[kind], a, b, threads=8)
    for lhs in (ca, to_device(ca)):
        out = eval_distance(FN[kind], lhs, cb)
        valid = va & vb
        np.testing.assert_array_equal(out.valid_mask(), valid)
        assert_bits(out.values()[valid], exp[valid])
    # a NULL constant gives NULL everywhere
    out = eval_distance(FN[kind], Column.vector_int8(a), const_vector(None, rows, dim=dim, dtype=abi.VEC_I8))
    assert not out.valid_mask().any()


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_distance_mixed_element_types(gpu, kind):
    """Int8 with Float32: dims are not compared, every row is 0.0 (non-nullable) or NULL."""
    rng = np.random.default_rng(5)
    a = rand_i8(rng, (300, 16))
    f = rng.standard_normal((300, 24)).astype(np.float32)
    for lhs, rhs in ((Column.vector_int8(a), Column.vector(f)), (Column.vector(f), Column.vector_int8(a)),
                     (Column.vector_int8(a), const_vector(f[0], 300))):
        out = eval_distance(FN[kind], lhs, rhs)
        assert out.validity is None
        np.testing.assert_array_equal(out.values().view(np.uint32), np.zeros(300, np.uint32))
    ca = Column.vector_int8(a)
    ca.validity = pack_bitmap(np.ones(300, bool))
    out = eval_distance(FN[kind], ca, Column.vector(f))
    assert not out.valid_mask().any()
    np.testing.assert_array_equal(out.values(), np.zeros(300, np.float32))


def test_distance_dim_mismatch(gpu):
    a, b = np.zeros((4, 8), np.int8), np.zeros((4, 9), np.int8)
    with pytest.raises(DbxError, match="Vector length not equal"):
        eval_distance("l2_distance", Column.vector_int8(a), Column.vector_int8(b))


# ---------------------------------------------------------------- kNN against the oracle
def oracle_topk(kind, corpus, q, k):
    d = oracle().distance_rows(KIND[kind], corpus, q, threads=8)
    key = np.where(np.isnan(d), np.inf, d)  # OrderedFloat: NaN last; ties by row id (stable)
    order = np.lexsort((np.arange(len(d)), np.isnan(d), key))[:k]
    return order, d[order]


def check_knn(kind, corpus, queries, k, op=None):
    own = op is None
    if own:
        op = VectorTopN(FN[kind], Column.vector_int8(corpus))
    idx, dist = op.search(Column.vector_int8(queries), k)
    st = op.stats()
    if own:
        op.close()
    kk = min(k, len(corpus))
    for i in range(len(queries)):
        ref_idx, ref_d = oracle_topk(kind, corpus, queries[i], kk)
        np.testing.assert_array_equal(idx[i, :kk], ref_idx, err_msg=f"query {i}")
        assert_bits(dist[i, :kk], ref_d)
        assert (idx[i, kk:] == -1).all()
    assert st["certified"] + st["exact_fallback"] == len(queries)
    return idx, dist, st


@pytest.mark.parametrize("kind", ["cosine", "l2"])
@pytest.mark.parametrize("dim", [8, 100, 768, 1024, 1025, 4096])
def test_knn_dims(gpu, kind, dim):
    rng = np.random.default_rng(dim + 7 * (kind == "l2"))
    corpus = special_rows(rand_i8(rng, (3000, dim)))
    queries = rand_i8(rng, (130, dim))
    op = VectorTopN(FN[kind], Column.vector_int8(corpus))
    for k in (1, 10, 128, 129):
        check_knn(kind, corpus, queries, k, op)
    op.close()


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_knn_k_and_batches(gpu, kind):
    rng = np.random.default_rng(21)
    corpus = rand_i8(rng, (5000, 100))
    queries = rand_i8(rng, (1024, 100))
    op = VectorTopN(FN[kind], Column.vector_int8(corpus))
    check_knn(kind, corpus, queries[:1], 1024, op)
    check_knn(kind, corpus, queries[:130], 1024, op)
    check_knn(kind, corpus, queries, 10, op)
    check_knn(kind, corpus, queries[:1], 10, op)
    op.close()


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_knn_corpus_spanning_passes(gpu, kind):
    rng = np.random.default_rng(300_001)
    corpus = rand_i8(rng, (300_001, 8))
    queries = rand_i8(rng, (3, 8))
    check_knn(kind, corpus, queries, 10)
    check_knn(kind, corpus, queries, 129)


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_knn_accumulator_headroom(gpu, kind):
    """Every value -128 at dim 4096: |ab| = 2^26 in each int32 accumulator."""
    rng = np.random.default_rng(4096)
    corpus = rand_i8(rng, (700, 4096))
    corpus[::3] = -128
    corpus[1::7] = 127
    queries = np.full((4, 4096), -128, np.int8)
    queries[1] = 127
    queries[2:] = rand_i8(rng, (2, 4096))
    check_knn(kind, corpus, queries, 10)
    check_knn(kind, corpus, queries, 300)


# ---------------------------------------------------------------- ties
@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_knn_duplicates_of_the_nearest_row(gpu, kind):
    rng = np.random.default_rng(8)
    dim = 64
    base = rand_i8(rng, (20_000, dim))
    q = rand_i8(rng, (1, dim))
    for n_dup in (8500, 10, 11):
        corpus = base.copy()
        rows = np.sort(rng.choice(len(corpus), n_dup, replace=False))
        corpus[rows] = q[0]
        check_knn(kind, corpus, q, 10)
        if n_dup == 8500:
            check_knn(kind, corpus, q, 1024)


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_knn_distinct_similarities_one_distance(gpu, kind):
    """Rows that differ from a target by a small step in one coordinate: many distinct exact integer
    similarities whose f32 distances coincide.  Cosine: the target is the query itself (distances
    within a few ulps of 0 of 1 - similarity).  L2: the target is 120 away in most coordinates, so
    S ~ 2^25.8 and the f32 fold rounds away the steps in the other coordinates."""
    rng = np.random.default_rng(12)
    n = 6000
    if kind == "cosine":
        dim = 1024
        q = rand_i8(rng, (1, dim), -120, 120)
        target, free = q[0].copy(), np.arange(dim)
        steps = np.array([-1, 1], np.int8)
    else:
        dim = 4096
        q = rand_i8(rng, (1, dim), -4, 5)
        target = q[0].copy()
        target[:4000] += 120
        free = np.arange(4000, dim)
        steps = np.array([-3, -2, -1, 0, 1, 2, 3], np.int8)  # S, S+1, S+4, S+9 -> three f32 sums
    corpus = np.repeat(target[None], n, 0)
    corpus[np.arange(n), rng.choice(free, n)] += rng.choice(steps, n)
    corpus = np.concatenate([corpus, rand_i8(rng, (2000, dim))])
    d = oracle().distance_rows(KIND[kind], corpus[:n], q[0], threads=8)
    c64, q64 = corpus[:n].astype(np.int64), q[0].astype(np.int64)
    if kind == "cosine":
        exact = np.unique(np.stack([c64 @ q64, (c64 * c64).sum(1)], 1), axis=0)
    else:
        exact = np.unique(((c64 - q64) ** 2).sum(1))
    assert len(np.unique(d)) < len(exact)  # the f32 distances really do collide
    for k in (10, 129):
        check_knn(kind, corpus, q, k)


def test_knn_zero_query_cosine(gpu):
    rng = np.random.default_rng(2)
    corpus = rand_i8(rng, (3000, 32))
    queries = np.concatenate([np.zeros((1, 32), np.int8), rand_i8(rng, (2, 32))])
    idx, dist, _ = check_knn("cosine", corpus, queries, 10)
    np.testing.assert_array_equal(idx[0], np.arange(10))
    assert np.isnan(dist[0]).all()


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_knn_zero_corpus(gpu, kind):
    corpus = np.zeros((2000, 48), np.int8)
    queries = rand_i8(np.random.default_rng(3), (3, 48))
    idx, _, _ = check_knn(kind, corpus, queries, 10)
    np.testing.assert_array_equal(idx, np.tile(np.arange(10), (3, 1)))


# ---------------------------------------------------------------- tensor-core pass vs references
@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_igmma_matches_cuda_core_reference(gpu, monkeypatch, kind):
    rng = np.random.default_rng(31)
    for n, dim in ((20_000, 100), (2000, 768)):
        corpus = rand_i8(rng, (n, dim))
        queries = rand_i8(rng, (130, dim))
        a = check_knn(kind, corpus, queries, 10)
        monkeypatch.setenv("DBX_KNN_REF_GEMM", "1")
        b = check_knn(kind, corpus, queries, 10)
        monkeypatch.delenv("DBX_KNN_REF_GEMM")
        np.testing.assert_array_equal(a[0], b[0])
        np.testing.assert_array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
        assert a[2]["certified"] == b[2]["certified"]


@pytest.fixture(scope="module")
def uniform_1m():
    rng = np.random.default_rng(1_000_000)
    return rand_i8(rng, (1_000_000, 768)), rand_i8(rng, (1024, 768))


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_same_answer_as_float32_and_no_fallback(gpu, uniform_1m, kind):
    """1e6 x 768, 1024 queries: the int8 search returns the Float32 search's ids and distance bits
    over the widened corpus, and on uniform data no query needs the exact fallback."""
    corpus, queries = uniform_1m
    op = VectorTopN(FN[kind], to_device(Column.vector_int8(corpus)))
    idx8, d8 = op.search(Column.vector_int8(queries), 10)
    st = op.stats()
    op.close()
    assert st["certified"] == 1024 and st["exact_fallback"] == 0, st
    opf = VectorTopN(FN[kind], to_device(Column.vector(corpus)))
    idxf, df = opf.search(Column.vector(queries), 10)
    stf = opf.stats()
    opf.close()
    assert stf["certified"] + stf["exact_fallback"] == 1024
    np.testing.assert_array_equal(idx8, idxf)
    np.testing.assert_array_equal(d8.view(np.uint32), df.view(np.uint32))
    for i in (0, 511, 1023):  # and the oracle for a few queries
        ref_idx, ref_d = oracle_topk(kind, corpus, queries[i], 10)
        np.testing.assert_array_equal(idx8[i], ref_idx)
        assert_bits(d8[i], ref_d)


# ---------------------------------------------------------------- refusals
def test_knn_refusals(gpu):
    rng = np.random.default_rng(1)
    corpus = rand_i8(rng, (500, 16))
    op = VectorTopN("cosine_distance", Column.vector_int8(corpus))
    with pytest.raises(DbxError) as e:
        op.search(Column.vector(corpus[:2].astype(np.float32)), 5)
    assert e.value.status == abi.ERR_INVALID
    with pytest.raises(DbxError, match="Vector length not equal"):
        op.search(Column.vector_int8(rand_i8(rng, (2, 17))), 5)
    q = Column.vector_int8(corpus[:2])
    q.validity = pack_bitmap([True, False])
    with pytest.raises(DbxError) as e:
        op.search(q, 5)
    assert e.value.status == abi.ERR_UNSUPPORTED
    op.close()
    c = Column.vector_int8(corpus)
    c.validity = pack_bitmap(np.ones(500, bool))
    with pytest.raises(DbxError) as e:
        VectorTopN("l2_distance", c)
    assert e.value.status == abi.ERR_UNSUPPORTED
    # a Float32 corpus refuses Int8 queries
    opf = VectorTopN("l2_distance", Column.vector(corpus.astype(np.float32)))
    with pytest.raises(DbxError) as e:
        opf.search(Column.vector_int8(corpus[:2]), 5)
    assert e.value.status == abi.ERR_INVALID
    opf.close()


def vec_block(n, seed=0):
    rng = np.random.default_rng(seed)
    return DataBlock([Column.from_data(np.arange(n, dtype=np.int32)), Column.vector_int8(rand_i8(rng, (n, 8)))], n)


def test_other_operators_refuse_vector_int8(gpu):
    """Filter, aggregate, top-k and join do not carry Vector(Int8): given one to read, they refuse it
    (dtype_size is 0 for it), they never misread its bytes as numbers."""
    blk = vec_block(100)
    types = schema_types(blk)

    def refused(make_and_push):
        with pytest.raises(DbxError):
            make_and_push()

    refused(lambda: TransformFilter(gt(col(0), lit(5)), types).transform(blk))
    refused(lambda: TransformPartialAggregate(AggregatorParams([1], [("count", 0)]), types).transform(blk))  # GROUP BY key
    refused(lambda: TransformPartialAggregate(AggregatorParams([0], [("sum", 1)]), types).transform(blk))    # argument
    refused(lambda: TransformTopN(1, True, False, 10, types).transform(blk))

    def join():  # the vector rides along as a build / probe payload column
        j = HashJoin(types, types, 0, 0)
        j.add_block(blk)
        j.final_build()
        j.probe_block(blk)
    refused(join)


# ---------------------------------------------------------------- block kernels
def int8_vec_block(n, seed, dims=(3, 8, 12), bit_off=5):
    rng = np.random.default_rng(seed)
    cols = [Column.from_data(rng.integers(-1000, 1000, n).astype(np.int64))]
    for j, d in enumerate(dims):
        c = Column.vector_int8(rand_i8(rng, (n, d)))
        if j != 1:
            c.validity, c.validity_bit_offset = pack_bitmap(rng.random(n) > 0.25, bit_off), bit_off
        cols.append(c)
    return DataBlock(cols, n)


def assert_rows(got: DataBlock, blk: DataBlock, rows):
    rows = np.asarray(rows, dtype=np.int64)
    assert got.num_rows == len(rows)
    for g, c in zip(got.columns, blk.columns):
        assert g.dtype == c.dtype and g.vec_dim == c.vec_dim
        m = c.valid_mask()[rows]
        np.testing.assert_array_equal(g.valid_mask(), m)
        np.testing.assert_array_equal(np.asarray(g.values())[m], np.asarray(c.values())[rows][m])


@pytest.mark.parametrize("device", [False, True])
def test_block_kernels_move_vector_int8(gpu, device):
    n = 5003
    blk = int8_vec_block(n, 1)
    src = DataBlock([to_device(c) for c in blk.columns], n) if device else blk
    rng = np.random.default_rng(2)
    idx = rng.integers(0, n, 7000)
    assert_rows(take(src, idx), blk, idx)
    ranges = [(0, 10), (4000, 5003), (17, 17), (250, 550)]  # [start, end)
    assert_rows(take_ranges(src, ranges), blk, np.concatenate([np.arange(s, e) for s, e in ranges]))
    part = rng.integers(0, 5, n)
    outs = scatter(src, part, 5)
    for p, o in enumerate(outs):
        assert_rows(o, blk, np.nonzero(part == p)[0])
    blk2 = int8_vec_block(777, 3, bit_off=0)
    src2 = DataBlock([to_device(c) for c in blk2.columns], 777) if device else blk2
    cat = concat([src, src2])
    assert_rows(DataBlock([c.slice(0, n) for c in cat.columns], n), blk, np.arange(n))
    assert_rows(DataBlock([c.slice(n, n + 777) for c in cat.columns], 777), blk2, np.arange(777))
