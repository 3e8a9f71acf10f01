"""Parity of the vector-distance functions and of brute-force kNN against the CPU oracle.

Row-wise `cosine_distance` / `l2_distance` (src/common/vector/src/distance.rs:19-35,65-80 via
scalars/vector.rs:497-556) must be BIT-EXACT with the oracle (f32, reference evaluation order) and
reproduce the reference's golden vectors (tests/golden/vector_distance.json).  kNN
(`ORDER BY distance LIMIT k`): returned row ids equal the oracle's ranking by (distance, row id),
returned distances are bit-identical to the row-wise function (tolerance 0; the bf16 tensor-core
pass only nominates candidates, and a certificate or the exact path guarantees the ranking)."""
import json
import os

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column
from databend_b200.transforms import to_device
from databend_b200.vector import VectorTopN, const_vector, eval_distance

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FN = {"cosine": "cosine_distance", "l2": "l2_distance"}
KIND = {"cosine": abi.DIST_COSINE, "l2": abi.DIST_L2}


def oracle():
    from oracle import oracle as orc
    return orc


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_f32_bits_equal(got, exp):
    g, e = np.asarray(got, np.float32), np.asarray(exp, np.float32)
    nan = np.isnan(e)
    np.testing.assert_array_equal(np.isnan(g), nan)
    np.testing.assert_array_equal(bits(g)[~nan], bits(e)[~nan])


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_distance_goldens(gpu, kind):
    """The reference's printed outputs, through the GPU row-wise kernel."""
    with open(os.path.join(GOLD, "vector_distance.json")) as f:
        cases = json.load(f)[kind]
    for c in cases:
        a = np.array([c["a"]], dtype=np.float32)
        b = np.array([c["b"]], dtype=np.float32)
        out = eval_distance(FN[kind], Column.vector(a), Column.vector(b)).values()
        exp = getattr(oracle(), FN[kind])(a[0], b[0])
        assert_f32_bits_equal(out, [exp])
        if c["out"] == "NaN":
            assert np.isnan(out[0]), c["src"]
        else:
            assert abs(float(out[0]) - float(c["out"])) <= 1e-6 * max(1.0, abs(float(c["out"]))), c["src"]


@pytest.mark.parametrize("kind", ["cosine", "l2"])
@pytest.mark.parametrize("dim", [1, 3, 7, 8, 9, 64, 100, 768])
def test_distance_rows_bit_exact(gpu, kind, dim):
    rng = np.random.default_rng(dim * 7 + (kind == "l2"))
    rows = 1000
    a = rng.standard_normal((rows, dim)).astype(np.float32)
    b = rng.standard_normal((rows, dim)).astype(np.float32)
    a[5] = 0.0  # zero vector -> NaN for cosine (vector.txt:28-34)
    exp = oracle().distance_rows(KIND[kind], a, b, threads=4)
    got = eval_distance(FN[kind], Column.vector(a), Column.vector(b)).values()
    assert_f32_bits_equal(got, exp)
    # const right-hand side (the `cosine_distance(col, [..])` form) and device-resident input
    q = b[3]
    exp = oracle().distance_rows(KIND[kind], a, q, threads=4)
    got = eval_distance(FN[kind], to_device(Column.vector(a)), const_vector(q, rows)).values()
    assert_f32_bits_equal(got, exp)
    exp = oracle().distance_rows(KIND[kind], q, a, threads=4)
    got = eval_distance(FN[kind], const_vector(q, rows), Column.vector(a)).values()
    assert_f32_bits_equal(got, exp)


def test_distance_null_and_errors(gpu):
    rng = np.random.default_rng(1)
    a = rng.standard_normal((40, 16)).astype(np.float32)
    b = rng.standard_normal((40, 16)).astype(np.float32)
    ca = Column.vector(a)
    valid = rng.random(40) > 0.3
    from databend_b200.block import pack_bitmap
    ca.validity, ca.validity_bit_offset = pack_bitmap(valid, 3), 3
    out = eval_distance("cosine_distance", ca, Column.vector(b))
    np.testing.assert_array_equal(out.valid_mask(), valid)
    exp = oracle().distance_rows(abi.DIST_COSINE, a, b)
    assert_f32_bits_equal(out.values()[valid], exp[valid])
    out = eval_distance("l2_distance", Column.vector(a), const_vector(None, 40, dim=16))
    assert not out.valid_mask().any()
    from databend_b200.lib import DbxError
    with pytest.raises(DbxError, match="Vector length not equal"):  # distance.rs:20-26
        eval_distance("cosine_distance", Column.vector(a), Column.vector(b[:, :8].copy()))


def oracle_knn(kind, corpus, queries, k):
    """Full ranking by the oracle: (OrderedFloat distance, row id), NaN last, -0 == +0."""
    idx = np.empty((len(queries), k), dtype=np.int64)
    dist = np.empty((len(queries), k), dtype=np.float32)
    for i, q in enumerate(queries):
        d = oracle().distance_rows(KIND[kind], corpus, q, threads=8)
        key = np.where(np.isnan(d), np.inf, d + 0.0)
        nan_last = np.isnan(d)
        order = np.lexsort((np.arange(len(d)), key, nan_last))[:k]
        idx[i, :len(order)] = order
        idx[i, len(order):] = -1
        dist[i, :len(order)] = d[order]
        dist[i, len(order):] = np.nan
    return idx, dist


def check_knn(kind, corpus, queries, k, device_resident=False, expect_exact=None):
    col = Column.vector(corpus)
    if device_resident:
        col = to_device(col)
    op = VectorTopN(FN[kind], col)
    idx, dist = op.search(Column.vector(queries), k)
    stats = op.stats()
    op.close()
    eidx, edist = oracle_knn(kind, corpus, queries, k)
    np.testing.assert_array_equal(idx, eidx)
    assert_f32_bits_equal(dist, edist)
    assert stats["certified"] + stats["exact_fallback"] == len(queries)
    if expect_exact is not None:
        assert stats["exact_fallback"] == expect_exact, stats
    return stats


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_knn_random_768(gpu, kind):
    """configs[4] shape at test size: 768-d N(0,1) corpus, k = 10; the certificate holds for every
    query, so the whole answer comes from the tensor-core path + exact re-rank."""
    rng = np.random.default_rng(42)
    corpus = rng.standard_normal((20000, 768)).astype(np.float32)
    queries = rng.standard_normal((70, 768)).astype(np.float32)
    stats = check_knn(kind, corpus, queries, 10, device_resident=True, expect_exact=0)
    assert stats["passes"] >= 1


@pytest.mark.parametrize("kind", ["cosine", "l2"])
@pytest.mark.parametrize("n,dim,nq,k", [(1, 8, 1, 1), (5, 3, 2, 10), (300, 100, 129, 7), (5000, 65, 3, 100), (4097, 128, 257, 1)])
def test_knn_ragged_shapes(gpu, kind, n, dim, nq, k):
    """dims that are not a multiple of the GEMM k-block, fewer rows than k, one row, query counts
    that straddle the 128-query tile."""
    rng = np.random.default_rng(n + dim)
    corpus = rng.standard_normal((n, dim)).astype(np.float32)
    queries = rng.standard_normal((nq, dim)).astype(np.float32)
    check_knn(kind, corpus, queries, k)


def test_knn_duplicates_zero_vectors_and_clusters(gpu):
    """Ties (duplicate rows) are ordered by row id; zero vectors give NaN (sorted last); a tight
    cluster defeats the bf16 candidate pass and must be caught by the certificate -> exact path."""
    rng = np.random.default_rng(7)
    base = rng.standard_normal((2000, 64)).astype(np.float32)
    corpus = np.concatenate([base, base[:500], np.zeros((3, 64), np.float32)])
    queries = np.concatenate([base[:4] + 0.01, np.zeros((1, 64), np.float32)]).astype(np.float32)
    check_knn("cosine", corpus, queries, 12)
    check_knn("l2", corpus, queries, 12)
    center = rng.standard_normal(64).astype(np.float32)
    cluster = (center + 1e-3 * rng.standard_normal((6000, 64))).astype(np.float32)
    stats = check_knn("cosine", cluster, (center + 1e-3 * rng.standard_normal((5, 64))).astype(np.float32), 5)
    assert stats["exact_fallback"] > 0


def test_knn_forced_exact_path(gpu, monkeypatch):
    rng = np.random.default_rng(3)
    corpus = rng.standard_normal((3000, 48)).astype(np.float32)
    queries = rng.standard_normal((9, 48)).astype(np.float32)
    monkeypatch.setenv("DBX_KNN_FORCE_EXACT", "1")
    check_knn("cosine", corpus, queries, 10, expect_exact=9)
    check_knn("l2", corpus, queries, 10, expect_exact=9)


def test_knn_tensor_core_pass_matches_cuda_core_reference(gpu, monkeypatch):
    """The wgmma similarity pass and the plain CUDA-core pass over the same bf16 operands must
    nominate candidate sets that give the same answer."""
    rng = np.random.default_rng(11)
    corpus = rng.standard_normal((9000, 200)).astype(np.float32)
    queries = rng.standard_normal((33, 200)).astype(np.float32)
    op = VectorTopN("cosine_distance", Column.vector(corpus))
    a = op.search(Column.vector(queries), 10)
    monkeypatch.setenv("DBX_KNN_REF_GEMM", "1")
    b = op.search(Column.vector(queries), 10)
    op.close()
    np.testing.assert_array_equal(a[0], b[0])
    assert_f32_bits_equal(a[1], b[1])


@pytest.mark.parametrize("mode", ["default", "shared_list", "sync", "tiny_lists"])
def test_knn_candidate_list_modes(gpu, monkeypatch, mode):
    """The three ways the candidate lists are run — per-query lists cut by one kernel per pass with
    no host check (default), one shared list cut by a radix sort without host checks, and the
    shared list with a host check after every pass — plus per-query lists so small that a pass
    overflows them (flagged on the device, the search is then repeated in checked mode): all give
    the oracle's answer."""
    if mode == "shared_list":
        monkeypatch.setenv("DBX_KNN_SHARED_LIST", "1")
    elif mode == "sync":
        monkeypatch.setenv("DBX_KNN_SYNC", "1")
    elif mode == "tiny_lists":
        monkeypatch.setenv("DBX_KNN_QCAP", "256")
    rng = np.random.default_rng(99)
    corpus = rng.standard_normal((60_000, 96)).astype(np.float32)
    queries = rng.standard_normal((130, 96)).astype(np.float32)
    k = 1 if mode == "tiny_lists" else 10
    for kind in ("cosine", "l2"):
        check_knn(kind, corpus, queries, k, device_resident=True)


def test_knn_one_million_rows_768(gpu):
    """configs[4] at 1e6 x 768 (a tenth of the benchmark's corpus): the returned neighbours of a
    query sample against the oracle's row-wise distances over ALL rows — ranking by (distance,
    row id) and distances bit for bit."""
    rng = np.random.default_rng(2024)
    n, dim, nq, k = 1_000_000, 768, 64, 10
    corpus = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((nq, dim), dtype=np.float32)
    op = VectorTopN("cosine_distance", to_device(Column.vector(corpus)))
    idx, dist = op.search(Column.vector(queries), k)
    stats = op.stats()
    op.close()
    assert stats["certified"] + stats["exact_fallback"] == nq
    sample = [0, 17, 63]
    eidx, edist = oracle_knn("cosine", corpus, queries[sample], k)
    np.testing.assert_array_equal(idx[sample], eidx)
    assert_f32_bits_equal(dist[sample], edist)
