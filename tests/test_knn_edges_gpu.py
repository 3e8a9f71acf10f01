"""Brute-force kNN where it can be wrong: the certificate at its error margin, k up to 1024 across
the candidate-list modes, embedding-size dims, large query batches, corpora beyond one pass chunk,
non-finite and extreme vectors, the device-output path and one handle reused across searches.

Every result is the oracle's ranking by (OrderedFloat distance, row id) with distances bit for
bit, and every query is either certified or answered exactly."""
import numpy as np
import pytest
import torch

from databend_b200 import abi
from databend_b200.block import Column
from databend_b200.lib import DbxError
from databend_b200.transforms import to_device
from databend_b200.vector import VectorTopN, const_vector, eval_distance
from knn_adversarial import Case
from test_knn_gpu import FN, KIND, assert_f32_bits_equal, check_knn, oracle

pytestmark = pytest.mark.gpu


def oracle_knn_many(kind, corpus, queries, k):
    """oracle_knn for many queries: a stable sort puts NaN last and keeps -0 == +0 in row order."""
    n = len(corpus)
    dist = np.empty((len(queries), n), dtype=np.float32)
    for i, q in enumerate(queries):
        dist[i] = oracle().distance_rows(KIND[kind], corpus, q, threads=8)
    order = np.argsort(dist, axis=1, kind="stable")[:, :k]
    idx = np.full((len(queries), k), -1, dtype=np.int64)
    out = np.full((len(queries), k), np.nan, dtype=np.float32)
    idx[:, :order.shape[1]] = order
    out[:, :order.shape[1]] = np.take_along_axis(dist, order, axis=1)
    return idx, out


def check_many(kind, corpus, queries, k, op=None):
    own = op is None
    if own:
        op = VectorTopN(FN[kind], Column.vector(corpus))
    idx, dist = op.search(Column.vector(queries), k)
    stats = op.stats()
    if own:
        op.close()
    eidx, edist = oracle_knn_many(kind, corpus, queries, k)
    np.testing.assert_array_equal(idx, eidx)
    assert_f32_bits_equal(dist, edist)
    assert stats["certified"] + stats["exact_fallback"] == len(queries)
    return stats


# ---------------------------------------------------------------- 1. certificate at its margin
@pytest.mark.parametrize("dim", [768, 1536, 4096])
@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_certificate_at_its_margin(gpu, kind, dim):
    """R's bf16 similarity is ~0.0077 below its exact similarity; decoys sit x below the anchor.
    For every x the answer must be R: either R stays a candidate or the query is answered exactly.
    A margin below the real error of R's approximate similarity would return the anchor."""
    certified_at = []
    for x in (0.0070, 0.0076, 0.0078, 0.0079, 0.00795, 0.0080, 0.0081, 0.0082, 0.0084, 0.0088, 0.0095):
        c = Case(dim, x, kind)
        stats = check_knn(kind, c.corpus, c.q[None], 1)
        if stats["certified"]:
            certified_at.append(x)
    print(f"{kind} dim {dim}: certified at x = {certified_at}")
    assert certified_at and max(certified_at) == 0.0095  # the certificate still works well above its margin


# ---------------------------------------------------------------- 2. k across the list modes
@pytest.fixture(scope="module")
def corpus_50k():
    rng = np.random.default_rng(5)
    return rng.standard_normal((50_000, 96)).astype(np.float32), rng.standard_normal((130, 96)).astype(np.float32)


@pytest.mark.parametrize("kind", ["cosine", "l2"])
@pytest.mark.parametrize("k", [1, 64, 128, 129, 300, 1024])
def test_k_across_list_modes(gpu, corpus_50k, kind, k):
    """k <= 128 keeps per-query candidate lists at these query counts, k >= 129 the shared list."""
    corpus, queries = corpus_50k
    for nq in (1, 130):
        check_many(kind, corpus, queries[:nq], k)


def test_k_above_limit_refused(gpu, corpus_50k):
    corpus, queries = corpus_50k
    op = VectorTopN("cosine_distance", Column.vector(corpus[:1000]))
    with pytest.raises(DbxError, match="k > 1024"):
        op.search(Column.vector(queries[:2]), 1025)
    op.close()


# ---------------------------------------------------------------- 3. embedding dims
@pytest.mark.parametrize("kind", ["cosine", "l2"])
@pytest.mark.parametrize("dim", [127, 129, 1024, 1536, 3072, 4095, 4096])
def test_embedding_dims(gpu, kind, dim):
    rng = np.random.default_rng(dim)
    corpus = rng.standard_normal((3000, dim)).astype(np.float32)
    queries = rng.standard_normal((5, dim)).astype(np.float32)
    for k in (10, 100):
        check_many(kind, corpus, queries, k)
    # the row-wise function at the same dims, column and const right-hand side
    a, b = corpus[:700], corpus[700:1400]
    assert_f32_bits_equal(eval_distance(FN[kind], Column.vector(a), Column.vector(b)).values(),
                          oracle().distance_rows(KIND[kind], a, b, threads=8))
    assert_f32_bits_equal(eval_distance(FN[kind], to_device(Column.vector(a)), const_vector(queries[0], len(a))).values(),
                          oracle().distance_rows(KIND[kind], a, queries[0], threads=8))


# ---------------------------------------------------------------- 4. query batches
@pytest.fixture(scope="module")
def small_corpus():
    rng = np.random.default_rng(17)
    return rng.standard_normal((400, 16)).astype(np.float32), rng.standard_normal((65_537, 16)).astype(np.float32)


@pytest.mark.parametrize("nq", [384, 1024, 4096, 8192, 65_536])
def test_query_batches(gpu, small_corpus, nq):
    """nq = 4096 still gets per-query lists at k = 10, 8192 the shared list, 65 536 is the limit."""
    corpus, queries = small_corpus
    for kind in ("cosine", "l2"):
        check_many(kind, corpus, queries[:nq], 10)


def test_query_batch_above_limit_refused(gpu, small_corpus):
    corpus, queries = small_corpus
    op = VectorTopN("l2_distance", Column.vector(corpus))
    with pytest.raises(DbxError, match="more than 65536 queries"):
        op.search(Column.vector(queries), 10)
    op.close()


@pytest.mark.parametrize("cluster,nq", [(4, 512), (8, 1024)])
def test_gemm_cluster_sizes(gpu, monkeypatch, cluster, nq):
    monkeypatch.setenv("DBX_KNN_CLUSTER", str(cluster))
    rng = np.random.default_rng(cluster)
    corpus = rng.standard_normal((20_000, 64)).astype(np.float32)
    queries = rng.standard_normal((nq, 64)).astype(np.float32)
    for kind in ("cosine", "l2"):
        op = VectorTopN(FN[kind], Column.vector(corpus))
        check_many(kind, corpus, queries, 10, op=op)
        assert op.stats()["cluster"] == cluster
        op.close()


# ---------------------------------------------------------------- 5. corpus sizes
def test_corpus_beyond_one_pass_chunk(gpu):
    """2^24 + 2^20 + 77 rows: passes stop growing at 2^24 rows, so this takes more than one capped
    pass."""
    n, dim = (1 << 24) + (1 << 20) + 77, 16
    rng = np.random.default_rng(24)
    corpus = rng.standard_normal((n, dim), dtype=np.float32)
    queries = rng.standard_normal((4, dim), dtype=np.float32)
    dev = to_device(Column.vector(corpus))
    for kind in ("cosine", "l2"):
        op = VectorTopN(FN[kind], dev)
        stats = check_many(kind, corpus, queries, 10, op=op)
        op.close()
        assert stats["passes"] >= 3


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_corpus_sizes_around_kprime(gpu, kind):
    rng = np.random.default_rng(3)
    queries = rng.standard_normal((3, 32)).astype(np.float32)
    # empty corpus: every slot is -1 / NaN, as for n < k
    op = VectorTopN(FN[kind], Column.vector(np.zeros((0, 32), np.float32)))
    idx, dist = op.search(Column.vector(queries), 5)
    op.close()
    assert (idx == -1).all() and np.isnan(dist).all()
    for k in (1, 10):
        kprime = max(8 * k, 64)
        kprime = (kprime + 63) // 64 * 64
        for n in (kprime - 1, kprime, kprime + 1):
            check_many(kind, rng.standard_normal((n, 32)).astype(np.float32), queries, k)


# ---------------------------------------------------------------- 6. non-finite and extreme vectors
def extreme_rows(rng, dim):
    base = rng.standard_normal((600, dim)).astype(np.float32)
    rows = [base]
    special = np.array(base[:24])
    special[0, 3] = np.nan
    special[1, 5] = np.inf
    special[2, 7] = -np.inf
    special[3] *= np.float32(3e19)           # squares overflow f32
    special[4] = np.float32(1e20)            # every component huge
    special[5] *= np.float32(1e-23)          # squares underflow to 0
    special[6] *= np.float32(1e-20)          # subnormal squares
    special[7] = np.float32(1e-45)           # subnormal components
    special[8] = 0.0
    special[9] = -0.0
    rows.append(special)
    # pairs equal after bf16 rounding but not in f32
    twin = base[40].copy()
    twin[::3] = np.nextafter(twin[::3], np.float32(np.inf))
    rows.append(twin[None])
    return np.concatenate(rows).astype(np.float32)


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_non_finite_and_extreme_vectors(gpu, kind):
    rng = np.random.default_rng(66)
    dim = 48
    corpus = extreme_rows(rng, dim)
    clean = corpus[:600]
    special = corpus[600:]
    queries = np.concatenate([special[:10], clean[40:41] + np.float32(1e-3), clean[:3] * np.float32(1e-23), clean[3:5] * np.float32(3e19)]).astype(np.float32)
    # extreme queries against a clean corpus, and all queries against the extreme corpus
    for k in (1, 10, 64, 700):
        check_many(kind, clean, queries, k)
        check_many(kind, corpus, queries, k)
    # the row-wise function on the same rows
    q = np.resize(queries, (len(corpus), dim)).astype(np.float32)
    assert_f32_bits_equal(eval_distance(FN[kind], Column.vector(corpus), Column.vector(q)).values(),
                          oracle().distance_rows(KIND[kind], corpus, q, threads=8))


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_bf16_twins_at_the_kth_position(gpu, kind):
    """Rows that are equal after bf16 rounding but not in f32, at and around the k-th position."""
    rng = np.random.default_rng(8)
    dim = 64
    q = rng.standard_normal(dim).astype(np.float32)
    base = (q + 0.3 * rng.standard_normal((20, dim))).astype(np.float32)
    twins = np.repeat(base, 4, axis=0)
    for j in range(1, 4):
        twins[j::4, j::5] = np.nextafter(twins[j::4, j::5], np.float32(np.inf * (1 if j % 2 else -1)))
    corpus = np.concatenate([rng.standard_normal((5000, dim)).astype(np.float32), twins]).astype(np.float32)
    for k in (2, 5, 9, 10, 40):
        check_many(kind, corpus, q[None], k)


# ---------------------------------------------------------------- 7. bench path and reuse
def test_search_into_device_outputs(gpu):
    """The benchmark's path: device-resident corpus and queries, results written to device buffers."""
    rng = np.random.default_rng(12)
    corpus = rng.standard_normal((30_000, 128)).astype(np.float32)
    queries = rng.standard_normal((256, 128)).astype(np.float32)
    op = VectorTopN("cosine_distance", to_device(Column.vector(corpus)))
    k = 10
    oi = torch.empty((len(queries), k), dtype=torch.int64, device="cuda")
    od = torch.empty((len(queries), k), dtype=torch.float32, device="cuda")
    op.search_into(to_device(Column.vector(queries)), k, oi.data_ptr(), od.data_ptr())
    torch.cuda.synchronize()
    stats = op.stats()
    op.close()
    eidx, edist = oracle_knn_many("cosine", corpus, queries, k)
    np.testing.assert_array_equal(oi.cpu().numpy(), eidx)
    assert_f32_bits_equal(od.cpu().numpy(), edist)
    assert stats["certified"] + stats["exact_fallback"] == len(queries)


@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_handle_reuse_across_searches(gpu, monkeypatch, kind):
    """One handle: the buffers grow, and the list mode changes from one search to the next."""
    rng = np.random.default_rng(31)
    corpus = rng.standard_normal((50_000, 96)).astype(np.float32)
    queries = rng.standard_normal((1500, 96)).astype(np.float32)
    op = VectorTopN(FN[kind], Column.vector(corpus))
    for nq, k in ((5, 10), (1500, 129), (3, 1024)):
        check_many(kind, corpus, queries[:nq], k, op=op)
    monkeypatch.setenv("DBX_KNN_QCAP", "256")  # per-query lists overflow: the search is repeated checked
    check_many(kind, corpus, queries[:130], 1, op=op)
    monkeypatch.delenv("DBX_KNN_QCAP")
    check_many(kind, corpus, queries[:200], 1, op=op)
    op.close()
