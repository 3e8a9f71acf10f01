"""The adversarial kNN inputs (tests/knn_adversarial.py) produce the bf16 shortfall they are built
for, emulated on the host: if they did not, the GPU test at the certificate's margin would prove
nothing."""
import numpy as np
import pytest

from databend_b200 import abi
from knn_adversarial import N_DECOYS, Case, bf16_rne


def test_bf16_rne_emulation():
    x = np.array([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -8 - 2.0 ** -20, 1.0 + 2.0 ** -8 + 2.0 ** -20, -3.0], np.float32)
    np.testing.assert_array_equal(bf16_rne(x), np.array([1.0, 1.0, 1.0 + 2 * 2.0 ** -7, 1.0, 1.0 + 2.0 ** -7, -3.0], np.float32))


@pytest.mark.parametrize("dim", [768, 1536, 4096])
@pytest.mark.parametrize("kind", ["cosine", "l2"])
def test_adversarial_construction(dim, kind):
    from oracle import oracle as orc
    x = 0.0070  # decoys between R's approximate and exact similarity
    c = Case(dim, x, kind)
    q = c.q.astype(np.float64)
    # q's normalised components sit just below a bf16 midpoint, with room for rsqrtf's error
    qn = q / np.linalg.norm(q)
    for rel in (-2e-6, 0.0, 2e-6):
        np.testing.assert_array_equal(bf16_rne((qn * (1 + rel)).astype(np.float32)), c.q_bf16)
    # R = q: the bf16 similarity falls short of 1 by close to the per-product maximum 0.0077670
    short = 1.0 - c.approx_similarity(c.r)
    assert 0.0076 < short < 0.0077670, short
    # decoys and anchor are exact in bf16 after normalisation (it moves them by < 1e-4)
    for row in list(c.decoys[:5]) + [c.anchor]:
        r = row.astype(np.float64)
        assert abs(np.linalg.norm(r) / (1.0 if kind == "cosine" else 2.0 ** 20) - 1.0) < 1e-3
        np.testing.assert_array_equal(bf16_rne((r / np.linalg.norm(r)).astype(np.float32)), (r / (1.0 if kind == "cosine" else 2.0 ** 20)).astype(np.float32))
    # every decoy has the same bf16 similarity, between R's approximate and exact similarity,
    # x below the anchor's exact similarity (to the finest step of the construction)
    ds = {c.approx_similarity(d) for d in c.decoys}
    assert len(ds) == 1
    dsim = ds.pop()
    assert dsim == c.decoy_similarity()
    assert 1.0 - short < dsim < 1.0
    assert abs(c.target - dsim) < 1e-6
    assert c.approx_similarity(c.anchor) > dsim + 0.003
    assert len({d.tobytes() for d in c.decoys}) == N_DECOYS
    # the oracle ranks R first, the anchor second, then the decoys
    kid = abi.DIST_COSINE if kind == "cosine" else abi.DIST_L2
    dist = orc.distance_rows(kid, c.corpus, c.q, threads=4)
    order = np.argsort(dist, kind="stable")
    assert order[0] == c.r_row and order[1] == c.anchor_row
    assert dist[c.anchor_row] < dist[:N_DECOYS].min()
