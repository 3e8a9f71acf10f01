"""Inputs that put the kNN certificate at the edge of its bf16 error budget (cosine and L2).

The similarity GEMM rounds both operands to bf16 (round to nearest even, u = 2^-8).  A value just
below a bf16 midpoint 2^e (1 + 2^-8) rounds DOWN by almost u/(1+u) of itself, so a product of two
such values loses almost 1 - (1+u)^-2 = 0.0077670.  The construction, for one query q and k = 1:

  * q: every component is 2^e_i * m with m = 1 + 2^-8 - 2^-15 (just below the midpoint, with a
    slack of 2^-15 that rsqrtf's few-ulp error in the normalisation cannot cross) and exponents
    chosen so that |q| = 1 to within 2e-5; its bf16 operand is exactly 2^e_i;
  * R = q: exact similarity 1, bf16 similarity sum(4^e_i) ~ 0.99247, short by ~0.0077;
  * an anchor with bf16-exact components 2^e_i or 2^e_i (1 + 2^-7) and |a| ~ 1 (so normalisation
    rounds back to the same bf16 values): exact similarity just below R's, bf16 similarity ~0.996;
  * decoys with components in {0, 2^e_i, 2^(e_i+1)} and |d| ~ 1: bf16-exact, and every product
    and partial sum of their bf16 dot product with q is a multiple of the finest 4^e_i below 2, so
    the tensor core computes their similarity D exactly, whatever its adder rounds;
  * D = S_anchor - x.  With at least k' - 1 decoys, R stays a candidate only if its approximate
    similarity is >= D.  The certificate accepts the anchor iff x >= margin.  So for every x, a
    sound margin gives R (R kept, or the query answered exactly); a margin smaller than the real
    error of R's similarity returns the anchor, certified.

The L2 form uses the same vectors times 2^20, where the absolute error of 2 q.c dominates.
"""
from __future__ import annotations

import math

import numpy as np

MID = 1.0 + 2.0 ** -8
Q_MANT = MID - 2.0 ** -15     # just below the midpoint: rounds down to 1
L2_SCALE = 2.0 ** 20
N_DECOYS = 80                  # >= k' - 1 = 63 at k = 1


def bf16_rne(x) -> np.ndarray:
    """float32 -> nearest bf16 (ties to even), returned as float32.  Finite inputs."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return r.astype(np.uint32).view(np.float32)


def _levels(dim: int) -> np.ndarray:
    """Exponents e_i with sum(4^e_i) * Q_MANT^2 = 1 to within 2e-5: most components at a base
    level b, some raised by 1-3 levels, and three components at each of the three levels below b
    (fine steps for the decoys' similarities)."""
    b = math.ceil(math.log(dim, 4)) + 2
    target = 1.0 / (Q_MANT * Q_MANT)
    e = np.full(dim, -b, dtype=np.int64)
    fine = np.array([-b - 1] * 3 + [-b - 2] * 3 + [-b - 3] * 3)
    e[dim - len(fine):] = fine
    w = 4.0 ** -b
    excess = round((target - float(np.sum(4.0 ** e))) / w)
    i = 0
    for step, up in ((63, 3), (15, 2), (3, 1)):
        while excess >= step and i < dim - len(fine):
            e[i] += up
            excess -= step
            i += 1
    if excess > 0:  # overshoot by < 3 units, then lower base components by 3/4 unit each
        e[i] += 1
        excess -= 3
        i += 1
    j = dim - len(fine) - 1
    while excess <= -0.375:
        e[j] -= 1
        excess += 0.75
        j -= 1
    return e


class Case:
    """One adversarial corpus for dim, kind and the gap x between the anchor and the decoys."""

    def __init__(self, dim: int, x: float, kind: str = "cosine"):
        self.dim, self.x, self.kind = dim, x, kind
        e = _levels(dim)
        self.e = e
        p2 = 2.0 ** e
        self.q = (p2 * Q_MANT).astype(np.float32)
        self.q_bf16 = p2.astype(np.float32)        # what the GEMM sees for q (and R)
        # anchor: 2^e (1 + 2^-7) on enough of the energy to bring |a| to ~1
        a = p2.copy()
        need = 1.0 - float(np.sum(p2 * p2))
        for i in np.argsort(-p2, kind="stable"):
            gain = p2[i] ** 2 * ((1 + 2.0 ** -7) ** 2 - 1)
            if need <= gain / 2:
                break
            a[i] *= 1 + 2.0 ** -7
            need -= gain
        self.anchor = a.astype(np.float32)
        s_anchor = float(np.dot(self.q.astype(np.float64), a) / (np.linalg.norm(self.q.astype(np.float64)) * np.linalg.norm(a)))
        self.target = s_anchor - x
        self.decoys = np.stack([self._decoy(seed) for seed in range(N_DECOYS)]).astype(np.float32)
        self.r = self.q.copy()
        if kind == "l2":
            self.q, self.r = self.q * np.float32(L2_SCALE), self.r * np.float32(L2_SCALE)
            self.anchor = self.anchor * np.float32(L2_SCALE)
            self.decoys = self.decoys * np.float32(L2_SCALE)
        # corpus rows: decoys, anchor, R last (largest row id: ties could only hide it)
        self.corpus = np.concatenate([self.decoys, self.anchor[None], self.r[None]]).astype(np.float32)
        self.r_row = len(self.corpus) - 1
        self.anchor_row = len(self.corpus) - 2

    def _decoy(self, seed: int) -> np.ndarray:
        """components in {0, 2^e, 2^(e+1)}, |d|^2 ~ 1, bf16 dot product with q exactly the decoy
        level: raise some components (+3 w energy, +w dot), zero others (-w, -w)."""
        rng = np.random.default_rng(1000 + seed)
        p2 = 2.0 ** self.e
        w = p2 * p2
        unit = float(w.min())
        d = p2.copy()
        dot = float(np.sum(w))
        want = math.floor(self.target / unit) * unit
        raise_by = (1.0 - want) / 2.0          # sum of w raised; then zeroed = dot + raised - want
        order = rng.permutation(len(d))
        used = np.zeros(len(d), dtype=bool)
        coarse = order[w[order] > unit * 16]
        for i in coarse:
            if raise_by < w[i]:
                continue
            d[i] *= 2.0
            dot += w[i]
            raise_by -= w[i]
            used[i] = True
        drop = dot - want
        for i in sorted(order, key=lambda j: -w[j]):
            if used[i] or drop < w[i]:
                continue
            d[i] = 0.0
            drop -= w[i]
            used[i] = True
        assert drop == 0.0, drop
        return d

    def approx_similarity(self, row: np.ndarray) -> float:
        """The GEMM's operand product before accumulation: sum of bf16(q^) * bf16(row^) in f64."""
        q = self.q.astype(np.float64)
        r = row.astype(np.float64)
        qn = bf16_rne((q / np.linalg.norm(q)).astype(np.float32)).astype(np.float64)
        rn = bf16_rne((r / np.linalg.norm(r)).astype(np.float32)).astype(np.float64)
        return float(np.dot(qn, rn))

    def decoy_similarity(self) -> float:
        return float(np.dot(self.q_bf16.astype(np.float64), (self.decoys[0] / (L2_SCALE if self.kind == "l2" else 1.0)).astype(np.float64)))
