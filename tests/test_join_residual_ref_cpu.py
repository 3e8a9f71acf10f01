"""The residual-predicate join reference (tests/join_residual_ref.py) without a GPU: with a constant-true
predicate it is the existing INNER / build-side / composite-key references, with a constant-false one every
kind degenerates as the reference's streams say, it agrees with a nested loop over all pairs, and it
reproduces the residual cases of the reference's SQL tests (tests/golden/join_residual.json)."""
import json
import os

import numpy as np
import pytest

from databend_b200 import abi, scalar_expr as S
from databend_b200.block import Column
from join_build_side_ref import hash_join_build_side
from join_multi_key_ref import hash_join_multi_key
from join_residual_ref import (GOLDEN_KINDS, golden_predicate, golden_rows, golden_table, hash_join_residual,
                               sort_rows)

HERE = os.path.dirname(os.path.abspath(__file__))
KINDS = [abi.JOIN_INNER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI, abi.JOIN_LEFT,
         abi.JOIN_RIGHT, abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL]
TRUE, FALSE = S.lit(True, abi.BOOL), S.lit(False, abi.BOOL)


def pairs(res):
    return sorted(zip(res[0].tolist(), res[1].tolist()))


def tables(seed, n_build=300, n_probe=500, key_range=120):
    """Build (k: I64 nullable, x: I32, y: F64 nullable) and probe (k: I32 nullable, z: I64) with duplicate keys."""
    rng = np.random.default_rng(seed)
    bk = rng.integers(0, key_range, n_build)
    pk = rng.integers(-5, key_range + 5, n_probe).astype(np.int32)
    bv, pv, yv = rng.random(n_build) > 0.1, rng.random(n_probe) > 0.1, rng.random(n_build) > 0.2
    build = [Column.from_data(bk, abi.I64, validity=bv), Column.from_data(rng.integers(-50, 50, n_build).astype(np.int32), abi.I32),
             Column.from_data(rng.standard_normal(n_build), abi.F64, validity=yv)]
    btypes = [abi.I64 | abi.NULLABLE, abi.I32, abi.F64 | abi.NULLABLE]
    probe = [Column.from_data(pk, abi.I32, validity=pv), Column.from_data(rng.integers(-50, 50, n_probe), abi.I64)]
    ptypes = [abi.I32 | abi.NULLABLE, abi.I64]
    return build, btypes, probe, ptypes


@pytest.mark.parametrize("kind", KINDS)
def test_constant_true_is_the_equi_join(kind):
    from oracle import oracle as orc
    build, btypes, probe, ptypes = tables(1)
    got = hash_join_residual(kind, build, btypes, probe, ptypes, 0, 0, TRUE)
    if kind in (abi.JOIN_INNER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI, abi.JOIN_LEFT):
        want = orc.hash_join(kind, build[0], probe[0])
    else:
        want = hash_join_build_side(kind, build[0], probe[0])
    assert pairs(got) == pairs(want)
    assert pairs(hash_join_residual(kind, build, btypes, probe, ptypes, 0, 0, None)) == pairs(want)


@pytest.mark.parametrize("kind", KINDS)
def test_constant_true_is_the_composite_key_join(kind):
    build, btypes, probe, ptypes = tables(2, key_range=8)
    build[1] = Column.from_data(np.asarray(build[1].values() % 3, dtype=np.int32), abi.I32)
    probe[1] = Column.from_data(np.asarray(probe[1].values() % 3, dtype=np.int64), abi.I64)
    got = hash_join_residual(kind, build, btypes, probe, ptypes, [0, 1], [0, 1], TRUE)
    want = hash_join_multi_key(kind, [build[0], build[1]], [probe[0], probe[1]])
    assert pairs(got) == pairs(want)


@pytest.mark.parametrize("kind", KINDS)
def test_constant_false(kind):
    build, btypes, probe, ptypes = tables(3)
    nb, npr = build[0].length, probe[0].length
    got = pairs(hash_join_residual(kind, build, btypes, probe, ptypes, 0, 0, FALSE))
    every_probe = [(p, -1) for p in range(npr)]
    every_build = [(-1, b) for b in range(nb)]
    want = {abi.JOIN_INNER: [], abi.JOIN_LEFT_SEMI: [], abi.JOIN_RIGHT_SEMI: [],
            abi.JOIN_LEFT: every_probe, abi.JOIN_LEFT_ANTI: every_probe,
            abi.JOIN_RIGHT: every_build, abi.JOIN_RIGHT_ANTI: every_build, abi.JOIN_FULL: every_probe + every_build}[kind]
    assert got == sorted(want)


def nested_loop(kind, build, probe, pred):
    """Every (probe, build) pair: equal non-NULL keys and pred(build row, probe row) is True (None = NULL)."""
    nb, npr = build[0].length, probe[0].length
    B = [[(float(c.values()[i]) if c.dtype == abi.F64 else int(c.values()[i])) if c.valid_mask()[i] else None for c in build] for i in range(nb)]
    P = [[int(c.values()[i]) if c.valid_mask()[i] else None for c in probe] for i in range(npr)]
    m = [(p, b) for p in range(npr) for b in range(nb)
         if P[p][0] is not None and B[b][0] is not None and P[p][0] == B[b][0] and pred(B[b], P[p]) is True]
    pm, bm = {p for p, _ in m}, {b for _, b in m}
    un_p = [(p, -1) for p in range(npr) if p not in pm]
    un_b = [(-1, b) for b in range(nb) if b not in bm]
    return sorted({abi.JOIN_INNER: m, abi.JOIN_LEFT: m + un_p, abi.JOIN_LEFT_SEMI: [(p, -1) for p in pm], abi.JOIN_LEFT_ANTI: un_p,
                   abi.JOIN_RIGHT: m + un_b, abi.JOIN_RIGHT_SEMI: [(-1, b) for b in bm], abi.JOIN_RIGHT_ANTI: un_b,
                   abi.JOIN_FULL: m + un_p + un_b}[kind])


@pytest.mark.parametrize("kind", KINDS)
def test_against_nested_loop(kind):
    build, btypes, probe, ptypes = tables(4, n_build=80, n_probe=120, key_range=20)
    # build.x < probe.z AND (build.y > 0 OR build.y IS NULL -> NULL): three-valued, NULL is not a match
    pred = S.call("and", S.call("lt", S.cast(S.col(1), abi.I64), S.col(4)), S.call("gt", S.col(2), S.lit(0.0, abi.F64)))

    def py(b, p):
        lt = b[1] < p[1]
        gt = None if b[2] is None else b[2] > 0.0
        if lt is False or gt is False:
            return False
        return True if (lt and gt) else None
    got = pairs(hash_join_residual(kind, build, btypes, probe, ptypes, 0, 0, pred))
    assert got == nested_loop(kind, build, probe, py)


def _golden():
    with open(os.path.join(HERE, "golden", "join_residual.json")) as f:
        return json.load(f)["cases"]


@pytest.mark.parametrize("case", _golden(), ids=lambda c: c["name"])
def test_reference_sql_cases(case):
    probe, ptypes = golden_table(case["probe"])
    build, btypes = golden_table(case["build"])
    pred = golden_predicate(case["residual"], btypes, ptypes)
    pi, bi = hash_join_residual(GOLDEN_KINDS[case["kind"]], build, btypes, probe, ptypes, case["build_key"], case["probe_key"], pred)
    assert golden_rows(case, pi.tolist(), bi.tolist()) == sort_rows(case["expect"])


def test_create_join_is_exported():
    assert "dbx_op_create_join" in abi.EXPORTS
