"""The build-side ("right") join kinds restated from right_join.rs / right_join_semi.rs /
right_join_anti.rs (a scan_map set during the probe walk, then a scan over every build row;
tests/join_build_side_ref.py) agree with the derivation from the C oracle's INNER pairs, and
reproduce the reference's SQL tests with the right child as the build side.  Also pins the C-ABI
additions.  No GPU needed."""
import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column
from join_build_side_ref import derive_build_side_join_rows, hash_join_build_side
from oracle import oracle as orc

KINDS = {"right": abi.JOIN_RIGHT, "right_semi": abi.JOIN_RIGHT_SEMI, "right_anti": abi.JOIN_RIGHT_ANTI, "full": abi.JOIN_FULL}


def _key(t):
    return (-1 if t[0] is None else t[0], -1 if t[1] is None else t[1])


@pytest.mark.parametrize("seed", [3, 11])
def test_oracle_build_side_kinds_agree_with_the_derivation(seed):
    """Random nullable keys on both sides, duplicate build keys, misses on both sides."""
    rng = np.random.default_rng(seed)
    nb, npr = 2000, 5000
    build = Column.from_data(rng.integers(0, 600, nb).astype(np.int64), validity=rng.random(nb) > 0.1)
    probe = Column.from_data(rng.integers(-50, 400, npr).astype(np.int64), validity=rng.random(npr) > 0.1)
    pairs = orc.hash_join_inner(build, probe)
    for name, kind in KINDS.items():
        p, b = hash_join_build_side(kind, build, probe)
        got = [((None if x < 0 else int(x)), (None if y < 0 else int(y))) for x, y in zip(p, b)]
        exp = derive_build_side_join_rows(name, npr, nb, pairs)
        assert sorted(got, key=_key) == sorted(exp, key=_key), name
    # a NULL-key build row is never matched: RIGHT / ANTI / FULL emit it, SEMI never does
    null_rows = set(np.nonzero(~build.valid_mask())[0].tolist())
    assert null_rows
    for name, kind in KINDS.items():
        final = {int(y) for x, y in zip(*hash_join_build_side(kind, build, probe)) if x < 0}
        assert (null_rows <= final) if name != "right_semi" else not (null_rows & final), name
    # duplicate build keys: RIGHT SEMI emits each matched build row once
    _, b = hash_join_build_side(abi.JOIN_RIGHT_SEMI, build, probe)
    assert len(b) == len(set(b.tolist()))


def _rows(kind, probe_cols, build_cols, pk=0, bk=0):
    """Output rows as tuples (probe columns then build columns; build columns only for SEMI / ANTI),
    None for NULL, sorted."""
    p, b = hash_join_build_side(KINDS[kind], build_cols[bk], probe_cols[pk])

    def val(c, i):
        return c.values()[i].item() if i >= 0 and c.valid_mask()[i] else None
    rows = []
    for x, y in zip(p, b):
        r = [] if kind in ("right_semi", "right_anti") else [val(c, x) for c in probe_cols]
        rows.append(tuple(r + [val(c, y) for c in build_cols]))
    return sorted(rows, key=lambda t: tuple((v is not None, v if v is not None else 0) for v in t))


def test_goldens_from_the_reference_sql_tests():
    I32 = abi.I32
    # left_outer.test:20-25  select * from t1 right join t2 on t1.a = t2.c
    t1 = [Column.from_data([1, 3, 7], I32), Column.from_data([2, 4, 8], I32)]
    t2 = [Column.from_data([1, 2, 6], I32), Column.from_data([4, 3, 8], I32)]
    assert _rows("right", t1, t2) == [(None, None, 2, 3), (None, None, 6, 8), (1, 2, 1, 4)]
    # right_outer.test:22-29  numbers(10) x right join numbers(5) y using(a): a = 0..4
    n10, n5, n1000 = (Column.from_data(np.arange(n, dtype=np.uint64)) for n in (10, 5, 1000))
    assert _rows("right", [n10], [n5]) == [(i, i) for i in range(5)]
    # right_outer.test:31-38  numbers(1000) x right join numbers(5) y on x.a = y.a
    assert _rows("right", [n1000], [n5]) == [(i, i) for i in range(5)]
    # join.test:7-25  right / right semi / right anti join against an empty build side: empty
    n100 = Column.from_data(np.arange(100, dtype=np.uint64))
    empty = Column.from_data(np.zeros(0, dtype=np.int32))
    for kind in ("right", "right_semi", "right_anti"):
        assert _rows(kind, [n100], [empty]) == [], kind
    # join.test:89-102  full join against an empty build side: every probe row, NULL build side
    assert _rows("full", [n10], [empty]) == [(i, None) for i in range(10)]
    # join.test:287-299  full outer join, then keep the rows whose `t` side is not NULL
    # ('A' stands in as the non-NULL marker column 65: string columns are out of scope)
    t = [Column.from_data([1, 2, 3], I32), Column.from_data([65, 65, 65], I32)]
    n5 = [Column.from_data(np.arange(5, dtype=np.uint64))]
    rows = [r for r in _rows("full", t, n5) if r[1] is not None]          # t1 full outer join t2 (t2 = build)
    assert rows == [(1, 65, 1), (2, 65, 2), (3, 65, 3)]
    rows = [r for r in _rows("full", n5, t) if r[2] is not None]          # t2 full outer join t1 (t1 = build)
    assert rows == [(1, 1, 65), (2, 2, 65), (3, 3, 65)]
    # the rows the filter drops: the unmatched side of both directions
    assert [r for r in _rows("full", t, n5) if r[1] is None] == [(None, None, 0), (None, None, 4)]
    assert [r for r in _rows("full", n5, t) if r[2] is None] == [(0, None, None), (4, None, None)]


def test_abi_pins_the_build_side_kinds_and_final_probe():
    import os
    import re
    assert (abi.JOIN_RIGHT, abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI, abi.JOIN_FULL) == (4, 5, 6, 7)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "dbx.h")) as f:
        header = f.read()
    for name, v in (("RIGHT", 4), ("RIGHT_SEMI", 5), ("RIGHT_ANTI", 6), ("FULL", 7)):
        assert re.search(rf"\bDBX_JOIN_{name} = {v}\b", header), name
    assert re.search(r"^int32_t dbx_join_final_probe\(dbx_op\* op\);", header, flags=re.M)
    assert "dbx_join_final_probe" in abi.EXPORTS
    from databend_b200 import build, lib
    build.build()
    assert hasattr(lib.load(), "dbx_join_final_probe")
