"""Reference results of hash joins on composite keys (ON b.x = p.x AND b.y = p.y ...; the reference's
HashMethodFixedKeys, new_hash_join/hashtable/fixed_keys.rs), reduced to the single-key references
the suite already pins:

  1. every key tuple on both sides gets a dense Int64 id by VALUE (Int16 -1 equals Int64 -1, UInt16
     65535 differs from Int32 -1), so equal tuples and only equal tuples share an id;
  2. a tuple with a NULL in any component gets a NULL id (such a row never matches);
  3. the ids are joined with oracle.hash_join (INNER, LEFT SEMI / ANTI, LEFT) or
     join_build_side_ref.hash_join_build_side (RIGHT, RIGHT SEMI / ANTI, FULL).

Values are compared as the pair (v >> 63, v & (2^63 - 1)), which identifies every integer in
[-2^63, 2^64) and so compares signed and unsigned columns of any width by value."""
import numpy as np

from databend_b200 import abi
from databend_b200.block import Column
from join_build_side_ref import hash_join_build_side

_LOW63 = np.int64(0x7FFFFFFFFFFFFFFF)


def _value_words(col):
    """(q, r) per row with value = q * 2^63 + r; unsigned 64-bit values >= 2^63 get q = 1."""
    v = col.values()
    if v.dtype.kind == "u":
        u = v.astype(np.uint64)
        return (u >> np.uint64(63)).astype(np.int64), (u & np.uint64(0x7FFFFFFFFFFFFFFF)).astype(np.int64)
    s = v.astype(np.int64)
    return s >> 63, s & _LOW63


def composite_ids(build_keys, probe_keys):
    """build_keys / probe_keys: equally long lists of key Columns.  Returns (build id Column, probe id
    Column): Int64, NULL where any component is NULL, equal exactly where the tuples are equal by value."""
    assert len(build_keys) == len(probe_keys) >= 1
    nb, npr = build_keys[0].length, probe_keys[0].length
    words, valid = [], np.ones(nb + npr, dtype=bool)
    for bc, pc in zip(build_keys, probe_keys):
        (bq, br), (pq, pr) = _value_words(bc), _value_words(pc)
        words += [np.concatenate([bq, pq]), np.concatenate([br, pr])]
        valid &= np.concatenate([bc.valid_mask(), pc.valid_mask()])
    if nb + npr:
        _, ids = np.unique(np.stack(words, axis=1), axis=0, return_inverse=True)
        ids = ids.reshape(-1).astype(np.int64)
    else:
        ids = np.zeros(0, dtype=np.int64)
    return (Column.from_data(ids[:nb], validity=valid[:nb]), Column.from_data(ids[nb:], validity=valid[nb:]))


GOLDEN_TYPES = {"Int32": abi.I32, "UInt64": abi.U64, "Int64": abi.I64}


def golden_table(t):
    """A table of tests/golden/join_multi_key.json as a list of Columns."""
    cols = []
    for i, ty in enumerate(t["types"]):
        vals = [r[i] for r in t["rows"]]
        valid = np.array([v is not None for v in vals])
        cols.append(Column.from_data([0 if v is None else v for v in vals], GOLDEN_TYPES[ty], validity=None if valid.all() else valid))
    return cols


def golden_result(query, rows):
    """Apply a golden query's WHERE and SELECT list to joined rows [(probe tuple, build tuple)] (None =
    NULL; a NULL comparison is not true) and return the sorted result rows."""
    def ref(r, x):
        return r[0 if x[0] == "probe" else 1][x[1]] if isinstance(x, list) else x
    side, col, op, rhs = query["where"]
    out = []
    for r in rows:
        a, b = ref(r, [side, col]), ref(r, rhs)
        if a is None or b is None or not {">": a > b, ">=": a >= b}[op]:
            continue
        out.append([ref(r, s) for s in query["select"]])
    return sort_rows(out)


def sort_rows(rows):
    """Result rows in one order (NULL first in each column), for comparing as multisets."""
    return sorted(rows, key=lambda t: [(v is not None, v if v is not None else 0) for v in t])


def hash_join_multi_key(kind: int, build_keys, probe_keys):
    """(probe_idx, build_idx) int64 arrays of the composite-key join, -1 on the side an output row
    does not carry; row order unspecified."""
    from oracle import oracle as orc
    b, p = composite_ids(build_keys, probe_keys)
    if kind in (abi.JOIN_INNER, abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI, abi.JOIN_LEFT):
        return orc.hash_join(kind, b, p)
    return hash_join_build_side(kind, b, p)
