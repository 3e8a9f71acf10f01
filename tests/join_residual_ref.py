"""Reference results of hash joins with a residual predicate (HashJoinDesc::other_predicate, the ON clause's
non-equi conditions ANDed and wrapped in is_true: service/src/pipelines/processors/transforms/hash_join/
desc.rs:60-63, 156-190) for the tests, restated from the reference's filtered join streams (paths relative
to service/src/pipelines/processors/transforms/new_hash_join/):

  INNER       memory/inner_join.rs:278-310 (InnerHashJoinFilterStream)   every matching pair
  LEFT        memory/left_join.rs:180-290 (the CONJUNCT stream)          every matching pair; each probe row
                                                                         with none once, build side NULL
  LEFT SEMI   memory/left_join_semi.rs (filtered stream)                 each probe row with a matching pair, once
  LEFT ANTI   memory/left_join_anti.rs:210-310 (LeftAntiFilterHashJoinStream)  each probe row with none,
                                                                         NULL-key rows included
  RIGHT       memory/right_join.rs (filtered stream)                     every matching pair, then the build
                                                                         rows in no matching pair
  RIGHT SEMI / RIGHT ANTI  memory/right_join_semi.rs, right_join_anti.rs the build rows in at least one / in
                                                                         no matching pair
  FULL        LEFT during the probe, then RIGHT's final scan

A candidate pair is a probe row and a build row whose keys are equal (64-bit key images, as in
join_build_side_ref.py; composite keys through join_multi_key_ref.composite_ids); a NULL key has none.  The
predicate is evaluated per candidate pair with conditional_oracle.evaluate over the gathered build and probe
columns (build column c is column c, probe column j is column n_build + j), and is_true makes NULL false: a
matching pair is a candidate pair on which it is true.  The matched map is set by matching pairs only."""
import numpy as np

from databend_b200 import abi
import computed_oracle as co
import conditional_oracle as cond
from join_build_side_ref import _key_words
from join_multi_key_ref import composite_ids


def candidate_pairs(build_keys, probe_keys):
    """All (probe_idx, build_idx) with equal non-NULL keys; build_keys / probe_keys are lists of Columns."""
    if len(build_keys) == 1:
        (bw, bvalid), (pw, pvalid) = _key_words(build_keys[0]), _key_words(probe_keys[0])
    else:
        b, p = composite_ids(build_keys, probe_keys)
        bw, bvalid, pw, pvalid = b.values(), b.valid_mask(), p.values(), p.valid_mask()
    inserted = np.nonzero(bvalid)[0]
    table = inserted[np.argsort(bw[inserted], kind="stable")]
    table_keys = bw[table]
    lo = np.searchsorted(table_keys, pw, side="left")
    hi = np.searchsorted(table_keys, pw, side="right")
    n_match = np.where(pvalid, hi - lo, 0)
    total = int(n_match.sum())
    first = np.cumsum(n_match) - n_match
    probe_idx = np.repeat(np.arange(len(pw), dtype=np.int64), n_match)
    build_idx = table[np.repeat(lo, n_match) + (np.arange(total) - np.repeat(first, n_match))].astype(np.int64)
    return probe_idx, build_idx


def _gathered(cols, types, rows):
    out = []
    for c, t in zip(cols, types):
        vals = c.values()[rows]
        valid = c.valid_mask()[rows] if t & abi.NULLABLE else None
        out.append((co.NAME[t & 0xFF], vals, valid))
    return out


def matching(predicate, build_cols, build_types, probe_cols, probe_types, probe_idx, build_idx):
    """Mask over the candidate pairs: is_true(predicate) on each.  predicate: scalar_expr.SExpr or None (true)."""
    if predicate is None:
        return np.ones(len(probe_idx), dtype=bool)
    if len(probe_idx) == 0:
        return np.zeros(0, dtype=bool)
    cols = _gathered(build_cols, build_types, build_idx) + _gathered(probe_cols, probe_types, probe_idx)
    t, _, vals, oks = cond.evaluate(co.to_tuple(predicate), cols)
    if t != "BOOL":
        raise ValueError("the residual predicate must be Boolean")
    return np.asarray(oks, dtype=bool) & np.asarray(vals, dtype=bool)


def hash_join_residual(kind, build_cols, build_types, probe_cols, probe_types, build_key, probe_key, predicate):
    """(probe_idx, build_idx) int64 arrays of the join with a residual predicate, -1 on the side an output
    row does not carry; row order unspecified.  build_key / probe_key: a column index or a list of them."""
    bkeys = [build_key] if isinstance(build_key, int) else list(build_key)
    pkeys = [probe_key] if isinstance(probe_key, int) else list(probe_key)
    n_build = build_cols[0].length if build_cols else 0
    n_probe = probe_cols[0].length if probe_cols else 0
    cp, cb = candidate_pairs([build_cols[i] for i in bkeys], [probe_cols[i] for i in pkeys])
    m = matching(predicate, build_cols, build_types, probe_cols, probe_types, cp, cb)
    mp, mb = cp[m], cb[m]
    probe_matched = np.zeros(n_probe, dtype=bool)
    probe_matched[mp] = True
    build_matched = np.zeros(n_build, dtype=bool)  # the matched map
    build_matched[mb] = True
    none = lambda n: np.full(n, -1, dtype=np.int64)  # noqa: E731

    def probe_rows(mask):
        r = np.nonzero(mask)[0].astype(np.int64)
        return r, none(len(r))

    def build_rows(mask):
        r = np.nonzero(mask)[0].astype(np.int64)
        return none(len(r)), r

    def cat(*parts):
        return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

    if kind == abi.JOIN_INNER:
        return mp, mb
    if kind == abi.JOIN_LEFT:
        return cat((mp, mb), probe_rows(~probe_matched))
    if kind == abi.JOIN_LEFT_SEMI:
        return probe_rows(probe_matched)
    if kind == abi.JOIN_LEFT_ANTI:
        return probe_rows(~probe_matched)
    if kind == abi.JOIN_RIGHT:
        return cat((mp, mb), build_rows(~build_matched))
    if kind == abi.JOIN_RIGHT_SEMI:
        return build_rows(build_matched)
    if kind == abi.JOIN_RIGHT_ANTI:
        return build_rows(~build_matched)
    if kind == abi.JOIN_FULL:
        return cat((mp, mb), probe_rows(~probe_matched), build_rows(~build_matched))
    raise ValueError(kind)


# ---- tests/golden/join_residual.json
GOLDEN_TYPES = {"Int32": abi.I32, "UInt64": abi.U64, "Int64": abi.I64}
GOLDEN_KINDS = {"INNER": abi.JOIN_INNER, "LEFT": abi.JOIN_LEFT, "LEFT_SEMI": abi.JOIN_LEFT_SEMI, "LEFT_ANTI": abi.JOIN_LEFT_ANTI,
                "RIGHT": abi.JOIN_RIGHT, "RIGHT_SEMI": abi.JOIN_RIGHT_SEMI, "RIGHT_ANTI": abi.JOIN_RIGHT_ANTI, "FULL": abi.JOIN_FULL}
_CMP = {">": "gt", ">=": "gte", "<": "lt", "<=": "lte", "=": "eq", "<>": "noteq"}


def golden_table(t):
    from databend_b200.block import Column
    cols, types = [], []
    for i, ty in enumerate(t["types"]):
        vals = [r[i] for r in t["rows"]]
        valid = np.array([v is not None for v in vals])
        cols.append(Column.from_data(np.array([0 if v is None else v for v in vals], dtype=co.NP[co.NAME[GOLDEN_TYPES[ty]]]),
                                     GOLDEN_TYPES[ty], validity=None if valid.all() else valid))
        types.append(GOLDEN_TYPES[ty] | (0 if valid.all() else abi.NULLABLE))
    return cols, types


def golden_predicate(tree, build_types, probe_types):
    """A golden comparison [op, a, b] as an SExpr over the join schema (build columns, then probe columns); a
    literal takes the type of the column it is compared with."""
    from databend_b200 import scalar_expr as S
    n_build = len(build_types)
    op, a, b = tree

    def side(x):
        return (x[1], build_types[x[1]]) if x[0] == "build" else (n_build + x[1], probe_types[x[1]])

    def operand(x, other):
        if isinstance(x, list):
            return S.col(side(x)[0])
        return S.lit(x, side(other)[1] & 0xFF)
    return S.call(_CMP[op], operand(a, b), operand(b, a))


def golden_rows(case, probe_idx, build_idx):
    """Apply a case's WHERE (a NULL comparison is not true) and SELECT list to joined index pairs; sorted rows."""
    pr, br = case["probe"]["rows"], case["build"]["rows"]
    out = []
    for p, b in zip(probe_idx, build_idx):
        def ref(x):
            if not isinstance(x, list):
                return x
            row = (pr[p] if p >= 0 else None) if x[0] == "probe" else (br[b] if b >= 0 else None)
            return None if row is None else row[x[1]]
        if case["where"] is not None:
            op, a, c = case["where"]
            x, y = ref(a), ref(c)
            if x is None or y is None or not {">": x > y, ">=": x >= y, "<": x < y, "<=": x <= y, "=": x == y, "<>": x != y}[op]:
                continue
        out.append([ref(s) for s in case["select"]])
    return sort_rows(out)


def sort_rows(rows):
    return sorted(rows, key=lambda t: [(v is not None, v if v is not None else 0) for v in t])
