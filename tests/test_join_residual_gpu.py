"""Hash joins with a residual predicate (dbx_op_create_join, HashJoinDesc::other_predicate) on the device
against tests/join_residual_ref.py, compared as multisets of rows (values bit for bit, NULL as None): all
eight kinds, single and composite keys, unique and duplicate build keys, every source a build slot reads
from, NULLs, floats, conditionals, the block / reset / out_mem lifecycle, runtime filters, the TPC-H Q21
shape and the refusals."""
import ctypes as C

import numpy as np
import pytest

from databend_b200 import abi, expr as E, scalar_expr as S
from databend_b200.block import Column, DataBlock
from databend_b200.lib import DbxError, check, load
from databend_b200.transforms import HashJoin, TransformFilter, schema_types, to_device
from join_residual_ref import hash_join_residual

pytestmark = pytest.mark.gpu

KINDS = {"inner": abi.JOIN_INNER, "left_semi": abi.JOIN_LEFT_SEMI, "left_anti": abi.JOIN_LEFT_ANTI, "left": abi.JOIN_LEFT,
         "right": abi.JOIN_RIGHT, "right_semi": abi.JOIN_RIGHT_SEMI, "right_anti": abi.JOIN_RIGHT_ANTI, "full": abi.JOIN_FULL}
PROBE_ONLY = (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI)
BUILD_ONLY = (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI)
NP = {abi.I8: np.int8, abi.I16: np.int16, abi.I32: np.int32, abi.I64: np.int64, abi.U8: np.uint8, abi.U16: np.uint16,
      abi.U32: np.uint32, abi.U64: np.uint64, abi.F32: np.float32, abi.F64: np.float64}


def _bits(vals):
    """Values as Python ints, floats by their bit pattern (NaN payloads and -0.0 compare exactly)."""
    v = np.asarray(vals)
    if v.dtype == np.float64:
        v = v.view(np.int64)
    elif v.dtype == np.float32:
        v = v.view(np.int32)
    return v.tolist()


def rows_of(cols):
    """[(values, valid)] per column -> sorted list of row tuples, None for NULL."""
    if not cols:
        return []
    per = [[x if ok else None for x, ok in zip(_bits(v), m.tolist())] for v, m in cols]
    rows = list(zip(*per))
    return sorted(rows, key=lambda t: [(x is not None, x if x is not None else 0) for x in t])


def take(col, idx):
    v, m = col.values(), col.valid_mask()
    if len(v) == 0:
        return np.zeros(len(idx), dtype=v.dtype), np.zeros(len(idx), dtype=bool)
    return v[np.maximum(idx, 0)], m[np.maximum(idx, 0)] & (idx >= 0)


def expected(kind, build, probe, bk, pk, pred):
    pi, bi = hash_join_residual(kind, build.columns, schema_types(build), probe.columns, schema_types(probe), bk, pk, pred)
    cols = [] if kind in BUILD_ONLY else [take(c, pi) for c in probe.columns]
    if kind not in PROBE_ONLY:
        cols += [take(c, bi) for c in build.columns]
    return rows_of(cols)


def host_rows(blocks):
    if not blocks:
        return []
    n = blocks[0].num_columns()
    return rows_of([(np.concatenate([b.columns[i].values() for b in blocks]), np.concatenate([b.columns[i].valid_mask() for b in blocks]))
                    for i in range(n)])


def device_rows(blocks, dtypes):
    """Rows of library-owned device blocks (copied out, then released)."""
    L = load()
    cols = [([], []) for _ in dtypes]
    for b in blocks:
        n = b.num_rows
        for i, dt in enumerate(dtypes):
            c = b.cols[i]
            if c.is_const:
                assert c.konst.is_null
                cols[i][0].append(np.zeros(n, NP[dt]))
                cols[i][1].append(np.zeros(n, bool))
                continue
            assert c.mem == abi.MEM_DEVICE
            v = np.empty(n, NP[dt])
            if n:
                check(L.dbx_memcpy_d2h(0, v.ctypes.data, c.data, v.nbytes))
            m = np.ones(n, bool)
            if c.validity and n:
                bits = np.empty((n + 7) // 8, np.uint8)
                check(L.dbx_memcpy_d2h(0, bits.ctypes.data, c.validity, bits.nbytes))
                m = np.unpackbits(bits, bitorder="little")[:n].astype(bool)
            cols[i][0].append(v)
            cols[i][1].append(m)
        check(L.dbx_block_release(C.byref(b)))
    return rows_of([(np.concatenate(v), np.concatenate(m)) for v, m in cols]) if blocks else []


def out_dtypes(kind, build, probe):
    d = [] if kind in BUILD_ONLY else [c.dtype for c in probe.columns]
    return d + ([] if kind in PROBE_ONLY else [c.dtype for c in build.columns])


def run(kind, build, probe, bk, pk, pred, split=None, out_mem=abi.MEM_HOST, device_probe=False, rounds=1):
    j = HashJoin(schema_types(build), schema_types(probe), bk, pk, kind=kind, other_predicate=pred)
    results = []
    for _ in range(rounds):
        j.reset()
        if build.num_rows:
            j.add_block(build)
        j.final_build()
        outs = []
        for p in (probe.split_by_rows(split) if split else [probe]):
            if device_probe:
                p = DataBlock([to_device(c) for c in p.columns], p.num_rows)
            outs += j.probe_block(p, out_mem)
        outs += j.final_probe(out_mem)
        results.append(device_rows(outs, out_dtypes(kind, build, probe)) if out_mem == abi.MEM_DEVICE else host_rows(outs))
    j.close()
    return results if rounds > 1 else results[0]


def check_join(kind, build, probe, bk, pk, pred, **kw):
    want = expected(kind, build, probe, bk, pk, pred)
    got = run(kind, build, probe, bk, pk, pred, **kw)
    if isinstance(got, list) and got and isinstance(got[0], list):
        for g in got:
            assert g == want
    else:
        assert got == want
    return want


# ---------------------------------------------------------------- data
def single_key_tables(seed, nb=3000, npr=5000, span=2000, unique=False):
    """build: k I64 (nullable), x I32 (-> p0), y F64 nullable (-> p1), w I64 nullable (gathered);
    probe: k I64 nullable, z I64, f F64 nullable."""
    rng = np.random.default_rng(seed)
    bk = rng.permutation(span)[:nb] if unique else rng.integers(0, span, nb)
    build = DataBlock([Column.from_data(bk.astype(np.int64), validity=rng.random(nb) > 0.05),
                       Column.from_data(rng.integers(-100, 100, nb).astype(np.int32)),
                       Column.from_data(rng.standard_normal(nb), validity=rng.random(nb) > 0.1),
                       Column.from_data(rng.integers(-100, 100, nb).astype(np.int64), validity=rng.random(nb) > 0.2)])
    probe = DataBlock([Column.from_data(rng.integers(-10, span + 10, npr).astype(np.int64), validity=rng.random(npr) > 0.05),
                       Column.from_data(rng.integers(-100, 100, npr).astype(np.int64)),
                       Column.from_data(rng.standard_normal(npr), validity=rng.random(npr) > 0.1)])
    return build, probe


NB = 4  # build columns of single_key_tables: probe column j is NB + j


def both_sides_pred():
    """(b.x < p.z OR b.w > p.z) AND (b.y <= p.f OR b.k >= 1000): every build source (key, p0, p1, gather)."""
    return S.call("and",
                  S.call("or", S.call("lt", S.cast(S.col(1), abi.I64), S.col(NB + 1)), S.call("gt", S.col(3), S.col(NB + 1))),
                  S.call("or", S.call("lte", S.col(2), S.col(NB + 2)), S.call("gte", S.col(0), S.lit(1000, abi.I64))))


PREDS = {
    "both": both_sides_pred,
    "probe_only": lambda: S.call("gt", S.col(NB + 1), S.lit(0, abi.I64)),
    "build_only": lambda: S.call("lt", S.col(1), S.lit(20, abi.I32)),
}


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("unique", [False, True], ids=["dup", "unique"])
def test_single_key_every_kind(gpu, kind, unique):
    build, probe = single_key_tables(1 + unique, span=4000 if unique else 2000, unique=unique)
    check_join(KINDS[kind], build, probe, 0, 0, both_sides_pred())


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("side", ["probe_only", "build_only"])
def test_one_side_predicates(gpu, kind, side):
    build, probe = single_key_tables(3)
    check_join(KINDS[kind], build, probe, 0, 0, PREDS[side]())


def composite_tables(seed, wide, nb=3000, npr=4000):
    """Keys (a, b): (I32, I16) packs into 64 bits, (I64, I32) into 128; one more build column c (p0)."""
    rng = np.random.default_rng(seed)
    ta, tb = (np.int64, np.int32) if wide else (np.int32, np.int16)
    build = DataBlock([Column.from_data(rng.integers(0, 40, nb).astype(ta), validity=rng.random(nb) > 0.05),
                       Column.from_data(rng.integers(-20, 20, nb).astype(tb)),
                       Column.from_data(rng.integers(-50, 50, nb).astype(np.int64), validity=rng.random(nb) > 0.1)])
    probe = DataBlock([Column.from_data(rng.integers(0, 42, npr).astype(ta)),
                       Column.from_data(rng.integers(-20, 20, npr).astype(tb), validity=rng.random(npr) > 0.05),
                       Column.from_data(rng.integers(-50, 50, npr).astype(np.int64))])
    return build, probe


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("wide", [False, True], ids=["64bit", "128bit"])
def test_composite_keys(gpu, kind, wide):
    build, probe = composite_tables(5 + wide, wide)
    # b.c < p.c AND b.b (a packed key field) <> 3 AND b.a (the other field) >= 2
    pred = S.call("and", S.call("and", S.call("lt", S.col(2), S.col(3 + 2)), S.call("noteq", S.col(1), S.lit(3, abi.I32 if wide else abi.I16))),
                  S.call("gte", S.col(0), S.lit(2, abi.I64 if wide else abi.I32)))
    check_join(KINDS[kind], build, probe, [0, 1], [0, 1], pred)


@pytest.mark.parametrize("kind", ["inner", "left", "right", "full"])
def test_many_to_many_takes_the_retry(gpu, kind):
    # ~60 build rows per key: ~60k candidate pairs, about half match: far beyond the probe's first out_cap
    rng = np.random.default_rng(7)
    nb, npr = 600, 1000
    build = DataBlock([Column.from_data(rng.integers(0, 10, nb).astype(np.int64)), Column.from_data(rng.integers(0, 100, nb).astype(np.int64))])
    probe = DataBlock([Column.from_data(rng.integers(0, 11, npr).astype(np.int64)), Column.from_data(rng.integers(0, 100, npr).astype(np.int64))])
    want = check_join(KINDS[kind], build, probe, 0, 0, S.call("lt", S.col(1), S.col(2 + 1)))
    assert len(want) > npr + npr // 8 + 1024


def float_tables():
    specials = [np.nan, -0.0, 0.0, 1.0, -1.0, np.inf, -np.inf, 2.5]
    rng = np.random.default_rng(11)
    nb, npr = 400, 600
    build = DataBlock([Column.from_data(rng.integers(0, 30, nb).astype(np.int32)),
                       Column.from_data(np.array(specials, np.float32)[rng.integers(0, 8, nb)], validity=rng.random(nb) > 0.1),
                       Column.from_data(np.array(specials)[rng.integers(0, 8, nb)])])
    probe = DataBlock([Column.from_data(rng.integers(0, 30, npr).astype(np.int32)),
                       Column.from_data(np.array(specials)[rng.integers(0, 8, npr)], validity=rng.random(npr) > 0.1),
                       Column.from_data(np.array(specials, np.float32)[rng.integers(0, 8, npr)])])
    return build, probe


@pytest.mark.parametrize("cmp", ["eq", "lt", "gte", "noteq"])
@pytest.mark.parametrize("kind", ["inner", "left_anti", "right_semi", "full"])
def test_float_compare_nan_and_signed_zero(gpu, kind, cmp):
    build, probe = float_tables()
    # cast(b.f32, F64) <cmp> p.f64 OR b.f64 <cmp> cast(p.f32, F64): OrderedFloat, NaN == NaN, -0 == +0
    pred = S.call("or", S.call(cmp, S.cast(S.col(1), abi.F64), S.col(3 + 1)), S.call(cmp, S.col(2), S.cast(S.col(3 + 2), abi.F64)))
    check_join(KINDS[kind], build, probe, 0, 0, pred)


@pytest.mark.parametrize("kind", ["inner", "left", "left_semi", "right_anti"])
def test_three_valued_logic_if_and_coalesce(gpu, kind):
    build, probe = single_key_tables(13, nb=1500, npr=2500)
    coal = S.call("gt", S.coalesce(S.col(3), S.col(NB + 1), dtype=abi.I64), S.lit(10, abi.I64))
    branch = S.if_(S.call("is_null", S.col(2)), S.call("gt", S.col(NB + 1), S.lit(0, abi.I64)), S.call("lt", S.col(2), S.col(NB + 2)))
    nullable_or = S.call("or", S.call("gt", S.col(2), S.col(NB + 2)), S.call("lt", S.col(3), S.lit(0, abi.I64)))
    check_join(KINDS[kind], build, probe, 0, 0, S.call("or", S.call("and", coal, branch), nullable_or))


@pytest.mark.parametrize("kind", list(KINDS))
def test_blocks_reset_device_output_and_empty_build(gpu, kind):
    build, probe = single_key_tables(17, nb=2000, npr=6000)
    pred = both_sides_pred()
    want = expected(KINDS[kind], build, probe, 0, 0, pred)
    # several probe blocks (device resident), then final_probe; reset and reuse keep the predicate
    for got in run(KINDS[kind], build, probe, 0, 0, pred, split=1000, device_probe=True, rounds=2):
        assert got == want
    assert run(KINDS[kind], build, probe, 0, 0, pred, split=2500, out_mem=abi.MEM_DEVICE) == want
    empty = DataBlock([Column.from_data(np.zeros(0, c.values().dtype), validity=np.zeros(0, bool) if c.validity is not None else None)
                       for c in build.columns], 0)
    assert run(KINDS[kind], empty, probe, 0, 0, pred, split=2500) == expected(KINDS[kind], empty, probe, 0, 0, pred)


def filtered(f, block, pk, types):
    mask = f.apply(block, pk)
    op = TransformFilter(E.bool_column(len(block.columns)), list(types) + [abi.BOOL])
    out = op.transform(DataBlock(block.columns + [mask], block.num_rows))
    op.close()
    return DataBlock(out.columns[:-1], out.num_rows)


@pytest.mark.parametrize("kind", ["inner", "left_semi", "right", "right_semi", "right_anti"])
@pytest.mark.parametrize("mode", ["apply", "in_probe"])
def test_runtime_filter(gpu, kind, mode):
    build, probe = single_key_tables(19, nb=500, npr=6000, span=20000)
    pred = both_sides_pred()
    ptypes = schema_types(probe)
    j = HashJoin(schema_types(build), ptypes, 0, 0, kind=KINDS[kind], other_predicate=pred)
    j.add_block(build)
    j.final_build()
    f = j.runtime_filter(in_probe=mode == "in_probe", build_table_rows=100 * build.num_rows)
    outs = []
    for p in probe.split_by_rows(2000):
        if mode == "apply":
            p = filtered(f, p, [0], ptypes)
            if p.num_rows == 0:
                continue
        outs += j.probe_block(p)
    outs += j.final_probe()
    info = f.info()
    f.close()
    j.close()
    assert host_rows(outs) == expected(KINDS[kind], build, probe, 0, 0, pred)
    assert (info.apply_rows_rejected if mode == "apply" else info.probe_rows_rejected) > 0


@pytest.mark.parametrize("kind", ["left_semi", "left_anti", "right_semi", "right_anti"])
def test_q21_semi_and_anti_with_noteq(gpu, kind):
    """EXISTS / NOT EXISTS (l2.l_orderkey = l1.l_orderkey AND l2.l_suppkey <> l1.l_suppkey): the build side
    (l2) has several lines per order, some orders a single supplier."""
    rng = np.random.default_rng(23)
    nb, npr = 8000, 6000
    orders = rng.integers(0, 2000, nb).astype(np.int64)
    supp = np.where(orders % 5 == 0, orders % 7, rng.integers(0, 7, nb)).astype(np.int32)  # every fifth order: one supplier
    build = DataBlock([Column.from_data(orders), Column.from_data(supp)])
    p_orders = rng.integers(0, 2100, npr).astype(np.int64)
    probe = DataBlock([Column.from_data(p_orders), Column.from_data(np.where(p_orders % 5 == 0, p_orders % 7, rng.integers(0, 7, npr)).astype(np.int32))])
    pred = S.call("noteq", S.col(1), S.col(2 + 1))
    want = check_join(KINDS[kind], build, probe, 0, 0, pred)
    assert 0 < len(want)


# ---------------------------------------------------------------- refusals
def _create(pred, build_types, probe_types, kind=abi.JOIN_INNER):
    p = abi.JoinParams()
    p.kind, p.build_key_col, p.probe_key_col, p.n_build_cols = kind, 0, 0, len(build_types)
    types = list(build_types) + list(probe_types)
    arr = (C.c_int32 * len(types))(*types)
    h = C.c_void_p()
    e = S.flatten(pred)
    st = load().dbx_op_create_join(C.byref(p), arr, len(types), C.byref(e), 0, C.byref(h))
    msg = (load().dbx_last_error(None) or b"").decode()
    if h:
        load().dbx_op_destroy(h)
    return st, msg


def test_refusals(gpu):
    bt, pt = [abi.I64] * 5, [abi.I64] * 5
    st, msg = _create(S.call("plus", S.col(1), S.col(6)), bt, pt)
    assert st == abi.ERR_INVALID and "Boolean" in msg
    st, msg = _create(S.call("gt", S.col(1), S.col(10)), bt, pt)
    assert st == abi.ERR_INVALID and "outside" in msg
    st, msg = _create(S.call("gt", S.col(1) / S.col(6), S.lit(1.0, abi.F64)), bt, pt)
    assert st == abi.ERR_UNSUPPORTED and "raise" in msg
    nine = S.call("gt", S.col(0), S.col(9))
    for c in range(1, 8):
        nine = S.call("and", nine, S.call("gt", S.col(c), S.lit(0, abi.I64)))
    st, msg = _create(nine, bt, pt)
    assert st == abi.ERR_UNSUPPORTED and "8" in msg
    # eight distinct columns fit; a nullable-Boolean result is accepted
    eight = S.call("gt", S.col(0), S.col(9))
    for c in range(1, 7):
        eight = S.call("and", eight, S.call("gt", S.col(c), S.lit(0, abi.I64)))
    assert _create(eight, bt, pt)[0] == abi.OK
    assert _create(S.call("gt", S.col(1), S.col(3)), [abi.I64, abi.I64 | abi.NULLABLE], [abi.I64, abi.I64])[0] == abi.OK
    # the Python wrapper raises with the library's message; create_computed still refuses joins
    with pytest.raises(DbxError):
        HashJoin([abi.I64, abi.I64], [abi.I64, abi.I64], 0, 0, other_predicate=S.call("plus", S.col(1), S.col(3)))
    p = abi.JoinParams()
    p.kind, p.n_build_cols = abi.JOIN_INNER, 1
    types = (C.c_int32 * 2)(abi.I64, abi.I64)
    comp = (abi.Expr * 1)(S.flatten(S.col(0)))
    h = C.c_void_p()
    assert load().dbx_op_create_computed(abi.OP_JOIN, C.cast(C.byref(p), C.c_void_p), types, 2, comp, 1, 0, C.byref(h)) == abi.ERR_UNSUPPORTED
    # no predicate (NULL or zero nodes) is the plain join
    p = abi.JoinParams()
    p.kind, p.n_build_cols = abi.JOIN_INNER, 1
    assert load().dbx_op_create_join(C.byref(p), types, 2, None, 0, C.byref(h)) == abi.OK
    load().dbx_op_destroy(h)
