"""The sorting join reference of tests/join_scale_ref.py is the C oracle's join, its verifier rejects
wrong outputs, and its slot construction builds the table runs the GPU tests rely on.  No GPU needed.

  * `JoinRef` against `oracle.hash_join` (INNER, LEFT, LEFT SEMI, LEFT ANTI) and `join_build_side_ref`
    (RIGHT, RIGHT SEMI, RIGHT ANTI, FULL), on random keys of mixed dtypes with NULLs, duplicates and
    misses, probed in several blocks;
  * the verifier accepts the reference's own output and rejects each single corruption of it;
  * keys computed for chosen home slots hash there, and a simulation of linear-probing insertion shows
    that the constructed runs cross slot cap - 1 -> 0 and hold many distinct keys."""
import numpy as np
import pytest
import torch

import join_scale_ref as R
from databend_b200 import abi
from databend_b200.block import Column
from join_build_side_ref import hash_join_build_side
from oracle import oracle as orc

DEV = "cpu"
PAIRS = [(abi.I64, abi.I64), (abi.I32, abi.I64), (abi.U16, abi.I32), (abi.U8, abi.I8), (abi.U64, abi.U32), (abi.I16, abi.U16)]


def random_key(dtype, n, rng, nvals):
    """Keys from a small range around 0 (duplicates and cross-type matches) plus the type's extremes."""
    nd = np.dtype(R.NP_DTYPE[dtype])
    info = np.iinfo(nd)
    lo = max(int(info.min), -nvals // 2)
    x = rng.integers(lo, min(lo + nvals, int(info.max) + 1), n).astype(nd)
    ext = rng.random(n) < 0.05
    x[ext] = rng.choice(np.array([info.min, info.max, -1 if info.min < 0 else 255], dtype=nd), int(ext.sum()))
    return x


def side(values, valid, dtype, tag_base=0):
    """Key column and tag column as a Side, plus the key as a host Column for the oracles."""
    n = len(values)
    key = R.Col(torch.from_numpy(np.ascontiguousarray(values).view(f"i{values.itemsize}")), dtype, torch.from_numpy(valid))
    tag = R.Col(torch.arange(tag_base, tag_base + n, dtype=torch.int64), abi.I64)
    return R.Side([key, tag], [0], 1, tag_base), Column.from_data(values, dtype, validity=valid)


def case(seed, bt, pt, nb=3000, npr=7000):
    rng = np.random.default_rng(seed)
    bv = random_key(bt, nb, rng, 900)
    pv = random_key(pt, npr, rng, 1200)
    bvalid, pvalid = rng.random(nb) > 0.08, rng.random(npr) > 0.08
    return (bv, bvalid), (pv, pvalid)


def ref_blocks(build: R.Side, pv, pvalid, pt, cuts):
    """Probe the reference in blocks; returns the JoinRef and per block (Side, lo, cnt)."""
    ref = R.JoinRef(build.key_images()[0], build.cols[0].valid)
    out = []
    for s, e in zip(cuts[:-1], cuts[1:]):
        ps, _ = side(pv[s:e], pvalid[s:e], pt, s)
        lo, cnt = ref.probe(ps.key_images()[0], ps.cols[0].valid)
        out.append((ps, lo, cnt))
    return ref, out


def _pairs_set(p, b):
    return sorted(zip(p.tolist(), b.tolist()))


@pytest.mark.parametrize("bt,pt", PAIRS)
@pytest.mark.parametrize("seed", [1, 2])
def test_reference_is_the_oracle_join(seed, bt, pt):
    (bv, bvalid), (pv, pvalid) = case(seed, bt, pt)
    build, bcol = side(bv, bvalid, bt)
    _, pcol = side(pv, pvalid, pt)
    cuts = [0, 1, 2500, 2501, len(pv)]
    ref, blocks = ref_blocks(build, pv, pvalid, pt, cuts)
    # probe-side kinds: the reference's pairs per block, in global probe rows
    ps, bs, cnts = [], [], []
    for s, (psd, lo, cnt) in zip(cuts, blocks):
        p, b = ref.pairs(lo, cnt)
        ps.append(p + s)
        bs.append(b)
        cnts.append(cnt)
    p, b, cnt = torch.cat(ps), torch.cat(bs), torch.cat(cnts)
    assert int(cnt.sum()) > 1000 and int((cnt > 1).sum()) > 100 and int((cnt == 0).sum()) > 100
    op, ob = orc.hash_join(abi.JOIN_INNER, bcol, pcol)
    assert _pairs_set(p, b) == _pairs_set(torch.from_numpy(op), torch.from_numpy(ob))
    op, ob = orc.hash_join(abi.JOIN_LEFT, bcol, pcol)
    un = (cnt == 0).nonzero().flatten()
    assert _pairs_set(torch.cat([p, un]), torch.cat([b, torch.full_like(un, -1)])) == _pairs_set(torch.from_numpy(op), torch.from_numpy(ob))
    for kind, sel in ((abi.JOIN_LEFT_SEMI, cnt > 0), (abi.JOIN_LEFT_ANTI, cnt == 0)):
        op, _ = orc.hash_join(kind, bcol, pcol)
        assert sorted(op.tolist()) == sel.nonzero().flatten().tolist(), R.KIND_NAMES[kind]
    # build-side kinds: the matched map accumulated over the blocks selects final_probe's rows
    m = ref.matched()
    assert int((~m).sum()) > 100 and int(m.sum()) > 100
    for kind in R.BUILD_SIDE_KINDS:
        hp, hb = hash_join_build_side(kind, bcol, pcol)
        final = np.sort(hb[hp < 0])
        if kind == abi.JOIN_FULL:  # FULL's unmatched probe rows carry build -1 too: keep the build rows only
            final = np.sort(hb[(hp < 0) & (hb >= 0)])
        exp = (m if kind == abi.JOIN_RIGHT_SEMI else ~m).nonzero().flatten().numpy()
        assert np.array_equal(final, exp), R.KIND_NAMES[kind]


# ---------------------------------------------------------------- the verifier rejects corruptions
def payload_case(seed=5):
    """Build: key (I32, nullable), btag (I64), F64 nullable, I16 nullable.  Probe: key (I64, nullable), ptag."""
    rng = np.random.default_rng(seed)
    nb, npr = 400, 900
    bkey = rng.integers(0, 150, nb).astype(np.int32)
    pkey = rng.integers(-20, 180, npr).astype(np.int64)
    bcols = [R.Col(torch.from_numpy(bkey), abi.I32, torch.from_numpy(rng.random(nb) > 0.1)),
             R.Col(torch.arange(nb, dtype=torch.int64), abi.I64),
             R.Col(torch.from_numpy(rng.standard_normal(nb)).view(torch.int64), abi.F64, torch.from_numpy(rng.random(nb) > 0.3)),
             R.Col(torch.from_numpy(rng.integers(-999, 999, nb).astype(np.int16)), abi.I16, torch.from_numpy(rng.random(nb) > 0.3))]
    pcols = [R.Col(torch.from_numpy(pkey), abi.I64, torch.from_numpy(rng.random(npr) > 0.1)),
             R.Col(torch.arange(npr, dtype=torch.int64), abi.I64)]
    return R.Side(bcols, [0], 1), R.Side(pcols, [0], 1)


def correct_output(kind, build, probe, lo, cnt, ref):
    """The output a correct join emits for the probe block, built from the reference's pairs."""
    p, b = ref.pairs(lo, cnt)
    with_valid = torch.ones_like(p, dtype=torch.bool)
    if kind in (abi.JOIN_LEFT_SEMI, abi.JOIN_LEFT_ANTI):
        rows = (cnt > 0 if kind == abi.JOIN_LEFT_SEMI else cnt == 0).nonzero().flatten()
        return [R.OutCol(c.values[rows].clone(), None if c.valid is None else c.valid[rows].clone()) for c in probe.cols]
    if kind in (abi.JOIN_LEFT, abi.JOIN_FULL):
        un = (cnt == 0).nonzero().flatten()
        p = torch.cat([p, un])
        b = torch.cat([b, torch.zeros_like(un)])
        with_valid = torch.cat([with_valid, torch.zeros_like(un, dtype=torch.bool)])
    out = [R.OutCol(c.values[p].clone(), None if c.valid is None else c.valid[p].clone()) for c in probe.cols]
    outer = kind in (abi.JOIN_LEFT, abi.JOIN_FULL)
    for c in build.cols:
        v = c.valid_or_ones()[b] & with_valid
        out.append(R.OutCol(c.values[b].clone(), v.clone() if (c.valid is not None or outer) else None))
    return out


def final_output(kind, build, matched):
    sel = (matched if kind == abi.JOIN_RIGHT_SEMI else ~matched).nonzero().flatten()
    npc = 2 if kind in (abi.JOIN_RIGHT, abi.JOIN_FULL) else 0
    out = [R.OutCol(None, None, True) for _ in range(npc)]
    for c in build.cols:
        out.append(R.OutCol(c.values[sel].clone(), None if (c.valid is None and kind != abi.JOIN_FULL) else c.valid_or_ones()[sel].clone()))
    return out


def _rows_where(out, keep):
    return [R.OutCol(None if c.values is None else c.values[keep], None if c.valid is None else c.valid[keep], c.const_null) for c in out]


def _append_row(out, i):
    return [R.OutCol(torch.cat([c.values, c.values[i:i + 1]]), None if c.valid is None else torch.cat([c.valid, c.valid[i:i + 1]])) for c in out]


def test_verifier_accepts_correct_outputs_of_every_kind():
    build, probe = payload_case()
    for kind in R.ALL_KINDS:
        ref = R.JoinRef(build.key_images()[0], build.key_valid())
        lo, cnt = ref.probe(probe.key_images()[0], probe.key_valid())
        blocks = [] if kind in (abi.JOIN_RIGHT_SEMI, abi.JOIN_RIGHT_ANTI) else [correct_output(kind, build, probe, lo, cnt, ref)]
        R.check_probe_output(kind, blocks, probe, build, cnt)
        R.check_final_output(kind, [final_output(kind, build, ref.matched())] if kind in R.BUILD_SIDE_KINDS else [], build, 2, ref.matched())


def test_verifier_rejects_each_corruption():
    build, probe = payload_case()
    ref = R.JoinRef(build.key_images()[0], build.key_valid())
    lo, cnt = ref.probe(probe.key_images()[0], probe.key_valid())
    good = correct_output(abi.JOIN_INNER, build, probe, lo, cnt, ref)
    n = good[0].values.shape[0]
    ptag = good[1].values
    multi = int((cnt > 1).nonzero()[0])  # a probe row with several matches
    rows = (ptag == multi).nonzero().flatten()
    keep = torch.ones(n, dtype=torch.bool)

    def rejects(kind, out, match):
        with pytest.raises(AssertionError, match=match):
            R.check_probe_output(kind, [out], probe, build, cnt)

    # a dropped pair
    k = keep.clone()
    k[rows[0]] = False
    rejects(abi.JOIN_INNER, _rows_where(good, k), "wrong number of output rows")
    # a duplicated pair, with another pair of the same probe row dropped: counts still equal
    dup = _rows_where(_append_row(good, int(rows[1])), torch.cat([k, torch.ones(1, dtype=torch.bool)]))
    rejects(abi.JOIN_INNER, dup, "repeated")
    # a wrong gathered payload (the I16 column, gathered by build row) and a wrong inlined one (F64)
    for c, what in ((5, "build column 3"), (4, "build column 2")):
        bad = [R.OutCol(x.values.clone(), None if x.valid is None else x.valid.clone()) for x in good]
        i = int(bad[c].valid.nonzero()[0])
        bad[c].values[i] += 1
        rejects(abi.JOIN_INNER, bad, f"{what}: values differ")
    # a wrong validity byte
    bad = [R.OutCol(x.values.clone(), None if x.valid is None else x.valid.clone()) for x in good]
    bad[5].valid[0] = ~bad[5].valid[0]
    rejects(abi.JOIN_INNER, bad, "build column 3: validity differs")
    # a pair whose build row has another key (btag swapped to a non-matching row)
    bad = [R.OutCol(x.values.clone(), None if x.valid is None else x.valid.clone()) for x in good]
    j = int((build.key_images()[0] != build.key_images()[0][int(bad[3].values[0])]).nonzero()[0])
    for c in range(2, 6):
        src = build.cols[c - 2]
        bad[c].values[0] = src.values[j]
        if bad[c].valid is not None:
            bad[c].valid[0] = src.valid_or_ones()[j]
    with pytest.raises(AssertionError):
        R.check_probe_output(abi.JOIN_INNER, [bad], probe, build, cnt)
    # LEFT: an unmatched probe row emitted twice
    left = correct_output(abi.JOIN_LEFT, build, probe, lo, cnt, ref)
    i = int((~left[3].valid).nonzero()[0])
    rejects(abi.JOIN_LEFT, _append_row(left, i), "wrong number of output rows")
    # LEFT: a matched row emitted with a NULL build side instead
    left2 = [R.OutCol(x.values.clone(), None if x.valid is None else x.valid.clone()) for x in left]
    for c in range(2, 6):
        left2[c].valid[0] = False
    rejects(abi.JOIN_LEFT, left2, "unmatched")
    # final_probe: an extra and a missing build row
    m = ref.matched()
    for kind in (abi.JOIN_RIGHT, abi.JOIN_RIGHT_ANTI, abi.JOIN_RIGHT_SEMI, abi.JOIN_FULL):
        fo = final_output(kind, build, m)
        npc = 2 if kind in (abi.JOIN_RIGHT, abi.JOIN_FULL) else 0
        nf = fo[npc].values.shape[0]
        missing = fo[:npc] + [R.OutCol(c.values[1:], None if c.valid is None else c.valid[1:]) for c in fo[npc:]]
        with pytest.raises(AssertionError, match="build rows"):
            R.check_final_output(kind, [missing], build, 2, m)
        other = int((m if kind != abi.JOIN_RIGHT_SEMI else ~m).nonzero()[0])  # a row the kind does not select
        extra = fo[:npc] + [R.OutCol(torch.cat([c.values, build.cols[i].values[other:other + 1]]),
                                     None if c.valid is None else torch.cat([c.valid, build.cols[i].valid_or_ones()[other:other + 1]]))
                            for i, c in enumerate(fo[npc:])]
        with pytest.raises(AssertionError, match="build rows"):
            R.check_final_output(kind, [extra], build, 2, m)
        assert nf > 0


# ---------------------------------------------------------------- slot construction
def test_hash_inverse_and_homes():
    rng = np.random.default_rng(0)
    x = rng.integers(0, 2**64, 10000, dtype=np.uint64, endpoint=False)
    assert np.array_equal(R.agg_hash_inv(R.agg_hash(x)), x)
    assert np.array_equal(R.agg_hash(R.agg_hash_inv(x)), x)
    assert (R.MUL * R.INV_MUL) % 2**64 == 1
    for cap in (1024, 1 << 21, 1 << 25):
        slots = rng.integers(0, cap, 1000)
        assert np.array_equal(R.home_slots(R.words_homed_at(slots, cap, rng), cap), slots)
        k0, k1 = R.wide_words_homed_at(slots, cap, rng)
        assert np.array_equal((R.agg_hash_wide(k0, k1) & np.uint64(cap - 1)).astype(np.int64), slots)
    for dt in (abi.I32, abi.U32, abi.I16):
        v = R.narrow_values_homed_in(1016, 1024, 1024, 50, dt)
        img = R.image(torch.from_numpy(v.view(f"i{v.itemsize}")), dt).numpy().view(np.uint64)
        h = R.home_slots(img, 1024)
        assert len(set(v.tolist())) == 50 and ((h >= 1016) & (h < 1024)).all()


def constructed_homes(slots, cap, rng):
    """Home slots of Int64 keys constructed for the given slots, through the join's hash."""
    return R.home_slots(R.words_homed_at(slots, cap, rng), cap)


def cluster_homes(cap, width, n_keys, copies, rng):
    """Homes of a cluster: n_keys distinct keys homed in the last `width` slots, `copies` entries each."""
    return np.repeat(constructed_homes(rng.integers(cap - width, cap, n_keys), cap, rng), copies)


@pytest.mark.parametrize("cap,width,n_keys,copies,n_other", [(1024, 8, 300, 1, 0), (1024, 8, 150, 2, 0),
                                                              (1 << 21, 4096, 8192, 1, 520_000), (1 << 21, 4096, 4096, 2, 520_000)])
def test_constructed_runs_wrap_and_mix_keys(cap, width, n_keys, copies, n_other):
    """The runs of the GPU tests' tables, simulated: the cluster's run crosses cap - 1 -> 0 whatever the
    insertion order, holds every cluster key (and keys homed in its wrapped part), and an absent key
    homed in the run walks across the wrap to the run's end."""
    rng = np.random.default_rng(cap + copies)
    homes = cluster_homes(cap, width, n_keys, copies, rng)
    wrapped = constructed_homes(rng.integers(0, 32, 16), cap, rng)  # keys homed inside the wrapped part
    other = R.home_slots(rng.integers(0, 2**64, n_other, dtype=np.uint64, endpoint=False), cap)
    all_homes = np.concatenate([homes, wrapped, other])
    owner = np.concatenate([np.repeat(np.arange(n_keys), copies), n_keys + np.arange(len(wrapped)), -1 - np.arange(n_other)])
    occ_sets = []
    for perm_seed in (0, 1):
        perm = np.random.default_rng(perm_seed).permutation(len(all_homes))
        slots = R.linear_probe_insert(all_homes[perm], cap)
        occ = np.zeros(cap, dtype=bool)
        occ[slots] = True
        occ_sets.append(occ)
        start, length = R.run_of(occ, cap - 1)
        assert occ[0] and start + length > cap, "the run does not cross cap - 1 -> 0"
        assert length >= len(homes) + len(wrapped)
        in_run = np.zeros(cap, dtype=bool)
        in_run[(start + np.arange(length)) % cap] = True
        keys_in_run = set(owner[perm][in_run[slots]].tolist())
        assert set(range(n_keys + len(wrapped))) <= keys_in_run  # every cluster key and every wrapped-home key
        if copies > 1:  # some key's entries are not adjacent: another key sits between two of them
            pos = {}
            for s, o in zip(slots.tolist(), owner[perm].tolist()):
                pos.setdefault(o, []).append((s - start) % cap)
            assert any(max(p) - min(p) >= len(p) for o, p in pos.items() if 0 <= o < n_keys)
        # an absent key homed at slot cap - width walks to the run's end, past slot 0
        walk = (start + length) - (cap - width)
        assert walk > width and (cap - width + walk) % cap < cap - width
    assert np.array_equal(occ_sets[0], occ_sets[1])  # the occupied set does not depend on the order


def test_straddling_duplicate_pair():
    """A key with two entries homed at cap - 1 and no other home there or at 0: its entries sit in
    slots cap - 1 and 0 in any insertion order."""
    cap = 1024
    rng = np.random.default_rng(9)
    others = constructed_homes(rng.integers(2, cap // 2, 200), cap, rng)
    homes = np.concatenate([constructed_homes(np.array([cap - 1, cap - 1]), cap, rng), others])
    for perm_seed in range(3):
        perm = np.random.default_rng(perm_seed).permutation(len(homes))
        slots = R.linear_probe_insert(homes[perm], cap)
        pair = sorted(slots[np.nonzero(perm < 2)[0]].tolist())
        assert pair == [0, cap - 1]
