"""The exact per-group reference of tests/float_agg_ref.py has teeth: on each dataset it accepts every
legitimate summation order (a sequential sum over a random row permutation, a pairwise tree, the C
oracle's row order) and rejects the kernel bugs it exists to catch (f32 accumulation, a dropped or
doubled row, NaN read as 0, flushed subnormals, a lossy f32 widening, +inf + -inf reported as inf)."""
import numpy as np
import pytest

import float_agg_ref as R
from databend_b200 import expr as E
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import AggregatorParams

SMALL = {
    "cancellation": lambda: R.cancellation_dataset(n=60_000, groups=800),
    "spread": lambda: R.spread_dataset(n=60_000),
    "specials": lambda: R.specials_dataset(n_background=20_000),
}
_cache = {}


def dataset(name):
    if name not in _cache:
        _cache[name] = SMALL[name]()
    return _cache[name]


def ref_of(name, col):
    key = (name, col)
    if key not in _cache:
        ds = dataset(name)
        _cache[key] = R.exact_reference(ds["k"], ds[col], R.counted_rows(ds, col))
    return _cache[key]


def _pairwise(a, rng=None):
    a = a.astype(np.float64)
    while len(a) > 1:
        if len(a) % 2:
            a = np.append(a, 0.0)
        a = a[0::2] + a[1::2]
    return a[0] if len(a) else 0.0


def _sequential(a, rng):
    return np.cumsum(np.concatenate([[0.0], rng.permutation(a.astype(np.float64))]))[-1]


def _f32_sequential(a, rng):
    return float(np.cumsum(np.concatenate([[np.float32(0)], rng.permutation(a).astype(np.float32)]), dtype=np.float32)[-1])


def group_slices(name, col):
    """(key, contributing values) per group, and the keys of groups without a non-NULL argument"""
    ds = dataset(name)
    rows = R.counted_rows(ds, col)
    k, x = ds["k"][rows], ds[col][rows]
    order = np.argsort(k, kind="stable")
    k, x = k[order], x[order]
    starts = np.flatnonzero(np.concatenate([[True], k[1:] != k[:-1]]))
    ends = np.append(starts[1:], len(k))
    null_groups = set(ds["k"][R.counted_rows(ds, col, nullable=False)].tolist()) - set(k.tolist())
    return [(int(k[lo]), x[lo:hi]) for lo, hi in zip(starts, ends)], null_groups


def group_results(name, col, how, mutate=lambda seg: seg, seed=0):
    """({key: sum}, {key: avg}) from summing each group's contributing rows with `how` after `mutate`"""
    slices, null_groups = group_slices(name, col)
    rng = np.random.default_rng(seed)
    sums, avgs = {}, {}
    with np.errstate(over="ignore", invalid="ignore"):
        for key, seg in slices:
            seg = mutate(seg)
            sums[key] = 0.0 + how(seg, rng)  # the state word starts at +0.0
            avgs[key] = sums[key] / len(seg)
    for key in null_groups:
        sums[key] = avgs[key] = None
    return sums, avgs


def minmax_results(name, col):
    """min / max as the reference computes them: the first row wins a tie"""
    out = {"min": {}, "max": {}}
    slices, null_groups = group_slices(name, col)
    for key, seg in slices:
        nan = np.isnan(seg)
        nonnan = seg[~nan]
        out["min"][key] = nonnan[np.argmin(nonnan)] if len(nonnan) else seg[0]
        out["max"][key] = seg[nan][0] if nan.any() else nonnan[np.argmax(nonnan)]
    for key in null_groups:
        out["min"][key] = out["max"][key] = None
    return out


DATASETS = list(SMALL)


@pytest.mark.parametrize("name", DATASETS)
@pytest.mark.parametrize("col", ["x", "y"])
@pytest.mark.parametrize("how", [_sequential, _pairwise], ids=["sequential_permuted", "pairwise_tree"])
def test_legitimate_orders_are_accepted(name, col, how):
    ref = ref_of(name, col)
    for seed in range(2):
        sums, avgs = group_results(name, col, how, seed=seed)
        assert R.sum_violations(ref, sums) == []
        assert R.avg_violations(ref, avgs) == []


@pytest.mark.parametrize("name", DATASETS)
@pytest.mark.parametrize("col", ["x", "y"])
def test_oracle_is_accepted(name, col):
    from oracle import oracle as orc
    ds = dataset(name)
    blk = DataBlock([Column.from_data(ds["k"]), Column.from_data(ds["v"]), Column.from_data(ds[col], validity=ds[col + "v"])])
    params = AggregatorParams([0], [("sum", 2), ("avg", 2), ("min", 2), ("max", 2), ("count", 2)])
    keys, _, aggs, valid, _ = orc.filter_group_agg(blk, params.to_c(E.ne(E.col(1) % E.lit(R.FILTER_MOD), E.lit(0))), threads=4)
    kk = keys[0].view(np.int64)
    got = [{int(kk[i]): (a[i] if valid[j][i] else None) for i in range(len(kk))} for j, a in enumerate(aggs)]
    ref = ref_of(name, col)
    assert R.sum_violations(ref, got[0]) == []
    assert R.avg_violations(ref, got[1]) == []
    assert R.minmax_violations(ref, got[2], "min", got_dtype=aggs[2].dtype) == []
    assert R.minmax_violations(ref, got[3], "max", got_dtype=aggs[3].dtype) == []
    for key, cnt in got[4].items():
        assert cnt == (ref.n[ref.index[key]] if key in ref.index else 0), key


@pytest.mark.parametrize("name", DATASETS)
@pytest.mark.parametrize("col", ["x", "y"])
def test_minmax_reference_orders_are_accepted(name, col):
    ref = ref_of(name, col)
    mm = minmax_results(name, col)
    for which in ("min", "max"):
        assert R.minmax_violations(ref, mm[which], which) == []


def _drop_last(seg):
    return seg[:-1] if len(seg) > 1 else seg


def _double_last(seg):
    return np.append(seg, seg[-1:])


def _nan_to_zero(seg):
    return np.where(np.isnan(seg), seg.dtype.type(0), seg)


def _flush_subnormals(seg):
    tiny = np.finfo(seg.dtype).tiny
    return np.where(np.abs(seg) < tiny, seg.dtype.type(0), seg)


def _bf16(seg):
    b = seg.astype(np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000  # round to nearest even on the upper 16 bits
    return b.astype(np.uint32).view(np.float32)


# (mutant, summation, datasets built to catch it, argument columns)
MUTANTS = [
    ("f32_accumulation", _f32_sequential, lambda s: s, ["cancellation", "spread"], ["x", "y"]),
    ("row_dropped", _sequential, _drop_last, ["cancellation", "spread", "specials"], ["x", "y"]),
    ("row_added_twice", _sequential, _double_last, ["cancellation", "spread", "specials"], ["x", "y"]),
    ("nan_as_zero", _sequential, _nan_to_zero, ["specials"], ["x", "y"]),
    ("subnormals_flushed", _sequential, _flush_subnormals, ["specials"], ["x", "y"]),
    ("f32_rounded_to_bf16", _sequential, _bf16, ["cancellation", "spread", "specials"], ["y"]),
]


@pytest.mark.parametrize("mutant,how,mutate,names,cols", MUTANTS, ids=[m[0] for m in MUTANTS])
def test_mutants_are_rejected(mutant, how, mutate, names, cols):
    for name in names:
        for col in cols:
            ref = ref_of(name, col)
            sums, avgs = group_results(name, col, how, mutate)
            assert R.sum_violations(ref, sums), (mutant, name, col)
            assert R.avg_violations(ref, avgs), (mutant, name, col)


@pytest.mark.parametrize("col", ["x", "y"])
def test_infinities_of_both_signs_reported_as_inf_are_rejected(col):
    ref = ref_of("specials", col)
    sums, avgs = group_results("specials", col, _sequential)
    both = R.SPECIAL_KEY0 + R.SPECIALS.index("both_inf")
    assert np.isnan(sums[both])
    sums[both], avgs[both] = np.inf, np.inf
    assert len(R.sum_violations(ref, sums)) == 1 and len(R.avg_violations(ref, avgs)) == 1


@pytest.mark.parametrize("col", ["x", "y"])
def test_special_groups_have_their_fixed_answers(col):
    """NaN in any form, infinities, all -0.0 -> +0.0, overflow pairs -> inf, NULL-only -> NULL"""
    ref = ref_of("specials", col)
    ix = {name: ref.index.get(R.SPECIAL_KEY0 + i) for i, name in enumerate(R.SPECIALS)}
    for name in ("nan", "nan_sign_bit", "nan_payload", "only_nan", "both_inf"):
        assert np.isnan(ref.special[ix[name]]), name
    assert ref.special[ix["pos_inf"]] == np.inf and ref.special[ix["neg_inf"]] == -np.inf
    if col == "x":
        assert ref.special[ix["overflow_pos"]] == np.inf and ref.special[ix["overflow_neg"]] == -np.inf
    assert ix["null_only"] is None
    assert ref.A[ix["all_neg_zero"]] == 0 and ref.both_zeros[ix["both_zeros"]]
    assert 0 < ref.s[ix["subnormal"]] < 2.0 ** -1000 if col == "x" else 0 < ref.s[ix["subnormal"]] < 2.0 ** -120
    sums, _ = group_results("specials", col, _sequential)
    key = R.SPECIAL_KEY0 + R.SPECIALS.index("all_neg_zero")
    assert R.sum_violations(ref, sums) == []
    sums[key] = -0.0  # the sign of the zero is part of the answer
    assert len(R.sum_violations(ref, sums)) == 1
    # the group without a non-NULL argument must stay NULL
    sums[key] = 0.0
    sums[R.SPECIAL_KEY0 + R.SPECIALS.index("null_only")] = 0.0
    assert len(R.sum_violations(ref, sums)) == 1


@pytest.mark.parametrize("col", ["x", "y"])
def test_minmax_device_rule(col):
    """zeros="device": -0.0 orders below +0.0 and every NaN result is the canonical quiet NaN"""
    ref = ref_of("specials", col)
    mm = minmax_results("specials", col)
    both = R.SPECIAL_KEY0 + R.SPECIALS.index("both_zeros")
    nan_key = R.SPECIAL_KEY0 + R.SPECIALS.index("nan_sign_bit")
    dt = ref.dtype.type
    mn, mx = dict(mm["min"]), dict(mm["max"])
    mn[both], mx[both] = dt(-0.0), dt(0.0)
    for d in (mn, mx):
        for k, v in d.items():
            if v is not None and np.isnan(v):
                d[k] = dt(np.nan)
    assert R.minmax_violations(ref, mn, "min", zeros="device") == []
    assert R.minmax_violations(ref, mx, "max", zeros="device") == []
    bad = dict(mn)
    bad[both] = dt(0.0)
    assert len(R.minmax_violations(ref, bad, "min", zeros="device")) == 1
    assert R.minmax_violations(ref, bad, "min", zeros="either") == []
    bad = dict(mx)
    bad[nan_key] = np.array([0xFFF8000000000000], dtype=np.uint64).view(np.float64)[0] if col == "x" else np.array([0xFFC00000], dtype=np.uint32).view(np.float32)[0]
    assert len(R.minmax_violations(ref, bad, "max", zeros="device")) == 1
    assert R.minmax_violations(ref, bad, "max", zeros="either") == []
    bad[nan_key] = dt(1.0)
    assert len(R.minmax_violations(ref, bad, "max", zeros="either")) == 1


def test_order_dependent_groups_are_refused():
    k = np.zeros(3, dtype=np.int64)
    rows = np.ones(3, dtype=bool)
    with pytest.raises(ValueError):  # DBL_MAX + DBL_MAX/4 - DBL_MAX: overflows in some orders only
        R.exact_reference(k, np.array([R.DBL_MAX, R.DBL_MAX / 4, -R.DBL_MAX]), rows)
    with pytest.raises(ValueError):  # +inf next to finite values that may overflow to -inf
        R.exact_reference(k, np.array([np.inf, -0.9 * R.DBL_MAX, -0.9 * R.DBL_MAX]), rows)
