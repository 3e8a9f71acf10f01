"""Order-independent reference for floating-point sum / avg / min / max per group (CPU only).

The device adds f64 state words in an order that changes from run to run: L2 reductions, shared-memory
compare-and-swap loops in the hot-group cache and the slice pass, warp shuffles, flushes and merges of
partial tables.  The C oracle adds in row order.  Comparing the two with an `rtol` says nothing under
cancellation, so this module checks a device result against the exact sum of each group instead:

  n = rows of the group that pass the filter and have a non-NULL argument (f32 widened exactly to f64)
  s = math.fsum(x)        the correctly rounded exact sum
  A = math.fsum(|x|)
  sum:  |ŝ − s| ≤ γ(n+1)·A,                      γ(k) = k·u / (1 − k·u), u = 2^-53
  avg:  |â − s/n| ≤ γ(n+1)·A/n + 3u·|s|/n

The sum bound holds for any binary tree of n − 1 additions; the +1 absorbs the rounding of s and A.
The avg bound adds the rounding of the device's quotient and of the reference's own s/n.  Special
values decide the result in every order:

  any NaN, or both +inf and −inf  -> NaN
  otherwise +inf or −inf present  -> that infinity
  two values of one sign each > DBL_MAX/2 and none of the other sign -> that sign's infinity (overflow)
  all values ±0.0                 -> +0.0 (the state starts at +0.0: NumberSumState, aggregate_sum.rs:93,108)

A group whose answer would depend on the order (a finite sum that could overflow, an infinity next to
finite values that could overflow the other way) raises ValueError: such a dataset proves nothing.

min / max follow OrderedFloat: NaN is the greatest value and all NaNs are equal, −0.0 == +0.0.  With
both zeros in a group the reference's answer depends on row order, so `zeros="either"` accepts both
signs and any NaN for a NaN result.  The device reduces one ordered image on every path, in which
−0.0 orders below +0.0 and every NaN maps to one canonical quiet NaN; `zeros="device"` checks that
rule bit for bit.  min / max of F32 stay F32.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import numpy as np

U = 2.0 ** -53
DBL_MAX = float(np.finfo(np.float64).max)
_REL_SLACK = 1.0 + 2.0 ** -40  # covers the float arithmetic that evaluates the bounds
_ABS_SLACK = 2.0 ** -1072      # four subnormal ulps: rounding of a bound that underflows
NAN_BITS = {np.dtype(np.float64): 0x7FF8000000000000, np.dtype(np.float32): 0x7FC00000}


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


@dataclass
class FloatAggRef:
    """Per-group exact reference over the rows that pass the filter with a non-NULL argument."""
    index: Dict[object, int]   # group key -> position
    dtype: np.dtype            # argument dtype (float32 or float64)
    n: np.ndarray              # contributing rows
    s: np.ndarray              # fsum of the finite values (0 where the result is special)
    A: np.ndarray              # fsum of their magnitudes
    special: np.ndarray        # result of sum that special values force: NaN / ±inf, or 0 when none
    min: np.ndarray            # argument dtype, OrderedFloat minimum
    max: np.ndarray
    both_zeros: np.ndarray     # the group holds both -0.0 and +0.0


def exact_reference(keys: np.ndarray, values: np.ndarray, rows: np.ndarray) -> FloatAggRef:
    """keys: one integer image per row (the group key; NULL keys as a value of their own chosen by the
    caller), values: float32 or float64 argument, rows: bool mask of the rows that count."""
    values = np.asarray(values)
    dt = values.dtype
    assert dt in (np.dtype(np.float32), np.dtype(np.float64)), dt
    k = np.asarray(keys)[rows]
    x = values[rows]
    order = np.argsort(k, kind="stable")
    k, x = k[order], x[order]
    if len(k) == 0:
        empty = np.zeros(0)
        return FloatAggRef({}, dt, empty.astype(np.int64), empty, empty, empty, empty.astype(dt), empty.astype(dt), empty.astype(bool))
    starts = np.flatnonzero(np.concatenate([[True], k[1:] != k[:-1]]))
    ends = np.append(starts[1:], len(k))
    w = x.astype(np.float64)  # exact widening
    nan = np.logical_or.reduceat(np.isnan(w), starts)
    pinf = np.logical_or.reduceat(w == np.inf, starts)
    ninf = np.logical_or.reduceat(w == -np.inf, starts)
    finite = np.isfinite(w)
    big_pos = np.add.reduceat(w > DBL_MAX / 2, starts)
    big_neg = np.add.reduceat(w < -DBL_MAX / 2, starts)
    has_pos = np.logical_or.reduceat(finite & (w > 0), starts)
    has_neg = np.logical_or.reduceat(finite & (w < 0), starts)
    neg0 = np.logical_or.reduceat((w == 0) & np.signbit(w), starts)
    pos0 = np.logical_or.reduceat((w == 0) & ~np.signbit(w), starts)

    G = len(starts)
    s = np.zeros(G)
    A = np.zeros(G)
    special = np.zeros(G)
    fw = np.where(finite, w, 0.0)
    for g in range(G):
        seg = fw[starts[g]:ends[g]]
        if nan[g] or (pinf[g] and ninf[g]):
            special[g] = np.nan
            continue
        if big_pos[g] >= 2 and not has_neg[g] and not ninf[g]:
            special[g] = np.inf
            continue
        if big_neg[g] >= 2 and not has_pos[g] and not pinf[g]:
            special[g] = -np.inf
            continue
        try:
            a = math.fsum(np.abs(seg))
        except OverflowError:
            a = math.inf
        if not a <= DBL_MAX / 4:
            raise ValueError(f"group {k[starts[g]]}: sum of magnitudes {a} may overflow in some orders and not in others")
        if pinf[g] or ninf[g]:
            special[g] = np.inf if pinf[g] else -np.inf
            continue
        s[g] = math.fsum(seg)
        A[g] = a

    # OrderedFloat: NaN is the greatest value
    nan_fill_lo = np.where(np.isnan(w), np.inf, w)
    nan_fill_hi = np.where(np.isnan(w), -np.inf, w)
    all_nan = np.logical_and.reduceat(np.isnan(w), starts)
    mn = np.minimum.reduceat(nan_fill_lo, starts)
    mn = np.where(all_nan, np.nan, mn)
    mx = np.maximum.reduceat(nan_fill_hi, starts)
    mx = np.where(nan, np.nan, mx)
    # a zero result takes the sign of the zeros present (either sign when both are: see `zeros`)
    zero_sign = np.where(neg0 & ~pos0, -0.0, 0.0)
    mn = np.where(mn == 0, zero_sign, mn)
    mx = np.where(mx == 0, zero_sign, mx)
    keys_out = [int(v) for v in k[starts]]
    return FloatAggRef({kk: i for i, kk in enumerate(keys_out)}, dt, ends - starts, s, A, special,
                       mn.astype(dt), mx.astype(dt), neg0 & pos0)


def _align(ref: FloatAggRef, got: Dict[object, Optional[float]], errors: List[str]):
    """positions of ref's groups in got order; groups without contributing rows must be NULL"""
    for key, v in got.items():
        if key not in ref.index and v is not None:
            errors.append(f"group {key}: no non-NULL argument, expected NULL, got {v!r}")
    vals = np.zeros(len(ref.index))
    present = np.zeros(len(ref.index), dtype=bool)
    missing = object()
    for key, i in ref.index.items():
        v = got.get(key, missing)
        if v is missing:
            errors.append(f"group {key}: missing")
        elif v is None:
            errors.append(f"group {key}: NULL, expected a value")
        else:
            vals[i] = v
            present[i] = True
    return vals, present


def _check_values(ref: FloatAggRef, got, expected_finite, bound, what: str) -> List[str]:
    errors: List[str] = []
    g, present = _align(ref, got, errors)
    keys = list(ref.index)
    sp = ref.special
    nan_exp = np.isnan(sp)
    inf_exp = np.isinf(sp)
    fin_exp = ~nan_exp & ~inf_exp
    with np.errstate(invalid="ignore", over="ignore"):
        err = np.abs(g - expected_finite)
    bad = present & (
        (nan_exp & ~np.isnan(g))
        | (inf_exp & (g != sp))
        | (fin_exp & ~(np.isfinite(g) & (err <= bound)))
        | (fin_exp & (ref.A == 0) & ((g != 0) | np.signbit(g))))  # all zeros: +0.0
    for i in np.flatnonzero(bad)[:20]:
        errors.append(f"{what} of group {keys[i]}: got {g[i]!r} ({float(g[i]).hex()}), exact {expected_finite[i]!r} "
                      f"special {sp[i]!r} n {ref.n[i]} bound {bound[i]:.3g} error {err[i]:.3g}")
    if bad.sum() > 20:
        errors.append(f"... {bad.sum()} {what} groups in all")
    return errors


def sum_violations(ref: FloatAggRef, got: Dict[object, Optional[float]]) -> List[str]:
    """got: {group key: device sum, or None for NULL}.  Returns one message per violating group."""
    bound = gamma(ref.n + 1) * ref.A * _REL_SLACK + _ABS_SLACK
    return _check_values(ref, got, ref.s, bound, "sum")


def avg_violations(ref: FloatAggRef, got: Dict[object, Optional[float]]) -> List[str]:
    c = np.maximum(ref.n, 1).astype(np.float64)
    q = ref.s / c
    bound = (gamma(ref.n + 1) * ref.A / c + 3 * U * np.abs(q)) * _REL_SLACK + _ABS_SLACK
    return _check_values(ref, got, q, bound, "avg")


def minmax_violations(ref: FloatAggRef, got: Dict[object, Optional[float]], which: str, zeros: str = "either",
                      got_dtype=None) -> List[str]:
    """which: "min" or "max".  zeros="either": the reference's semantics (either zero when a group holds both,
    any NaN for a NaN result); zeros="device": −0.0 < +0.0 and the canonical quiet NaN, bit for bit."""
    assert which in ("min", "max") and zeros in ("either", "device")
    errors: List[str] = []
    if got_dtype is not None and np.dtype(got_dtype) != ref.dtype:
        errors.append(f"{which}: result dtype {np.dtype(got_dtype)}, argument dtype {ref.dtype}")
    g, present = _align(ref, got, errors)
    dt = ref.dtype
    ub = np.uint64 if dt.itemsize == 8 else np.uint32
    g = g.astype(dt)
    exp = (ref.min if which == "min" else ref.max).copy()
    if zeros == "device":
        exp[ref.both_zeros & (exp == 0)] = dt.type(-0.0) if which == "min" else dt.type(0.0)
    gb, eb = g.view(ub), exp.view(ub)
    nan_exp = np.isnan(exp)
    if zeros == "device":
        ok = np.where(nan_exp, gb == ub(NAN_BITS[dt]), gb == eb)
    else:
        ok = np.where(nan_exp, np.isnan(g), (gb == eb) | (ref.both_zeros & (exp == 0) & (g == 0)))
    keys = list(ref.index)
    for i in np.flatnonzero(present & ~ok)[:20]:
        errors.append(f"{which} of group {keys[i]}: got {g[i]!r} (bits {int(gb[i]):#x}), expected {exp[i]!r} (bits {int(eb[i]):#x})")
    return errors


# ---------------------------------------------------------------- seeded datasets
# Each dataset is a dict of row arrays: `k` Int64 group key, `v` Int64 filter column, `x` Float64 and `y`
# Float32 arguments with validity `xv` / `yv`.  FILTER_MOD is the filter `v % FILTER_MOD <> 0`.
FILTER_MOD = 5
SPECIAL_KEY0 = 10 ** 7  # dedicated groups of the specials dataset: SPECIAL_KEY0 + SPECIALS.index(name)
SPECIALS = ["nan", "nan_sign_bit", "nan_payload", "only_nan", "pos_inf", "neg_inf", "both_inf", "all_neg_zero",
            "both_zeros", "subnormal", "overflow_pos", "overflow_neg", "null_only", "small_next_to_large"]


def _f64_real(rng, n, e_lo=-40, e_hi=40):
    """±m·2^e with a 53-bit m and e in [e_lo, e_hi]"""
    m = rng.integers(2 ** 52, 2 ** 53, n, dtype=np.int64).astype(np.float64)
    x = np.ldexp(m, rng.integers(e_lo, e_hi + 1, n) - 52)
    return np.where(rng.random(n) < 0.5, -x, x)


def _f32_real(rng, n, subnormal_share=0.01):
    """±m·2^e with a 24-bit m and e in [-30, 30], and some f32 subnormals"""
    m = rng.integers(2 ** 23, 2 ** 24, n).astype(np.float64)
    y = np.ldexp(m, rng.integers(-30, 31, n) - 23).astype(np.float32)
    sub = rng.random(n) < subnormal_share
    y[sub] = rng.integers(1, 2 ** 23, int(sub.sum())).astype(np.uint32).view(np.float32)
    return np.where(rng.random(n) < 0.5, -y, y).astype(np.float32)


def _finish(rng, k, x, y, null_share, v=None, xv=None):
    n = len(k)
    if v is None:
        v = rng.integers(0, 1 << 40, n).astype(np.int64)
    if xv is None:
        xv = rng.random(n) >= null_share
    perm = rng.permutation(n)  # spread every group over tiles, warps and blocks
    return {"k": np.asarray(k, dtype=np.int64)[perm], "v": v[perm], "x": np.asarray(x, dtype=np.float64)[perm],
            "y": np.asarray(y, dtype=np.float32)[perm], "xv": xv[perm], "yv": (rng.random(n) >= null_share)[perm]}


def cancellation_dataset(n=300_000, groups=4000, seed=1, null_share=0.1):
    """x: values ±m·2^e (53-bit m, e in [-40, 40]) in pairs that cancel within their group exactly or up to
    a relative 2^-30, plus a tenth of unpaired rows with e in [-40, 0], so |s| << A; y: f32 arguments with
    full 24-bit mantissas, exponents in [-30, 30] and 1 % f32 subnormals."""
    rng = np.random.default_rng(seed)
    n0 = n * 9 // 20
    k0 = rng.integers(0, groups, n0)
    x0 = _f64_real(rng, n0)
    xn = -(x0 * (1.0 + rng.integers(-1, 2, n0) * 2.0 ** -30))
    k = np.concatenate([k0, k0, rng.integers(0, groups, n - 2 * n0)])
    x = np.concatenate([x0, xn, _f64_real(rng, n - 2 * n0, -40, 0)])
    v0, xv0 = rng.integers(0, 1 << 40, n0), rng.random(n0) >= null_share  # a pair is counted or dropped as one
    v = np.concatenate([v0, v0, rng.integers(0, 1 << 40, n - 2 * n0)])
    xv = np.concatenate([xv0, xv0, rng.random(n - 2 * n0) >= null_share])
    return _finish(rng, k, x, _f32_real(rng, n), null_share, v, xv)


def spread_dataset(n=300_000, seed=2, null_share=0.1):
    """group sizes from one group holding half of the rows, through P(k) ~ 1/k over 10^5 keys, to 20 000
    groups of 1-3 rows; real-valued x and y"""
    rng = np.random.default_rng(seed)
    tail = np.repeat(200_000 + np.arange(20_000), rng.integers(1, 4, 20_000))
    m = n - len(tail)
    log_uniform = np.minimum((np.exp(rng.random(m) * np.log(1e5)) - 1).astype(np.int64), 99_999)
    k = np.concatenate([np.where(rng.random(m) < n / 2 / m, 7, log_uniform), tail])
    return _finish(rng, k, _f64_real(rng, len(k), -20, 20), _f32_real(rng, len(k)), null_share)


def specials_dataset(n_background=200_000, seed=3, null_share=0.1):
    """background groups of real values plus one dedicated group per SPECIALS entry (rows that pass the
    filter; the filter still drops background rows).  The NULL rows of `null_only` hold NaN in their value
    slot: they must not count."""
    rng = np.random.default_rng(seed)
    ks, xs, ys, vs = [rng.integers(0, 3000, n_background)], [_f64_real(rng, n_background)], [_f32_real(rng, n_background)], []
    vs.append(rng.integers(0, 1 << 40, n_background))
    nulls = []
    f64 = lambda bits: np.array(bits, dtype=np.uint64).view(np.float64)
    f32 = lambda bits: np.array(bits, dtype=np.uint32).view(np.float32)
    for i, name in enumerate(SPECIALS):
        m = 64
        x, y = _f64_real(rng, m), _f32_real(rng, m, 0.0)
        if name in ("nan", "nan_sign_bit", "nan_payload"):
            j = rng.choice(m, 3, replace=False)
            x[j] = f64({"nan": 0x7FF8000000000000, "nan_sign_bit": 0xFFF8000000000000, "nan_payload": 0x7FF8000000000123}[name])
            y[j] = f32({"nan": 0x7FC00000, "nan_sign_bit": 0xFFC00000, "nan_payload": 0x7FC00123}[name])
        elif name == "only_nan":
            x[:] = f64([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF80000000ABCDE, 0x7FF8000000000000] * (m // 4))
            y[:] = f32([0x7FC00000, 0xFFC00000, 0x7FC0ABCD, 0x7FC00000] * (m // 4))
        elif name in ("pos_inf", "neg_inf", "both_inf"):
            j = rng.choice(m, 4, replace=False)
            x[j[:2]] = y[j[:2]] = -np.inf if name == "neg_inf" else np.inf
            x[j[2:]] = y[j[2:]] = np.inf if name == "pos_inf" else -np.inf
        elif name == "all_neg_zero":
            x[:] = y[:] = -0.0
        elif name == "both_zeros":
            x[:] = y[:] = np.where(rng.random(m) < 0.5, -0.0, 0.0)
            x[:2] = y[:2] = [-0.0, 0.0]
        elif name == "subnormal":
            x[:] = rng.integers(1, 2 ** 52, m, dtype=np.uint64).view(np.float64)
            y[:] = rng.integers(1, 2 ** 23, m).astype(np.uint32).view(np.float32)
        elif name in ("overflow_pos", "overflow_neg"):
            sign = 1.0 if name == "overflow_pos" else -1.0
            x[:] = sign * np.abs(x)
            x[:2] = sign * np.array([0.75, 0.9]) * DBL_MAX
        elif name == "small_next_to_large":  # one large value, the rest about 2^-40 of it
            x[:] = 1.0 + rng.random(m)
            x[0] = 2.0 ** 40
            y[:] = (1.0 + rng.random(m)).astype(np.float32)
            y[0] = 2.0 ** 24
        ks.append(np.full(m, SPECIAL_KEY0 + i))
        xs.append(x)
        ys.append(y)
        vs.append(np.ones(m, dtype=np.int64))
        nulls.append((len(np.concatenate(ks)) - m, m) if name == "null_only" else None)
    k, x, y, v = (np.concatenate(a) for a in (ks, xs, ys, vs))
    n = len(k)
    xv, yv = rng.random(n) >= null_share, rng.random(n) >= null_share
    special_rows = k >= SPECIAL_KEY0
    xv[special_rows] = yv[special_rows] = True
    for span in nulls:
        if span:
            lo, m = span
            xv[lo:lo + m] = yv[lo:lo + m] = False
            x[lo:lo + m] = np.nan
            y[lo:lo + m] = np.nan
    perm = rng.permutation(n)
    return {"k": k[perm].astype(np.int64), "v": v[perm].astype(np.int64), "x": x[perm], "y": y[perm].astype(np.float32),
            "xv": xv[perm], "yv": yv[perm]}


def counted_rows(ds, col, nullable=True, filtered=True):
    """rows that pass `v % FILTER_MOD <> 0` and have a non-NULL `col`"""
    rows = ds["v"] % FILTER_MOD != 0 if filtered else np.ones(len(ds["k"]), dtype=bool)
    return rows & ds[col + "v"] if nullable else rows
