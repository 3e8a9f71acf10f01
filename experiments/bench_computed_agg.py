"""Fused computed columns against materialising them first, on device-resident synthetic columns.

For each shape: fused = one operator created with dbx_op_create_computed; materialised = dbx_eval_scalar
of every expression into a device column, then the plain operator over inputs + those columns.  After
warm-up, two times per query: the aggregate kernel(s) of the push from the operator's CUDA events
(dbx_op_last_kernel_ms), and the whole query on the host clock from the first launch to the finished
device-resident result (every call ends in a stream synchronisation; the host pull of the result is
outside).  The materialised query adds dbx_eval_scalar, which synchronises per expression.  Results of
both ways are compared.  Algorithmic
bytes per row: the inputs only for fused, plus 16 B per materialised column (written once, read once).

  python experiments/bench_computed_agg.py [--q1-rows 5e8] [--rows 2e8] [--reps 5]
"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databend_b200 import abi, expr as E, scalar_expr as S  # noqa: E402
from databend_b200.block import Column, DataBlock  # noqa: E402
from databend_b200.lib import check, load  # noqa: E402
from databend_b200.transforms import (AggregatorParams, DeviceBuffer, TransformFinalAggregate, TransformPartialAggregate,  # noqa: E402
                                      _block_from_c)

HBM_BPS = 3.35e12  # H100 SXM data sheet (700 W)


def dev_col(kind, seed, a, n, dtype, np_dtype=None):
    buf = DeviceBuffer(max(1, n * 8))
    check(load().dbx_synth_fill(0, kind, seed, a, 0, n, buf.ptr))
    col = Column(dtype, n, dev_ptr=buf.ptr)
    col._keep.append(buf)
    return col


def run(params, filt, blk, types):
    part = TransformPartialAggregate(params, types, filt)
    fin = TransformFinalAggregate(params, types)
    load().dbx_device_synchronize(0)
    t0 = time.perf_counter()
    part.transform(blk)
    part.on_finish()
    fin.transform(part)
    fin.finish()
    fin.synchronize()
    dt = time.perf_counter() - t0
    kms = part.last_kernel_ms()
    out = _block_from_c(fin.pull_c(abi.MEM_HOST), 0)
    part.close()
    fin.close()
    return dt, kms, out


def materialise(blk, exprs):
    cols, dts, t = list(blk.columns), [], 0.0
    for e in exprs:
        load().dbx_device_synchronize(0)
        t0 = time.perf_counter()
        b, dt = S.eval_scalar(blk, e, out_mem=abi.MEM_DEVICE)
        t += time.perf_counter() - t0
        c = b.cols[0]
        col = Column(dt & 0xFF, c.len, dev_ptr=c.data)
        col._keep.append(b)
        cols.append(col)
        dts.append(dt)
    return DataBlock(cols, blk.num_rows), dts, t


def same_results(a, b):
    return all(np.allclose(np.sort(a.columns[i].values()), np.sort(b.columns[i].values()), rtol=1e-9, equal_nan=True)
               for i in range(a.num_columns()))


def shape(name, n, blk, types, params_f, params_m, filt, exprs, in_bytes, reps, params_a=None):
    """params_a: an optional third variant, a fused form of the same query written without IF."""
    for _ in range(2):
        run(params_f, filt, blk, types)
    runs = [run(params_f, filt, blk, types) for _ in range(reps)]
    tf, kf, out_f = min(r[0] for r in runs), min(r[1] for r in runs), runs[-1][2]
    variants = []
    if params_a is not None:
        run(params_a, filt, blk, types)
        runs_a = [run(params_a, filt, blk, types) for _ in range(reps)]
        variants.append(("fused-arith", min(r[0] for r in runs_a), min(r[1] for r in runs_a), in_bytes, same_results(out_f, runs_a[-1][2])))
    tm_best, km_best, out_m = None, None, None
    for _ in range(reps + 1):
        mblk, dts, t_eval = materialise(blk, exprs)
        t_agg, k_agg, out_m = run(params_m, filt, mblk, types + dts)
        tm_best = t_eval + t_agg if tm_best is None else min(tm_best, t_eval + t_agg)
        km_best = k_agg if km_best is None else min(km_best, k_agg)
        del mblk
    same = same_results(out_f, out_m)
    for how, t, k, bpr, same in [("fused", tf, kf, in_bytes, same), ("materialised", tm_best, km_best, in_bytes + 16 * len(exprs), same)] + variants:
        print(f"{name:10s} {how:13s} rows {n:.3g}  query {t * 1e3:9.2f} ms  {n / t / 1e9:7.2f} G rows/s  {bpr:3d} B/row  "
              f"query share of HBM bound {n * bpr / t / HBM_BPS:5.2f}  aggregate kernel {k:8.2f} ms (events)  results equal: {same}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--q1-rows", type=float, default=5e8)
    ap.add_argument("--rows", type=float, default=2e8)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    one = S.lit(1.0, abi.F64)
    # Q1: four (flag, status) groups, heavily skewed onto the hot-group cache
    n = int(a.q1_rows)
    cols = [dev_col(0, 1, 2, n, abi.I64), dev_col(0, 2, 2, n, abi.I64), dev_col(2, 3, 5, n, abi.F64), dev_col(2, 4, 17, n, abi.F64),
            dev_col(3, 5, 0, n, abi.F64), dev_col(3, 6, 0, n, abi.F64), dev_col(0, 7, 2600, n, abi.I64)]
    blk = DataBlock(cols, n)
    types = [abi.I64, abi.I64, abi.F64, abi.F64, abi.F64, abi.F64, abi.I64]
    dp = S.col(3) * (one - S.col(4))
    ch = dp * (one + S.col(5))
    filt = E.le(E.col(6), E.lit(2500))
    pf = AggregatorParams([0, 1], [("sum", 2), ("sum", 3), ("sum", dp), ("sum", ch), ("avg", 2), ("avg", 3), ("avg", 4), ("count", None)])
    pm = AggregatorParams([0, 1], [("sum", 2), ("sum", 3), ("sum", 7), ("sum", 8), ("avg", 2), ("avg", 3), ("avg", 4), ("count", None)])
    shape("Q1", n, blk, types, pf, pm, filt, [dp, ch], 56, a.reps)
    del blk, cols
    # Q6: no GROUP BY
    n = int(a.rows)
    cols = [dev_col(2, 11, 17, n, abi.F64), dev_col(3, 12, 0, n, abi.F64), dev_col(2, 13, 6, n, abi.F64)]
    blk = DataBlock(cols, n)
    types = [abi.F64] * 3
    filt = E.lt(E.col(2), E.lit(24.0))
    shape("Q6", n, blk, types, AggregatorParams([], [("sum", S.col(0) * S.col(1))]), AggregatorParams([], [("sum", 3)]), filt,
          [S.col(0) * S.col(1)], 24, a.reps)
    del blk, cols
    # 1e6 groups: SELECT k, sum(v * x), avg(x + v) WHERE v % 3 = 0
    cols = [dev_col(0, 21, 1_000_000, n, abi.I64), dev_col(1, 22, 0, n, abi.I64), dev_col(2, 23, 20, n, abi.F64)]
    blk = DataBlock(cols, n)
    types = [abi.I64, abi.I64, abi.F64]
    e1, e2 = S.col(1) * S.col(2), S.col(2) + S.col(1)
    filt = E.eq(E.col(1) % E.lit(3), E.lit(0))
    shape("1e6-group", n, blk, types, AggregatorParams([0], [("sum", e1), ("avg", e2)]), AggregatorParams([0], [("sum", 3), ("avg", 4)]),
          filt, [e1, e2], 24, a.reps)
    del blk, cols
    # Q12-shaped (ship modes and priorities as integer codes): SELECT mode, sum(if(prio = 0 or prio = 1, 1, 0)),
    # sum(if(prio > 1, 1, 0)) WHERE (mode = 0 OR mode = 1) AND receipt < 1000 GROUP BY mode
    cols = [dev_col(0, 31, 7, n, abi.I64), dev_col(0, 32, 5, n, abi.I64), dev_col(0, 33, 2600, n, abi.I64)]
    blk = DataBlock(cols, n)
    types = [abi.I64] * 3
    zero, one64 = S.lit(0, abi.I64), S.lit(1, abi.I64)
    high = S.call("or", S.call("eq", S.col(1), zero), S.call("eq", S.col(1), one64))
    low = S.call("gt", S.col(1), one64)
    h, lo = S.if_(high, one64, zero), S.if_(low, one64, zero)
    filt = E.and_(E.or_(E.eq(E.col(0), E.lit(0)), E.eq(E.col(0), E.lit(1))), E.lt(E.col(2), E.lit(1000)))
    shape("Q12", n, blk, types, AggregatorParams([0], [("sum", h), ("sum", lo)]), AggregatorParams([0], [("sum", 3), ("sum", 4)]), filt,
          [h, lo], 24, a.reps, AggregatorParams([0], [("sum", S.cast(high, abi.I64)), ("sum", S.cast(low, abi.I64))]))
    del blk, cols
    # Q14-shaped, no GROUP BY: sum(if(ptype < 25, price * (1 - disc), 0.0)), sum(price * (1 - disc)) over a ship-date range
    cols = [dev_col(2, 41, 17, n, abi.F64), dev_col(3, 42, 0, n, abi.F64), dev_col(0, 43, 150, n, abi.I64), dev_col(0, 44, 2600, n, abi.I64)]
    blk = DataBlock(cols, n)
    types = [abi.F64, abi.F64, abi.I64, abi.I64]
    rev = S.col(0) * (one - S.col(1))
    promo_c = S.call("lt", S.col(2), S.lit(25, abi.I64))
    promo = S.if_(promo_c, rev, S.lit(0.0, abi.F64))
    filt = E.and_(E.ge(E.col(3), E.lit(1000)), E.lt(E.col(3), E.lit(1030)))
    shape("Q14", n, blk, types, AggregatorParams([], [("sum", promo), ("sum", rev)]), AggregatorParams([], [("sum", 4), ("sum", 5)]), filt,
          [promo, rev], 32, a.reps, AggregatorParams([], [("sum", rev * S.cast(promo_c, abi.F64)), ("sum", rev)]))


if __name__ == "__main__":
    main()
