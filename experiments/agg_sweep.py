"""Sweeps the tuning knobs of the fused filter->hash-agg kernel in ONE process (columns generated
once): the persisting-L2 window and the bisecting modes of DBX_AGG_DEBUG.  Every variant's result
is compared bit for bit with the first one (keys, sums, counts, avgs after sorting by key).
The kernel launcher reads DBX_AGG_GRID once per process: compare grid sizes with one run per value.
usage: python experiments/agg_sweep.py [rows] [n_keys] [reps] [quick]"""
import ctypes as C
import os
import sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databend_b200 import abi, build, lib, expr as E
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import AggregatorParams, DeviceBuffer, TransformFinalAggregate, TransformPartialAggregate

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000_000
n_keys = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
build.build()
L = lib.load()
lib.require_device()
bufs = [DeviceBuffer(rows * 8) for _ in range(3)]
lib.check(L.dbx_synth_fill(0, 0, 42, n_keys, 0, rows, bufs[0].ptr))
lib.check(L.dbx_synth_fill(0, 1, 43, 0, 0, rows, bufs[1].ptr))
lib.check(L.dbx_synth_fill(0, 2, 44, 20, 0, rows, bufs[2].ptr))
blk = DataBlock([Column.device(abi.I64, rows, bufs[0].ptr), Column.device(abi.I64, rows, bufs[1].ptr),
                 Column.device(abi.F64, rows, bufs[2].ptr)], rows)
params = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2)])
filt = E.eq(E.col(1) % E.lit(3), E.lit(0))
types = [abi.I64, abi.I64, abi.F64]
KNOBS = ["DBX_AGG_L2_PERSIST", "DBX_AGG_DEBUG"]
ref = None


def run(name, **env):
    global ref
    for k in KNOBS:
        os.environ.pop(k, None)
    for k, v in env.items():
        os.environ[k] = str(v)
    part = TransformPartialAggregate(params, types, filt)
    fin = TransformFinalAggregate(params, types)
    best = 1e9
    res = None
    for i in range(reps):
        part.reset(); fin.reset()
        part.transform(blk)
        ms = part.last_kernel_ms()
        fin.transform(part.on_finish())
        if i == 0:
            res = fin.on_finish()[0]
        else:
            out = fin.on_finish(abi.MEM_DEVICE)
            L.dbx_block_release(C.byref(out[0]))
        best = min(best, ms)
    part.close(); fin.close()
    order = np.argsort(res.columns[3].values(), kind="stable")
    sig = [res.columns[i].values()[order].view(np.uint64) for i in range(4)]
    ok = "ref"
    if ref is None:
        ref = sig
    elif "DBX_AGG_DEBUG" not in env:
        ok = "same" if all(np.array_equal(a, b) for a, b in zip(sig, ref)) else "DIFFERENT"
    else:
        ok = "debug"
    print(f"{name:44s} {best:8.3f} ms  {rows/best/1e6:7.1f} Grows/s  {24*rows/best/1e6:7.1f} GB/s  frac {24*rows/best/1e6/6572.2:.3f}  groups {res.num_rows}  {ok}", flush=True)


print(f"rows {rows} keys {n_keys} reps {reps}", flush=True)
run("plain RED kernel, no L2 window", DBX_AGG_L2_PERSIST=0)
run("plain RED kernel, L2 window")
run("plain kernel front end only (dbg 2)", DBX_AGG_DEBUG=2)
run("plain kernel probe only (dbg 1)", DBX_AGG_DEBUG=1)
