"""Window-function benchmark: DBX_OP_WINDOW over device-generated (seeded, dbx_synth_fill) columns.

Shapes (2^28 rows by default):
  partition  PARTITION BY k (1e6 keys) ORDER BY t: row_number, rank, running sum(v), lag(v)
  running    no PARTITION BY, ORDER BY t: running sum(v)
  moving     PARTITION BY k ORDER BY t: avg(x) ROWS BETWEEN 100 PRECEDING AND CURRENT ROW over Float64
k is uniform in [0, 1e6), t a permutation of the rows, v uniform 32-bit integers as Int64, x uniform
[0, 1) doubles.  The columns are pushed as device blocks of 2^24 rows and the result stays on the device.

Per shape one JSON line: rows/s over push + finish, and the device ms of each phase: ingest (the
pushes: one device copy per block; host clock around the pushes and a synchronise), sort (key images
+ stable radix sorts), scans (boundary kernel + partition / peer index scans), emit (argument gathers,
aggregate scans, one emit kernel per function), gather (the input columns into window order; the call
is synchronous, so this is its wall time).  The times are medians over --steps runs after --warmup.
For the non-sort phases, algorithmic bytes (the reads and writes the phase needs at least, computed
below from the shape) over the phase's time, against the H100 SXM data sheet's 3.35 TB/s HBM3.  The
card's name and power limit are read by the same process; without a GPU nothing is measured."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databend_b200 import abi, lib  # noqa: E402
from databend_b200.block import Column, DataBlock  # noqa: E402
from databend_b200.transforms import TransformWindow, WindowFunc  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BLOCK = 1 << 24

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=1 << 28)
ap.add_argument("--keys", type=int, default=1_000_000)
ap.add_argument("--steps", type=int, default=3)
ap.add_argument("--warmup", type=int, default=1)
ap.add_argument("--shapes", default="partition,running,moving")
a = ap.parse_args()

L = lib.load()
lib.require_device()
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
n = a.rows


def synth(kind, seed, arg):
    p = C.c_void_p()
    lib.check(L.dbx_device_alloc(0, n * 8, C.byref(p)))
    lib.check(L.dbx_synth_fill(0, kind, seed, arg, 0, n, p))
    return p


bufs = {"k": synth(0, 1, a.keys), "t": synth(5, 2, max(1, (n - 1).bit_length())), "v": synth(1, 3, 0), "x": synth(3, 4, 0)}
lib.check(L.dbx_device_synchronize(0))
DTYPES = {"k": abi.I64, "t": abi.I64, "v": abi.I64, "x": abi.F64}

SHAPES = {
    "partition": (["k", "t", "v"], [0], [(1, True, False)],
                  [WindowFunc("row_number"), WindowFunc("rank"), WindowFunc("sum", arg=2, frame=("rows", "unbounded_preceding", "current_row")),
                   WindowFunc("lag", arg=2, n=1)]),
    "running": (["t", "v"], [], [(0, True, False)], [WindowFunc("sum", arg=1, frame=("rows", "unbounded_preceding", "current_row"))]),
    "moving": (["k", "t", "x"], [0], [(1, True, False)], [WindowFunc("avg", arg=2, frame=("rows", ("preceding", 100), "current_row"))]),
}


def algorithmic_bytes(names, n_part, n_order, funcs):
    """Least bytes the non-sort phases move, from the shape."""
    nk = n_part + n_order
    scans = n * (4 + nk * 2 * 12 + 6) + 5 * n * (2 * 1 + 4)  # boundary kernel; five index scans (flags read twice, u32 written)
    emit = 0
    for f in funcs:
        out = 8 + (1 if f.name in ("sum", "avg", "lag") else 0)
        emit += n * (5 * 4 + out)                      # row indices read, value (+ validity byte) written
        if f.arg >= 0:
            emit += n * (4 + 8 + 9)                    # row id, argument value read, gathered value + validity written
            if f.name in ("sum", "avg"):
                emit += 2 * n * (2 * 9 + 8)            # prefix count and prefix sum scans
                emit += n * 2 * 8                      # frame ends' prefix values
    gather = n * 4 + 2 * n * sum(8 for _ in names)     # row ids, every input column read and written
    return scans, emit, gather


def run_once(names, pb, ob, funcs):
    op = TransformWindow(pb, ob, funcs, [DTYPES[c] for c in names])
    t0 = time.perf_counter()
    for s in range(0, n, BLOCK):
        m = min(BLOCK, n - s)
        cols = [Column.device(DTYPES[c], m, bufs[c].value + s * 8) for c in names]
        op.transform(DataBlock(cols, m))
    lib.check(L.dbx_device_synchronize(0))
    t1 = time.perf_counter()
    op.finish()
    t2 = time.perf_counter()
    phases = [op.kernel_ms(b) for b in (3, 2, 1, 0)]  # sort, scans, emit, gather
    out = op.pull_c(abi.MEM_DEVICE)
    assert out.num_rows == n and out.num_cols == len(names) + len(funcs)
    L.dbx_block_release(C.byref(out))
    op.close()
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3, phases


for shape in a.shapes.split(","):
    names, pb, ob, funcs = SHAPES[shape]
    for _ in range(a.warmup):
        run_once(names, pb, ob, funcs)
    runs = [run_once(names, pb, ob, funcs) for _ in range(a.steps)]
    med = lambda xs: sorted(xs)[len(xs) // 2]
    ingest = med([r[0] for r in runs])
    finish = med([r[1] for r in runs])
    sort_ms, scan_ms, emit_ms, gather_ms = (med([r[2][i] for r in runs]) for i in range(4))
    b_scan, b_emit, b_gather = algorithmic_bytes(names, len(pb), len(ob), funcs)
    frac = lambda b, ms: round(b / (ms * 1e-3) / HBM_BYTES_PER_S, 3) if ms > 0 else None
    print(json.dumps({
        "shape": shape, "rows": n, "keys": a.keys if pb else 0, "functions": [f.name for f in funcs], "card": card,
        "rows_per_s": round(n / ((ingest + finish) * 1e-3)),
        "ms": {"ingest": round(ingest, 2), "sort": round(sort_ms, 2), "bounds_scans": round(scan_ms, 2), "emit": round(emit_ms, 2),
               "gather": round(gather_ms, 2), "finish_wall": round(finish, 2)},
        "hbm_fraction": {"bounds_scans": frac(b_scan, scan_ms), "emit": frac(b_emit, emit_ms), "gather": frac(b_gather, gather_ms)},
        "steps": a.steps}), flush=True)

for p in bufs.values():
    L.dbx_device_free(0, p)
