"""Times the phases of the two-pass aggregation of configs[1] (filter v % 3 = 0, sum / count / avg GROUP BY k)
separately: pass 1 (filter_partition_kernel, or its build for the plan dbx_jit_agg_part), pass 2 (slice_agg_kernel or
dbx_jit_agg_slice, or the fused kernel per L2 region for tables with too many slices) and the deferred rows (the fused kernel over a row list), each against its byte
floor at the data-sheet HBM bandwidth and at the copy rate this card reaches (a device-to-device torch copy_
that reads and writes 4 GiB each, best of five, timed with CUDA events).  Kernel times come from torch.profiler
(CUDA activities) over `steps` queries after one warm-up query; the card's name, power limit and SM clock are
printed with them, and the operator's variant text says which pass-1 kernel ran (DBX_AGG_PART_RING=0: the
plain kernel instead of the bulk-copy ring).
usage: python experiments/agg_two_pass_phases.py [rows] [n_keys] [steps]"""
import collections
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databend_b200 import abi, build, lib, expr as E
from databend_b200.block import Column, DataBlock
from databend_b200.transforms import AggregatorParams, DeviceBuffer, TransformFinalAggregate, TransformPartialAggregate

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet

rows = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000_000
n_keys = int(sys.argv[2]) if len(sys.argv) > 2 else 1_000_000
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
build.build()
L = lib.load()
lib.require_device()
card = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
bufs = [DeviceBuffer(rows * 8) for _ in range(3)]
lib.check(L.dbx_synth_fill(0, 0, 42, n_keys, 0, rows, bufs[0].ptr))
lib.check(L.dbx_synth_fill(0, 1, 43, 0, 0, rows, bufs[1].ptr))
lib.check(L.dbx_synth_fill(0, 2, 44, 20, 0, rows, bufs[2].ptr))
blk = DataBlock([Column.device(abi.I64, rows, bufs[0].ptr), Column.device(abi.I64, rows, bufs[1].ptr),
                 Column.device(abi.F64, rows, bufs[2].ptr)], rows)
survivors = 0
step = 1 << 27
for i in range(0, rows, step):  # rows passing the filter, counted on the device in slices of the v column
    m = min(step, rows - i)
    t = torch.empty(m, dtype=torch.int64, device="cuda:0")
    lib.check(L.dbx_memcpy_d2d(0, t.data_ptr(), bufs[1].ptr + 8 * i, 8 * m))
    survivors += int(((t % 3) == 0).sum())
    del t
params = AggregatorParams([0], [("sum", 1), ("count", 1), ("avg", 2)])
filt = E.eq(E.col(1) % E.lit(3), E.lit(0))
types = [abi.I64, abi.I64, abi.F64]
part = TransformPartialAggregate(params, types, filt)
fin = TransformFinalAggregate(params, types)


def copy_rate():
    """bytes per second a device-to-device copy moves (read + write) on this card"""
    n = 4 << 30
    src = torch.empty(n, dtype=torch.uint8, device="cuda:0").fill_(1)
    dst = torch.empty_like(src)
    dst.copy_(src)
    best = float("inf")
    for _ in range(5):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        dst.copy_(src)
        t1.record()
        t1.synchronize()
        best = min(best, t0.elapsed_time(t1) / 1e3)
    del src, dst
    torch.cuda.empty_cache()
    return 2 * n / best


def query():
    part.reset(); fin.reset()
    part.transform(blk)
    fin.transform(part.on_finish())
    out = fin.on_finish(abi.MEM_DEVICE)
    g = out[0].num_rows
    L.dbx_block_release(C.byref(out[0]))
    return g


copy_bytes_per_s = copy_rate()
query()
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
        groups = query()
    torch.cuda.synchronize()
ms = collections.defaultdict(float)
for e in prof.events():
    if e.device_type == torch.autograd.DeviceType.CUDA:
        name = e.name
        if "filter_partition_kernel" in name or "filter_partition_ring_kernel" in name or "dbx_jit_agg_part" in name:
            key = "pass1 filter_partition_kernel"
        elif "slice_agg_kernel" in name or "dbx_jit_agg_slice" in name:
            key = "pass2 slice_agg_kernel"
        elif "filter_group_agg_kernel" in name and "true" in name.split(",")[2]:
            key = "deferred rows (fused kernel, row list)"
        elif "filter_group_agg" in name or "dbx_jit_agg" in name:
            key = "fused kernel (direct rows)"
        else:
            key = "other: " + name.split("(")[0][:60]
        ms[key] += e.device_time_total / 1e3 / steps
variant = part.kernel_variant()
part.close(); fin.close()
table_bytes = (2 ** 21 + 2) * 32  # config 2's default table: 2^21 slots x (key + 3 state words)
chunks = (rows + (1 << 28) - 1) >> 28
moved = {
    "pass1 filter_partition_kernel": 24 * rows + 24 * survivors,
    "pass2 slice_agg_kernel": 24 * survivors + 2 * table_bytes * chunks,
}
floors = {k: b / HBM_BYTES_PER_S * 1e3 for k, b in moved.items()}
copy_floors = {k: b / copy_bytes_per_s * 1e3 for k, b in moved.items()}
ring = variant.split("pass 1 on the bulk-copy ring: ")[1].split(";")[0] if "bulk-copy ring" in variant else "n/a"
report = {"card": card, "rows": rows, "keys": n_keys, "survivors": survivors, "groups": groups, "steps": steps, "kernel_variant": variant,
          "pass1_on_ring": ring, "copy_rate_TB/s": round(copy_bytes_per_s / 1e12, 3),
          "ms_per_query": {k: round(x, 3) for k, x in sorted(ms.items())},
          "floor_ms_at_3.35TB/s": {k: round(x, 3) for k, x in floors.items()},
          "share_of_floor": {k: round(floors[k] / ms[k], 3) for k in floors if ms.get(k)},
          "floor_ms_at_copy_rate": {k: round(x, 3) for k, x in copy_floors.items()},
          "share_of_copy_rate_floor": {k: round(copy_floors[k] / ms[k], 3) for k in copy_floors if ms.get(k)}}
print(json.dumps(report, indent=1), flush=True)
