"""Hash join with a residual (non-equi) ON condition, on device-resident inputs at config-3 sizes.

  band_fused    fact (fk Int64 uniform over the dim keys, ts Int64 in [0, 1000)) INNER JOIN dim (dk unique,
                lo in [0, 900), hi = lo + 100) ON fk = dk AND ts BETWEEN lo AND hi, the band evaluated inside
                the probe (dbx_op_create_join); about 10 % of the fact rows match;
  band_filter   the same join without the residual, then DBX_OP_FILTER (ts >= lo AND ts <= hi) on every
                materialised output block: the write and re-read of the candidate pairs the fused form saves;
  equi          the join without the residual (its output is every candidate pair);
  q21_semi / q21_anti   TPC-H Q21's EXISTS / NOT EXISTS shape: fact (ok, supp) LEFT SEMI / ANTI JOIN a build
                side with about four lines per order ON ok = ok AND b.supp <> p.supp (ten suppliers).
Per mode: the probe kernels' device time (CUDA events summed over the fact blocks; band_filter adds the
filter kernels) and fact rows per second of that time, best of --reps, modes interleaved per repetition.
band_fused and band_filter must return the same rows (count and sum of ts)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from databend_b200 import abi, expr as E, scalar_expr as S  # noqa: E402
from databend_b200.block import Column, DataBlock  # noqa: E402
from databend_b200.distributed import _dev_tensor  # noqa: E402
from databend_b200.lib import check, load  # noqa: E402
from databend_b200.transforms import DeviceBuffer, HashJoin, TransformFilter  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--fact-rows", type=int, default=1_000_000_000)
ap.add_argument("--dim-rows", type=int, default=10_000_000)
ap.add_argument("--block-rows", type=int, default=1 << 26)
ap.add_argument("--reps", type=int, default=2)
ap.add_argument("--modes", default="band_fused,band_filter,equi,q21_semi,q21_anti")
a = ap.parse_args()
L = load()
dev = 0
torch.cuda.set_device(dev)
F, D = a.fact_rows, a.dim_rows
I64 = abi.I64


def fill(kind, seed, aa, n):
    b = DeviceBuffer(max(1, n * 8), dev)
    check(L.dbx_synth_fill(dev, kind, seed, aa, 0, n, b.ptr))
    return b


def tensor(buf, n):
    return _dev_tensor(buf.ptr, n * 8, dev).view(torch.int64)


def dcol(buf, n):
    return Column.device(I64, n, buf.ptr)


# band join inputs
fk, fts = fill(0, 7, D, F), fill(0, 8, 1000, F)
dk, dlo, dhi = DeviceBuffer(D * 8, dev), fill(0, 9, 900, D), DeviceBuffer(D * 8, dev)
g = torch.Generator(device=f"cuda:{dev}").manual_seed(3)
tensor(dk, D).copy_(torch.randperm(D, device=f"cuda:{dev}", generator=g))
tensor(dhi, D).copy_(tensor(dlo, D) + 100)
dim = DataBlock([dcol(dk, D), dcol(dlo, D), dcol(dhi, D)], D)
fact = DataBlock([dcol(fk, F), dcol(fts, F)], F)
# Q21 inputs: about four build lines per order, ten suppliers
NO = max(1, D // 4)
qk, qs = fill(0, 11, NO, D), fill(0, 12, 10, D)
pk, ps = fill(0, 13, NO, F), fill(0, 14, 10, F)
q_build = DataBlock([dcol(qk, D), dcol(qs, D)], D)
q_fact = DataBlock([dcol(pk, F), dcol(ps, F)], F)

BAND = S.call("and", S.call("gte", S.col(3 + 1), S.col(1)), S.call("lte", S.col(3 + 1), S.col(2)))
NOTEQ = S.call("noteq", S.col(1), S.col(2 + 1))
torch.cuda.synchronize()


def drain(j, out, filt=None):
    """Pull every joined block; with filt, push it through the filter first.  Returns the filter's kernel ms."""
    ms = 0.0
    while True:
        ob = j.pull_c(abi.MEM_DEVICE)
        if ob is None:
            return ms
        if filt is not None and ob.num_rows:
            check(L.dbx_op_push(filt.handle, C.byref(ob)), filt.handle)
            fo = filt.pull_c(abi.MEM_DEVICE)
            filt.inputs_consumed()
            ms += filt.last_kernel_ms()
            check(L.dbx_block_release(C.byref(ob)))
            if fo is None:
                continue
            ob = fo
        n = ob.num_rows
        if n:
            out[0] += n
            out[1] += int(_dev_tensor(ob.cols[1].data, n * 8, dev).view(torch.int64).sum().item())
        check(L.dbx_block_release(C.byref(ob)))


def run(mode):
    torch.cuda.synchronize()
    if mode.startswith("q21"):
        build, probe, pred = q_build, q_fact, NOTEQ
        kind = abi.JOIN_LEFT_SEMI if mode == "q21_semi" else abi.JOIN_LEFT_ANTI
    else:
        build, probe, kind = dim, fact, abi.JOIN_INNER
        pred = BAND if mode == "band_fused" else None
    bt, pt = [I64] * build.num_columns(), [I64] * probe.num_columns()
    j = HashJoin(bt, pt, 0, 0, dev, kind=kind, other_predicate=pred)
    j.add_block(build)
    j.final_build()
    filt = None
    if mode == "band_filter":  # output (fk, ts, dk, lo, hi)
        filt = TransformFilter(E.and_(E.ge(E.col(1), E.col(3)), E.le(E.col(1), E.col(4))), [I64] * 5, dev)
    out = [0, 0]
    probe_ms = filter_ms = 0.0
    t0 = time.perf_counter()
    for s in range(0, F, a.block_rows):
        blk = probe.slice(s, min(s + a.block_rows, F))
        b, keep = blk.as_c()
        check(L.dbx_join_probe(j.handle, C.byref(b)), j.handle)
        probe_ms += j.last_kernel_ms()
        filter_ms += drain(j, out, filt)
        del keep
    j.synchronize()
    wall = time.perf_counter() - t0
    if filt:
        filt.close()
    j.close()
    kernel_ms = probe_ms + filter_ms
    return {"probe_kernel_ms": round(probe_ms, 3), "filter_kernel_ms": round(filter_ms, 3), "kernel_ms": round(kernel_ms, 3),
            "fact_rows_per_s": F / (kernel_ms / 1e3) if kernel_ms else None, "probe_wall_ms": round(wall * 1e3, 1),
            "rows": out[0], "sum_col1": out[1]}


def gpu_name():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


modes = a.modes.split(",")
for m in modes:  # warm-up: module load, pools, every kernel instantiation the timed runs use
    run(m)
best = {}
for rep in range(a.reps):
    for m in modes:
        r = run(m)
        if m not in best or r["kernel_ms"] < best[m]["kernel_ms"]:
            best[m] = r
if "band_fused" in best and "band_filter" in best:
    assert (best["band_fused"]["rows"], best["band_fused"]["sum_col1"]) == (best["band_filter"]["rows"], best["band_filter"]["sum_col1"])
print(json.dumps({"op": "join_residual", "gpu": gpu_name(), "fact_rows": F, "dim_rows": D, "block_rows": a.block_rows,
                  "reps": a.reps, "modes": best}), flush=True)
