"""Per-operator measurements for the configs that are not bench.py's headline line:
configs[2] hash join, configs[3] top-k, configs[0]-style standalone filter.  One JSON line per
operator; under torchrun the join is hash-partitioned across the ranks (one all-to-all per side
and column over NCCL) and the top-k is row-range partitioned + all-gather + final merge.
Timing: CUDA events on the operator's stream where one kernel dominates, host wall clock (with
device synchronisation on both sides, max over ranks) for the multi-step paths."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from databend_b200 import abi, expr as E  # noqa: E402
from databend_b200.block import Column, DataBlock, np_dtype  # noqa: E402
from databend_b200.lib import check, load  # noqa: E402
from databend_b200.transforms import DeviceBuffer, HashJoin, TransformFilter, TransformTopN  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--ops", default="join,topk,sort,filter,eval")
ap.add_argument("--sort-rows", type=int, default=250_000_000)
ap.add_argument("--join-shuffle", default="peer", choices=["peer", "nccl"])
ap.add_argument("--join-kind", default="inner", choices=["inner", "left", "right", "right_semi", "right_anti", "full"])
# key layout of the join (the same unique key either way): one Int64 column; split into two Int32
# columns (lo, hi; the 64-bit packed key); or two Int64 columns (k, -k; the 128-bit packed key)
ap.add_argument("--join-keys", default="i64", choices=["i64", "2xi32", "2xi64"])
ap.add_argument("--round-rows", type=int, default=32 << 20)
ap.add_argument("--fact-rows", type=int, default=1_000_000_000)
ap.add_argument("--dim-rows", type=int, default=10_000_000)
ap.add_argument("--topk-rows", type=int, default=1_000_000_000)
# ORDER BY keys of the top-k leg: "f64" (one key), "f64,i64" (a high-cardinality first key) or
# "i8,f64" (7 distinct first-key values: the later key is read for most rows); single GPU only
# for several keys
ap.add_argument("--topk-keys", default="f64", choices=["f64", "f64,i64", "i8,f64"])
ap.add_argument("--filter-rows", type=int, default=500_000_000)
ap.add_argument("--block-rows", type=int, default=1 << 26)
ap.add_argument("--reps", type=int, default=3)
a = ap.parse_args()
L = load()
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
dev = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(dev)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
HBM = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
    os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 6650.0


def sync_all():
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        torch.cuda.synchronize()


def max_over_ranks(x):
    if world == 1:
        return x
    t = torch.tensor([x], dtype=torch.float64, device=f"cuda:{dev}")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def fill(kind, seed, aa, first, n, width=8):
    b = DeviceBuffer(max(1, n * width), dev)
    check(L.dbx_synth_fill(dev, kind, seed, aa, first, n, b.ptr))
    return b


def emit(d):
    if rank == 0:
        print(json.dumps(d), flush=True)


ops = a.ops.split(",")

if "join" in ops:
    # configs[2]: fact(fk uniform over the dim keys, fv) JOIN dim(dk = 0..D-1 hashed anyway, dv); every fact row matches once.
    # The other kinds use a second dim variant: every 10th dim key is moved out of the facts' range
    # (dk = i + D for i % 10 == 9), so 10 % of the dim rows are never matched (RIGHT / RIGHT ANTI /
    # FULL have a final stream) and 10 % of the fact rows find no dim row.
    join_kind = {"inner": abi.JOIN_INNER, "left": abi.JOIN_LEFT, "right": abi.JOIN_RIGHT, "right_semi": abi.JOIN_RIGHT_SEMI,
                 "right_anti": abi.JOIN_RIGHT_ANTI, "full": abi.JOIN_FULL}[a.join_kind]
    F, D = a.fact_rows, a.dim_rows
    f0, f1 = F * rank // world, F * (rank + 1) // world
    d0, d1 = D * rank // world, D * (rank + 1) // world
    nf, nd = f1 - f0, d1 - d0
    fk, fv = fill(0, 7, D, f0, nf), fill(1, 8, 0, f0, nf)
    dk = DeviceBuffer(max(1, nd * 8), dev)
    dkeys = np.arange(d0, d1, dtype=np.int64)
    if join_kind != abi.JOIN_INNER:
        dkeys[dkeys % 10 == 9] += D
    dk.upload(dkeys)
    dv = fill(1, 9, 0, d0, nd)
    key_hold = []  # device tensors behind the derived key columns

    def key_cols(buf, n):
        """the join key columns of one side in the --join-keys layout (the first one is unique: the shuffle key)"""
        if a.join_keys == "i64":
            return [Column.device(abi.I64, n, buf.ptr)]
        from databend_b200.distributed import _dev_tensor
        k = _dev_tensor(buf.ptr, n * 8, dev).view(torch.int64)
        if a.join_keys == "2xi32":
            parts, dt = [(k & 0xFFFFFFFF).to(torch.int32), (k >> 32).to(torch.int32)], abi.I32
        else:
            parts, dt = [k.clone(), -k], abi.I64
        key_hold.extend(parts)
        return [Column.device(dt, n, t.data_ptr()) for t in parts]
    dim_keys, fact_keys = key_cols(dk, nd), key_cols(fk, nf)
    torch.cuda.synchronize(dev)
    n_keys = len(dim_keys)
    key_ids = list(range(n_keys)) if n_keys > 1 else 0
    side_types = [c.dtype for c in dim_keys] + [abi.I64]
    key_bytes = sum(np_dtype(c.dtype).itemsize for c in fact_keys)
    dim = DataBlock(dim_keys + [Column.device(abi.I64, nd, dv.ptr)], nd)
    fact = DataBlock(fact_keys + [Column.device(abi.I64, nf, fv.ptr)], nf)
    best = None
    best_stats = None
    pj = None
    if world > 1 and a.join_shuffle == "peer":  # collective set-up (receive buffers, IPC mapping) once, outside the timed region
        from databend_b200.distributed import PartitionedHashJoin
        mx = torch.tensor([nd, nf], dtype=torch.int64, device=f"cuda:{dev}")
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        pj = PartitionedHashJoin(side_types, side_types, key_ids, key_ids, dev, rank, world, int(mx[0]), int(mx[1]), a.round_rows, kind=join_kind)
    for rep in range(a.reps):
        sync_all()
        t0 = time.perf_counter()
        keep = None
        if world > 1 and a.join_shuffle == "peer":
            st = {}
            outs, j = pj.run(dim, fact, abi.MEM_DEVICE, st)
            out_rows = 0
            for ob in outs:
                out_rows += ob.num_rows
                L.dbx_block_release(C.byref(ob))
            sync_all()
            total = time.perf_counter() - t0
            j.close()
            rec = (max_over_ranks(total), max_over_ranks((st["shuffle_send"] + st["shuffle_wait"]) * 1e-3), max_over_ranks(st["build"] * 1e-3),
                   max_over_ranks(st["probe"] * 1e-3), max_over_ranks(st["probe"]), out_rows, max_over_ranks(st["final_probe"]))
            if best is None or rec[0] < best[0]:
                best = rec
                best_stats = {k_: max_over_ranks(v_) for k_, v_ in st.items()}
            continue
        if world > 1:
            from databend_b200.distributed import shuffle_by_key
            dim_l, k1 = shuffle_by_key(dim, 0, dev)
            fact_l, k2 = shuffle_by_key(fact, 0, dev)
            keep = (k1, k2)
            torch.cuda.synchronize()
        else:
            dim_l, fact_l = dim, fact
        t_shuffle = time.perf_counter() - t0
        j = HashJoin(side_types, side_types, key_ids, key_ids, dev, join_kind)
        tb = time.perf_counter()
        j.add_block(dim_l)
        j.final_build()
        j.synchronize()
        t_build = time.perf_counter() - tb
        tp = time.perf_counter()
        out_rows, probe_ms = 0, 0.0
        for s in range(0, fact_l.num_rows, a.block_rows):
            blk = fact_l.slice(s, min(s + a.block_rows, fact_l.num_rows))
            outs = j.probe_block(blk, abi.MEM_DEVICE)
            probe_ms += j.last_kernel_ms()
            for ob in outs:
                out_rows += ob.num_rows
                L.dbx_block_release(C.byref(ob))
        # Join::final_probe (build-side kinds): a counting pass over the matched map, then, when rows
        # are selected, the compacting pass; both are timed with events (kernel_ms(0) is the last)
        final_ms = 0.0
        if join_kind >= abi.JOIN_RIGHT:
            fouts = j.final_probe(abi.MEM_DEVICE)
            final_ms = j.kernel_ms(0) + (j.kernel_ms(1) if fouts else 0.0)
            for ob in fouts:
                out_rows += ob.num_rows
                L.dbx_block_release(C.byref(ob))
        j.synchronize()
        t_probe = time.perf_counter() - tp
        sync_all()
        total = time.perf_counter() - t0
        j.close()
        del keep
        rec = (max_over_ranks(total), max_over_ranks(t_shuffle), max_over_ranks(t_build), max_over_ranks(t_probe), max_over_ranks(probe_ms), out_rows,
               max_over_ranks(final_ms))
        if best is None or rec[0] < best[0]:
            best = rec
    if pj is not None:
        pj.close()
    total, t_shuffle, t_build, t_probe, probe_ms, out_rows, final_ms = best
    ot = torch.tensor([out_rows], dtype=torch.int64, device=f"cuda:{dev}")
    if world > 1:
        dist.all_reduce(ot)
    rows_per_gpu = F / world
    kind_fields = {} if join_kind == abi.JOIN_INNER else {
        "join_kind": a.join_kind, "final_probe_ms": final_ms,
        "dim_variant": "every 10th dim key moved out of the facts' range: 10 % of dim rows unmatched, 10 % of fact rows without a dim row",
        "final_probe_timing": "multi-GPU: host wall clock of final_probe per rank" if world > 1 and a.join_shuffle == "peer" else
                              "CUDA events: counting pass + compacting pass of the final scan (probe_kernel_ms covers the probe blocks only)"}
    key_fields = {} if a.join_keys == "i64" else {
        "join_keys": a.join_keys, "key_bytes_per_fact_row": key_bytes,
        "key_layout": "two Int32 columns (lo, hi) of the unique key: 64-bit packed key" if a.join_keys == "2xi32" else
                      "two Int64 columns (k, -k): 128-bit packed key, one inlined build column"}
    emit({"op": "hash_join", "workload": "configs[2]: fact 1e9 x dim 1e7 inner join on int64 key, (fk, fv, dk, dv) materialised", "n_gpus": world, **kind_fields, **key_fields,
          "fact_rows": F, "dim_rows": D, "joined_rows": int(ot.item()), "rows_per_s": F / total, "total_ms": total * 1e3,
          "shuffle_ms": t_shuffle * 1e3, "build_ms": t_build * 1e3, "probe_wall_ms": t_probe * 1e3, "probe_kernel_ms": probe_ms,
          "roofline": {"bound": "hbm", "bytes_per_fact_row": 64, "note": "read fk,fv (16) + table bucket (32-byte sector) + write 4 x 8 (32) = 80 with dk materialised; 56 by SURVEY 8d (3 output columns, dim row gather)",
                       "achieved_GBs_per_gpu": 56.0 * rows_per_gpu / (probe_ms * 1e-3) / 1e9, "peak": HBM, "frac": 56.0 * rows_per_gpu / (probe_ms * 1e-3) / 1e9 / HBM},
          "shuffle_phases_ms": best_stats,
          "parallelism": "single GPU" if world == 1 else (f"hash-partition x{world}: fused partition + store-to-peer kernel over NVLink (dbx_shuffle), {a.round_rows} rows per rank and round" if a.join_shuffle == "peer" else f"hash-partition x{world}: dbx_hash_partition + NCCL all-to-all per side and column")})
    for b_ in (fk, fv, dk, dv):
        b_.free()

if "topk" in ops and a.topk_keys != "f64" and world == 1:
    # ORDER BY k0, k1 LIMIT 1000 (streaming top-k on the composite image) next to the single-key
    # top-k over the same first column in the same run
    N = a.topk_rows
    from databend_b200.distributed import _dev_tensor
    hold = []
    if a.topk_keys == "f64,i64":
        b0, b1 = fill(3, 11, 0, 0, N), fill(1, 12, 0, 0, N)
        c0, c1 = Column.device(abi.F64, N, b0.ptr), Column.device(abi.I64, N, b1.ptr)
        types, widths = [abi.F64, abi.I64], (8, 8)
    else:
        kb = fill(0, 13, 7, 0, N)  # uniform over 0..6
        t8 = _dev_tensor(kb.ptr, N * 8, dev).view(torch.int64).to(torch.int8)
        kb.free()
        hold.append(t8)
        b1 = fill(3, 11, 0, 0, N)
        c0, c1 = Column.device(abi.I8, N, t8.data_ptr()), Column.device(abi.F64, N, b1.ptr)
        types, widths = [abi.I8, abi.F64], (1, 8)

    def run_leg(op, blk):
        best, kms, res = None, None, None
        for rep in range(a.reps + 1):
            op.reset()
            sync_all()
            t0 = time.perf_counter()
            op.transform(blk)
            res = op.on_finish()
            k_ms = op.last_kernel_ms()
            sync_all()
            dt = time.perf_counter() - t0
            if rep and (best is None or dt < best):
                best, kms = dt, k_ms
        op.close()
        return best * 1e3, kms, res

    multi_ms, multi_kms, res = run_leg(TransformTopN(0, True, False, 1000, types, dev, extra_keys=[(1, True, False)]), DataBlock([c0, c1], N))
    single_ms, single_kms, _ = run_leg(TransformTopN(0, True, False, 1000, types[:1], dev), DataBlock([c0], N))
    PEAK = 3350.0  # H100 SXM HBM3 GB/s
    rows = res.columns[1].values()
    emit({"op": "topk_multi_key", "keys": a.topk_keys, "workload": f"ORDER BY {a.topk_keys.replace(',', ', ')} LIMIT 1000", "rows": N,
          "total_ms": multi_ms, "scan_ms_incl_candidate_cuts": multi_kms,
          "floor_first_key": {"bytes_per_row": widths[0], "ms": widths[0] * N / PEAK / 1e6, "frac_of_3350GBs": widths[0] * N / (multi_kms * 1e-3) / 1e9 / PEAK},
          "floor_all_keys": {"bytes_per_row": sum(widths), "ms": sum(widths) * N / PEAK / 1e6, "frac_of_3350GBs": sum(widths) * N / (multi_kms * 1e-3) / 1e9 / PEAK},
          "single_key_same_first_column": {"total_ms": single_ms, "scan_ms_incl_candidate_cuts": single_kms},
          "result_rows_sum": int(rows.sum()), "result_rows_head": [int(x) for x in rows[:4]]})
    for b_ in (b0, b1) if a.topk_keys == "f64,i64" else (b1,):
        b_.free()
    ops = [o for o in ops if o != "topk"]

if "topk" in ops:
    N = a.topk_rows
    r0, r1 = N * rank // world, N * (rank + 1) // world
    n = r1 - r0
    xb = fill(3, 11, 0, r0, n)
    col = Column.device(abi.F64, n, xb.ptr)
    op = TransformTopN(0, True, False, 1000, [abi.F64], dev)
    fop = TransformTopN(0, True, False, 1000, [abi.F64], dev) if world > 1 else None
    best, kms = None, None
    for rep in range(a.reps + 1):
        op.reset()
        sync_all()
        t0 = time.perf_counter()
        op.transform(DataBlock([col], n))
        if world > 1:
            from databend_b200.distributed import topk_merge_device
            res = topk_merge_device(op, r0, 1000, fop, dev)
        else:
            res = op.on_finish()
        k_ms = op.last_kernel_ms()
        sync_all()
        dt = max_over_ranks(time.perf_counter() - t0)
        if rep and (best is None or dt < best):
            best, kms = dt, max_over_ranks(k_ms)
    op.close()
    emit({"op": "topk", "workload": "configs[3]: ORDER BY float64 LIMIT 1000 over 1e9 rows", "n_gpus": world, "rows": N, "rows_per_s": N / best,
          "total_ms": best * 1e3, "scan_ms_incl_candidate_cuts": kms, "first_key": float(res.columns[0].values()[0]),
          "roofline": {"bound": "hbm", "bytes_per_row": 8, "achieved_GBs_per_gpu": 8.0 * n / (kms * 1e-3) / 1e9, "peak": HBM,
                       "frac": 8.0 * n / (kms * 1e-3) / 1e9 / HBM},
          "parallelism": "single GPU" if world == 1 else f"row ranges x{world} + device all-gather of 1000 candidates per rank + final top-k"})
    xb.free()

if "sort" in ops and world == 1:
    # ORDER BY float64 without LIMIT: hand-written onesweep LSD radix sort of (ordered key, row id)
    n = a.sort_rows
    xb = fill(3, 13, 0, 0, n)
    col = Column.device(abi.F64, n, xb.ptr)
    op = TransformTopN(0, True, False, 0, [abi.F64], dev)
    best = None
    for rep in range(a.reps):
        op.reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        op.transform(DataBlock([col], n))
        op.finish()
        ob = op.pull_c(abi.MEM_DEVICE)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        first = DeviceBuffer.__new__(DeviceBuffer)
        first.device, first.nbytes, first.ptr = dev, 16, ob.cols[0].data
        head = first.download(np.float64, 2)
        first.ptr = 0
        L.dbx_block_release(C.byref(ob))
        if best is None or dt < best:
            best = dt
    op.close()
    # 8 digit passes x (8 + 4 B read + 8 + 4 B written) + one histogram read + ingest/emit
    emit({"op": "sort", "workload": "ORDER BY float64 (no LIMIT): full device radix sort, keys + row ids out", "rows": n,
          "rows_per_s": n / best, "total_ms": best * 1e3, "first_keys": [float(head[0]), float(head[1])],
          "roofline": {"bound": "hbm", "bytes_per_row": 8 * 24 + 8 + 28 + 24, "note": "8 LSD passes x 24 B + histogram 8 B + ingest (8 read, 20 written) + emit (12 + 8 gather read, 16 written)",
                       "achieved_GBs": (8 * 24 + 8 + 28 + 24 + 12) * n / best / 1e9, "peak": HBM, "frac": (8 * 24 + 8 + 28 + 36) * n / best / 1e9 / HBM}})
    xb.free()

if "filter" in ops and world == 1:
    n = a.filter_rows
    kb, vb, xb = fill(0, 1, 1_000_000, 0, n), fill(1, 2, 0, 0, n), fill(2, 3, 20, 0, n)
    blk = DataBlock([Column.device(abi.I64, n, kb.ptr), Column.device(abi.I64, n, vb.ptr), Column.device(abi.F64, n, xb.ptr)], n)
    op = TransformFilter(E.eq(E.col(1) % E.lit(3), E.lit(0)), [abi.I64, abi.I64, abi.F64], dev)
    best, rows_out = None, 0
    for rep in range(a.reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        op.push(blk)
        ob = op.pull_c(abi.MEM_DEVICE)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        kms = op.last_kernel_ms()
        rows_out = ob.num_rows
        L.dbx_block_release(C.byref(ob))
        if rep and (best is None or kms < best[1]):
            best = (dt, kms)
    op.close()
    moved = 8.0 * n + 24.0 * n + 24.0 * rows_out  # predicate column + every column read once + selected rows written
    emit({"op": "filter", "workload": "WHERE v % 3 = 0 over (k,v,x) int64/int64/float64, order-preserving select + take", "rows": n,
          "rows_out": rows_out, "rows_per_s": n / (best[1] * 1e-3), "kernel_ms": best[1], "wall_ms": best[0] * 1e3,
          "roofline": {"bound": "hbm", "algorithmic_bytes": moved, "achieved_GBs": moved / (best[1] * 1e-3) / 1e9, "peak": HBM,
                       "frac": moved / (best[1] * 1e-3) / 1e9 / HBM}})

if "eval" in ops and world == 1:
    # Evaluator::run of one nested expression over device-resident columns: (k * v + v) % 7 > cast(x / 3 as Int64) and v > 5
    from databend_b200 import scalar_expr as sx
    n = a.filter_rows
    kb, vb, xb = fill(0, 1, 1_000_000, 0, n), fill(1, 2, 0, 0, n), fill(2, 3, 20, 0, n)
    blk = DataBlock([Column.device(abi.I64, n, kb.ptr), Column.device(abi.I64, n, vb.ptr), Column.device(abi.F64, n, xb.ptr)], n)
    k_, v_, x_ = sx.col(0), sx.col(1), sx.col(2)
    e = sx.call("and", sx.call("gt", sx.cast((k_ * v_ + v_) % sx.lit(7, abi.U8), abi.I64), sx.cast(x_ / sx.lit(3, abi.U8), abi.I64)), sx.call("gt", v_, sx.lit(5, abi.I64)))
    best = None
    for rep in range(a.reps + 2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ob, odt = sx.eval_scalar(blk, e, dev, abi.MEM_DEVICE)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        L.dbx_block_release(C.byref(ob))
        if rep and (best is None or dt < best):
            best = dt
    moved = 24.0 * n + n / 8.0  # three 8-byte columns read once, one Boolean bitmap written
    emit({"op": "eval_scalar", "workload": "(k * v + v) % 7 > CAST(x / 3 AS Int64) AND v > 5 over int64/int64/float64 (11-node tree, one fused kernel + bit packing)",
          "rows": n, "rows_per_s": n / best, "wall_ms": best * 1e3, "timing": "host wall clock around dbx_eval_scalar (stream create, launch, first-error read-back, synchronise)",
          "roofline": {"bound": "hbm", "algorithmic_bytes": moved, "achieved_GBs": moved / best / 1e9, "peak": HBM, "frac": moved / best / 1e9 / HBM,
                       "note": "the reference materialises one column per tree node: 11 passes over memory"}})

if world > 1:
    dist.barrier()
    dist.destroy_process_group()
