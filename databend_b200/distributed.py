"""Multi-GPU drivers for the operators that shard across the GPUs of one box (SURVEY 8e).
One process per GPU; torch.distributed (NCCL on GPUs, gloo in the CPU tests) is the plumbing,
every row-touching step is a libdbx kernel.

  hash join   both sides hash-partitioned by key (dbx_hash_partition) -> one all-to-all per side
              and column -> local DBX_OP_JOIN; the result stays partitioned by key
              (reference: flight_scatter_hash.rs + physical_hash_join.rs exchange on the join keys)
  top-k       row-range shards -> local TransformTopN -> all-gather of k candidates per rank ->
              a final TransformTopN over the gathered candidates (sorts/sort_merge*.rs, top_n/)
"""
from __future__ import annotations

import ctypes as C
from typing import List, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import abi
from .block import Column, DataBlock, np_dtype
from .lib import check, load
from .transforms import HashJoin, TransformTopN, schema_types

_TORCH_BYTES = torch.uint8


def hash_partition(block: DataBlock, key_col: int, n_parts: int, device: int = 0) -> Tuple[List[torch.Tensor], List[int]]:
    """dbx_hash_partition over a device-resident block: returns one uint8 tensor per column holding
    the permuted values, and the partition offsets (n_parts + 1)."""
    n = block.num_rows
    outs, ptrs = [], (C.c_void_p * len(block.columns))()
    for i, c in enumerate(block.columns):
        t = torch.empty(max(1, n * np_dtype(c.dtype).itemsize), dtype=_TORCH_BYTES, device=f"cuda:{device}")
        outs.append(t)
        ptrs[i] = t.data_ptr()
    offs = (C.c_int64 * (n_parts + 1))()
    b, keep = block.as_c()
    check(load().dbx_hash_partition(device, C.byref(b), key_col, n_parts, ptrs, offs))
    return outs, list(offs)


def all_to_all_columns(cols: Sequence[torch.Tensor], widths: Sequence[int], offsets: Sequence[int], group=None):
    """One all-to-all per column: `cols[i]` holds rows laid out partition after partition
    (`offsets`), `widths[i]` bytes per value.  Returns (received byte tensors, rows received)."""
    world = dist.get_world_size(group)
    send_counts = [offsets[i + 1] - offsets[i] for i in range(world)]
    dev = cols[0].device
    sc = torch.tensor(send_counts, dtype=torch.int64, device=dev)
    rc = torch.empty_like(sc)
    dist.all_to_all_single(rc, sc, group=group)
    recv_counts = [int(v) for v in rc.tolist()]
    n_recv, n_send = sum(recv_counts), sum(send_counts)
    out = []
    for t, w in zip(cols, widths):
        r = torch.empty(max(1, n_recv * w), dtype=_TORCH_BYTES, device=dev)
        dist.all_to_all_single(r[: n_recv * w], t[: n_send * w], [c * w for c in recv_counts], [c * w for c in send_counts], group=group)
        out.append(r)
    return out, n_recv


def shuffle_by_key(block: DataBlock, key_col: int, device: int, group=None) -> Tuple[DataBlock, list]:
    """Hash-partition a device-resident block and exchange the partitions: afterwards this rank
    holds every row whose key it owns.  Returns the received block (device columns) and the
    tensors backing it (keep them alive)."""
    world = dist.get_world_size(group)
    parts, offs = hash_partition(block, key_col, world, device)
    widths = [np_dtype(c.dtype).itemsize for c in block.columns]
    recv, n = all_to_all_columns(parts, widths, offs, group)
    cols = [Column.device(c.dtype, n, t.data_ptr()) for c, t in zip(block.columns, recv)]
    return DataBlock(cols, n), recv


def _first_key(key) -> int:
    return int(key) if isinstance(key, (int, np.integer)) else int(key[0])


def partitioned_hash_join(build: DataBlock, probe: DataBlock, build_key, probe_key, device: int, group=None,
                          out_mem: int = abi.MEM_HOST, kind: int = abi.JOIN_INNER):
    """Join of two row-range-sharded tables: shuffle both sides by key, then join locally.
    Returns the joined blocks of this rank (probe columns then build columns).  Each rank owns
    every build row of its keys, so its final_probe stream (the build-side kinds) is complete.
    build_key / probe_key: a column index or equally long lists (composite keys, see HashJoin).
    Both sides are shuffled on the FIRST key pair only: rows equal on every key are equal on the
    first, and both sides hash the same 64-bit image of it.  A first key with few distinct values
    therefore puts most rows on few ranks."""
    b_local, keep_b = shuffle_by_key(build, _first_key(build_key), device, group)
    p_local, keep_p = shuffle_by_key(probe, _first_key(probe_key), device, group)
    torch.cuda.synchronize(device)
    j = HashJoin(schema_types(b_local), schema_types(p_local), build_key, probe_key, device, kind)
    j.add_block(b_local)
    j.final_build()
    out = j.probe_block(p_local, out_mem)
    out += j.final_probe(out_mem)
    return out, j, (keep_b, keep_p)


def _pack_i64(vals: np.ndarray) -> np.ndarray:
    if vals.dtype.itemsize == 8:
        return np.ascontiguousarray(vals).view(np.int64)
    return vals.astype(np.float64).view(np.int64) if vals.dtype.kind == "f" else vals.astype(np.int64)


def _unpack_i64(raw: np.ndarray, dtype: np.dtype) -> np.ndarray:
    if dtype.itemsize == 8:
        return raw.view(dtype)
    return raw.view(np.float64).astype(dtype) if dtype.kind == "f" else raw.astype(dtype)


def topk_merge(local: DataBlock, row_base: int, k: int, asc: bool, nulls_first: bool, device: int = 0, group=None,
               final_op: TransformTopN = None, extra_keys: Sequence[Tuple[Column, bool, bool]] = ()) -> DataBlock:
    """All-gather every rank's top-k block ([key, row id], already in output order) and run the
    final TransformTopN over the gathered candidates.  Candidates are concatenated in rank order,
    so equal keys keep ascending GLOBAL row ids (rank r's rows precede rank r+1's).

    extra_keys: the later keys of ORDER BY a, b, ... as (column, asc, nulls_first), each column
    holding the rank's candidate values in the block's row order (taken by row id from the local
    input, e.g. with kernels.take).  The final TransformTopN then breaks ties on them, so equal
    composite keys keep ascending global row ids.  A caller-supplied final_op must be built with
    the same extra keys at offsets 1, 2, ...."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    keys = local.columns[0]
    cols_l = [keys] + [c for c, _, _ in extra_keys]
    vals_l = [c.values() for c in cols_l]
    valid_l = [c.valid_mask() for c in cols_l]
    rows_l = local.columns[1].values().astype(np.int64) + row_base
    nk = len(cols_l)
    if world > 1:
        # fixed-size tensors (k slots per rank and per array, count in front): one all_gather, no pickling
        n = len(rows_l)
        width = 1 + (2 * nk + 1) * k
        dev = torch.device("cuda", device) if dist.get_backend(group) == "nccl" else torch.device("cpu")
        buf = torch.zeros(width, dtype=torch.int64, device=dev)
        pack = np.zeros(width, dtype=np.int64)
        pack[0] = n
        for j in range(nk):
            pack[1 + 2 * j * k:1 + 2 * j * k + n] = _pack_i64(vals_l[j])
            pack[1 + (2 * j + 1) * k:1 + (2 * j + 1) * k + n] = valid_l[j].astype(np.int64)
        pack[1 + 2 * nk * k:1 + 2 * nk * k + n] = rows_l
        buf.copy_(torch.from_numpy(pack))
        out = torch.empty(world * width, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(out, buf, group=group)
        g = out.cpu().numpy().reshape(world, width)
        vs, ms, rs = [[] for _ in range(nk)], [[] for _ in range(nk)], []
        for r in range(world):
            m = int(g[r, 0])
            for j in range(nk):
                vs[j].append(_unpack_i64(g[r, 1 + 2 * j * k:1 + 2 * j * k + m], vals_l[j].dtype))
                ms[j].append(g[r, 1 + (2 * j + 1) * k:1 + (2 * j + 1) * k + m].astype(bool))
            rs.append(g[r, 1 + 2 * nk * k:1 + 2 * nk * k + m])
        vals, valid, rows = [np.concatenate(v) for v in vs], [np.concatenate(m) for m in ms], np.concatenate(rs)
    else:
        vals, valid, rows = vals_l, valid_l, rows_l
    cand_cols = []
    for j, c in enumerate(cols_l):
        nullable = c.validity is not None or not valid[j].all()
        cand_cols.append(Column.from_data(vals[j], c.dtype, validity=valid[j] if nullable else None))
    cand = DataBlock(cand_cols, len(rows))
    op = final_op or TransformTopN(0, asc, nulls_first, k, schema_types(cand), device,
                                   extra_keys=[(1 + j, a, nf) for j, (_, a, nf) in enumerate(extra_keys)])
    if final_op is not None:
        op.reset()
    op.transform(cand)
    out = op.on_finish()
    if final_op is None:
        op.close()
    pos = out.columns[1].values()
    return DataBlock([out.columns[0], Column.from_data(rows[pos])], out.num_rows)


def allreduce_single_state(partial, final, device: int = 0, group=None, out_mem: int = abi.MEM_HOST) -> DataBlock:
    """Aggregation WITHOUT GROUP BY across ranks (SURVEY 8e row 2; PartialSingleStateAggregator ->
    FinalSingleStateAggregator, transform_single_key.rs:93-141,232-278): every rank's partial state is
    one fixed-width row [key][kind][state words]; the rows are all-gathered (a few dozen bytes per
    rank — the reference's `allReduce` of 1-2 scalars) and every rank merges ALL of them in rank
    order with one device thread (dbx_agg_final_merge_rows on a no-GROUP-BY plan), so integer
    results are exact and f64 sums are reproducible and identical on every rank."""
    L = load()
    partial.on_finish()
    rows_ptr, offs, rb = C.c_void_p(), (C.c_int64 * 2)(), C.c_int32(0)
    check(L.dbx_agg_partial_partition(partial.handle, 1, C.byref(rows_ptr), offs, C.byref(rb)), partial.handle)
    n_rows, row_bytes = offs[1], rb.value
    assert n_rows == 1, "a no-GROUP-BY partial holds exactly one state row"
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    host = np.empty(row_bytes // 8, dtype=np.int64)
    check(L.dbx_memcpy_d2h(device, host.ctypes.data, rows_ptr, row_bytes))
    check(L.dbx_device_free(device, rows_ptr))
    if world > 1:
        nccl = dist.get_backend(group) == "nccl"
        t = torch.from_numpy(host)
        if nccl:
            t = t.to(f"cuda:{device}")
        g = torch.empty(world * len(host), dtype=torch.int64, device=t.device)
        dist.all_gather_into_tensor(g, t, group=group)
        allrows = g.cpu().numpy()
    else:
        allrows = host
    buf = C.c_void_p()
    check(L.dbx_device_alloc(device, allrows.nbytes, C.byref(buf)))
    try:
        check(L.dbx_memcpy_h2d(device, buf, allrows.ctypes.data, allrows.nbytes))
        final.merge_rows(buf.value, world)
        out = final.on_finish(out_mem)
    finally:
        check(L.dbx_device_free(device, buf))
    return out[0]


class PartitionedHashJoin:
    """Partitioned hash join with the FUSED shuffle (BASELINE configs[2]): both sides are
    hash-partitioned by key and stored straight into the owners' HBM over NVLink by one kernel per
    round (dbx_shuffle_send; no pack pass, no per-column library all-to-all), `round_rows` rows per
    rank and round; every received region is handed to the local join as a device block.
    Reference: flight_scatter_hash.rs:86-125 (scatter) + new_hash_join/memory/inner_join.rs:122-262.
    The constructor is collective (receive buffers + IPC mapping, once per schema); `run` joins one
    pair of row-range-sharded tables.  Composite keys (lists of column indices, see HashJoin) are
    shuffled on their first pair, as in partitioned_hash_join: a low-cardinality first key skews
    the ranks."""

    def __init__(self, build_types: Sequence[int], probe_types: Sequence[int], build_key, probe_key, device: int, rank: int,
                 world: int, max_build_rows: int, max_probe_rows: int, round_rows: int = 32 << 20, group=None, kind: int = abi.JOIN_INNER):
        from .exchange import PeerShuffle
        self.device, self.rank, self.world, self.round_rows = device, rank, world, round_rows
        self.build_types, self.probe_types, self.build_key, self.probe_key, self.kind = list(build_types), list(probe_types), build_key, probe_key, kind
        self.max_build, self.max_probe = max_build_rows, max_probe_rows
        self.sb = PeerShuffle(device, rank, world, [t & 0xFF for t in build_types], _first_key(build_key), max(1, min(round_rows, max_build_rows)))
        self.sp = PeerShuffle(device, rank, world, [t & 0xFF for t in probe_types], _first_key(probe_key), max(1, min(round_rows, max_probe_rows)))
        if world > 1:
            self.sb.connect(group)
            self.sp.connect(group)
        else:
            self.sb.connect_local([self.sb])
            self.sp.connect_local([self.sp])

    def _rounds(self, shuf, blk, total_max, each, j, ms):
        import time
        step = max(1, min(self.round_rows, total_max))
        for lo in range(0, max(total_max, 1), step):
            a = min(lo, blk.num_rows)
            shuf.send(blk.slice(a, max(min(blk.num_rows, lo + step), a)))
            got = shuf.recv()
            lm = shuf.last_ms()
            ms["shuffle_send"] += lm["send"]
            ms["shuffle_wait"] += lm["wait"]
            t0 = time.perf_counter()
            for b in got:
                if b.num_rows:
                    each(b)
            j.synchronize()  # the regions may be overwritten two sends from now: be done reading them
            yield (time.perf_counter() - t0) * 1e3

    def run(self, build: DataBlock, probe: DataBlock, out_mem: int = abi.MEM_HOST, stats: dict = None):
        """-> (joined blocks of this rank, join operator); close the operator when done with the blocks."""
        import time
        j = HashJoin(self.build_types, self.probe_types, self.build_key, self.probe_key, self.device, self.kind,
                     expected_build_rows=int(self.max_build * 1.25) + 1024)
        ms = {"shuffle_send": 0.0, "shuffle_wait": 0.0, "build": 0.0, "probe": 0.0}
        for m in self._rounds(self.sb, build, self.max_build, j.add_block, j, ms):
            ms["build"] += m
        t0 = time.perf_counter()
        j.final_build()
        ms["build"] += (time.perf_counter() - t0) * 1e3
        outs = []
        for m in self._rounds(self.sp, probe, self.max_probe, lambda b: outs.extend(j.probe_block(b, out_mem)), j, ms):
            ms["probe"] += m
        # Join::final_probe after the last round: this rank owns every build row of its keys, so its
        # matched map is complete (a no-op for INNER and the LEFT kinds)
        t0 = time.perf_counter()
        outs.extend(j.final_probe(out_mem))
        ms["final_probe"] = (time.perf_counter() - t0) * 1e3
        if stats is not None:
            stats.update(ms)
        return outs, j

    def close(self):
        self.sb.close()
        self.sp.close()


def partitioned_hash_join_peer(build: DataBlock, probe: DataBlock, build_key, probe_key, device: int, rank: int, world: int,
                               round_rows: int = 32 << 20, out_mem: int = abi.MEM_HOST, group=None, kind: int = abi.JOIN_INNER,
                               stats: dict = None):
    """One-shot form of PartitionedHashJoin (set-up included): returns (joined blocks, join op, [the object to close])."""
    t = torch.tensor([build.num_rows, probe.num_rows], dtype=torch.int64)
    if world > 1:
        if dist.get_backend(group) == "nccl":
            t = t.to(f"cuda:{device}")
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    max_build, max_probe = [int(v) for v in t.tolist()]
    pj = PartitionedHashJoin(schema_types(build), schema_types(probe), build_key, probe_key, device, rank, world, max_build, max_probe,
                             round_rows, group, kind)
    outs, j = pj.run(build, probe, out_mem, stats)
    return outs, j, (pj,)


def _dev_tensor(ptr: int, nbytes: int, device: int) -> torch.Tensor:
    """uint8 view of library-owned device memory (no copy)."""
    class _H:
        pass
    h = _H()
    h.__cuda_array_interface__ = {"shape": (max(nbytes, 0),), "typestr": "|u1", "data": (ptr, False), "version": 2}
    return torch.as_tensor(h, device=f"cuda:{device}")


def topk_merge_device(local_op: TransformTopN, row_base: int, k: int, final_op: TransformTopN, device: int = 0, group=None) -> DataBlock:
    """Multi-GPU top-k merge without the host in the data path (non-nullable keys): every rank's
    sorted top-k stays in HBM (dbx_op_pull with DBX_MEM_DEVICE), keys and GLOBAL row ids are
    all-gathered as device tensors, and the final TransformTopN consumes the gathered candidates as
    one device-resident block.  Candidates are concatenated in rank order and each rank's block is
    already in output order, so equal keys keep ascending global row ids.  Only the k result rows
    reach the host."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    local_op.finish()
    b = local_op.pull_c(abi.MEM_DEVICE)
    n = b.num_rows
    kcol, rcol = b.cols[0], b.cols[1]
    key_dtype = kcol.dtype  # (the descriptors die with the block below)
    esz = np_dtype(key_dtype).itemsize
    if kcol.validity:
        check(load().dbx_block_release(C.byref(b)))
        raise ValueError("topk_merge_device: nullable keys take the host merge (topk_merge)")
    pad_k = torch.zeros(k * esz, dtype=torch.uint8, device=f"cuda:{device}")
    pad_r = torch.zeros(k, dtype=torch.int64, device=f"cuda:{device}")
    if n:
        pad_k[: n * esz] = _dev_tensor(kcol.data, n * esz, device)
        pad_r[:n] = _dev_tensor(rcol.data, n * 8, device).view(torch.int64) + row_base
    check(load().dbx_block_release(C.byref(b)))
    cnt = torch.tensor([n], dtype=torch.int64, device=f"cuda:{device}")
    if world > 1:
        gk = torch.empty(world * k * esz, dtype=torch.uint8, device=f"cuda:{device}")
        gr = torch.empty(world * k, dtype=torch.int64, device=f"cuda:{device}")
        gc = torch.empty(world, dtype=torch.int64, device=f"cuda:{device}")
        dist.all_gather_into_tensor(gk, pad_k, group=group)
        dist.all_gather_into_tensor(gr, pad_r, group=group)
        dist.all_gather_into_tensor(gc, cnt, group=group)
        counts = gc.tolist()
        if all(c == k for c in counts):
            keys, rows = gk, gr
        else:  # ragged (a rank with fewer than k rows): compact on the device
            keys = torch.cat([gk[r * k * esz: r * k * esz + counts[r] * esz] for r in range(world)])
            rows = torch.cat([gr[r * k: r * k + counts[r]] for r in range(world)])
    else:
        keys, rows = pad_k[: n * esz], pad_r[:n]
    m = rows.numel()
    torch.cuda.current_stream().synchronize()
    final_op.reset()
    final_op.transform(DataBlock([Column.device(key_dtype, m, keys.data_ptr())], m))
    out = final_op.on_finish()
    pos = torch.from_numpy(out.columns[1].values().astype(np.int64)).to(f"cuda:{device}")
    return DataBlock([out.columns[0], Column.from_data(rows[pos].cpu().numpy())], out.num_rows)
