"""Partial -> final exchange across GPUs: ONE variable-size all-to-all of partial group rows.

Replaces the reference's cluster shuffle of aggregate partials
(src/query/service/src/pipelines/processors/transforms/aggregator/build_partition_bucket.rs:41-131
within a node, Arrow-Flight exchange between nodes: servers/flight/v1/exchange/*) with
torch.distributed (NCCL over NVLink on GPUs, gloo in the CPU tests): a count exchange followed by
the payload exchange.  Only plumbing lives here; partitioning and merging are CUDA kernels behind
dbx_agg_partial_partition / dbx_agg_final_merge_rows.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import abi
from .lib import DbxError, load

_M64 = (1 << 64) - 1
_NULL_HASH = 0xd1cefa08eb382d69
_EMPTY_KEY = 0x8000000000000000


def agg_hash_np(x: np.ndarray) -> np.ndarray:
    """group_hash.rs:555-570 on a uint64 array (host restatement used by host-side tests)."""
    x = x.astype(np.uint64).copy()
    c = np.uint64(0xd6e8feb86659fd93)
    s = np.uint64(32)
    with np.errstate(over="ignore"):
        x ^= x >> s
        x *= c
        x ^= x >> s
        x *= c
        x ^= x >> s
    return x


def owner_of(keys: np.ndarray, key_kind: np.ndarray, n_parts: int) -> np.ndarray:
    """Owner rank of a group: top 32 hash bits scaled to n_parts (same rule as the device kernel
    `owner_of` in csrc/agg_kernels.cuh; radix partitioning on hash bits like
    partitioned_payload.rs:44-57 generalised to any partition count)."""
    k = np.where(key_kind == 1, np.uint64(_EMPTY_KEY), keys.astype(np.uint64))
    h = agg_hash_np(k)
    h = np.where(key_kind == 2, np.uint64(_NULL_HASH), h)
    return (((h >> np.uint64(32)) * np.uint64(n_parts)) >> np.uint64(32)).astype(np.int64)


def all_to_all_rows(send: torch.Tensor, send_counts: Sequence[int], row_bytes: int, group=None) -> Tuple[torch.Tensor, List[int]]:
    """Exchange fixed-width rows.  `send` is a uint8 tensor holding sum(send_counts) rows laid out
    partition after partition; returns (recv uint8 tensor, recv_counts)."""
    world = dist.get_world_size(group)
    assert len(send_counts) == world
    dev = send.device
    sc = torch.tensor(list(send_counts), dtype=torch.int64, device=dev)
    rc = torch.empty_like(sc)
    dist.all_to_all_single(rc, sc, group=group)
    recv_counts = [int(v) for v in rc.tolist()]
    total_recv = sum(recv_counts)
    recv = torch.empty(max(total_recv, 1) * row_bytes, dtype=torch.uint8, device=dev)
    total_send = sum(send_counts)
    dist.all_to_all_single(recv[: total_recv * row_bytes], send[: total_send * row_bytes],
                           [c * row_bytes for c in recv_counts], [c * row_bytes for c in send_counts], group=group)
    return recv, recv_counts


class PeerExchange:
    """Partial -> final shuffle through peer memory (NVLink), the GPU-native replacement of the
    all-to-all above: `scatter(partial)` partitions the partial's groups and stores every row
    straight into its owner's receive buffer, `merge(final)` waits on the device for all sources
    and merges.  Only the one-time exchange of the 64-byte IPC handles goes through
    torch.distributed.  One instance per rank; `connect()` is collective."""

    def __init__(self, partial, rank: int, world: int, region_rows: int = 0):
        self.rank, self.world = rank, world
        self._h = C.c_void_p()
        self._handle = (C.c_ubyte * 64)()
        st = load().dbx_agg_exchange_create(partial.handle, rank, world, region_rows, C.byref(self._h), self._handle)
        self._check(st, created=False)

    def _check(self, st, created=True):
        if st != abi.OK:
            msg = load().dbx_agg_exchange_last_error(self._h if created else None)
            raise DbxError(st, (msg or b"").decode("utf-8", "replace"))

    def ipc_handle(self) -> bytes:
        return bytes(self._handle)

    def local_buffer(self) -> Tuple[int, int, int]:
        base, rows, rb = C.c_void_p(), C.c_int64(0), C.c_int32(0)
        self._check(load().dbx_agg_exchange_local_buffer(self._h, C.byref(base), C.byref(rows), C.byref(rb)))
        return base.value, rows.value, rb.value

    def connect(self, group=None):
        """Collective: all-gather the IPC handles and map every peer's receive buffer."""
        handles: List[Optional[bytes]] = [None] * self.world
        dist.all_gather_object(handles, self.ipc_handle(), group=group)
        blob = b"".join(handles)
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._check(load().dbx_agg_exchange_connect(self._h, buf, None))

    def connect_local(self, peers: Sequence["PeerExchange"]):
        """Ranks simulated inside one process (tests): wire the receive buffers directly."""
        ptrs = (C.c_void_p * self.world)(*[p.local_buffer()[0] for p in peers])
        self._check(load().dbx_agg_exchange_connect(self._h, None, ptrs))

    def scatter(self, partial):
        self._check(load().dbx_agg_exchange_scatter(self._h, partial.handle))

    def merge(self, final):
        self._check(load().dbx_agg_exchange_merge(self._h, final.handle))

    def phase_ms(self) -> dict:
        """Device times (ms) of the last scatter / wait / merge / finalize (call after the final's on_finish)."""
        out = (C.c_float * 8)()
        self._check(load().dbx_agg_exchange_phase_ms(self._h, out))
        return {"scatter": out[0], "wait_flags": out[1], "merge": out[2], "finalize": out[3], "wait_spin": out[4]}

    def close(self):
        if self._h:
            load().dbx_agg_exchange_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PeerShuffle:
    """Hash-partitioned row shuffle over peer memory (include/dbx.h: dbx_shuffle_*): the exchange in
    front of a partitioned hash join.  `send(block)` partitions a device-resident block by the
    owner of its key column and stores the rows straight into the owners' HBM over NVLink;
    `recv()` returns one device-resident block per source rank.  Collective: every rank alternates
    send / recv the same number of times.  One instance per rank and schema; `connect()` is collective."""

    def __init__(self, device: int, rank: int, world: int, col_types: Sequence[int], key_col: int, region_rows: int):
        self.device, self.rank, self.world, self.col_types = device, rank, world, list(col_types)
        self._h = C.c_void_p()
        self._handle = (C.c_ubyte * 64)()
        types = (C.c_int32 * len(col_types))(*col_types)
        st = load().dbx_shuffle_create(device, rank, world, types, len(col_types), key_col, region_rows, C.byref(self._h), self._handle)
        self._check(st, created=False)

    def _check(self, st, created=True):
        if st != abi.OK:
            msg = load().dbx_shuffle_last_error(self._h if created else None)
            raise DbxError(st, (msg or b"").decode("utf-8", "replace"))

    def connect(self, group=None):
        handles: List[Optional[bytes]] = [None] * self.world
        dist.all_gather_object(handles, bytes(self._handle), group=group)
        blob = b"".join(handles)
        buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
        self._check(load().dbx_shuffle_connect(self._h, buf, None))

    def connect_local(self, peers: Sequence["PeerShuffle"]):
        ptrs = (C.c_void_p * self.world)()
        for i, p in enumerate(peers):
            base = C.c_void_p()
            p._check(load().dbx_shuffle_local_buffer(p._h, C.byref(base)))
            ptrs[i] = base.value
        self._check(load().dbx_shuffle_connect(self._h, None, ptrs))

    def send(self, block):
        b, keep = block.as_c()
        self._check(load().dbx_shuffle_send(self._h, C.byref(b)))
        self._keep = (block, keep)

    def recv(self):
        """-> list of `world` device-resident DataBlocks (views into the receive buffer)."""
        from .block import Column, DataBlock
        n_cols = len(self.col_types)
        blocks = (abi.Block * self.world)()
        cols = (abi.Column * (self.world * n_cols))()
        self._check(load().dbx_shuffle_recv(self._h, blocks, cols))
        out = []
        for r in range(self.world):
            n = blocks[r].num_rows
            out.append(DataBlock([Column.device(self.col_types[c], n, cols[r * n_cols + c].data or 0) for c in range(n_cols)], n))
        return out

    def last_ms(self):
        a, b = C.c_float(0), C.c_float(0)
        self._check(load().dbx_shuffle_last_ms(self._h, C.byref(a), C.byref(b)))
        return {"send": a.value, "wait": b.value}

    def close(self):
        if self._h:
            load().dbx_shuffle_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
