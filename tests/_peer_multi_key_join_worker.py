"""Worker of tests/test_peer_multi_key_join_procs_gpu.py: ONE rank of partitioned INNER, LEFT and FULL
hash joins on composite keys (2 x Int32 and 2 x Int64) with the fused peer-memory shuffle.  Both
sides are shuffled on the first key pair; every rank joins its share on all key pairs."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYOUTS = ("2xI32", "2xI64")


def tables(layout):
    """Same tables on every rank: unique dimension tuples (k0, k1), 10 % of them referenced by no fact;
    every 40th fact tuple differs from its dimension tuple in the second key only (equal on the
    shuffle key).  No NULLs: the peer-memory shuffle takes non-nullable columns."""
    rng = np.random.default_rng(8765)
    n_dim, n_fact = 40_000, 300_000
    k = rng.permutation(n_dim).astype(np.int64) * 3 - 9000
    dt = np.int32 if layout == "2xI32" else np.int64
    d0, d1 = (k % 1000).astype(dt), (k // 1000).astype(dt)
    dv = rng.integers(-2**40, 2**40, n_dim).astype(np.int64)
    pick = rng.integers(0, n_dim * 9 // 10, n_fact)
    f0, f1 = d0[pick].copy(), d1[pick].copy()
    f1[::40] += 1
    fv = rng.integers(0, 2**31, n_fact).astype(np.int32)
    return d0, d1, dv, f0, f1, fv


def main():
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    out_dir = sys.argv[1]
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from databend_b200 import abi, lib
    from databend_b200.block import Column, DataBlock
    from databend_b200.distributed import partitioned_hash_join_peer
    from databend_b200.transforms import to_device
    n_dev = lib.require_device()
    dev = rank % n_dev
    for layout in LAYOUTS:
        d0, d1, dv, f0, f1, fv = tables(layout)
        n_dim, n_fact = len(d0), len(f0)
        b_lo, b_hi = n_dim * rank // world, n_dim * (rank + 1) // world
        p_lo, p_hi = n_fact * rank // world, n_fact * (rank + 1) // world
        build = DataBlock([to_device(Column.from_data(c[b_lo:b_hi]), dev) for c in (d0, d1, dv)], b_hi - b_lo)
        probe = DataBlock([to_device(Column.from_data(f0[p_lo:p_hi]), dev),
                           to_device(Column.from_data(f1[p_lo:p_hi]), dev),
                           to_device(Column.from_data(fv[p_lo:p_hi]), dev)], p_hi - p_lo)
        for name, kind in (("inner", abi.JOIN_INNER), ("left", abi.JOIN_LEFT), ("full", abi.JOIN_FULL)):
            outs, j, shufs = partitioned_hash_join_peer(build, probe, [0, 1], [0, 1], dev, rank, world, round_rows=30_000, kind=kind)
            res = {}
            for i, c in enumerate(("f0", "f1", "fv", "d0", "d1", "dv")):
                res[c] = np.concatenate([o.columns[i].values().astype(np.int64) for o in outs]) if outs else np.empty(0, np.int64)
                res[c + "_valid"] = np.concatenate([o.columns[i].valid_mask() for o in outs]) if outs else np.empty(0, bool)
            np.savez(os.path.join(out_dir, f"{layout}_{name}_r{rank}.npz"), **res)
            dist.barrier()
            for s in shufs:
                s.close()
            j.close()
            dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
