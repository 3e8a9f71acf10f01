"""Worker of tests/test_peer_right_join_procs_gpu.py: ONE rank of the partitioned RIGHT and FULL
hash joins with the fused peer-memory shuffle (real CUDA-IPC mapping between processes; handles
travel over gloo).  Each rank owns the build rows of its keys, so its final_probe stream is its
share of the unmatched dimension rows."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def tables():
    """Same tables on every rank: 10 % of the dimension keys are referenced by no fact, and every
    50th fact key matches no dimension row."""
    rng = np.random.default_rng(4321)
    n_dim, n_fact = 50_000, 400_000
    dk = rng.permutation(n_dim).astype(np.int64) * 3 - 7000
    dv = rng.integers(-2**40, 2**40, n_dim).astype(np.int64)
    fk = dk[rng.integers(0, n_dim * 9 // 10, n_fact)].copy()
    fk[::50] = 10**12
    fv = rng.integers(0, 2**31, n_fact).astype(np.int32)
    return dk, dv, fk, fv


def main():
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    out_dir = sys.argv[1]
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from databend_b200 import abi, lib
    from databend_b200.block import Column, DataBlock
    from databend_b200.distributed import partitioned_hash_join_peer
    from databend_b200.exchange import owner_of
    from databend_b200.transforms import to_device
    n_dev = lib.require_device()
    dev = rank % n_dev
    dk, dv, fk, fv = tables()
    n_dim, n_fact = len(dk), len(fk)
    b_lo, b_hi = n_dim * rank // world, n_dim * (rank + 1) // world
    p_lo, p_hi = n_fact * rank // world, n_fact * (rank + 1) // world
    build = DataBlock([to_device(Column.from_data(dk[b_lo:b_hi]), dev), to_device(Column.from_data(dv[b_lo:b_hi]), dev)], b_hi - b_lo)
    probe = DataBlock([to_device(Column.from_data(fk[p_lo:p_hi]), dev), to_device(Column.from_data(fv[p_lo:p_hi]), dev)], p_hi - p_lo)
    for name, kind in (("right", abi.JOIN_RIGHT), ("full", abi.JOIN_FULL)):
        # small rounds: several send/recv rounds per side, so both parities of the regions are reused
        outs, j, shufs = partitioned_hash_join_peer(build, probe, 0, 0, dev, rank, world, round_rows=40_000, kind=kind)
        res = {}
        for i, c in enumerate(("fk", "fv", "dk", "dv")):
            res[c] = np.concatenate([o.columns[i].values().astype(np.int64) for o in outs]) if outs else np.empty(0, np.int64)
            res[c + "_valid"] = np.concatenate([o.columns[i].valid_mask() for o in outs]) if outs else np.empty(0, bool)
        # every row sits on the owner of its key (the build key where the probe side is NULL)
        key = np.where(res["fk_valid"], res["fk"], res["dk"])
        assert (owner_of(key.view(np.uint64), np.zeros(len(key), np.int64), world) == rank).all()
        np.savez(os.path.join(out_dir, f"{name}_r{rank}.npz"), **res)
        dist.barrier()
        for s in shufs:
            s.close()
        j.close()
        dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
