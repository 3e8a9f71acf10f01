"""Partitioned RIGHT and FULL hash joins over REAL ranks with the fused peer-memory shuffle: the
union of the ranks' results (probe blocks plus each rank's final_probe stream) equals the CPU
restatement's (tests/join_build_side_ref.py) as a multiset, and every unmatched dimension row appears exactly once across the ranks."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from databend_b200 import abi
from databend_b200.block import Column

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rows(cols):
    a = np.stack([np.where(m, v, 0) for v, m in cols] + [m.astype(np.int64) for _, m in cols], axis=1)
    return a[np.lexsort(a.T[::-1])]


@pytest.mark.parametrize("world", [1, 2, 3])
def test_partitioned_right_and_full_join_between_processes(gpu, tmp_path, world):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from _peer_right_join_worker import tables
    from join_build_side_ref import hash_join_build_side
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), DBX_EXCH_SPIN_MS="30000")
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_peer_right_join_worker.py"), str(tmp_path)], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            outs.append(p.communicate(timeout=600)[0])
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, f"rank {r} failed:\n{o[-3000:]}"
    dk, dv, fk, fv = tables()
    unmatched_dims = np.setdiff1d(dk, fk)
    assert len(unmatched_dims) >= len(dk) // 10
    for name, kind in (("right", abi.JOIN_RIGHT), ("full", abi.JOIN_FULL)):
        pi, bi = hash_join_build_side(kind, Column.from_data(dk), Column.from_data(fk))
        exp = []
        for arr, idx in ((fk, pi), (fv.astype(np.int64), pi), (dk, bi), (dv, bi)):
            exp.append((arr[np.maximum(idx, 0)], idx >= 0))
        parts = [np.load(os.path.join(tmp_path, f"{name}_r{r}.npz")) for r in range(world)]
        got = [(np.concatenate([d[c] for d in parts]), np.concatenate([d[c + "_valid"] for d in parts])) for c in ("fk", "fv", "dk", "dv")]
        assert len(got[0][0]) == len(pi), name
        np.testing.assert_array_equal(_rows(got), _rows(exp), err_msg=name)
        # every unmatched dimension row exactly once across the ranks (rows whose probe side is NULL)
        final_dk = got[2][0][~got[0][1]]
        np.testing.assert_array_equal(np.sort(final_dk), np.sort(unmatched_dims), err_msg=name)
