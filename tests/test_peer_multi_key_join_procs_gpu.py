"""Partitioned INNER, LEFT and FULL hash joins on composite keys over REAL ranks with the fused
peer-memory shuffle (shuffled on the first key pair): the union of the ranks' results equals the
reduction to single-key joins (tests/join_multi_key_ref.py) as a multiset, and every unmatched
dimension row appears exactly once across the ranks."""
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
def test_partitioned_multi_key_joins_between_processes(gpu, tmp_path, world):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from _peer_multi_key_join_worker import LAYOUTS, tables
    from join_multi_key_ref import hash_join_multi_key
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), DBX_EXCH_SPIN_MS="30000")
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "_peer_multi_key_join_worker.py"), str(tmp_path)], env=env,
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
    for layout in LAYOUTS:
        d0, d1, dv, f0, f1, fv = tables(layout)
        bcols = [Column.from_data(d0), Column.from_data(d1)]
        pcols = [Column.from_data(f0), Column.from_data(f1)]
        for name, kind in (("inner", abi.JOIN_INNER), ("left", abi.JOIN_LEFT), ("full", abi.JOIN_FULL)):
            pi, bi = hash_join_multi_key(kind, bcols, pcols)
            exp = []
            for arr, idx in ((f0, pi), (f1, pi), (fv, pi), (d0, bi), (d1, bi), (dv, bi)):
                exp.append((arr.astype(np.int64)[np.maximum(idx, 0)], idx >= 0))
            parts = [np.load(os.path.join(tmp_path, f"{layout}_{name}_r{r}.npz")) for r in range(world)]
            got = [(np.concatenate([d[c] for d in parts]), np.concatenate([d[c + "_valid"] for d in parts])) for c in ("f0", "f1", "fv", "d0", "d1", "dv")]
            assert len(got[0][0]) == len(pi), (layout, name)
            np.testing.assert_array_equal(_rows(got), _rows(exp), err_msg=f"{layout} {name}")
            if name == "full":  # every unmatched dimension row exactly once across the ranks
                matched = np.zeros(len(d0), dtype=bool)
                matched[bi[(bi >= 0) & (pi >= 0)]] = True
                final = ~got[0][1]  # rows whose probe side is NULL
                key = got[3][0][final] * 10**6 + got[4][0][final]
                want = d0.astype(np.int64)[~matched] * 10**6 + d1.astype(np.int64)[~matched]
                np.testing.assert_array_equal(np.sort(key), np.sort(want), err_msg=layout)
                assert (~matched).sum() >= len(d0) // 10
