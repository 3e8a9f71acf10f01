"""Int8 kNN benchmark: a device-generated uniform int8 corpus (seeded), one batch of queries, both
distance kinds.  Reports the similarity-pass time (CUDA events inside the library), its achieved
TOPS against the data sheet's dense INT8 rate, QPS and the certificate's counts; then runs the
Float32 path on the widened corpus (bf16 similarity pass) in the same process, reports its pass
time for comparison and asserts identical ids and distance bits.

Memory at the default shape (1e7 x 768): int8 corpus 7.7 GB + its padded operand copy 7.7 GB, then
the f32 corpus 30.7 GB + its bf16 copy 15.4 GB (the int8 handle is closed first)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from databend_b200 import abi  # noqa: E402
from databend_b200.block import Column  # noqa: E402
from databend_b200.vector import VectorTopN  # noqa: E402

INT8_DENSE_TOPS = 1979.0  # H100 SXM data sheet, dense INT8
BF16_DENSE_TFLOPS = 989.0

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=10_000_000)
ap.add_argument("--dim", type=int, default=768)
ap.add_argument("--nq", type=int, default=1024)
ap.add_argument("--k", type=int, default=10)
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--out", default=None, help="also write the records as a JSON list to this file")
a = ap.parse_args()

gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip().splitlines()[0]
gen = torch.Generator(device="cuda").manual_seed(20261018)
c8 = torch.randint(-128, 128, (a.n, a.dim), dtype=torch.int8, device="cuda", generator=gen)
q8 = torch.randint(-128, 128, (a.nq, a.dim), dtype=torch.int8, device="cuda", generator=gen)
torch.cuda.synchronize()
ops = 2.0 * a.nq * a.n * a.dim


def run(fn, corpus_col, q_col, label):
    t0 = time.time()
    op = VectorTopN(fn, corpus_col)
    create_s = time.time() - t0
    op.search(q_col, a.k)  # warm-up: module load, per-search buffers
    walls, gemms = [], []
    for _ in range(a.reps):
        t0 = time.time()
        idx, dist = op.search(q_col, a.k)
        walls.append(time.time() - t0)
        gemms.append(op.last_gemm_ms()[0])
    st = op.stats()
    op.close()
    gemm_ms = float(np.median(gemms))
    wall = float(np.median(walls))
    peak = INT8_DENSE_TOPS if label == "int8" else BF16_DENSE_TFLOPS
    rec = {"path": label, "fn": fn, "n": a.n, "dim": a.dim, "nq": a.nq, "k": a.k, "gpu": gpu, "create_s": round(create_s, 2),
           "gemm_ms": round(gemm_ms, 2), "gemm_ms_all": [round(x, 2) for x in gemms],
           "achieved_tops": round(ops / (gemm_ms * 1e-3) / 1e12, 1),
           "share_of_dense_peak": round(ops / (gemm_ms * 1e-3) / 1e12 / peak, 3),
           "search_wall_ms": round(wall * 1e3, 1), "qps": round(a.nq / wall, 1),
           "certified": st["certified"], "exact_fallback": st["exact_fallback"], "candidates": st["candidates"],
           "passes": st["passes"], "us_passes": st["us_passes"], "us_rerank": st["us_rerank"]}
    print(json.dumps(rec), flush=True)
    return idx, dist, rec


records = []
for fn in ("cosine_distance", "l2_distance"):
    idx8, d8, r8 = run(fn, Column.device(abi.VEC_I8, a.n, c8.data_ptr(), vec_dim=a.dim),
                       Column.device(abi.VEC_I8, a.nq, q8.data_ptr(), vec_dim=a.dim), "int8")
    cf = c8.float()
    qf = q8.float()
    torch.cuda.synchronize()
    idxf, df, rf = run(fn, Column.device(abi.VEC_F32, a.n, cf.data_ptr(), vec_dim=a.dim),
                       Column.device(abi.VEC_F32, a.nq, qf.data_ptr(), vec_dim=a.dim), "float32")
    del cf, qf
    torch.cuda.empty_cache()
    assert np.array_equal(idx8, idxf), f"{fn}: int8 and float32 ids differ"
    assert np.array_equal(d8.view(np.uint32), df.view(np.uint32)), f"{fn}: int8 and float32 distances differ"
    print(json.dumps({"fn": fn, "identical_to_float32": True, "int8_pass_speedup_vs_bf16": round(rf["gemm_ms"] / r8["gemm_ms"], 2)}),
          flush=True)
    records += [r8, rf]

if a.out:
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(records, f, indent=1)
