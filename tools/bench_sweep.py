"""The tensor-core embedding sweep (emb_gemm_kernel, K2) alone: a vector search over a 1M x 768-d store in fp32 and in
bf16, at B = 128 / 256 / 1024, limit 10.  For every case: the median / min / max over --calls calls of
oc_last_timing.scan_sweep_ms (CUDA events around the sweep launch, inputs resident, after --warmup calls), and the
traffic the sweep needs, computed from the shapes and the tile constants:

  * L2 -> SM bytes: each CTA reads its 128-query block (A) for every row tile it sweeps, the rows (B) are read once
    per query group, or once per CTA pair when the groups run in pairs that share each row tile by multicast; plus
    the rows' inverse norms, once per consumer warpgroup and tile;
  * HBM bytes: the store and its inverse norms once;
  * FLOPs: 2 x padded B x rows x stride (what the tensor core executes);

and the rates achieved.  B = 128 is one query group and never paired.  The card's name, power limit and SM clock limit
are read in the same process.  --tile-rows / --cluster describe the build being measured (default: this tree's
GEMM_N = 256 and CTA pairs; a build with 128-row tiles and no pairs: --tile-rows 128 --cluster 1).  Writes nothing
into the tree.

    python tools/bench_sweep.py [--calls 30] [--warmup 3] [--tile-rows 256] [--cluster 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oramacore_b200 as ob  # noqa: E402
from oramacore_b200 import synth  # noqa: E402

N, DIM, LIMIT = 1_000_000, 768, 10
BATCHES = (128, 256, 1024)
GEMM_M = 128            # queries per CTA (emb_gemm.cuh)
CONSUMER_WG = 2         # consumer warpgroups per CTA, each loading the tile's inverse norms


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def traffic(B, esz, tile_rows, cluster):
    stride = DIM   # 768 is a multiple of 128: no padding
    n_qg = (B + GEMM_M - 1) // GEMM_M
    paired = cluster > 1 and n_qg % cluster == 0
    tiles = (N + tile_rows - 1) // tile_rows
    row_bytes = tiles * tile_rows * stride * esz
    l2_rows = row_bytes * n_qg // (cluster if paired else 1)
    l2_queries = n_qg * tiles * GEMM_M * stride * esz
    l2_norms = n_qg * CONSUMER_WG * tiles * tile_rows * 4
    return dict(paired=paired, l2_sm_bytes=l2_rows + l2_queries + l2_norms, l2_rows_bytes=l2_rows,
                l2_queries_bytes=l2_queries, hbm_bytes=N * stride * esz + N * 4, flop=2 * n_qg * GEMM_M * N * stride)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tile-rows", type=int, default=256)
    ap.add_argument("--cluster", type=int, default=2)
    a = ap.parse_args()
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi(name, power.limit, clocks.max.sm)": card(),
            "library": os.environ.get("OC_SO_PATH", "tree")}
    rows = synth.make_vectors(N, DIM)
    qv = {B: synth.make_vector_queries(rows[:1 << 18], B)[0] for B in BATCHES}
    ids = np.arange(N, dtype=np.uint64)
    for dtype, esz in (("f32", 4), ("bf16", 2)):
        emb = ob.EmbeddingFieldStorage(ctx, "BGEBase", dtype=dtype)
        emb.reserve(N)
        for i in range(0, N, 1 << 18):
            emb.insert_batch(ids[i:i + (1 << 18)], rows[i:i + (1 << 18)])
        tsc = ob.TokenScoreContext(ctx, emb, None)
        p = ob.TokenScoreParams(mode=ob.MODE_VECTOR, limit_hint=LIMIT, similarity=0.0)
        for B in BATCHES:
            for _ in range(a.warmup):
                tsc.execute_batch_arrays(p, None, qv[B])
            t = []
            for _ in range(a.calls):
                tsc.execute_batch_arrays(p, None, qv[B])
                lt = ctx.last_timing()
                assert lt["scan_tensor_core"], "the tensor-core sweep did not run"
                t.append(lt["scan_sweep_ms"])
            ms = float(np.median(t))
            tr = traffic(B, esz, a.tile_rows, a.cluster)
            print(json.dumps({"dtype": dtype, "B": B, "limit": LIMIT, "scan_sweep_ms": {"median": ms, "min": float(np.min(t)),
                                                                                         "max": float(np.max(t))},
                              **tr, "l2_sm_TBps": tr["l2_sm_bytes"] / ms / 1e9, "hbm_TBps": tr["hbm_bytes"] / ms / 1e9,
                              "TFLOPps": tr["flop"] / ms / 1e9, "tile_rows": a.tile_rows, "cluster": a.cluster, **info}),
                  flush=True)
        emb.close()
    ctx.close()


if __name__ == "__main__":
    main()
