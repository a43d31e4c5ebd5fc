"""Cost and effect of oc_emb_compact (EmbeddingFieldStorage.compact) on synthetic stores.

For a 1M x 768 fp32 store (with its fp16 copy) and a 1M x 1024 bf16 store, one document per row, and three delete
patterns — 10 % and 50 % of the documents uniformly spread, and the newest 10 % — the script reports
  * the compaction's `device_ms` (CUDA events around its device work), median / min / max of --reps compactions, each of
    a freshly built store (a compaction cannot be repeated on the same store), after a warm-up compaction of a small
    store of each dtype so that no timed call loads a kernel;
  * the algorithmic bytes of the move (per moved row: read + write of the row, of its fp16 copy when kept, and of its
    16 B of per-row arrays) and that figure over `device_ms`;
  * `workspace_bytes`;
  * the device time (`oc_last_timing().device_ms`, median of --calls after two warm-up calls) of a B = 256, limit 10
    vector `oc_search` before the deletes, after them, and after the compaction, and whether the three returned the
    same bytes.
`--windows` repeats the fp32 / 50 % case at other staging-window sizes (OC_EMB_COMPACT_WINDOW).
The card's name, power limit and SM clock limit are read in the same process, as found.  Writes nothing into the tree.

    python tools/bench_emb_compact.py [--rows 1000000] [--reps 3] [--calls 7] [--windows 4,8,32,64]
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

B, LIMIT = 256, 10


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}


def moved_bytes(st, stride, esz, f16):
    """Algorithmic bytes of a compaction: every moved row is read once and written once, in every per-row array."""
    return st["rows_moved"] * 2 * (stride * esz + (stride * 2 + 4 if f16 else 0) + 12)


def search_ms(ctx, emb, qv, calls):
    t = []
    hits = None
    for i in range(calls + 2):
        hits = ob.search(ctx, emb, None, "vector", q_vecs=qv, limit=LIMIT, similarity=0.0)
        if i >= 2:
            t.append(ctx.last_timing()["device_ms"])
    sig = [(h.count, h.doc_ids.tobytes(), np.asarray(h.scores, np.float32).tobytes()) for h in hits]
    return stats(t), sig


def dead_docs(pattern, n):
    if pattern == "10% spread":
        return np.flatnonzero(np.random.default_rng(1).random(n) < 0.10).astype(np.uint64)
    if pattern == "50% spread":
        return np.flatnonzero(np.random.default_rng(2).random(n) < 0.50).astype(np.uint64)
    return np.arange(n - n // 10, n, dtype=np.uint64)   # the newest 10 %


def warm_up(ctx):
    for dtype in ("f32", "bf16"):
        emb = ob.EmbeddingFieldStorage(ctx, dim=128, dtype=dtype)
        emb.insert_batch(np.arange(20000, dtype=np.uint64), synth.make_vectors(20000, 128, seed=1))
        emb.delete(np.arange(0, 20000, 3, dtype=np.uint64))
        emb.compact(shrink=True)
        emb.close()


def run_case(ctx, rows, dtype, pattern, reps, calls, qv, with_search=True):
    n, dim = rows.shape
    ids = np.arange(n, dtype=np.uint64)
    dead = dead_docs(pattern, n)
    ms, out = [], {}
    for rep in range(reps):
        emb = ob.EmbeddingFieldStorage(ctx, dim=dim, dtype=dtype)
        emb.insert_batch(ids, rows)
        first = rep == 0 and with_search
        if first:
            out["search_ms_before_deletes"], sig0 = search_ms(ctx, emb, qv, calls)
        emb.delete(dead)
        if first:
            out["search_ms_with_tombstones"], sig1 = search_ms(ctx, emb, qv, calls)
        st = emb.compact()
        ms.append(st["device_ms"])
        if first:
            out["search_ms_after_compaction"], sig2 = search_ms(ctx, emb, qv, calls)
            out["search_bytes_unchanged_by_compaction"] = sig1 == sig2
        if rep == 0:
            stride = (dim + 127) // 128 * 128
            esz = 2 if dtype == "bf16" else 4
            f16 = dtype == "f32" and os.environ.get("OC_EMB_F16", "1")[0] != "0"
            out.update(rows_before=st["rows_before"], rows_after=st["rows_after"], rows_moved=st["rows_moved"],
                       workspace_bytes=st["workspace_bytes"], moved_bytes=moved_bytes(st, stride, esz, f16))
        emb.close()
    out["compact_device_ms"] = stats(ms)
    out["moved_GB_per_s"] = out["moved_bytes"] / (out["compact_device_ms"]["median"] * 1e-3) / 1e9 if out["rows_moved"] else 0.0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--calls", type=int, default=7)
    ap.add_argument("--windows", default="", help="comma-separated staging-window sizes in MiB for the fp32 / 50 %% case")
    a = ap.parse_args()
    ctx = ob.Context(0)   # no device: an error, there is nothing to measure without one
    print(json.dumps({"card": card(), "rows": a.rows, "B": B, "limit": LIMIT, "reps": a.reps, "calls": a.calls}), flush=True)
    warm_up(ctx)
    for dtype, dim in (("f32", 768), ("bf16", 1024)):
        rows = synth.make_vectors(a.rows, dim, seed=21)
        qv, _ = synth.make_vector_queries(rows, B, seed=22)
        for pattern in ("10% spread", "50% spread", "newest 10%"):
            r = run_case(ctx, rows, dtype, pattern, a.reps, a.calls, qv)
            print(json.dumps({"store": f"{a.rows} x {dim} {dtype}", "deleted": pattern, **r}), flush=True)
        if dtype == "f32":
            for w in [int(x) for x in a.windows.split(",") if x]:
                os.environ["OC_EMB_COMPACT_WINDOW"] = str(w << 20)
                r = run_case(ctx, rows, dtype, "50% spread", a.reps, a.calls, qv, with_search=False)
                print(json.dumps({"store": f"{a.rows} x {dim} {dtype}", "deleted": "50% spread", "window_MiB": w, **r}), flush=True)
            os.environ.pop("OC_EMB_COMPACT_WINDOW", None)
        del rows
    ctx.close()


if __name__ == "__main__":
    main()
