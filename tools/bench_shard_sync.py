"""Per-rank fulltext stage time of a sharded index after a commit: the counted-df route (OC_SHARD_COUNT_DF, what a
shard without a df table needs) against the synced route (oc_str_sync_global rebuilt the tables), and the sync's own
cost next to the commit's.

W = 2 contexts on one GPU joined by the in-process transport (Context.comm_init_local) hold the two halves of a
t1-shaped Zipf corpus (bench.py's t1: 10 M documents, 1 M terms, B = 256), each loaded without df tables and committed.
Then every rank syncs, and the two routes run alternated, --calls times each, on one thread per rank.  Reported per
rank: the medians of oc_timing.bm25_ms and device_ms of each route, the sync's and the commit's device_ms / wall_ms;
every pair of calls is compared byte for byte (doc ids, score bits, counts).  The local transport stages every
collective through host memory, so these are per-rank device times, not an end-to-end rate and not NVLink figures.
The card's name and power limit are read in the same run.  Nothing is written into the tree.

    python tools/bench_shard_sync.py [--docs 10000000] [--vocab 1000000] [--batch 256] [--calls 30]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def on_ranks(W, fn):
    out, errs = [None] * W, [None] * W

    def go(r):
        try:
            out[r] = fn(r)
        except Exception as e:   # noqa: BLE001 - reported below
            errs[r] = e
    th = [threading.Thread(target=go, args=(r,)) for r in range(W)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if any(e is not None for e in errs):
        raise RuntimeError(f"rank errors: {errs}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--calls", type=int, default=30)
    a = ap.parse_args()
    import oramacore_b200 as ob
    from oramacore_b200 import synth
    from oramacore_b200.engine import TokenScoreContext, TokenScoreParams
    from oramacore_b200.sharding import shard_range, shard_string_index
    from oramacore_b200.types import MODE_FULLTEXT

    W = 2
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    t0 = time.perf_counter()
    data = synth.make_text_corpus(a.docs, a.vocab)
    texts = synth.make_text_queries(a.vocab, a.batch, seed=synth.SEED_TQUERIES)
    ctxs = [ob.Context(0) for _ in range(W)]
    ob.Context.comm_init_local(ctxs)
    stores = []
    for r in range(W):
        sd, _ = shard_string_index(data, *shard_range(a.docs, r, W))
        stores.append(ob.StringFieldStorage(ctxs[r], sd))   # no df table: as after a commit
    setup_s = time.perf_counter() - t0
    commits = [s.commit() for s in stores]
    tscs = [TokenScoreContext(ctxs[r], None, stores[r]) for r in range(W)]

    def search(count_df):
        p = TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, sharded=True, shard_count_df=count_df)
        return on_ranks(W, lambda r: (tscs[r].execute_batch_arrays(p, texts), ctxs[r].last_timing()))

    before = search(True)   # the only route a committed shard has without tables
    syncs = on_ranks(W, lambda r: stores[r].sync_global())
    for _ in range(3):      # warm-up of both routes
        search(True)
        search(False)
    tim = {"counted": [[] for _ in range(W)], "synced": [[] for _ in range(W)]}
    mismatches = 0
    for _ in range(a.calls):
        got = {}
        for route, flag in (("counted", True), ("synced", False)):
            res = search(flag)
            got[route] = res
            for r in range(W):
                tim[route][r].append((res[r][1]["bm25_ms"], res[r][1]["device_ms"], res[r][1]["bm25_dense_items"]))
        for r in range(W):
            for x, y in zip(got["counted"][r][0], got["synced"][r][0]):
                mismatches += not np.array_equal(x.view(np.uint8), y.view(np.uint8))
    for r in range(W):   # the counted route before the sync answered the same
        for x, y in zip(before[r][0], got["synced"][r][0]):
            mismatches += not np.array_equal(x.view(np.uint8), y.view(np.uint8))
    out = {"card": card, "docs": a.docs, "vocab": a.vocab, "batch": a.batch, "calls": a.calls, "world": W,
           "setup_s": round(setup_s, 1), "outputs_equal": mismatches == 0, "ranks": []}
    for r in range(W):
        row = {"rank": r, "rows": stores[r].info()["total_documents"],
               "commit": {k: commits[r][k] for k in ("device_ms", "wall_ms")},
               "sync": {k: syncs[r][k] for k in ("device_ms", "wall_ms", "bytes_reduced")}}
        for route in ("counted", "synced"):
            t = np.asarray(tim[route][r])
            row[route] = {"bm25_ms_median": float(np.median(t[:, 0])), "device_ms_median": float(np.median(t[:, 1])),
                          "bm25_dense_items": int(t[-1, 2])}
        row["bm25_speedup"] = row["counted"]["bm25_ms_median"] / max(row["synced"]["bm25_ms_median"], 1e-9)
        row["device_speedup"] = row["counted"]["device_ms_median"] / max(row["synced"]["device_ms_median"], 1e-9)
        out["ranks"].append(row)
    print(json.dumps(out))
    for s in stores:
        s.close()
    for c in ctxs:
        c.close()
    if mismatches:
        sys.exit(1)


if __name__ == "__main__":
    main()
