"""What a batch in which every query has its own where-filter, sortBy and pin rules (oc_search_q_sorted) costs, on the
h1 shape: hybrid, 1M x 768-d fp32 + BM25 over 1M synthetic documents, top 10.  Each query gets its own range-leaf
`where` on a number field, a sort from the mix none / number ASC / number DESC / date DESC, and 0-3 promote items.

  (a) oc_search_q_sorted at B = 256;
  (c) oc_search_sorted at B = 256 with one sort and no filter (the single-sort path);
  (b) the same 256 queries of (a), each alone through oc_search_sorted / oc_search_pinned with its filter: the sum of
      the 256 device times per round (what a batcher that cannot merge sorted requests does);
  (e) end-to-end QPS of 256 threads, each issuing its (a) query through SearchBatcher.search_sorted, against the same
      threads calling the library directly (one single-query call each).
Rows (a)-(c): the median / min / max over --calls calls of oc_last_timing.device_ms (CUDA events, inputs resident).
The card's name and power limit are read in the same process.  Writes nothing into the tree.

    python tools/bench_sorted_batch.py [--calls 20] [--rounds 3]
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

import oramacore_b200 as ob  # noqa: E402
from oramacore_b200 import synth  # noqa: E402

N, DIM, VOCAB, B, LIMIT = 1_000_000, 768, 200_000, 256, 10


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3, help="end-to-end rounds of 256 requests per arm in (e)")
    a = ap.parse_args()
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi": card()}
    rng = np.random.default_rng(8)
    rows = synth.make_vectors(N, DIM)
    emb = ob.EmbeddingFieldStorage(ctx, "BGEBase")
    emb.reserve(N)
    ids = np.arange(N, dtype=np.uint64)
    for i in range(0, N, 1 << 18):
        emb.insert_batch(ids[i:i + (1 << 18)], rows[i:i + (1 << 18)])
    qv, _ = synth.make_vector_queries(rows[:1 << 18], B)
    del rows
    strs = ob.StringFieldStorage(ctx, synth.make_text_corpus(N, VOCAB))
    texts = synth.make_text_queries(VOCAB, B)
    batch = ob.TextQueryBatch(texts)
    tsc = ob.TokenScoreContext(ctx, emb, strs)
    st = ob.FacetStore(ctx, N)
    price_v = rng.random(N) * 100.0
    st.add_number_field("price", ids, price_v)
    price = ob.SortField(ctx, N, ids, price_v, "number")
    date = ob.SortField(ctx, N, ids, (1_600_000_000_000 + rng.integers(0, 3650, N) * 86_400_000).astype(np.int64), "date")

    def where(lo, width):
        return ob.evaluate_where(ob.parse_where({"price": {"between": [lo, lo + width]}}), st, {}, N, [])
    filters = [where(float(rng.uniform(0, 50)), float(w)) for w in np.exp(rng.uniform(np.log(1.0), np.log(50.0), B))]
    mix = [None, (price, "ASC"), (price, "DESC"), (date, "DESC")]
    sorts = [mix[i % 4] for i in range(B)]
    promote = [[(int(rng.integers(0, N)), int(rng.integers(0, 10))) for _ in range(int(rng.integers(0, 4)))] for _ in range(B)]

    def timed(name, fn, **extra):
        fn()
        t = []
        for _ in range(a.calls):
            fn()
            t.append(ctx.last_timing()["device_ms"])
        s = stats(t)
        print(json.dumps({"case": name, "B": B, "limit": LIMIT, "device_ms": s, "qps": B / s["median"] * 1e3, **extra, **info}),
              flush=True)
        return s

    pq = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filters=filters)
    p0 = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0)
    res = {}
    res["a"] = timed("(a) oc_search_q_sorted, 256 filters / sorts / pin sets",
                     lambda: ob.search_q_sorted_arrays(tsc, pq, sorts, promote, batch, qv))
    res["c"] = timed("(c) oc_search_sorted, one sort (price ASC), no filter, no pins",
                     lambda: ob.search_sorted_arrays(tsc, p0, price, "ASC", None, batch, qv))

    def alone(q):
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=filters[q])
        if sorts[q] is None:
            return ob.search_pinned_arrays(tsc, p, [promote[q]], [texts[q]], qv[q:q + 1])
        return ob.search_sorted_arrays(tsc, p, sorts[q][0], sorts[q][1], [promote[q]], [texts[q]], qv[q:q + 1])
    for q in range(B):   # warm-up of every shape
        alone(q)
    tot = []
    for _ in range(a.calls):
        s = 0.0
        for q in range(B):
            alone(q)
            s += ctx.last_timing()["device_ms"]
        tot.append(s)
    res["b"] = stats(tot)
    print(json.dumps({"case": "(b) the same 256 queries alone (oc_search_sorted / oc_search_pinned)", "B": 1, "calls_per_round": B,
                      "device_ms_per_round": res["b"], "qps": B / res["b"]["median"] * 1e3, **info}), flush=True)
    print(json.dumps({"headline": "(b) / (a) device time", "speedup": res["b"]["median"] / res["a"]["median"], **info}), flush=True)

    # (e) 256 threads, one request each per round: through the batcher vs. each calling the library directly
    bat = ob.SearchBatcher(tsc, max_batch=B, max_wait_us=2000)

    def via_batcher(q):
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=filters[q])
        bat.search_sorted(p, sorts[q], promote[q] or None, texts[q], qv[q])

    def run_threads(fn):
        go = threading.Barrier(B + 1)

        def w(q):
            go.wait()
            fn(q)
        th = [threading.Thread(target=w, args=(q,)) for q in range(B)]
        for x in th:
            x.start()
        go.wait()
        t0 = time.perf_counter()
        for x in th:
            x.join()
        return time.perf_counter() - t0
    for fn in (via_batcher, alone):   # warm-up
        run_threads(fn)
    e2e = {"batcher": [], "direct": []}
    for _ in range(a.rounds):   # alternated
        e2e["batcher"].append(run_threads(via_batcher))
        e2e["direct"].append(run_threads(alone))
    st_b = bat.stats()
    for k, v in e2e.items():
        print(json.dumps({"case": f"(e) 256 threads, end to end, {k}", "rounds": a.rounds, "seconds_per_round": stats(v),
                          "qps": B / float(np.median(v)), **({"batcher_stats": st_b} if k == "batcher" else {}), **info}), flush=True)
    bat.close()
    for f in filters:
        f.close()
    price.close(); date.close(); st.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
