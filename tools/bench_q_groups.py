"""What a batch in which every query has its own groupBy, where-filter, sortBy and pin rules (oc_search_q_groups)
costs, on the h1 shape: hybrid, 1M x 768-d fp32 + BM25 over 1M synthetic documents, top 10.  Each query gets its own
range-leaf `where` on a number field (1-50 % of the documents), a group handle from string_filter with 10 keys /
bool x string_filter (20 groups) / none, max_results 1, 3 or 10, a sort from the mix of bench_sorted_batch.py (none /
number ASC / number DESC / date DESC) and 0-3 promote items.

  (a) oc_search_q_groups at B = 256;
  (b) the same 256 queries, each alone through the single call it stands for (oc_search_groups / _pinned / _sorted, or
      oc_search_q_sorted without groups): the sum of the 256 device times per round;
  (c) end-to-end QPS of 256 threads, each issuing its (a) query through SearchBatcher.search_groups, against the same
      threads calling the library directly (one single-query call each).
Rows (a) and (b): the median / min / max over --calls calls of oc_last_timing.device_ms (CUDA events, inputs resident).
The card's name and power limit are read in the same process.  Writes nothing into the tree.

    python tools/bench_q_groups.py [--calls 20] [--rounds 3]
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
    ap.add_argument("--rounds", type=int, default=3, help="end-to-end rounds of 256 requests per arm in (c)")
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
    cat = rng.integers(0, 10, N)
    st.add_string_field("cat", {f"c{k}": ids[cat == k] for k in range(10)})
    flag = rng.random(N) < 0.5
    st.add_bool_field("flag", ids[flag], ids[~flag])
    g10, g20 = ob.GroupBy(st, ["cat"]), ob.GroupBy(st, ["flag", "cat"])
    price = ob.SortField(ctx, N, ids, price_v, "number")
    date = ob.SortField(ctx, N, ids, (1_600_000_000_000 + rng.integers(0, 3650, N) * 86_400_000).astype(np.int64), "date")

    def where(lo, width):
        return ob.evaluate_where(ob.parse_where({"price": {"between": [lo, lo + width]}}), st, {}, N, [])
    filters = [where(float(rng.uniform(0, 50)), float(w)) for w in np.exp(rng.uniform(np.log(1.0), np.log(50.0), B))]
    mix = [None, (price, "ASC"), (price, "DESC"), (date, "DESC")]
    handles = [g10, g20, None]
    reqs = [(handles[int(rng.integers(0, 3))], [1, 3, 10][int(rng.integers(0, 3))], mix[i % 4]) for i in range(B)]
    promote = [[(int(rng.integers(0, N)), int(rng.integers(0, 10))) for _ in range(int(rng.integers(0, 4)))] for _ in range(B)]
    mixinfo = {"groups": {"cat (10)": sum(r[0] is g10 for r in reqs), "flag x cat (20)": sum(r[0] is g20 for r in reqs),
                          "none": sum(r[0] is None for r in reqs)}}

    pq = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filters=filters)
    ob.search_q_groups_arrays(tsc, pq, reqs, promote, batch, qv)
    t = []
    for _ in range(a.calls):
        ob.search_q_groups_arrays(tsc, pq, reqs, promote, batch, qv)
        t.append(ctx.last_timing()["device_ms"])
    res = {"a": stats(t)}
    print(json.dumps({"case": "(a) oc_search_q_groups, 256 groupBy / filters / sorts / pin sets", "B": B, "limit": LIMIT,
                      "device_ms": res["a"], "qps": B / res["a"]["median"] * 1e3, **mixinfo, **info}), flush=True)

    def alone(q):
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=filters[q])
        gb, m, sort = reqs[q]
        if gb is None:
            if sort is None:
                return ob.search_pinned_arrays(tsc, p, [promote[q]], [texts[q]], qv[q:q + 1])
            return ob.search_sorted_arrays(tsc, p, sort[0], sort[1], [promote[q]], [texts[q]], qv[q:q + 1])
        if sort is None:
            return ob.search_groups_arrays(tsc, gb, p, m, [texts[q]], qv[q:q + 1], promote=[promote[q]] if promote[q] else None)
        return ob.search_groups_arrays(tsc, gb, p, m, [texts[q]], qv[q:q + 1], promote=[promote[q]], sort_by=sort)
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
    print(json.dumps({"case": "(b) the same 256 queries alone (their single calls)", "B": 1, "calls_per_round": B,
                      "device_ms_per_round": res["b"], "qps": B / res["b"]["median"] * 1e3, **info}), flush=True)
    print(json.dumps({"headline": "(b) / (a) device time", "speedup": res["b"]["median"] / res["a"]["median"], **info}), flush=True)

    # (c) 256 threads, one request each per round: through the batcher vs. each calling the library directly
    bat = ob.SearchBatcher(tsc, max_batch=B, max_wait_us=2000)

    def via_batcher(q):
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=filters[q])
        bat.search_groups(p, reqs[q], promote[q] or None, texts[q], qv[q])

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
        print(json.dumps({"case": f"(c) 256 threads, end to end, {k}", "rounds": a.rounds, "seconds_per_round": stats(v),
                          "qps": B / float(np.median(v)), **({"batcher_stats": st_b} if k == "batcher" else {}), **info}), flush=True)
    bat.close()
    for f in filters:
        f.close()
    g10.close(); g20.close(); price.close(); date.close(); st.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
