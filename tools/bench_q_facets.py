"""What per-query facets in the batched call (oc_search_q_facets) cost, on the h1 shape: hybrid, 1M x 768-d fp32 + BM25
over 1M synthetic documents, B = 256, top 10.  Each query asks for 1-3 facet fields drawn from a bool field, a 10-key
string_filter field and a number field with 5 ranges; half the queries get a range `where` on the number field, a third
get a groupBy (10 groups, max_results 3).

  (a) oc_search_q_facets at B = 256;
  (b) today's path without it: each query alone through oc_search_q_groups + oc_search_facets, summed per round;
  (c) today's best batched workaround: oc_search_q_groups at B = 256 plus oc_search_facets at B = 256 over the union of
      all the queries' requests;
  (d) end-to-end QPS of 256 threads through SearchBatcher.search_faceted, against the same threads calling the library
      directly (the two calls of (b) each).
Rows (a)-(c): median / min / max over --calls calls of the host time of the calls, which end in a stream synchronise.

  --facets-only: (e) oc_search_facets alone at B = 256 over the union of the requests, fulltext over the same 1M
      documents (the counting does not depend on the vector stage): call time, and with --profile the device time of the
      facet counting kernel from torch.profiler (run it in a process of its own; for an A/B, run this file from a tree of
      the other build).

The card's name and power limit are read in the same process.  Writes nothing into the tree.

    python tools/bench_q_facets.py [--calls 20] [--rounds 3] [--facets-only [--profile]]
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
RANGES = [{"from": 0, "to": 10}, {"from": 10, "to": 25}, {"from": 25, "to": 50}, {"from": 50, "to": 80}, {"from": 80, "to": 100}]
FIELDS = {"flag": {"true": True, "false": True}, "cat": {}, "price": {"ranges": RANGES}}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}


def timed(fn, calls):
    fn()
    t = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return stats(t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3, help="end-to-end rounds of 256 requests per arm in (d)")
    ap.add_argument("--facets-only", action="store_true")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi": card(), "library": ob.SO_PATH}
    rng = np.random.default_rng(8)
    ids = np.arange(N, dtype=np.uint64)
    emb, qv = None, None
    if not a.facets_only:
        rows = synth.make_vectors(N, DIM)
        emb = ob.EmbeddingFieldStorage(ctx, "BGEBase")
        emb.reserve(N)
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
    g10 = ob.GroupBy(st, ["cat"])
    names = list(FIELDS)
    facets = [{k: FIELDS[k] for k in rng.choice(names, int(rng.integers(1, 4)), replace=False)} for _ in range(B)]
    union = {k: FIELDS[k] for k in names if any(k in f for f in facets)}
    fr = getattr(ob, "facet_requests", None)   # absent from builds before oc_search_q_facets (the --facets-only A/B)
    mixinfo = {} if fr is None else {"facet_requests": sum(len(fr(st, f)[0]) for f in facets), "union_requests": len(fr(st, union)[0])}

    if a.facets_only:   # (e)
        p = ob.TokenScoreParams(mode=ob.MODE_FULLTEXT, limit_hint=LIMIT)
        row = {"case": "(e) oc_search_facets, B = 256, fulltext, union of the requests", **mixinfo, **info,
               "call_ms": timed(lambda: ob.search_facets(tsc, st, p, union, batch), a.calls)}
        if a.profile:
            import torch
            from torch.profiler import ProfilerActivity, profile
            torch.cuda.init()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.calls):
                    ob.search_facets(tsc, st, p, union, batch)
            k = [e for e in prof.key_averages() if "facet" in e.key and "count" in e.key]
            row["kernels"] = {e.key: {"calls": e.count, "device_us_per_call": e.device_time_total / max(e.count, 1)} for e in k}
        print(json.dumps(row), flush=True)
        st.close(); g10.close(); strs.close(); ctx.close()
        return

    def where(lo, width):
        return ob.evaluate_where(ob.parse_where({"price": {"between": [lo, lo + width]}}), st, {}, N, [])
    filters = [where(float(rng.uniform(0, 50)), float(rng.uniform(1, 50))) if b % 2 == 0 else None for b in range(B)]
    groups = [(g10, 3) if b % 3 == 0 else None for b in range(B)]
    mixinfo.update(filtered=sum(f is not None for f in filters), grouped=sum(g is not None for g in groups))
    pq = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filters=filters)
    res = {"a": timed(lambda: ob.search_q_facets_arrays(tsc, st, pq, facets, groups, None, batch, qv), a.calls)}
    print(json.dumps({"case": "(a) oc_search_q_facets, B = 256", "B": B, "limit": LIMIT, "call_ms": res["a"],
                      "qps": B / res["a"]["median"] * 1e3, **mixinfo, **info}), flush=True)

    def alone(q):
        p1 = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filters=[filters[q]])
        ob.search_q_groups_arrays(tsc, p1, [groups[q]], None, [texts[q]], qv[q:q + 1])
        p2 = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0)
        ob.search_facets(tsc, st, p2, facets[q], [texts[q]], qv[q:q + 1])

    def all_alone():
        for q in range(B):
            alone(q)
    res["b"] = timed(all_alone, max(3, a.calls // 4))
    print(json.dumps({"case": "(b) each query alone: oc_search_q_groups + oc_search_facets, summed", "calls_per_round": 2 * B,
                      "call_ms_per_round": res["b"], "qps": B / res["b"]["median"] * 1e3, **info}), flush=True)

    def workaround():
        ob.search_q_groups_arrays(tsc, pq, groups, None, batch, qv)
        ob.search_facets(tsc, st, ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0), union, batch, qv)
    res["c"] = timed(workaround, a.calls)
    print(json.dumps({"case": "(c) oc_search_q_groups B = 256 + oc_search_facets B = 256 over the union", "call_ms": res["c"],
                      "qps": B / res["c"]["median"] * 1e3, **info}), flush=True)
    print(json.dumps({"headline": "(b) / (a) and (c) / (a)", "speedup_b": res["b"]["median"] / res["a"]["median"],
                      "speedup_c": res["c"]["median"] / res["a"]["median"], **info}), flush=True)

    bat = ob.SearchBatcher(tsc, max_batch=B, max_wait_us=2000)

    def via_batcher(q):
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=filters[q])
        bat.search_faceted(st, p, facets[q], groups[q], None, texts[q], qv[q])

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
        print(json.dumps({"case": f"(d) 256 threads, end to end, {k}", "rounds": a.rounds, "seconds_per_round": stats(v),
                          "qps": B / float(np.median(v)), **({"batcher_stats": st_b} if k == "batcher" else {}), **info}), flush=True)
    bat.close()
    for f in filters:
        if f is not None:
            f.close()
    g10.close(); st.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
