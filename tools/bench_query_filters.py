"""What per-query where-filters in one batch (oc_search_params.q_filters) cost, against the alternatives, on the h1
shape: hybrid, 1M x 768-d fp32 + BM25 over 1M synthetic documents, top 10.

  (a) B = 256, no filter;
  (b) B = 256, one batch-wide `where` filter (p->filter);
  (c) B = 256, 256 distinct per-query `where` filters of mixed selectivity (1 % - 50 %);
  (d) the same 256 queries, each issued alone with its filter (what a batcher without per-query filters does);
  (e) B = 256 with one filtered query and 255 unfiltered ones (the cost of routing the whole batch as filtered);
  (f) B = 256 with 256 distinct 0.05 % filters (the selective path: every passing row is gathered, overflow re-runs).
The filters are range leaves of a number field (FacetStore + evaluate_where), one handle per query.  Every row: the
median / min / max over --calls calls of oc_last_timing.device_ms (CUDA events, inputs resident); for (d) the sum of
the 256 single-query device times per round.  QPS = 256 / median.  A separate run under torch.profiler reports the
device time of rows_ok_kernel (the per-slot row bitmaps) in one (c) call.  The card's name and power limit are read in
the same process.  Writes nothing into the tree.

    python tools/bench_query_filters.py [--calls 20] [--no-profile]
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

N, DIM, VOCAB, B, LIMIT = 1_000_000, 768, 200_000, 256, 10


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--no-profile", action="store_true")
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
    st.add_number_field("price", ids, rng.random(N) * 100.0)

    def where(lo, width):
        return ob.evaluate_where(ob.parse_where({"price": {"between": [lo, lo + width]}}), st, {}, N, [])
    wide = where(20.0, 30.0)
    mixed = [where(float(rng.uniform(0, 50)), float(w)) for w in np.exp(rng.uniform(np.log(1.0), np.log(50.0), B))]
    tiny = [where(float(rng.uniform(0, 99.9)), 0.05) for _ in range(B)]
    one = [mixed[0]] + [None] * (B - 1)

    def batched(name, **kw):
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, **kw)
        tsc.execute_batch_arrays(p, batch, qv)
        t, unproven = [], 0
        for _ in range(a.calls):
            tsc.execute_batch_arrays(p, batch, qv)
            lt = ctx.last_timing()
            t.append(lt["device_ms"]); unproven = max(unproven, lt["scan_unproven"])
        s = stats(t)
        print(json.dumps({"case": name, "B": B, "limit": LIMIT, "device_ms": s, "qps": B / s["median"] * 1e3,
                          "scan_unproven_max": unproven, **info}), flush=True)
        return s

    res = {}
    res["a"] = batched("(a) no filter")
    res["b"] = batched("(b) one batch-wide where filter", device_filter=wide)
    res["c"] = batched("(c) 256 distinct per-query filters, 1-50 %", device_filters=mixed)
    # (d): each query alone with its filter
    for q in range(B):   # warm-up of every shape
        tsc.execute_batch_arrays(ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=mixed[q]),
                                 [texts[q]], qv[q:q + 1])
    tot = []
    for _ in range(a.calls):
        s = 0.0
        for q in range(B):
            tsc.execute_batch_arrays(ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=mixed[q]),
                                     [texts[q]], qv[q:q + 1])
            s += ctx.last_timing()["device_ms"]
        tot.append(s)
    res["d"] = stats(tot)
    print(json.dumps({"case": "(d) the same 256 queries alone, each with its filter", "B": 1, "calls_per_round": B,
                      "device_ms_per_round": res["d"], "qps": B / res["d"]["median"] * 1e3, **info}), flush=True)
    res["e"] = batched("(e) one filtered query, 255 unfiltered", device_filters=one)
    res["f"] = batched("(f) 256 distinct 0.05 % filters", device_filters=tiny)
    print(json.dumps({"headline": "(c) / (d) throughput", "speedup": res["d"]["median"] / res["c"]["median"], **info}), flush=True)

    if not a.no_profile:
        try:
            import torch
            from torch.profiler import ProfilerActivity, profile
            p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filters=mixed)
            tsc.execute_batch_arrays(p, batch, qv)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                tsc.execute_batch_arrays(p, batch, qv)
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if "rows_ok_kernel" in e.name]
            us = [getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) for e in ev]
            print(json.dumps({"profile": "rows_ok_kernel in one (c) call", "launches": len(ev), "device_us": [float(x) for x in us],
                              **info}), flush=True)
        except Exception as e:   # the measurement above stands without the breakdown
            print(json.dumps({"profile": "unavailable", "error": repr(e)}), flush=True)

    for f in [wide] + mixed + tiny:
        f.close()
    st.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
