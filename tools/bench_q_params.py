"""What a batch in which every query has its own mode, limit, offset, similarity and threshold (oc_search_params.q_params)
costs, on the h1 shape: 1M x 768-d fp32 + BM25 over 1M synthetic documents, B = 256.  A third of the queries are
fulltext, a third vector, a third hybrid; limit 5-50, offset 0-40, similarity {0, 0.5, 0.7}, threshold {None, 0.5}.

  (a) one oc_search with q_params;
  (b) the same requests split by the scalars (the batcher's default key) into uniform calls, summed;
  (c) each request alone, summed;
  (d) the uniform h1 batch (hybrid, limit 10, similarity 0), the reference point;
  (e) 256 threads, one request each per round, through SearchBatcher without and with mixed=True: queries per batch and
      end-to-end QPS.
Rows (a)-(d): median / min / max over --calls calls of oc_last_timing.device_ms (CUDA events; (b), (c): the sum over a
round's calls).  The card's name and power limit are read in the same process.  Writes nothing into the tree.

    python tools/bench_q_params.py [--calls 20] [--rounds 3]
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

N, DIM, VOCAB, B = 1_000_000, 768, 200_000, 256


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
    rng = np.random.default_rng(9)
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
    modes = (ob.MODE_FULLTEXT, ob.MODE_VECTOR, ob.MODE_HYBRID)
    entries = [ob.QueryParams(mode=modes[i % 3], limit=int(rng.integers(5, 51)), offset=int(rng.integers(0, 41)),
                              similarity=float(rng.choice([0.0, 0.5, 0.7])),
                              threshold=None if rng.random() < 0.5 else 0.5) for i in range(B)]

    def one_params(e):
        return ob.TokenScoreParams(mode=e.mode, limit_hint=e.limit, offset=e.offset, similarity=e.similarity, threshold=e.threshold)

    def timed(fn):
        fn()
        t = []
        for _ in range(a.calls):
            t.append(fn())
        return stats(t)

    def call_a():
        tsc.execute_batch_arrays(ob.TokenScoreParams(mode=ob.MODE_HYBRID, query_params=entries), batch, qv)
        return ctx.last_timing()["device_ms"]
    res = {"a": timed(call_a)}
    print(json.dumps({"case": "(a) one oc_search with q_params", "B": B, "device_ms": res["a"],
                      "qps": B / res["a"]["median"] * 1e3, **info}), flush=True)

    groups = {}
    for i, e in enumerate(entries):
        groups.setdefault((e.mode, e.limit, e.offset, e.similarity, e.threshold), []).append(i)

    def call_b():
        s = 0.0
        for (m, lim, off, sim, thr), qs in groups.items():
            p = ob.TokenScoreParams(mode=m, limit_hint=lim, offset=off, similarity=sim, threshold=thr)
            tsc.execute_batch_arrays(p, [texts[q] for q in qs] if m != ob.MODE_VECTOR else None,
                                     qv[qs] if m != ob.MODE_FULLTEXT else None)
            s += ctx.last_timing()["device_ms"]
        return s
    res["b"] = timed(call_b)
    print(json.dumps({"case": "(b) split by the scalars into uniform calls, summed", "calls_per_round": len(groups),
                      "device_ms_per_round": res["b"], "qps": B / res["b"]["median"] * 1e3, **info}), flush=True)

    def call_c():
        s = 0.0
        for q, e in enumerate(entries):
            tsc.execute_batch_arrays(one_params(e), [texts[q]] if e.mode != ob.MODE_VECTOR else None,
                                     qv[q:q + 1] if e.mode != ob.MODE_FULLTEXT else None)
            s += ctx.last_timing()["device_ms"]
        return s
    res["c"] = timed(call_c)
    print(json.dumps({"case": "(c) each request alone, summed", "calls_per_round": B, "device_ms_per_round": res["c"],
                      "qps": B / res["c"]["median"] * 1e3, **info}), flush=True)

    def call_d():
        tsc.execute_batch_arrays(ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=10, similarity=0.0), batch, qv)
        return ctx.last_timing()["device_ms"]
    res["d"] = timed(call_d)
    print(json.dumps({"case": "(d) the uniform h1 batch (hybrid, limit 10)", "B": B, "device_ms": res["d"],
                      "qps": B / res["d"]["median"] * 1e3, **info}), flush=True)
    print(json.dumps({"headline": "device time (b) / (a), (c) / (a)", "split_over_mixed": res["b"]["median"] / res["a"]["median"],
                      "alone_over_mixed": res["c"]["median"] / res["a"]["median"], **info}), flush=True)

    def run_threads(bat):
        go = threading.Barrier(B + 1)

        def w(q):
            e = entries[q]
            go.wait()
            bat.search(one_params(e), texts[q] if e.mode != ob.MODE_VECTOR else None, qv[q] if e.mode != ob.MODE_FULLTEXT else None)
        th = [threading.Thread(target=w, args=(q,)) for q in range(B)]
        for x in th:
            x.start()
        go.wait()
        t0 = time.perf_counter()
        for x in th:
            x.join()
        return time.perf_counter() - t0
    bats = {"default key": ob.SearchBatcher(tsc, max_batch=B, max_wait_us=2000),
            "mixed": ob.SearchBatcher(tsc, max_batch=B, max_wait_us=2000, mixed=True)}
    for bat in bats.values():   # warm-up
        run_threads(bat)
    before = {k: b.stats() for k, b in bats.items()}
    e2e = {k: [] for k in bats}
    for _ in range(a.rounds):   # alternated
        for k, bat in bats.items():
            e2e[k].append(run_threads(bat))
    for k, bat in bats.items():
        s1, s0 = bat.stats(), before[k]
        nq, nb, nd = s1["queries"] - s0["queries"], s1["batches"] - s0["batches"], s1["direct"] - s0["direct"]
        print(json.dumps({"case": f"(e) 256 threads through SearchBatcher, {k}", "rounds": a.rounds,
                          "seconds_per_round": stats(e2e[k]), "qps": B / float(np.median(e2e[k])),
                          "queries_per_batch": nq / max(nb, 1), "direct": nd, **info}), flush=True)
        bat.close()
    emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
