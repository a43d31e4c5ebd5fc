"""Cost of groupBy on the h1 shape (1M x 768-d fp32 embeddings + BM25 over 1M synthetic docs, hybrid, B = 256, top 10).

Runs the same batches through oc_search and through oc_search_groups for
  * one string_filter field with 10 keys, with 1000 keys, and a bool x string_filter (10 keys) grouping,
  * max_results 1 and 10,
and prints one JSON line per configuration with the per-call device time (oc_last_timing.device_ms, CUDA events;
for oc_search_groups it includes the group stage).  With --profile it instead runs each configuration under
torch.profiler and prints the group kernel's own time.  The card's name and power limit are read in the same
process.  Writes nothing into the tree.

    python tools/bench_groups.py [--calls 20] [--profile]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi": card()}
    rows = synth.make_vectors(N, DIM)
    emb = ob.EmbeddingFieldStorage(ctx, "BGEBase")
    emb.reserve(N)
    ids = np.arange(N, dtype=np.uint64)
    for i in range(0, N, 1 << 18):
        emb.insert_batch(ids[i:i + (1 << 18)], rows[i:i + (1 << 18)])
    qv, _ = synth.make_vector_queries(rows[:1 << 18], B)
    del rows
    strs = ob.StringFieldStorage(ctx, synth.make_text_corpus(N, VOCAB))
    texts = ob.TextQueryBatch(synth.make_text_queries(VOCAB, B))
    tsc = ob.TokenScoreContext(ctx, emb, strs)
    params = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0)
    rng = np.random.default_rng(5)
    st = ob.FacetStore(ctx, N)
    for k in (10, 1000):
        key = rng.integers(0, k, size=N)
        order = np.argsort(key, kind="stable")
        bounds = np.searchsorted(key[order], np.arange(k + 1))
        st.add_string_field(f"s{k}", {f"k{j}": ids[order[bounds[j]:bounds[j + 1]]] for j in range(k)})
    flag = rng.random(N) < 0.5
    st.add_bool_field("b", ids[flag], ids[~flag])
    configs = [(["s10"], 1), (["s10"], 10), (["s1000"], 1), (["s1000"], 10), (["b", "s10"], 1), (["b", "s10"], 10)]

    def device_ms(fn):
        fn()   # warm-up of this shape
        t = []
        for _ in range(a.calls):
            fn()
            t.append(ctx.last_timing()["device_ms"])
        return float(np.median(t)), float(np.min(t)), float(np.max(t))

    if not a.profile:
        base = device_ms(lambda: tsc.execute_batch_arrays(params, texts, qv))
        print(json.dumps({"call": "oc_search", "B": B, "limit": LIMIT, "device_ms_median": base[0], "device_ms_min": base[1],
                          "device_ms_max": base[2], **info}), flush=True)
    for props, m in configs:
        gb = ob.GroupBy(st, props)
        run = lambda: ob.search_groups_arrays(tsc, gb, params, m, texts=texts, q_vecs=qv)  # noqa: E731
        if a.profile:
            import torch
            from torch.profiler import ProfilerActivity, profile
            run()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.calls):
                    run()
                torch.cuda.synchronize()
            ev = [e for e in prof.key_averages() if "group_topk_kernel" in e.key]
            us = (sum(e.device_time_total for e in ev) / a.calls) if ev else float("nan")
            print(json.dumps({"call": "group_topk_kernel", "groups": props, "n_groups": gb.n_groups, "max_results": m,
                              "kernel_ms_per_call": us / 1e3, **info}), flush=True)
        else:
            t = device_ms(run)
            print(json.dumps({"call": "oc_search_groups", "groups": props, "n_groups": gb.n_groups, "max_results": m, "B": B,
                              "limit": LIMIT, "device_ms_median": t[0], "device_ms_min": t[1], "device_ms_max": t[2], **info}), flush=True)
        gb.close()
    st.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
