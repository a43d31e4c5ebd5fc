"""Cost of sortBy on the h1 shape (1M x 768-d fp32 embeddings + BM25 over 1M synthetic docs, hybrid, B = 256, top 10).

A random number field holds one value for every document.  Runs
  * oc_search and oc_search_sorted (ASC) on the same batches, and oc_search_sorted with 3 promote items per query;
  * the full walk: fulltext queries of one rare term each whose matches all rank last in a second field, so the walk
    passes every ranked document before it has its top 10;
  * oc_search_groups and oc_search_groups_sorted (max_results 10) over a string_filter field with 10 and 1000 keys,
and prints one JSON line per configuration with the per-call device time (oc_last_timing.device_ms, CUDA events;
median / min / max of --calls calls after one warm-up call).  With --profile it instead runs each sorted configuration
under torch.profiler and prints the device time per call of the kernels the sorted path adds (sort_walk_kernel,
group_sort_topk_kernel, and the pin kernels it reuses to score and page).  The card's name and power limit are read in
the same process.  Writes nothing into the tree.

    python tools/bench_sort.py [--calls 20] [--profile]
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

N, DIM, VOCAB, B, LIMIT, MAX_RESULTS = 1_000_000, 768, 200_000, 256, 10, 10


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
    promote = [[(int(d), int(p)) for d, p in zip(rng.integers(0, N, size=3), rng.integers(0, 20, size=3))] for _ in range(B)]
    field = ob.SortField(ctx, N, ids, rng.random(N), "number")
    # the full walk: one rare term per query (at most 1024 matches each, found by a plain search), all ranked last
    ft = ob.TokenScoreContext(ctx, None, strs)
    rare = ob.TextQueryBatch([ob.TextQuery.single_terms([t]) for t in range(VOCAB - B, VOCAB)])
    all_p = ob.TokenScoreParams(mode=ob.MODE_FULLTEXT, limit_hint=1024)
    d, _, n, cnt = ft.execute_batch_arrays(all_p, rare)
    last = np.zeros(N)
    for q in range(B):
        last[d[q, :n[q]].astype(np.int64)] = 1.0
    info["full_walk_queries_with_all_keys_known"] = int((cnt <= 1024).sum())
    info["full_walk_queries_with_a_match"] = int((cnt > 0).sum())
    field_last = ob.SortField(ctx, N, ids, last, "number")
    ft_params = ob.TokenScoreParams(mode=ob.MODE_FULLTEXT, limit_hint=LIMIT)
    st = ob.FacetStore(ctx, N)
    for k in (10, 1000):
        key = rng.integers(0, k, size=N)
        order = np.argsort(key, kind="stable")
        bounds = np.searchsorted(key[order], np.arange(k + 1))
        st.add_string_field(f"s{k}", {f"k{j}": ids[order[bounds[j]:bounds[j + 1]]] for j in range(k)})

    def device_ms(fn):
        fn()   # warm-up of this shape
        t = []
        for _ in range(a.calls):
            fn()
            t.append(ctx.last_timing()["device_ms"])
        return {"device_ms_median": float(np.median(t)), "device_ms_min": float(np.min(t)), "device_ms_max": float(np.max(t))}

    def sort_kernels_ms(fn):
        import torch
        from torch.profiler import ProfilerActivity, profile
        fn()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.calls):
                fn()
            torch.cuda.synchronize()
        return {e.key: e.device_time_total / a.calls / 1e3 for e in prof.key_averages() if "sort_" in e.key or "pin_" in e.key}

    configs = [("oc_search", None, lambda: tsc.execute_batch_arrays(params, texts, qv)),
               ("oc_search_sorted", None, lambda: ob.search_sorted_arrays(tsc, params, field, "ASC", texts=texts, q_vecs=qv)),
               ("oc_search_sorted", {"items_per_query": 3},
                lambda: ob.search_sorted_arrays(tsc, params, field, "ASC", promote=promote, texts=texts, q_vecs=qv)),
               ("oc_search", {"mode": "fulltext", "queries": "rare terms"}, lambda: ft.execute_batch_arrays(ft_params, rare)),
               ("oc_search_sorted", {"mode": "fulltext", "queries": "rare terms", "walk": "full"},
                lambda: ob.search_sorted_arrays(ft, ft_params, field_last, "ASC", texts=rare))]
    gbs = []
    for k in (10, 1000):
        gb = ob.GroupBy(st, [f"s{k}"])
        gbs.append(gb)
        configs.append(("oc_search_groups", {"n_groups": gb.n_groups, "max_results": MAX_RESULTS},
                        lambda gb=gb: ob.search_groups_arrays(tsc, gb, params, MAX_RESULTS, texts=texts, q_vecs=qv)))
        configs.append(("oc_search_groups_sorted", {"n_groups": gb.n_groups, "max_results": MAX_RESULTS},
                        lambda gb=gb: ob.search_groups_arrays(tsc, gb, params, MAX_RESULTS, texts=texts, q_vecs=qv,
                                                              sort_by=(field, "ASC"))))
    for name, extra, fn in configs:
        row = {"call": name, **(extra or {}), "B": B, "limit": LIMIT}
        if a.profile:
            if "sorted" not in name:
                continue
            row["kernels_ms_per_call"] = sort_kernels_ms(fn)
        else:
            row.update(device_ms(fn))
        print(json.dumps({**row, **info}), flush=True)
    for gb in gbs:
        gb.close()
    field.close(); field_last.close(); st.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
