"""Cost of pin rules on the h1 shape (1M x 768-d fp32 embeddings + BM25 over 1M synthetic docs, hybrid, B = 256, top 10).

Runs the same batches through
  * oc_search, and oc_search_pinned with 0, 3 and 50 promote items per query (random documents, positions 0-19);
  * oc_search_groups and oc_search_groups_pinned (3 items per query, max_results 10) over one string_filter field
    with 10 keys and with 1000 keys,
and prints one JSON line per configuration with the per-call device time (oc_last_timing.device_ms, CUDA events).
With --profile it instead runs each pinned configuration under torch.profiler and prints the device time per call of
every kernel whose name contains "pin_" (pin_score_kernel, pin_splice_kernel, group_pin_splice_kernel).  The card's
name and power limit are read in the same process.  Writes nothing into the tree.

    python tools/bench_pins.py [--calls 20] [--profile]
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
    promote = {k: [[(int(d), int(p)) for d, p in zip(rng.integers(0, N, size=k), rng.integers(0, 20, size=k))] for _ in range(B)]
               for k in (0, 3, 50)}
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

    def pin_kernels_ms(fn):
        import torch
        from torch.profiler import ProfilerActivity, profile
        fn()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.calls):
                fn()
            torch.cuda.synchronize()
        return {e.key: e.device_time_total / a.calls / 1e3 for e in prof.key_averages() if "pin_" in e.key}

    configs = [("oc_search", None, lambda: tsc.execute_batch_arrays(params, texts, qv))]
    for k in (0, 3, 50):
        configs.append(("oc_search_pinned", {"items_per_query": k},
                        lambda k=k: ob.search_pinned_arrays(tsc, params, promote[k], texts=texts, q_vecs=qv)))
    gbs = []
    for k in (10, 1000):
        gb = ob.GroupBy(st, [f"s{k}"])
        gbs.append(gb)
        configs.append(("oc_search_groups", {"n_groups": gb.n_groups, "max_results": MAX_RESULTS},
                        lambda gb=gb: ob.search_groups_arrays(tsc, gb, params, MAX_RESULTS, texts=texts, q_vecs=qv)))
        configs.append(("oc_search_groups_pinned", {"n_groups": gb.n_groups, "max_results": MAX_RESULTS, "items_per_query": 3},
                        lambda gb=gb: ob.search_groups_arrays(tsc, gb, params, MAX_RESULTS, texts=texts, q_vecs=qv, promote=promote[3])))
    for name, extra, fn in configs:
        row = {"call": name, **(extra or {}), "B": B, "limit": LIMIT}
        if a.profile:
            if "pinned" not in name:
                continue
            row["pin_kernels_ms_per_call"] = pin_kernels_ms(fn)
        else:
            row.update(device_ms(fn))
        print(json.dumps({**row, **info}), flush=True)
    for gb in gbs:
        gb.close()
    st.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
