"""Where the fulltext stage's time goes in the h1 call shape, and what the dense-array cache of hot terms saves.

The h1 workload of bench.py (1M x 768 fp32 embeddings, BM25 over the same 1M synthetic documents, hybrid, B = 256,
limit 10) runs through `execute_batch_arrays` over the same 8 rotating seeded batches as bench.py, in four
configurations: the dense-array cache on (OC_BM25_DENSE_CACHE_MB unset: the default budget) and off (= 0, every call
builds its hot terms' arrays from scratch), each with the side stream on and off (OC_SIDE_STREAM=0).  Per
configuration the script reports
  * per call: `device_ms` and the stage times of `last_timing()` (median / min / max of --calls calls after a warm-up
    pass over the 8 batches);
  * from a separate `torch.profiler` run over 8 calls: every kernel, memset and copy by name and stream (count and
    device ms per call), and per call the device time inside the call's window when nothing ran on any stream (idle);
  * per batch the number of hot terms (a posting in at least every 16th row) and the bytes of their dense arrays
    (with their summaries: presence bitmap and tile maxima), from the corpus, as the library selects them;
  * per call: the dense passes of the register-folded scorers and the share of them replaced by a count pass
    (`bm25_dense_items` / `bm25_dense_skipped` of `last_timing()`).
The card's name, power limit and SM clock limit are read in the same process.  Writes nothing into the tree (the
traces go to a temporary directory unless --trace-dir names one).

    python tools/bench_ft_stage.py [--calls 40] [--n-docs 1000000] [--trace-dir DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oramacore_b200 as ob  # noqa: E402
from oramacore_b200 import synth  # noqa: E402

B, LIMIT, DIM, VOCAB, N_BATCHES = 256, 10, 768, 200_000, 8
TILE = 8192   # BM25_TILE
CONFIGS = [("cache", None, None), ("no-cache", "0", None), ("cache, no side stream", None, "0"),
           ("no-cache, no side stream", "0", "0")]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}


def hot_terms(data, texts, n_rows):
    """Per batch: the distinct hot terms (list length >= max(512, n_rows / 16)) and the bytes of their dense arrays."""
    offs = data.fields[0].term_offsets
    dense_min = max(512, n_rows // 16)
    n_tiles = (n_rows + TILE - 1) // TILE
    rows_pad = n_tiles * TILE
    arr_bytes = rows_pad * 4 + rows_pad // 8 + (n_tiles * 4 + 255) // 256 * 256   # bm25_dense_bytes
    out = []
    for batch in texts:
        ids = set()
        for q in batch:
            for t in q.term_id.tolist():
                if int(offs[t + 1] - offs[t]) >= dense_min:
                    ids.add(t)
        out.append({"n_dense": len(ids), "dense_bytes": len(ids) * arr_bytes})
    return out


def set_env(cache, side):
    for k, v in (("OC_BM25_DENSE_CACHE_MB", cache), ("OC_SIDE_STREAM", side)):
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def timed(ctx, step, calls):
    for k in range(N_BATCHES):   # warm-up: every batch once (the cache, when on, is filled here)
        step(k)
    t, items, skipped = {}, 0, 0
    for k in range(calls):
        step(k)
        lt = ctx.last_timing()
        for key, v in lt.items():
            if key.endswith("_ms"):
                t.setdefault(key, []).append(v)
        items += lt["bm25_dense_items"]
        skipped += lt["bm25_dense_skipped"]
    out = {k: stats(v) for k, v in t.items() if max(v) > 0}
    out["dense_items_per_call"] = items / calls
    out["dense_skipped_fraction"] = skipped / items if items else 0.0
    return out


def profiled(step, trace_dir, tag):
    import torch
    from torch.profiler import ProfilerActivity, profile
    for k in range(N_BATCHES):
        step(k)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        for k in range(N_BATCHES):
            step(k)
        torch.cuda.synchronize()
    path = os.path.join(trace_dir, tag.replace(", ", "_").replace(" ", "-") + ".pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    dev = [e for e in ev if e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy") and "dur" in e]
    dev.sort(key=lambda e: e["ts"])
    per = {}
    for e in dev:
        name = e["name"].split("(")[0].split("<")[0].replace("void ", "").strip()
        if e["cat"] != "kernel":
            name = e["cat"] + ": " + name
        key = f"{name} [stream {e.get('args', {}).get('stream', '?')}]"
        p = per.setdefault(key, [0, 0.0])
        p[0] += 1
        p[1] += e["dur"] / 1e3
    # idle: a call's window runs from the first device event after the previous call's last one; calls are separated
    # by the host gap between them (every call ends in a synchronise), found as the N_BATCHES - 1 widest gaps
    gaps = [(dev[i + 1]["ts"] - max(d["ts"] + d["dur"] for d in dev[:i + 1]), i) for i in range(len(dev) - 1)]
    cuts = sorted(i for _, i in sorted(gaps, reverse=True)[:N_BATCHES - 1])
    idle, bounds, lo = [], [], 0
    for hi in cuts + [len(dev) - 1]:
        win = dev[lo:hi + 1]
        busy, end = 0.0, None
        for d in win:
            s, t = d["ts"], d["ts"] + d["dur"]
            if end is None or s >= end:
                busy += t - s
                end = t
            elif t > end:
                busy += t - end
                end = t
        span = max(d["ts"] + d["dur"] for d in win) - win[0]["ts"]
        idle.append((span - busy) / 1e3)
        bounds.append(span / 1e3)
        lo = hi + 1
    return {"per_call": {k: {"count": v[0] / N_BATCHES, "ms": v[1] / N_BATCHES}
                         for k, v in sorted(per.items(), key=lambda kv: -kv[1][1])},
            "call_window_ms": stats(bounds), "idle_in_window_ms": stats(idle)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=40)
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--trace-dir", default=None, help="keep the torch.profiler traces here")
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    ctx = ob.Context(0)   # no device: an error, there is nothing to measure without one
    print(json.dumps({"card": card(), "workload": "h1", "n_docs": a.n_docs, "B": B, "limit": LIMIT,
                      "calls": a.calls}), flush=True)
    rows = synth.make_vectors(a.n_docs, DIM)
    qv = [synth.make_vector_queries(rows, B, seed=synth.SEED_VQUERIES + i)[0] for i in range(N_BATCHES)]
    data = synth.make_text_corpus(a.n_docs, VOCAB)
    texts = [synth.make_text_queries(VOCAB, B, seed=synth.SEED_TQUERIES + i) for i in range(N_BATCHES)]
    for i, h in enumerate(hot_terms(data, texts, a.n_docs)):
        print(json.dumps({"batch": i, **h}), flush=True)
    emb = ob.EmbeddingFieldStorage(ctx, dim=DIM, model="BGEBase")
    emb.reserve(a.n_docs)
    ids = np.arange(a.n_docs, dtype=np.uint64)
    for i in range(0, a.n_docs, 1 << 18):
        emb.insert_batch(ids[i:i + (1 << 18)], rows[i:i + (1 << 18)])
    del rows
    strs = ob.StringFieldStorage(ctx, data)
    tsc = ob.TokenScoreContext(ctx, emb, strs)
    params = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0)
    packed = [ob.TextQueryBatch(t) for t in texts]
    qv_host = []
    for q in qv:
        h = ob.pinned_empty(q.shape, np.float32)
        h[...] = q
        qv_host.append(h)

    def step(k):
        return tsc.execute_batch_arrays(params, packed[k % N_BATCHES], qv_host[k % N_BATCHES])

    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        trace_dir = a.trace_dir or tmp
        os.makedirs(trace_dir, exist_ok=True)
        for tag, cache, side in CONFIGS:
            set_env(cache, side)
            r = {"config": tag, **timed(ctx, step, a.calls)}
            outs[tag] = [np.ascontiguousarray(x).tobytes() for k in range(N_BATCHES) for x in step(k)]
            print(json.dumps(r), flush=True)
            if not a.no_profile:
                print(json.dumps({"config": tag, "profile": profiled(step, trace_dir, tag)}), flush=True)
    set_env(None, None)
    ref = outs[CONFIGS[1][0]]
    print(json.dumps({"outputs_identical_to_no_cache": {t: o == ref for t, o in outs.items()}}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
