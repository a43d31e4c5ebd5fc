"""One oc_search_indexes call against n per-index oc_search calls plus the host merge, on the h1 shape (1M x 768-d fp32
embeddings + BM25 over 1M synthetic docs, hybrid, B = 256, top 10) split by doc id mod n into n = 2 and 4 indexes.

Per configuration it alternates the two paths over the same batch and prints one JSON line with, per path, the
median wall time of a whole search (host clock around calls that end in a device synchronise), the device time
(oc_last_timing.device_ms, summed over the n calls for the per-index path) and the bytes copied back to the host; and
whether the two outputs are byte-identical.  The card's name and power limit are read in the same process.  Writes
nothing into the tree.

    python tools/bench_multi_index.py [--calls 20] [--indexes 2 4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oramacore_b200 as ob  # noqa: E402
from oramacore_b200 import synth  # noqa: E402
from oramacore_b200.types import FieldPostings, StringIndexData  # noqa: E402

N, DIM, VOCAB, B, LIMIT = 1_000_000, 768, 200_000, 256, 10


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def split_text(data, parts, i):
    """documents d with d % parts == i as one index (own row space, own average length and document count)."""
    f = data.fields[0]
    term_of = np.repeat(np.arange(f.n_terms, dtype=np.int64), np.diff(f.term_offsets.astype(np.int64)))
    docs = np.arange(i, data.n_rows, parts, dtype=np.uint64)
    sel = (f.post_row % parts) == i
    offs = np.zeros(f.n_terms + 1, np.uint64)
    offs[1:] = np.cumsum(np.bincount(term_of[sel], minlength=f.n_terms)).astype(np.uint64)
    lens = np.zeros(data.n_rows, np.int64)
    lens[f.post_row[sel]] = f.post_len[sel]
    fp = FieldPostings(float(lens[docs.astype(np.int64)].mean()), offs, (f.post_row[sel] // parts).astype(np.uint32),
                       f.post_tf[sel].copy(), f.post_len[sel].copy())
    return StringIndexData([fp], docs.shape[0], docs.shape[0], docs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--indexes", type=int, nargs="+", default=[2, 4])
    a = ap.parse_args()
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi": card()}
    rows = synth.make_vectors(N, DIM)
    qv, _ = synth.make_vector_queries(rows[:1 << 18], B)
    data = synth.make_text_corpus(N, VOCAB)
    texts = ob.TextQueryBatch(synth.make_text_queries(VOCAB, B))
    params = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0)
    per_params = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, offset=0, vector_limit=LIMIT, similarity=0.0)
    for n in a.indexes:
        stores, parts = [], []
        for i in range(n):
            docs = np.arange(i, N, n, dtype=np.uint64)
            e = ob.EmbeddingFieldStorage(ctx, "BGEBase")
            e.reserve(docs.shape[0])
            for s in range(0, docs.shape[0], 1 << 18):
                e.insert_batch(docs[s:s + (1 << 18)], rows[docs[s:s + (1 << 18)].astype(np.int64)])
            st = ob.StringFieldStorage(ctx, split_text(data, n, i))
            stores.append((e, st))
            parts.append(ob.IndexPart(ob.TokenScoreContext(ctx, e, st), texts, qv))

        def per_index():
            t0 = time.perf_counter()
            per, dev, d2h = [], 0.0, 0
            for p in parts:
                per.append(p.tsc.execute_batch_arrays(per_params, texts, qv))
                t = ctx.last_timing()
                dev += t["device_ms"]; d2h += t["d2h_bytes"]
            hits = ob.merge_index_results(per, LIMIT, 0)
            return (time.perf_counter() - t0) * 1e3, dev, d2h, hits

        def one_call():
            t0 = time.perf_counter()
            d, s, _, nn, c, _, _ = ob.search_indexes_arrays(ctx, parts, params)
            wall = (time.perf_counter() - t0) * 1e3
            t = ctx.last_timing()
            hits = [ob.SearchHits(d[q, :nn[q]].copy(), s[q, :nn[q]].copy(), int(c[q])) for q in range(B)]
            return wall, t["device_ms"], t["d2h_bytes"], hits

        for _ in range(3):   # warm every shape
            per_index(); one_call()
        res = {"per_index": [], "one_call": []}
        same = True
        for _ in range(a.calls):
            x, y = per_index(), one_call()
            res["per_index"].append(x[:3]); res["one_call"].append(y[:3])
            same = same and all(np.array_equal(h.doc_ids, g.doc_ids) and np.array_equal(h.scores.view(np.uint32), g.scores.view(np.uint32))
                                and h.count == g.count for h, g in zip(x[3], y[3]))
        out = dict(info, indexes=n, batch=B, limit=LIMIT, calls=a.calls, byte_identical=bool(same))
        for k, v in res.items():
            arr = np.asarray(v)
            out[k] = {"wall_ms_median": float(np.median(arr[:, 0])), "device_ms_median": float(np.median(arr[:, 1])),
                      "d2h_bytes": int(arr[0, 2])}
        print(json.dumps(out), flush=True)
        for e, st in stores:
            e.close(); st.close()
    ctx.close()


if __name__ == "__main__":
    main()
