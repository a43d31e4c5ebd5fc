"""One oc_search_indexes call against n per-index oc_search calls plus the host merge, on the h1 shape (1M x 768-d fp32
embeddings + BM25 over 1M synthetic docs, hybrid, B = 256, top 10) split by doc id mod n into n = 2 and 4 indexes.

Per configuration it alternates the two paths over the same batch and prints one JSON line with, per path, the
median wall time of a whole search (host clock around calls that end in a device synchronise), the device time
(oc_last_timing.device_ms, summed over the n calls for the per-index path) and the bytes copied back to the host; and
whether the two outputs are byte-identical.  The card's name and power limit are read in the same process.  Writes
nothing into the tree.

Two more arms per configuration (--arms): "grouped" groups by 4 categories x 8 number values (max_results 5) and
"faceted" counts three facet fields (a string_filter field, number ranges, a bool).  Their per-index path is
oc_search_q_groups / oc_search_q_facets per index plus the host merge of the group rows (oc_merge_results over the
collection's rows) or the host sum of the counts by label; the one call is oc_search_indexes_ex.  Their lines add the
host planning time of each path (the key union and key maps, or the facet slots, and the host merge or sum).

    python tools/bench_multi_index.py [--calls 20] [--indexes 2 4] [--arms flat grouped faceted]
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
GROUP_MAX = 5
FACETS = {"cat": {}, "num": {"ranges": [{"from": 0, "to": 3}, {"from": 4, "to": 7}]}, "flag": {"true": True, "false": True}}


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
    ap.add_argument("--arms", nargs="+", default=["flat", "grouped", "faceted"])
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
            fs = ob.FacetStore(ctx, N)
            di = docs.astype(np.int64)
            fs.add_string_field("cat", {f"c{k}": di[di % 4 == k] for k in range(4)})
            fs.add_number_field("num", di, (di % 8).astype(np.float64))
            fs.add_bool_field("flag", di[di % 3 == 0], di[di % 3 != 0])
            stores.append((e, st, fs))
            parts.append(ob.IndexPart(ob.TokenScoreContext(ctx, e, st), texts, qv, None, fs))

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

        gbs = [ob.GroupBy(p.store, ["cat", "num"]) for p in parts]
        groups = [(gbs, GROUP_MAX)] * B

        def per_index_grouped():
            t0 = time.perf_counter()
            per, dev, d2h, host = [], 0.0, 0, 0.0
            for p, gb in zip(parts, gbs):
                per.append(ob.search_q_groups_arrays(p.tsc, per_params, [(gb, GROUP_MAX)] * B, texts=texts, q_vecs=qv))
                t = ctx.last_timing()
                dev += t["device_ms"]; d2h += t["d2h_bytes"]
            h0 = time.perf_counter()
            keys, maps = ob.collection_group_keys(gbs)
            K = len(keys)
            lists = []
            for r, m in zip(per, maps):   # each index's rows scattered to the collection's rows (b, key)
                gd, gs, gn = r[7], r[8], r[10]
                G = gd.shape[0] // B
                dst = (np.arange(B)[:, None] * K + m[None, :G]).ravel()
                d = np.zeros((B * K, GROUP_MAX), np.uint64); s_ = np.zeros((B * K, GROUP_MAX), np.float32)
                nn = np.zeros(B * K, np.uint32)
                d[dst], s_[dst], nn[dst] = gd[:, :GROUP_MAX], gs[:, :GROUP_MAX], gn
                lists.append((d, s_, nn, np.zeros(B * K, np.uint64)))
            merged = ob.merge_index_results(lists, GROUP_MAX, 0)
            host += (time.perf_counter() - h0) * 1e3
            return (time.perf_counter() - t0) * 1e3, dev, d2h, host, merged

        def one_call_grouped():
            t0 = time.perf_counter()
            got = ob.search_indexes_arrays(ctx, parts, params, groups=groups)
            wall = (time.perf_counter() - t0) * 1e3
            t = ctx.last_timing()
            h0 = time.perf_counter()
            ob.collection_group_keys(gbs)   # the host planning of the call's Python side
            host = (time.perf_counter() - h0) * 1e3
            gd, gs, gn = got[7], got[8], got[10]
            return wall, t["device_ms"], t["d2h_bytes"], host, (gd, gs, gn)

        def same_grouped(x, y):
            gd, gs, gn = y
            return all(int(gn[r]) == len(h.doc_ids) and np.array_equal(gd[r, :gn[r]], h.doc_ids)
                       and np.array_equal(gs[r, :gn[r]].view(np.uint32), h.scores.view(np.uint32)) for r, h in enumerate(x))

        def per_index_faceted():
            t0 = time.perf_counter()
            per, dev, d2h = [], 0.0, 0
            for p in parts:
                per.append(ob.search_q_facets_arrays(p.tsc, p.store, per_params, [FACETS] * B, texts=texts, q_vecs=qv))
                t = ctx.last_timing()
                dev += t["device_ms"]; d2h += t["d2h_bytes"]
            h0 = time.perf_counter()
            tot = [{} for _ in range(B)]
            for r in per:
                fc, foff, labels = r[12], r[13], r[14]
                for b in range(B):
                    for j, lab in enumerate(labels[b]):
                        tot[b][lab] = tot[b].get(lab, 0) + int(fc[foff[b] + j])
            host = (time.perf_counter() - h0) * 1e3
            return (time.perf_counter() - t0) * 1e3, dev, d2h, host, tot

        def one_call_faceted():
            t0 = time.perf_counter()
            got = ob.search_indexes_arrays(ctx, parts, params, facets=[FACETS] * B)
            wall = (time.perf_counter() - t0) * 1e3
            t = ctx.last_timing()
            h0 = time.perf_counter()
            ob.collection_facet_requests([p.store for p in parts], FACETS)   # the host planning of the call's Python side
            host = (time.perf_counter() - h0) * 1e3
            fc, foff, labels = got[13], got[14], got[15]
            return wall, t["device_ms"], t["d2h_bytes"], host, [{lab: int(fc[foff[b] + j]) for j, lab in enumerate(labels[b])}
                                                                for b in range(B)]

        def same_flat(x, y):
            return all(np.array_equal(h.doc_ids, g.doc_ids) and np.array_equal(h.scores.view(np.uint32), g.scores.view(np.uint32))
                       and h.count == g.count for h, g in zip(x, y))

        arms = {"flat": (per_index, one_call, same_flat), "grouped": (per_index_grouped, one_call_grouped, same_grouped),
                "faceted": (per_index_faceted, one_call_faceted, lambda x, y: x == y)}
        for arm in a.arms:
            pa, oc, eq = arms[arm]
            for _ in range(3):   # warm every shape
                pa(); oc()
            res = {"per_index": [], "one_call": []}
            same = True
            for _ in range(a.calls):
                x, y = pa(), oc()
                res["per_index"].append(x[:-1]); res["one_call"].append(y[:-1])
                same = same and eq(x[-1], y[-1])
            out = dict(info, arm=arm, indexes=n, batch=B, limit=LIMIT, calls=a.calls, byte_identical=bool(same))
            for k, v in res.items():
                arr = np.asarray(v)
                out[k] = {"wall_ms_median": float(np.median(arr[:, 0])), "device_ms_median": float(np.median(arr[:, 1])),
                          "d2h_bytes": int(arr[0, 2])}
                if arr.shape[1] > 3:
                    out[k]["host_plan_ms_median"] = float(np.median(arr[:, 3]))
            print(json.dumps(out), flush=True)
        for g in gbs:
            g.close()
        for e, st, fs in stores:
            e.close(); st.close(); fs.close()
    ctx.close()


if __name__ == "__main__":
    main()
