"""Cost of where-filter leaves over filter fields (oc_filter_facet_range / oc_filter_facet_variant), of a whole `where`
clause, and of searching under one.

Runs, at 1M and 10M documents (one value per document in each field):
  * a range leaf of a number field at 0.1 / 10 / 50 / 100 % selectivity, a bool leaf and a string_filter leaf, each
    against what a caller does without them: numpy `searchsorted` over the sorted values (or the variant's id list)
    plus `oc_filter_from_ids` of the same ids, which uploads 8 B per id;
  * one 4-leaf `where` (number range, bool, string, NOT of another range) with 1000 uncommitted deletes, end to end
    (parse, compile, deletes handle, one oc_filter_from_where), through `evaluate_where`;
  * at 1M only, the h1 oc_search (hybrid, 1M x 768-d fp32 + BM25 over 1M synthetic docs, B = 256, top 10) without a
    filter, under that `where`, and under the same documents built with `from_ids`.
Leaves and clauses: host wall time of the whole synchronous call, median / min / max of --calls calls after one
warm-up call.  Searches: oc_last_timing.device_ms (CUDA events).  The card's name and power limit are read in the same
process.  Writes nothing into the tree.

    python tools/bench_where.py [--calls 20] [--skip-search]
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

N, DIM, VOCAB, B, LIMIT = 1_000_000, 768, 200_000, 256, 10


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}


def timed(make, calls):
    make().close()   # warm-up of this shape
    t = []
    for _ in range(calls):
        t0 = time.perf_counter()
        f = make()
        t.append((time.perf_counter() - t0) * 1e3)
        if f is not None:
            f.close()
    return stats(t)


def build_store(ctx, n, rng):
    ids = np.arange(n, dtype=np.uint64)
    price = rng.random(n) * 1000.0
    st = ob.FacetStore(ctx, n)
    st.add_number_field("price", ids, price)
    ok = rng.random(n) < 0.5
    st.add_bool_field("ok", ids[ok], ids[~ok])
    cat = rng.integers(0, 8, n)
    st.add_string_field("cat", {f"c{k}": ids[cat == k] for k in range(8)})
    host = {"price_sorted": np.sort(price), "price_order": ids[np.argsort(price, kind="stable")], "ok": ids[ok],
            "cat3": ids[cat == 3]}
    return st, host


WHERE = {"price": {"between": [100, 700]}, "ok": True, "cat": "c3", "not": {"price": {"gt": 650}}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--skip-search", action="store_true")
    a = ap.parse_args()
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi": card()}
    rng = np.random.default_rng(4)
    for n in (1_000_000, 10_000_000):
        st, host = build_store(ctx, n, rng)
        for sel in (0.001, 0.1, 0.5, 1.0):
            hi = 1000.0 * sel
            leaf = st.leaf("price", ob.parse_where({"price": {"lte": hi}}).filter_on_fields[0][1])
            docs = leaf.count()
            leaf.close()
            flt = ob.parse_where({"price": {"lte": hi}}).filter_on_fields[0][1]
            vs, order = host["price_sorted"], host["price_order"]

            def by_ids():
                k = np.searchsorted(vs, hi, side="right")
                return ob.DeviceFilter.from_ids(ctx, order[:k], n)
            row = {"leaf": "range", "documents": n, "selectivity": sel, "documents_in_leaf": docs,
                   "facet_range_ms": timed(lambda: st.leaf("price", flt), a.calls),
                   "searchsorted_from_ids_ms": timed(by_ids, a.calls)}
            print(json.dumps({**row, **info}), flush=True)
        for name, key, flt, ids in [("bool", "ok", True, host["ok"]), ("string", "cat", "c3", host["cat3"])]:
            row = {"leaf": name, "documents": n, "documents_in_leaf": int(ids.shape[0]),
                   "facet_variant_ms": timed(lambda: st.leaf(key, flt), a.calls),
                   "from_ids_ms": timed(lambda: ob.DeviceFilter.from_ids(ctx, ids, n), a.calls)}
            print(json.dumps({**row, **info}), flush=True)
        deleted = rng.choice(n, 1000, replace=False)
        f = ob.evaluate_where(ob.parse_where(WHERE), st, {}, n, deleted)
        row = {"where": WHERE, "documents": n, "deletes": 1000, "documents_in_filter": f.count(),
               "evaluate_where_ms": timed(lambda: ob.evaluate_where(ob.parse_where(WHERE), st, {}, n, deleted), a.calls)}
        f.close()
        print(json.dumps({**row, **info}), flush=True)
        if n == N and not a.skip_search:
            search_rows(ctx, st, deleted, a.calls, info)
        st.close()
    ctx.close()


def search_rows(ctx, st, deleted, calls, info):
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
    wf = ob.evaluate_where(ob.parse_where(WHERE), st, {}, N, deleted)
    bits = wf.read()
    same = ob.DeviceFilter.from_ids(ctx, np.flatnonzero(np.unpackbits(bits.view(np.uint8), bitorder="little")[:N]), N)
    for name, f in [("oc_search", None), ("oc_search under the where filter", wf),
                    ("oc_search under an id leaf, same documents", same)]:
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=f)
        tsc.execute_batch_arrays(p, texts, qv)
        t = []
        for _ in range(calls):
            tsc.execute_batch_arrays(p, texts, qv)
            t.append(ctx.last_timing()["device_ms"])
        row = {"call": name, "B": B, "limit": LIMIT, "documents_in_filter": None if f is None else f.count(),
               "device_ms": stats(t)}
        print(json.dumps({**row, **info}), flush=True)
    wf.close(); same.close(); emb.close(); strs.close()


if __name__ == "__main__":
    main()
