"""Cost of `where` clauses evaluated inside the search call (where programs, oc_search_params.q_where) against the
handle path (one handle per clause, then q_filters).

Runs:
  * at 1M and 10M documents, the 4-leaf `where` of tools/bench_where.py with 1000 uncommitted deletes: evaluate_where
    (which builds NOT(deletes) on every call, then evaluates the clause's program with oc_filter_from_where) and
    compile_where + oc_filter_from_where (NOT(deletes) built once, as IndexLoader keeps it per set of deletes).  Host
    wall time of the whole synchronous work, median / min / max of --calls after one warm-up.
  * the h1 shape (hybrid, 1M x 768-d fp32 + BM25 over 1M synthetic docs, B = 256, top 10) with 256 distinct 4-leaf
    clauses: building 256 handles with evaluate_where + oc_search(q_filters), against compiling 256 programs + one
    oc_search(q_where).
    Wall time of the whole request path; the search's own wall time; and, from one torch.profiler run of each search,
    the summed device time of every kernel of the call and of its where kernels alone.  The outputs of both paths are
    compared byte for byte.
The card's name and power limit are read in the same process.  Writes nothing into the tree.

    python tools/bench_where_program.py [--calls 10] [--skip-search]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import oramacore_b200 as ob  # noqa: E402
from oramacore_b200 import synth  # noqa: E402
from oramacore_b200.where import compile_where, filter_from_program  # noqa: E402
from bench_where import WHERE, build_store, card, stats  # noqa: E402

N, DIM, VOCAB, B, LIMIT = 1_000_000, 768, 200_000, 256, 10


def wall(fn, calls):
    fn()   # warm-up of this shape
    t = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return stats(t)


def live_of(ctx, deleted, n):
    d = ob.DeviceFilter.from_ids(ctx, deleted, n)
    try:
        return ~d
    finally:
        d.close()


def clauses(rng, k):
    """k distinct 4-leaf clauses of WHERE's shape."""
    out = []
    for i in range(k):
        lo = float(rng.integers(0, 500)) + i * 1e-3
        out.append({"price": {"between": [lo, lo + 400]}, "ok": bool(i % 2), "cat": f"c{i % 8}",
                    "not": {"price": {"gt": lo + 350}}})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--skip-search", action="store_true")
    a = ap.parse_args()
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi": card()}
    rng = np.random.default_rng(4)
    for n in (1_000_000, 10_000_000):
        st, _ = build_store(ctx, n, rng)
        deleted = rng.choice(n, 1000, replace=False)
        live = live_of(ctx, deleted, n)
        w = ob.parse_where(WHERE)
        ref = ob.evaluate_where(w, st, {}, n, deleted)
        got = filter_from_program(ctx, compile_where(w, st, {}, n, live))
        same = ref.read().tobytes() == got.read().tobytes()
        ref.close(); got.close()
        row = {"where": WHERE, "documents": n, "deletes": 1000, "bit_identical": same,
               "evaluate_where_ms": wall(lambda: ob.evaluate_where(ob.parse_where(WHERE), st, {}, n, deleted).close(), a.calls),
               "compile_where_filter_from_where_ms": wall(
                   lambda: filter_from_program(ctx, compile_where(ob.parse_where(WHERE), st, {}, n, live)).close(), a.calls)}
        print(json.dumps({**row, **info}), flush=True)
        if n == N and not a.skip_search:
            search_rows(ctx, st, deleted, live, a.calls, info, rng)
        live.close()
        st.close()
    ctx.close()


def profiled(fn):
    """Summed device time (ms) of every kernel of fn's calls, and of the where / filter kernels among them."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    total = where = 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        total += us
        if "where_" in e.name or "filter_" in e.name:
            where += us
    return total / 1e3, where / 1e3


def search_rows(ctx, st, deleted, live, calls, info, rng):
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
    ws = [ob.parse_where(x) for x in clauses(rng, B)]
    kw = dict(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0)

    def handles_path():
        hs = [ob.evaluate_where(w, st, {}, N, deleted) for w in ws]
        try:
            return tsc.execute_batch_arrays(ob.TokenScoreParams(device_filters=hs, **kw), texts, qv)
        finally:
            for h in hs:
                h.close()

    def program_path():
        ps = [compile_where(w, st, {}, N, live) for w in ws]
        return tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=ps, **kw), texts, qv)

    a, b = handles_path(), program_path()
    same = all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    hs = [ob.evaluate_where(w, st, {}, N, deleted) for w in ws]
    ps = [compile_where(w, st, {}, N, live) for w in ws]
    p_h, p_w = ob.TokenScoreParams(device_filters=hs, **kw), ob.TokenScoreParams(where_programs=ps, **kw)
    search_h = lambda: tsc.execute_batch_arrays(p_h, texts, qv)  # noqa: E731
    search_w = lambda: tsc.execute_batch_arrays(p_w, texts, qv)  # noqa: E731
    for name, path, search, build_note in [
            ("256 handles (evaluate_where) + oc_search(q_filters)", handles_path, search_h, "evaluate_where x 256 inside"),
            ("256 programs (compile_where) + oc_search(q_where)", program_path, search_w, "compile_where x 256 inside")]:
        row = {"call": name, "B": B, "limit": LIMIT, "outputs_identical": same,
               "request_path_wall_ms": wall(path, calls), "search_wall_ms": wall(search, calls), "path": build_note}
        try:
            search()
            total, where = profiled(search)
            row.update(search_kernels_device_ms=total, where_and_filter_kernels_device_ms=where)
        except Exception as e:   # the profiler is optional: the wall times stand alone
            row["profiler"] = f"unavailable: {e}"
        print(json.dumps({**row, **info}), flush=True)
    for h in hs:
        h.close()
    emb.close(); strs.close()


if __name__ == "__main__":
    main()
