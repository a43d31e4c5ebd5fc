"""End-to-end throughput of concurrent SINGLE-QUERY callers through the micro-batching front
(oc_batcher_*): the reference's request shape (one search per task) on the h1 corpus.  Native threads
(tools/callers_drive.cpp) submit one query per call; results of the last pass are compared with the direct
batched oc_search.  Run on a GPU machine:  python tools/bench_callers.py --callers 256 --max-batch 256 --wait-us 200
Not part of bench.py's contract (that one times the batch API); this is the number a drop-in user sees."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build_driver():
    out = os.path.join(tempfile.mkdtemp(prefix="oc_callers_"), "libcallers_drive.so")
    libdir = os.path.join(ROOT, "oramacore_b200")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-pthread", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tools", "callers_drive.cpp"), "-o", out, "-L", libdir, "-loramacore_b200",
                    f"-Wl,-rpath,{libdir}"], check=True)
    return C.CDLL(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--callers", type=int, default=256)
    ap.add_argument("--max-batch", type=int, default=256)
    ap.add_argument("--wait-us", type=int, default=200)
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--n-docs", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--vocab", type=int, default=200_000)
    args = ap.parse_args()
    import oramacore_b200 as ob
    from oramacore_b200 import synth
    from oramacore_b200.engine import _p   # noqa: PLC2701  (ctypes pointer helper)
    ob.build()
    drv = build_driver()
    ctx = ob.Context(0)
    rows = synth.make_vectors(args.n_docs, args.dim, seed=1)
    qv, _ = synth.make_vector_queries(rows, args.queries, seed=2)
    data = synth.make_text_corpus(args.n_docs, args.vocab, seed=3)
    tq_list = synth.make_text_queries(args.vocab, args.queries, seed=4)
    texts = ob.TextQueryBatch(tq_list)
    emb = ob.EmbeddingFieldStorage(ctx, "BGEBase" if args.dim == 768 else "BGESmall")
    emb.insert_batch(np.arange(args.n_docs, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(ctx, data)
    tsc = ob.TokenScoreContext(ctx, emb, strs)
    params = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=10, similarity=0.0)
    Q, L = args.queries, 10
    ref_d, ref_s, ref_n, ref_c = [], [], [], []
    for lo in range(0, Q, 256):   # reference answer: the direct batched call
        d, s, n, c = tsc.execute_batch_arrays(params, tq_list[lo:lo + 256], qv[lo:lo + 256])
        ref_d.append(d); ref_s.append(s); ref_n.append(n); ref_c.append(c)
    bat = ob.SearchBatcher(tsc, max_batch=args.max_batch, max_wait_us=args.wait_us)
    docs = np.zeros((Q, L), np.uint64); scores = np.zeros((Q, L), np.float32)
    n = np.zeros(Q, np.uint32); cnt = np.zeros(Q, np.uint64)
    el = C.c_double()
    qvc = np.ascontiguousarray(qv, np.float32)
    drv.callers_drive.argtypes = [C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float,
                                  C.c_float, C.c_float] + [C.c_void_p] * 10 + [C.POINTER(C.c_double)]
    for warm in (True, False):
        rc = drv.callers_drive(bat._h, ob.MODE_HYBRID, args.callers, 1 if warm else args.rounds, Q, args.dim, L, 0.0,
                               ob.BM25_K, ob.BM25_B, _p(qvc), _p(texts.q_token_offsets), _p(texts.token_term_offsets),
                               _p(texts.term_field), _p(texts.term_id), _p(texts.term_weight), _p(docs), _p(scores), _p(n),
                               _p(cnt), C.byref(el))
        assert rc == 0, rc
    st = bat.stats()
    line = {"metric": "hybrid_search_qps_single_query_callers", "value": Q * args.rounds / el.value, "unit": "queries/s",
            "callers": args.callers, "max_batch": args.max_batch, "max_wait_us": args.wait_us,
            "mean_batch": st["queries"] / max(st["batches"], 1), "n_docs": args.n_docs, "dim": args.dim}
    if ref_d:
        rd, rs = np.concatenate(ref_d), np.concatenate(ref_s)
        line["identical_to_batched_call"] = int(sum(np.array_equal(docs[i], rd[i]) and np.array_equal(scores[i], rs[i]) for i in range(Q)))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
