"""Cost of building a sort field from a facet store's number field: the recipe a caller had before the device build
(`recipe`: oc_facets_read_field back to the host, then oc_sort_field_create) against oc_sort_field_from_facets
(`from_facets`), for this tree and, alternated with it in the same run, for another checkout given by path (--other:
a tree of the parent commit with its library built, whose oc_sort_field_create sorts on the host).  Each tree runs in
its own process, with its own Python package and library.

Workloads: 1 M documents with one number value each (the h1 scale), the same with three values on every fifth
document, and 10 M documents (the t1 scale).
  (a) per path: wall time of the whole call (median, min, max of --reps), the device time of one call (the sum of its
      kernels, copies and memsets in a torch.profiler trace of its own) and the workspace the layout in
      sort_field_build needs (CUB's temporary storage not counted);
  (b) the latency of a B = 256 sorted fulltext search (200 K documents, limit 10) on the same ctx, alone and while
      another thread runs the builds back to back: the build holds the ctx lock, so that is what a searching user
      notices (median, p99 and max over --window seconds).
The card's name, power limit and SM clock limit are read in the same run.  Nothing is written into the tree.

    python tools/bench_sort_field.py [--other /path/to/other/checkout] [--reps 7] [--window 3]
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

WORKLOADS = {"h1_1M": (1_000_000, False), "h1_1M_multi": (1_000_000, True), "t1_10M": (10_000_000, False)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def workspace_bytes(n, nbits):
    """sort_field_build's workspace for n device-resident entries (from_facets; create uploads 16 B more per entry)."""
    al = lambda x: (x + 255) & ~255  # noqa: E731
    return al(n * 4) * 2 + al(n * 8) * 3 + al(nbits * 4) + 2 * al((n + 1) * 4)


def stats(xs):
    xs = sorted(xs)
    return {"median": round(float(np.median(xs)), 3), "min": round(xs[0], 3), "max": round(xs[-1], 3),
            "p99": round(float(np.percentile(xs, 99)), 3), "n": len(xs)}


def device_ms(fn):
    import torch
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
    return sum(e.self_device_time_total for e in prof.key_averages()) / 1000.0


def worker(args):
    sys.path.insert(0, args.root)
    import oramacore_b200 as ob
    from oramacore_b200 import synth
    from oramacore_b200.types import MODE_FULLTEXT
    has_ff = hasattr(ob.SortField, "from_facets")
    ctx = ob.Context(0)
    out = {"tree": args.root, "workloads": {}}
    # the search of (b): its own store and sort field on the same ctx
    ns, vocab = 200_000, 5000
    strs = ob.StringFieldStorage(ctx, synth.make_text_corpus(ns, vocab, seed=5))
    tsc = ob.TokenScoreContext(ctx, None, strs)
    texts = synth.make_text_queries(vocab, 256, seed=6)
    sf = ob.SortField(ctx, ns, np.arange(ns), np.random.default_rng(7).random(ns), "number")
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10)

    def search_latencies(stop_after):
        lat, t_end = [], time.perf_counter() + stop_after
        while time.perf_counter() < t_end:
            t0 = time.perf_counter()
            ob.search_sorted_arrays(tsc, p, sf, "ASC", texts=texts)
            lat.append((time.perf_counter() - t0) * 1e3)
        return lat

    search_latencies(0.5)   # warm-up
    out["search_alone_ms"] = stats(search_latencies(args.window))
    rng = np.random.default_rng(11)
    for name, (n, multi) in WORKLOADS.items():
        d = np.arange(n, dtype=np.uint64)
        v = rng.integers(0, 1_000_000, size=n).astype(np.float64)
        if multi:
            d = np.concatenate([d, d[::5], d[::5]])
            v = np.concatenate([v, rng.random(d.shape[0] - n) * 1e6])
        st = ob.FacetStore(ctx, n)
        st.add_number_field("p", d, v)
        paths = {"recipe": lambda: ob.SortField(ctx, n, *(lambda x: (x["doc_ids"], x["values"]))(st.read_field("p")), "number")}
        if has_ff:
            paths["from_facets"] = lambda: ob.SortField.from_facets(st, "p")
        res = {"entries": int(d.shape[0]), "nbits": n}
        for k, fn in paths.items():
            fn().close()   # warm-up
            walls = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                f = fn()
                walls.append((time.perf_counter() - t0) * 1e3)
                f.close()
            holder = []
            dev = device_ms(lambda: holder.append(fn()))
            holder[0].close()
            stop, lat = threading.Event(), []

            def builds():
                while not stop.is_set():
                    fn().close()
            th = threading.Thread(target=builds)
            th.start()
            lat = search_latencies(args.window)
            stop.set()
            th.join()
            res[k] = {"wall_ms": stats(walls), "device_ms": round(dev, 3), "search_during_builds_ms": stats(lat)}
            if has_ff:
                res[k]["workspace_bytes"] = workspace_bytes(int(d.shape[0]), n) + (16 * int(d.shape[0]) if k == "recipe" else 0)
        out["workloads"][name] = res
        st.close()
    sf.close(); strs.close(); ctx.close()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", default=None, help="another checkout with its library built, alternated with this one")
    ap.add_argument("--root", default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--window", type=float, default=3.0, help="seconds of searches per latency measurement")
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the builds")
    ap.add_argument("--worker", action="store_true")
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    print(json.dumps({"card": card()}), flush=True)
    trees = [ROOT] + ([os.path.abspath(args.other)] if args.other else [])
    for r in range(args.rounds):
        for tree in trees:
            env = dict(os.environ)
            env.pop("OC_SO_PATH", None)
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--root", tree, "--reps", str(args.reps), "--window",
                   str(args.window)]
            p = subprocess.run(cmd, env=env, capture_output=True, text=True)
            if p.returncode != 0:
                raise RuntimeError(p.stdout + p.stderr)
            print(json.dumps({"round": r, **json.loads(p.stdout.strip().splitlines()[-1])}), flush=True)


if __name__ == "__main__":
    main()
