"""Query-term resolution on the host walk vs. on the device (oc_dict_resolve_q with a ctx).

Two shapes: 256 queries x 3 random words of a 200 K-term vocabulary (h1) and of a 1 M-term vocabulary (t1), words of
4-10 letters a-z.  For tolerance 1 and 2 the script times the whole resolve call (wall clock; the device path ends in
a synchronise) with ctx = NULL (the host walk, threaded over the host cores) and with a ctx, alternating the two, and
checks that both return the same bytes.  It also times prefix expansion (exact = false, no tolerance), which always
runs on the host, next to the device path's floor: one query of one token with tolerance 1.  The first device call
of each vocabulary builds the mirror; it is reported apart (`mirror_build_ms`) with the mirror's device bytes.
The card's name and power limit are read in the same process, and the host's core count is printed.
Writes nothing into the tree.

    python tools/bench_resolve.py [--reps 5] [--batch 256]
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


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def vocabulary(n, seed):
    rng = np.random.default_rng(seed)
    m = int(n * 1.1)
    lens = rng.integers(4, 11, size=m)
    buf = rng.integers(97, 123, size=int(lens.sum()), dtype=np.uint8).tobytes().decode()
    offs = np.concatenate([[0], np.cumsum(lens)])
    words = list(dict.fromkeys(buf[offs[i]:offs[i + 1]] for i in range(m)))[:n]
    assert len(words) == n
    return words


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def same(a, b):
    return all(np.array_equal(getattr(a, k), getattr(b, k)) for k in ("q_token_offsets", "token_term_offsets", "term_field", "term_id")) \
        and np.array_equal(a.term_weight.view(np.uint32), b.term_weight.view(np.uint32))


def stats(t):
    return {"best": float(np.min(t)), "median": float(np.median(t)), "max": float(np.max(t))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=256)
    a = ap.parse_args()
    ctx = ob.Context(0)   # no device: an error, there is nothing to measure without one
    print(json.dumps({"card": card(), "host_cores": os.cpu_count(), "batch": a.batch, "tokens_per_query": 3, "reps": a.reps}), flush=True)
    for name, n, seed in (("h1", 200_000, 1), ("t1", 1_000_000, 2)):
        words = vocabulary(n, seed)
        d = ob.TermDictionary(1)
        d.add_terms(0, words)
        rng = np.random.default_rng(seed + 10)
        texts = [" ".join(words[int(i)] for i in rng.integers(0, n, size=3)) for _ in range(a.batch)]
        d.resolve_batch(texts[:1])                                          # the sorted index
        build_ms, _ = timed(lambda: d.resolve_batch(texts[:1], tolerance=1, ctx=ctx))
        row = {"vocabulary": name, "terms": n, "mirror_build_ms": build_ms, "mirror_device_bytes": d.device_bytes(ctx)}
        for tol in (1, 2):
            d.resolve_batch(texts, tolerance=tol, ctx=ctx)                  # warm: kernel shapes of this tolerance
            host_t, dev_t, equal, n_terms = [], [], True, 0
            for _ in range(a.reps):
                th, h = timed(lambda: d.resolve_batch(texts, tolerance=tol))
                td, g = timed(lambda: d.resolve_batch(texts, tolerance=tol, ctx=ctx))
                host_t.append(th); dev_t.append(td)
                equal = equal and same(h, g)
                n_terms = int(g.term_id.size)
            row[f"tolerance{tol}"] = {"host_ms": stats(host_t), "device_ms": stats(dev_t), "outputs_equal": equal,
                                      "expanded_terms": n_terms, "host_over_device": float(np.median(host_t) / np.median(dev_t))}
        prefix = [timed(lambda: d.resolve_batch(texts))[0] for _ in range(a.reps)]
        floor = [timed(lambda: d.resolve_batch(texts[:1], tolerance=1, ctx=ctx))[0] for _ in range(a.reps)]
        one = [timed(lambda: d.resolve_batch([texts[0].split()[0]], tolerance=1, ctx=ctx))[0] for _ in range(a.reps)]
        row["prefix_host_ms"] = stats(prefix)
        row["device_one_query_ms"] = stats(floor)
        row["device_one_token_ms"] = stats(one)
        print(json.dumps(row), flush=True)
        d.close()
    ctx.close()


if __name__ == "__main__":
    main()
