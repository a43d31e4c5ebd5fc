"""Cost of geopoint where-filter leaves (oc_filter_geo_radius / oc_filter_geo_polygon) and of searching under one.

Runs
  * radius leaves (1000 km around random centres) over 1M and 10M points uniform on the sphere;
  * polygon leaves of 4, 64 and 1024 vertices (a star-shaped region of ~40 degrees across, so the bounding-box
    pre-test keeps a few percent of the points) over the same fields;
  * the h1 oc_search (hybrid, 1M x 768-d fp32 + BM25 over 1M synthetic docs, B = 256, top 10) without a filter, under
    a radius leaf over one point per document (5000 km, about a sixth of the documents), and under a filter of the
    same documents uploaded as a bitmap (what any filter of that size costs the search);
  * the same leaves restated in numpy on the CPU (an f64 haversine, a vectorised PNPOLY), labelled as such: that is a
    CPU restatement, not the reference.
For every leaf it prints the kernel's device time (torch.profiler, CUDA activity of where_geo_kernel, per call) and the
host wall time of the whole synchronous call (bitmap allocation, plan upload, zeroing, the kernel, the copy into the
handle, the synchronise); for the searches oc_last_timing.device_ms (CUDA events).  Median / min / max of --calls calls
after one warm-up call.  The card's name and power limit are read in the same process.  Writes nothing into the tree.

    python tools/bench_geo.py [--calls 20] [--skip-search]
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
R = 6371000.0


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def sphere(n, rng):
    return np.degrees(np.arcsin(rng.uniform(-1, 1, n))), rng.uniform(-180, 180, n)


def star(nv, clat=20.0, clon=-40.0, r1=20.0, r2=8.0):
    a = np.linspace(0, 2 * np.pi, nv, endpoint=False)
    r = np.where(np.arange(nv) % 2 == 0, r1, r2) if nv > 4 else np.full(nv, r1)
    return [(float(np.float32(clat + rr * np.sin(t))), float(np.float32(clon + rr * np.cos(t)))) for t, rr in zip(a, r)]


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t))}


def np_haversine_docs(lat, lon, clat, clon, r):
    p1, p2 = np.radians(lat), np.radians(clat)
    a = np.sin((p2 - p1) / 2) ** 2 + np.cos(p1) * np.cos(p2) * np.sin(np.radians(clon - lon) / 2) ** 2
    return 2 * R * np.arcsin(np.sqrt(np.minimum(a, 1.0))) <= r


def np_pnpoly(verts, lat, lon):
    inside = np.zeros(lat.shape, bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(len(verts)):
            (yi, xi), (yj, xj) = verts[i], verts[i - 1]
            inside ^= ((yi > lat) != (yj > lat)) & (lon < (xj - xi) * (lat - yi) / (yj - yi) + xi)
    return inside


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--skip-search", action="store_true")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    ctx = ob.Context(0)
    info = {"device": ctx.device_info()["name"], "nvidia_smi": card()}
    rng = np.random.default_rng(3)

    def leaf_cost(make):
        make().close()   # warm-up of this shape
        wall = []
        for _ in range(a.calls):
            t0 = time.perf_counter()
            f = make()
            wall.append((time.perf_counter() - t0) * 1e3)
            f.close()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.calls):
                make().close()
            torch.cuda.synchronize()
        k = {e.key: e.device_time_total / a.calls / 1e3 for e in prof.key_averages() if "geo_" in e.key}
        return {"kernel_ms": k, "call_wall_ms": stats(wall)}

    def cpu_cost(fn, reps=3):
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            fn()
            t.append((time.perf_counter() - t0) * 1e3)
        return stats(t)

    for n in (1_000_000, 10_000_000):
        lat, lon = sphere(n, rng)
        g = ob.GeoPointField(ctx, n, np.arange(n, dtype=np.uint64), lat, lon)
        centres = [sphere(1, rng) for _ in range(4)]
        it = iter(range(1 << 30))

        def radius_leaf():
            c = centres[next(it) % 4]
            return g.radius(float(c[0][0]), float(c[1][0]), 1000, "km")
        f = radius_leaf()
        row = {"leaf": "radius", "points": n, "radius_km": 1000, "documents_in_leaf": f.count(), **leaf_cost(radius_leaf)}
        f.close()
        c = centres[0]
        row["numpy_cpu_restatement_ms"] = cpu_cost(lambda: np_haversine_docs(lat, lon, float(c[0][0]), float(c[1][0]), 1e6))
        print(json.dumps({**row, **info}), flush=True)
        for nv in (4, 64, 1024):
            verts = star(nv)
            f = g.polygon(verts)
            vl, vo = np.array([v[0] for v in verts]), np.array([v[1] for v in verts])
            in_box = float(((lat >= vl.min()) & (lat <= vl.max()) & (lon >= vo.min()) & (lon <= vo.max())).mean())
            row = {"leaf": "polygon", "points": n, "vertices": nv, "bbox_fraction": in_box, "documents_in_leaf": f.count(),
                   **leaf_cost(lambda: g.polygon(verts))}
            f.close()
            if n == 1_000_000:
                row["numpy_cpu_restatement_ms"] = cpu_cost(lambda: np_pnpoly(verts, lat, lon), reps=1 if nv == 1024 else 3)
            print(json.dumps({**row, **info}), flush=True)
        g.close()
        del lat, lon

    if a.skip_search:
        ctx.close()
        return
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
    lat, lon = sphere(N, rng)
    g = ob.GeoPointField(ctx, N, ids, lat, lon)
    leaf = g.radius(30.0, 10.0, 5000, "km")
    same = ob.DeviceFilter.from_bits(ctx, leaf.read(), N)   # the same documents as an id leaf: the filtered search's own cost
    for name, f in [("oc_search", None), ("oc_search under a radius leaf", leaf), ("oc_search under an id leaf, same documents", same)]:
        p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=LIMIT, similarity=0.0, device_filter=f)
        tsc.execute_batch_arrays(p, texts, qv)
        t = []
        for _ in range(a.calls):
            tsc.execute_batch_arrays(p, texts, qv)
            t.append(ctx.last_timing()["device_ms"])
        row = {"call": name, "B": B, "limit": LIMIT, "documents_in_filter": None if f is None else f.count(),
               "device_ms": stats(t)}
        print(json.dumps({**row, **info}), flush=True)
    leaf.close(); same.close(); g.close(); emb.close(); strs.close(); ctx.close()


if __name__ == "__main__":
    main()
