"""Cost of publishing the filter fields at a commit: IndexLoader.refresh_facets() on the device commit (`new`) against
the host rebuild it replaced (`rebuild`: per-document Python dicts of every filter value, and a new FacetStore and
GeoPointField built from all of them at each commit).

Set-up: h1's 1 M documents with one bool, one number, one date, one string_filter (1000 keys) and one geopoint field.
Workloads: (a) rounds of 300 new documents + 30 deletes, one commit each; (b) one commit of 100 K new documents;
(c) a store of 100 documents, a commit of 10 new ones.  Each path runs in its own process (its peak RSS is its own),
alternated: rebuild, new, rebuild, new.  Prints one JSON line per run and the card's name and limits.

    python tools/bench_filter_commit.py [--docs 1000000] [--reps 2]"""
import argparse
import json
import os
import resource
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class Rebuild:
    """The host rebuild: IndexLoader.refresh_facets() before the device commit, for the five field kinds used here."""

    def __init__(self, ctx):
        import oramacore_b200 as ob
        self.ob, self.ctx = ob, ctx
        self.b, self.n, self.d, self.s, self.g = {}, {}, {}, {}, {}
        self.max_doc, self.st, self.geo = -1, None, None

    def index(self, d, b, n, dt, s, lat, lon):
        self.max_doc = max(self.max_doc, d)
        self.b[d] = b
        self.n.setdefault(d, []).append(n)
        self.d.setdefault(d, []).append(dt)
        self.s.setdefault(d, []).append(s)
        self.g.setdefault(d, []).append((lat, lon))

    def delete(self, d):
        for m in (self.b, self.n, self.d, self.s, self.g):
            m.pop(d, None)

    def refresh(self):
        ob, nb = self.ob, self.max_doc + 2
        if self.geo is not None:
            self.geo.close(); self.st.close()
        self.geo = ob.GeoPointField(self.ctx, nb, [d for d, ps in self.g.items() for _ in ps], [p[0] for ps in self.g.values() for p in ps],
                                    [p[1] for ps in self.g.values() for p in ps])
        st = ob.FacetStore(self.ctx, nb)
        st.add_bool_field("b", [d for d, x in self.b.items() if x], [d for d, x in self.b.items() if not x])
        st.add_number_field("n", [d for d, vs in self.n.items() for _ in vs], [x for vs in self.n.values() for x in vs])
        keys = {}
        for d, ks in self.s.items():
            for k in ks:
                keys.setdefault(k, []).append(d)
        st.add_string_field("s", {k: keys[k] for k in sorted(keys)})
        st.add_date_field("d", [d for d, ms in self.d.items() for _ in ms], [x for ms in self.d.values() for x in ms])
        self.st = st
        return {}

    def close(self):
        if self.st is not None:
            self.st.close(); self.geo.close()


class New:
    """IndexLoader's own filter path: values queued on the device handles, refresh_facets() commits them."""

    def __init__(self, ctx):
        from oramacore_b200.loader import IndexLoader
        self.ld = IndexLoader(ctx, ["text"], bool_fields=["b"], number_fields=["n"], string_filter_fields=["s"], date_fields=["d"],
                              geopoint_fields=["g"])

    def bulk(self, ids, b, n, dt, s, lat, lon):   # set-up only: the same queue apply() fills, in a few calls
        f = self.ld.facets
        self.ld.max_doc_id = max(self.ld.max_doc_id, int(ids.max()))
        if "s" not in f.fields:
            f.add_string_field("s", {s[0]: []})
        f.insert_variants("b", ids, b.tolist())
        f.insert_numbers("n", ids, n)
        f.insert_numbers("d", ids, dt)
        f.insert_variants("s", ids, s)
        self.ld.geo["g"].insert(ids, lat, lon)

    def index(self, d, b, n, dt, s, lat, lon):
        self.ld.apply({"type": "Index", "doc_id": d, "indexed_values": [
            {"type": "FilterBool", "field": "b", "value": b}, {"type": "FilterNumber", "field": "n", "value": n},
            {"type": "FilterDate", "field": "d", "value": dt}, {"type": "FilterString", "field": "s", "value": s},
            {"type": "FilterGeoPoint2", "field": "g", "value": {"Plain": {"lat": lat, "lon": lon}}}]})

    def delete(self, d):
        self.ld.apply({"type": "DeleteDocuments", "doc_ids": [d]})

    def refresh(self):
        return self.ld.refresh_facets()

    def close(self):
        self.ld.close()


def _values(rng, n, base):
    ids = np.arange(base, base + n, dtype=np.uint64)
    return (ids, rng.random(n) < 0.5, rng.integers(0, 1000, n).astype(np.float64), rng.integers(0, 10**12, n),
            [f"k{int(x)}" for x in rng.integers(0, 1000, n)], rng.uniform(-80, 80, n), rng.uniform(-170, 170, n))


def _run(path, n_docs):
    import oramacore_b200 as ob
    ctx = ob.Context(0)
    rng = np.random.default_rng(1)
    out = {"path": path}

    def make(n):
        p = Rebuild(ctx) if path == "rebuild" else New(ctx)
        ids, b, n_, dt, s, la, lo = _values(rng, n, 0)
        if path == "rebuild":
            for i in range(n):
                p.index(int(ids[i]), bool(b[i]), float(n_[i]), int(dt[i]), s[i], float(la[i]), float(lo[i]))
        else:
            p.bulk(ids, b, n_, dt, s, la, lo)
        p.refresh()
        return p

    def commit(p):
        t = time.perf_counter()
        st = p.refresh()   # both paths end in a device synchronise
        wall = (time.perf_counter() - t) * 1e3
        dev = sum(v["device_ms"] for v in st.values()) if st else None
        ws = max((v["workspace_bytes"] for v in st.values()), default=0) if st else None
        return wall, dev, ws

    def feed(p, n, base, n_del, hi):
        ids, b, n_, dt, s, la, lo = _values(rng, n, base)
        for i in range(n):
            p.index(int(ids[i]), bool(b[i]), float(n_[i]), int(dt[i]), s[i], float(la[i]), float(lo[i]))
        for d in rng.integers(0, hi, n_del):
            p.delete(int(d))

    p = make(n_docs)
    base = n_docs
    rounds = []
    for r in range(6):
        feed(p, 300, base, 30, base)
        base += 300
        rounds.append(commit(p))
    out["a_rounds"] = {"wall_ms": [x[0] for x in rounds[1:]], "device_ms": [x[1] for x in rounds[1:]], "workspace_bytes": rounds[-1][2]}
    feed(p, 100000, base, 0, base)
    base += 100000
    out["b_100k"] = dict(zip(("wall_ms", "device_ms", "workspace_bytes"), commit(p)))
    p.close()
    t = make(100)
    cs = []
    for r in range(6):
        feed(t, 10, 100 + 10 * r, 2, 100 + 10 * r)
        cs.append(commit(t))
    out["c_tiny"] = {"wall_ms": [x[0] for x in cs[1:]], "device_ms": [x[1] for x in cs[1:]]}
    t.close()
    out["peak_rss_mb"] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024
    ctx.close()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--path", choices=["rebuild", "new"])
    a = ap.parse_args()
    if a.path:
        _run(a.path, a.docs)
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    for _ in range(a.reps):
        for path in ("rebuild", "new"):
            r = subprocess.run([sys.executable, __file__, "--docs", str(a.docs), "--path", path], capture_output=True, text=True)
            sys.stdout.write(r.stdout)
            if r.returncode:
                sys.stdout.write(r.stderr[-3000:])
                sys.exit(r.returncode)


if __name__ == "__main__":
    main()
