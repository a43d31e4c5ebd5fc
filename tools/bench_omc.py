"""OMC from the device-resident store (p->omc, OmcStore) against the per-call host arrays (omc_doc_ids / omc_mult), and
the cost of the store's commit.

Search: h1's shape (1 M documents, 768-d fp32 embeddings, 200 K-term vocabulary, hybrid top-10, batch 256) with a
multiplier on every document, on 1 % of them and on none.  Per case, the array path and the store path alternate call by
call; the line reports the median per-call device_ms (oc_last_timing) and wall time (host clock around the call, which
ends in a device synchronise), and checks both paths give the same bytes.
Commit: (a) rounds of 300 new multipliers and 30 deletes on a 1 M-entry map; (b) one commit of 100 K entries into an
empty store; (c) a 100-entry map, a commit of 10.  Row list: the first search with the store after an oc_str_commit
(it rebuilds the list of OMC string rows) against the next one.

    python tools/bench_omc.py [--docs 1000000] [--calls 30]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")])) if r.returncode == 0 else {}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--batch", type=int, default=256)
    a = ap.parse_args()
    import oramacore_b200 as ob
    from oramacore_b200 import synth
    from oramacore_b200.engine import OmcStore, TokenScoreContext, TokenScoreParams
    from oramacore_b200.types import MODE_HYBRID

    n, B = a.docs, a.batch
    print(json.dumps({"card": card()}), flush=True)
    ctx = ob.Context(0)
    rows = synth.make_vectors(n, 768, seed=1)
    qv, _ = synth.make_vector_queries(rows, B, seed=2)
    data = synth.make_text_corpus(n, 200_000, seed=3)
    texts = synth.make_text_queries(200_000, B, seed=4)
    emb = ob.EmbeddingFieldStorage(ctx, "BGEBase")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    del rows
    strs = ob.StringFieldStorage(ctx, data)
    tsc = TokenScoreContext(ctx, emb, strs)
    rng = np.random.default_rng(5)

    def call(kw):
        t0 = time.perf_counter()
        out = tsc.execute_batch_arrays(TokenScoreParams(mode=MODE_HYBRID, limit_hint=10, similarity=0.0, **kw), texts, qv)
        wall = (time.perf_counter() - t0) * 1e3
        return out, wall, ctx.last_timing()["device_ms"]

    for frac in (1.0, 0.01, 0.0):
        k = int(round(n * frac))
        od = np.sort(rng.choice(n, size=k, replace=False)).astype(np.uint64)
        om = rng.choice([0.5, 1.5, 2.0, 3.0], size=k).astype(np.float32)
        st = OmcStore(ctx)
        st.set(od, om)
        st.commit()
        kws = {"arrays": dict(omc_doc_ids=od, omc_mult=om) if k else {}, "store": dict(omc_store=st)}
        res = {p: {"wall": [], "dev": []} for p in kws}
        for _ in range(3):   # warm-up: modules, workspaces, the store's row list
            outs = {p: call(kw)[0] for p, kw in kws.items()}
        same = all(x.tobytes() == y.tobytes() for x, y in zip(outs["arrays"], outs["store"]))
        for _ in range(a.calls):
            for p, kw in kws.items():
                _, w, d = call(kw)
                res[p]["wall"].append(w)
                res[p]["dev"].append(d)
        line = {"case": "search", "omc_entries": k, "fraction": frac, "identical": same}
        for p in kws:
            line[f"{p}_wall_ms"] = round(float(np.median(res[p]["wall"])), 3)
            line[f"{p}_device_ms"] = round(float(np.median(res[p]["dev"])), 3)
        print(json.dumps(line), flush=True)
        if frac == 1.0:   # row list: the first search after an oc_str_commit against the next one
            rl = []
            for r in range(5):
                for j in range(300):
                    strs.insert(n + 1000 * r + j, 0, 5, {int(t): 1 for t in rng.choice(1000, 3, replace=False)})
                strs.commit()
                first = call(kws["store"])[1]
                rl.append((first, call(kws["store"])[1]))
            print(json.dumps({"case": "row_list_rebuild", "omc_entries": k,
                              "first_wall_ms": round(float(np.median([x for x, _ in rl])), 3),
                              "next_wall_ms": round(float(np.median([y for _, y in rl])), 3)}), flush=True)
        st.close()

    def commits(name, base, rounds, n_set, n_del):
        st = OmcStore(ctx)
        if base:
            st.set(np.arange(base, dtype=np.uint64) * 2, np.full(base, 2.0, np.float32))
            st.commit()
        dev, wall = [], []
        for _ in range(rounds):
            st.set(rng.integers(0, 4 * max(base, n_set), n_set).astype(np.uint64), rng.random(n_set).astype(np.float32))
            if n_del:
                st.delete((rng.integers(0, max(base, 1), n_del) * 2).astype(np.uint64))
            s = st.commit()
            dev.append(s["device_ms"]); wall.append(s["wall_ms"])
        print(json.dumps({"case": "commit", "name": name, "map": base, "set": n_set, "delete": n_del, "rounds": rounds,
                          "device_ms": round(float(np.median(dev)), 3), "wall_ms": round(float(np.median(wall)), 3),
                          "entries_after": int(st.read()[0].shape[0])}), flush=True)
        st.close()
    commits("rounds_on_1M", 1_000_000, 20, 300, 30)
    commits("one_100K", 0, 1, 100_000, 0)
    commits("map_100", 100, 20, 10, 0)
    print(json.dumps({"card_after": card()}), flush=True)
    strs.close(); emb.close(); ctx.close()


if __name__ == "__main__":
    main()
