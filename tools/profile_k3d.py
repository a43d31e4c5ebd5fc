"""Phase profile of the warp BM25 scorer (bm25_warp_kernel, K3d) on bench.py's h1 batches.

Builds (or takes with --so) the library variant compiled with OC_BM25_PHASE_PROFILE (csrc/Makefile `phaseprof`),
whose K3d appends one record per (tile, query) item — the clock64 cycles of each phase and the item's class — and
one record per warp (start / finish in %globaltimer ns).  Runs the 8 seeded h1 batches once each after a warm-up and
prints one JSON object: the phase split over all items, the split per item class, and the ragged end of each launch.
The hooks add registers and stores to the scorer: spans are its shape, not the production kernel's times.

    python tools/profile_k3d.py [--so PATH] [--n-docs N] [--out FILE]
"""
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

PHASES = ["desc", "mark", "count_or_scan", "fold", "clear", "keep_top", "emit"]
ITEM_DT = np.dtype([("item", "<u4"), ("cls", "<u4"), ("postings", "<u4"), ("cand", "<u4"),
                    ("span", "<u4", (len(PHASES),)), ("smid", "<u4")])
WARP_DT = np.dtype([("t0", "<u8"), ("t1", "<u8"), ("c0", "<u8"), ("c1", "<u8"), ("smid", "<u4"), ("items", "<u4"),
                    ("pad", "<u4", (2,))])


def build_so():
    out = os.path.join(tempfile.mkdtemp(prefix="oc_phaseprof_"), "liboramacore_b200_phaseprof.so")
    subprocess.run(["make", "-C", os.path.join(ROOT, "oramacore_b200", "csrc"), "phaseprof", f"PROF_OUT={out}"], check=True)
    return out


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def classes(it):
    nd, nl, skip, passes = it["cls"] & 15, (it["cls"] >> 4) & 15, (it["cls"] >> 8) & 1, it["cls"] >> 12
    return {
        "list_only": nd == 0,
        "count_only": (nd > 0) & (skip == 1) & (nl == 0),
        "count_with_lists": (nd > 0) & (skip == 1) & (nl > 0),
        "scan": (nd > 0) & (skip == 0),
        "redo": passes > 1,
    }, nd, nl


def summarise(items, warps_per_launch):
    span = items["span"].astype(np.float64)
    tot = span.sum()
    out = {"items": int(len(items)),
           "phase_share": {ph: float(span[:, i].sum() / tot) for i, ph in enumerate(PHASES)},
           "cycles_per_item": float(span.sum(1).mean())}
    masks, nd, nl = classes(items)
    out["classes"] = {}
    for name, m in masks.items():
        if not m.any():
            continue
        s = span[m]
        out["classes"][name] = {
            "items": int(m.sum()), "share_of_cycles": float(s.sum() / tot),
            "cycles_per_item": float(s.sum(1).mean()),
            "phase_cycles_per_item": {ph: float(s[:, i].mean()) for i, ph in enumerate(PHASES)},
            "dense_tokens_mean": float(nd[m].mean()), "list_tokens_mean": float(nl[m].mean()),
            "list_postings_mean": float(items["postings"][m].mean()),
        }
    ragged = []
    for w in warps_per_launch:
        t0, t1 = int(w["t0"].min()), int(w["t1"].max())
        ends = (w["t1"] - t0) / 1e3
        span_us = (t1 - t0) / 1e3
        ragged.append({"warps": int(len(w)), "span_us": span_us,
                       "finish_us_p10_p50_p90": [float(x) for x in np.percentile(ends, [10, 50, 90])],
                       "idle_warp_share": float(((t1 - w["t1"]) / 1e3).sum() / (len(w) * span_us)),
                       "sm_clock_mhz": float(((w["c1"] - w["c0"]) / np.maximum(w["t1"] - w["t0"], 1)).mean() * 1e3)})
    out["launches"] = ragged
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--so", default=None, help="prebuilt phase-profile library (default: build one in a temp dir)")
    ap.add_argument("--n-docs", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    os.environ["OC_SO_PATH"] = args.so or build_so()

    import torch
    import bench
    import oramacore_b200 as ob
    from oramacore_b200 import _lib

    w = dict(bench.WORKLOADS["h1"])
    n_docs = args.n_docs or w["n_docs"]
    wl = bench.make_workload(w, n_docs, w["batch"], 0, 1, keep_all=False)
    ctx = ob.Context(0)
    emb = ob.EmbeddingFieldStorage(ctx, dim=w["dim"], model="BGEBase")
    emb.reserve(n_docs)
    ids = np.arange(n_docs, dtype=np.uint64)
    for i in range(0, n_docs, 1 << 18):
        emb.insert_batch(ids[i:i + (1 << 18)], wl["rows"][i:i + (1 << 18)])
    strs = ob.StringFieldStorage(ctx, wl["data_all"])
    tsc = ob.TokenScoreContext(ctx, emb, strs)
    params = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=10, similarity=0.0)
    packed = [ob.TextQueryBatch(t) for t in wl["texts"]]
    qv = []
    for q in wl["qv"]:
        h = ob.pinned_empty(q.shape, np.float32)
        h[...] = q
        qv.append(h)

    L = _lib.lib()
    if not hasattr(L, "oc_bm25_phase_profile"):
        raise RuntimeError(f"{os.environ['OC_SO_PATH']} was not built with OC_BM25_PHASE_PROFILE")
    L.oc_bm25_phase_profile.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    cap_items, cap_warps = 1 << 17, 1 << 14
    d_items = torch.zeros(cap_items * ITEM_DT.itemsize, dtype=torch.uint8, device="cuda")
    d_warps = torch.zeros(cap_warps * WARP_DT.itemsize, dtype=torch.uint8, device="cuda")
    d_cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    for k in range(len(packed)):   # warm-up (module load, kept dense arrays), nothing recorded
        tsc.execute_batch_arrays(params, packed[k], qv[k])
    torch.cuda.synchronize()
    assert L.oc_bm25_phase_profile(d_items.data_ptr(), cap_items, d_warps.data_ptr(), cap_warps, d_cnt.data_ptr()) == 0

    items, launches = [], []
    for k in range(len(packed)):
        d_cnt.zero_()
        torch.cuda.synchronize()
        tsc.execute_batch_arrays(params, packed[k], qv[k])
        torch.cuda.synchronize()
        ni, nw = (int(x) for x in d_cnt.cpu())
        assert ni <= cap_items and nw <= cap_warps, (ni, nw)
        items.append(np.frombuffer(d_items[:ni * ITEM_DT.itemsize].cpu().numpy().tobytes(), ITEM_DT))
        launches.append(np.frombuffer(d_warps[:nw * WARP_DT.itemsize].cpu().numpy().tobytes(), WARP_DT))
    res = summarise(np.concatenate(items), launches)
    res.update(card=card(), batches=len(packed), n_docs=n_docs, batch=w["batch"])
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
