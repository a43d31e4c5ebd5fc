"""Cost of oc_str_commit on the h1 corpus (1 M documents, 200 K terms, 32 M postings, loaded with oc_str_load_field),
for this build and, alternated with it in the same run, for any other build of the library given by path (--other:
a liboramacore_b200.so built from another commit).  Each build runs in its own process through minimal ctypes
bindings of calls every build has (oc_init, oc_device_info, oc_str_*), so two builds of different ABIs compare.

Workloads:
  (a) the reference's commit cadence (a commit every insert_batch_commit_size = 300 ops): rounds of 270 new documents,
      20 re-inserts and 10 deletes, each followed by a commit; median / min / max of the commit call's wall time over
      --rounds rounds after 3 warm-up rounds;
  (b) one commit of 100 K new documents;
  (c) a tiny store: 10 new documents per commit on an empty store, median of 50 commits (the floor of launches and
      copies).
Where the build has oc_str_commit_ex, its device_ms and workspace_bytes are reported for (a) and (b).  Each process
also reports its peak resident host memory.  The card's name, power limit and SM clock limit are read in the same run.
The corpora are generated once into a temporary directory; nothing is written into the tree.

    python tools/bench_str_commit.py [--other /path/to/liboramacore_b200.so] [--rounds 40] [--reps 2]
"""
import argparse
import ctypes as C
import json
import os
import resource
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_DOCS, VOCAB, N_EXTRA = 1_000_000, 200_000, 100_000


class StrCommit(C.Structure):   # oc_str_commit_t
    _fields_ = [("rows_before", C.c_uint64), ("rows_after", C.c_uint64), ("postings_before", C.c_uint64),
                ("postings_after", C.c_uint64), ("pending_postings", C.c_uint64), ("workspace_bytes", C.c_uint64),
                ("device_ms", C.c_float), ("wall_ms", C.c_float)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def stats(t):
    return {"median": float(np.median(t)), "min": float(np.min(t)), "max": float(np.max(t)), "n": len(t)}


def corpora(tmp):
    """h1 and the documents the workloads insert, as npz files in `tmp` (made once)."""
    from oramacore_b200 import synth
    out = []
    for name, n, seed in (("h1", N_DOCS, None), ("extra", N_EXTRA, 12)):
        p = os.path.join(tmp, f"{name}.npz")
        if not os.path.exists(p):
            d = synth.make_text_corpus(n, VOCAB) if seed is None else synth.make_text_corpus(n, VOCAB, seed=seed)
            f = d.fields[0]
            np.savez(p, off=f.term_offsets, row=f.post_row, tf=f.post_tf, ln=f.post_len, avg=np.float32(f.avg_field_len))
        out.append(p)
    return out


class Lib:
    def __init__(self, path):
        L = self.L = C.CDLL(path)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.oc_init.argtypes = [C.c_int, C.POINTER(vp)]
        L.oc_device_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
        L.oc_str_create.argtypes = [vp, u32, C.POINTER(vp)]
        L.oc_str_destroy.argtypes = [vp]
        L.oc_str_destroy.restype = None
        L.oc_str_set_rows.argtypes = [vp, u64, vp, u64]
        L.oc_str_load_field.argtypes = [vp, u32, C.c_float, u32, vp, vp, vp, vp, vp]
        L.oc_str_insert.argtypes = [vp, u32, u64, C.c_uint16, u32, vp, vp]
        L.oc_str_delete.argtypes = [vp, vp, u64]
        L.oc_str_commit.argtypes = [vp]
        self.has_ex = hasattr(L, "oc_str_commit_ex")
        if self.has_ex:
            L.oc_str_commit_ex.argtypes = [vp, C.POINTER(StrCommit)]
        L.oc_last_error.restype = C.c_char_p
        self.ctx = vp()
        self.ok(L.oc_init(0, C.byref(self.ctx)))

    def ok(self, rc):
        if rc != 0:
            raise RuntimeError(f"error {rc}: {self.L.oc_last_error().decode()}")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Docs:
    """The documents of a corpus file, row by row: (term ids, tfs, field length)."""

    def __init__(self, path):
        z = np.load(path)
        off = z["off"].astype(np.int64)
        term = np.repeat(np.arange(off.shape[0] - 1, dtype=np.uint32), np.diff(off))
        o = np.argsort(z["row"], kind="stable")
        self.row, self.term, self.tf = z["row"][o], term[o], z["tf"][o]
        n = int(self.row[-1]) + 1
        self.start = np.searchsorted(self.row, np.arange(n + 1))
        self.len = np.zeros(n, np.uint16)
        self.len[z["row"]] = z["ln"]

    def insert(self, lib, s, doc_id, r):
        a, b = self.start[r], self.start[r + 1]
        lib.ok(lib.L.oc_str_insert(s, 0, int(doc_id), int(self.len[r]), int(b - a), _p(self.term[a:b]), _p(self.tf[a:b])))


def commit(lib, s, use_ex):
    st = StrCommit()
    t0 = time.perf_counter()
    lib.ok(lib.L.oc_str_commit_ex(s, C.byref(st)) if use_ex else lib.L.oc_str_commit(s))
    return (time.perf_counter() - t0) * 1e3, st


def child(so, workload, h1, extra, rounds):
    lib = Lib(so)
    L = lib.L
    ex = Docs(extra)
    out = {"so": so, "workload": workload}
    s = C.c_void_p()
    lib.ok(L.oc_str_create(lib.ctx, 1, C.byref(s)))
    if workload == "tiny":
        t = []
        for i in range(60):
            for k in range(10):
                ex.insert(lib, s, i * 10 + k, i * 10 + k)
            ms, _ = commit(lib, s, False)
            if i >= 10:
                t.append(ms)
        out["commit_ms"] = stats(t)
    else:
        z = np.load(h1)
        lib.ok(L.oc_str_set_rows(s, N_DOCS, None, N_DOCS))
        lib.ok(L.oc_str_load_field(s, 0, float(z["avg"]), int(z["off"].shape[0] - 1), _p(z["off"]), _p(z["row"]), _p(z["tf"]),
                                   _p(z["ln"]), None))
        out["postings"] = int(z["off"][-1])
        del z
        rng = np.random.default_rng(5)
        if workload == "cadence":
            t, dev, nxt = [], [], 0
            live = list(range(N_DOCS))
            for i in range(rounds + 3):
                for _ in range(270):
                    ex.insert(lib, s, N_DOCS + nxt, nxt % N_EXTRA)
                    live.append(N_DOCS + nxt)
                    nxt += 1
                for d in rng.choice(len(live), 20, replace=False):
                    ex.insert(lib, s, live[d], int(rng.integers(0, N_EXTRA)))
                dead = np.asarray([live.pop(int(j)) for j in sorted(rng.choice(len(live), 10, replace=False), reverse=True)], np.uint64)
                lib.ok(L.oc_str_delete(s, _p(dead), 10))
                ms, st = commit(lib, s, lib.has_ex and i >= 3 + rounds // 2)   # the last half also reads the statistics
                if i >= 3:
                    t.append(ms)
                    if lib.has_ex and i >= 3 + rounds // 2:
                        dev.append(st.device_ms)
                        out["workspace_bytes"] = st.workspace_bytes
            out["commit_ms"] = stats(t)
            if dev:
                out["device_ms"] = stats(dev)
        else:   # bulk
            for r in range(N_EXTRA):
                ex.insert(lib, s, N_DOCS + r, r)
            ms, st = commit(lib, s, lib.has_ex)
            out["commit_ms"] = ms
            if lib.has_ex:
                out.update(device_ms=st.device_ms, workspace_bytes=st.workspace_bytes, postings_after=st.postings_after,
                           pending_postings=st.pending_postings)
    L.oc_str_destroy(s)
    out["peak_rss_mb"] = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", default=None, help="another build of liboramacore_b200.so to alternate with this one")
    ap.add_argument("--rounds", type=int, default=40)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--child", nargs=5, metavar=("SO", "WORKLOAD", "H1", "EXTRA", "ROUNDS"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        so, w, h1, ex, r = a.child
        return child(so, w, h1, ex, int(r))
    mine = os.path.join(ROOT, "oramacore_b200", "liboramacore_b200.so")
    builds = [("this", mine)] + ([("other", a.other)] if a.other else [])
    print(json.dumps({"card": card()}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        h1, extra = corpora(tmp)
        for w in ("tiny", "cadence", "bulk"):
            for rep in range(a.reps):
                for name, so in (builds if rep % 2 == 0 else builds[::-1]):
                    r = subprocess.run([sys.executable, __file__, "--child", so, w, h1, extra, str(a.rounds)],
                                       capture_output=True, text=True)
                    if r.returncode != 0:
                        raise RuntimeError(f"{name} {w}: {r.stderr[-2000:]}")
                    res = json.loads(r.stdout.strip().splitlines()[-1])
                    res["build"] = name
                    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
