"""Launch census: a fixed matrix of calls through every public search entry point, on small seeded stores.

Per call it prints one line: the return code, the oc_launch_count() delta, oc_last_timing's h2d_bytes / d2h_bytes
and a sha256 of every output array.  Then every oc_batcher_search* function runs rounds of B single-query requests,
direct (max_batch = 1) and merged into one call, and mixed rounds (plain, plain with sorted / pinned, grouped) on each
filter variant; per request it prints the return code and output digest, per round the same counters and the
oc_batcher_stats delta.  Two builds that do the same device work print the same lines, so a host-side
change is checked by running this under OC_SO_PATH for each build and diffing the two outputs:

    OC_SO_PATH=/path/to/parent/liboramacore_b200.so python tools/launch_census.py > parent.txt
    python tools/launch_census.py > new.txt && diff parent.txt new.txt

Needs an sm_90 GPU.  Writes nothing.
"""
import ctypes as C
import hashlib
import itertools
import os
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oramacore_b200 as ob  # noqa: E402
from oramacore_b200 import _lib, engine as E, synth  # noqa: E402

N, DIM, VOCAB, B = 6000, 64, 400, 6
MODES = {"fulltext": ob.MODE_FULLTEXT, "vector": ob.MODE_VECTOR, "hybrid": ob.MODE_HYBRID}


def digest(arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes() if isinstance(a, np.ndarray) else repr(a).encode())
    return h.hexdigest()[:16]


def main():
    ctx = ob.Context(0)
    rows = synth.make_vectors(N, DIM, seed=21)
    qv, _ = synth.make_vector_queries(rows, B, seed=22)
    data = synth.make_text_corpus(N, VOCAB, seed=23)
    texts = synth.make_text_queries(VOCAB, B, seed=24)
    emb = ob.EmbeddingFieldStorage(ctx, "BGEBase", dim=DIM)
    emb.insert_batch(np.arange(N, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(ctx, data)
    tsc = ob.TokenScoreContext(ctx, emb, strs)
    rng = np.random.default_rng(25)
    store = ob.FacetStore(ctx, N)
    store.add_bool_field("flag", np.arange(0, N, 3), np.arange(1, N, 3))
    store.add_string_field("color", {k: np.flatnonzero(rng.integers(0, 4, N) == i) for i, k in enumerate(["r", "g", "b"])})
    store.add_number_field("price", np.arange(N), rng.integers(0, 50, N).astype(np.float64))
    gb = ob.GroupBy(store, ["color"])
    gb2 = ob.GroupBy(store, ["flag", "color"])
    sf = E.SortField(ctx, N, np.arange(N), rng.normal(size=N), "number")
    f_a = ob.DeviceFilter.from_ids(ctx, np.arange(0, N, 2), N)
    f_b = ob.DeviceFilter.from_ids(ctx, np.arange(0, N // 2), N)
    host_bits = np.zeros((N + 63) // 64, np.uint64)
    host_bits[: len(host_bits) // 2] = np.uint64(0x5555555555555555)
    promote = [[(5, 0), (17, 2)], [], [(3, 1)], [(40, 0), (41, 1), (42, 2)], [], [(9, 4)]]
    facets = [{"flag": {"true": True, "false": True}}, None, {"color": {}}, {"price": {"ranges": [{"from": 0, "to": 20}]}},
              {"color": {}, "flag": {"true": True}}, None]
    sorts = [(sf, "ASC"), None, (sf, "DESC"), None, (sf, "ASC"), None]
    qgroups = [(gb, 3), None, (gb2, 2, (sf, "DESC")), (gb, 1), None, (None, 0, (sf, "ASC"))]

    def params(mode, flt, extra, limit=8, offset=1):
        kw = {}
        if flt == "filter":
            kw["device_filter"] = f_a
        elif flt == "bits":
            kw.update(filtered_doc_ids=host_bits, filter_nbits=N)
        elif flt == "q_filters":
            kw["device_filters"] = [f_a, None, f_b, f_a, None, f_b]
        if extra == "omc":
            kw.update(omc_doc_ids=np.arange(0, N, 7, dtype=np.uint64), omc_mult=np.full(len(range(0, N, 7)), 1.5, np.float32))
        if extra == "threshold":
            kw["threshold"] = 0.5
        return ob.TokenScoreParams(mode=MODES[mode], limit_hint=limit, offset=offset, similarity=0.0, **kw)

    def items(extra):
        return promote if extra == "items" else None

    calls = {
        "oc_search": lambda p, x: tsc.execute_batch_arrays(p, texts, qv),
        "oc_search_facets": lambda p, x: E.search_facets(tsc, store, p, {"flag": {"true": True, "false": True}, "color": {}}, texts, qv),
        "oc_search_groups": lambda p, x: E.search_groups_arrays(tsc, gb, p, 3, texts, qv),
        "oc_search_pinned": lambda p, x: E.search_pinned_arrays(tsc, p, promote if x == "items" else [[]] * B, texts, qv),
        "oc_search_groups_pinned": lambda p, x: E.search_groups_arrays(tsc, gb2, p, 2, texts, qv, promote=promote if x == "items" else [[]] * B),
        "oc_search_sorted": lambda p, x: E.search_sorted_arrays(tsc, p, sf, "DESC", items(x), texts, qv),
        "oc_search_groups_sorted": lambda p, x: E.search_groups_arrays(tsc, gb, p, 2, texts, qv, items(x), (sf, "ASC")),
        "oc_search_q_sorted": lambda p, x: E.search_q_sorted_arrays(tsc, p, sorts, items(x), texts, qv),
        "oc_search_q_groups": lambda p, x: E.search_q_groups_arrays(tsc, p, qgroups, items(x), texts, qv),
        "oc_search_q_facets": lambda p, x: E.search_q_facets_arrays(tsc, store, p, facets, qgroups, items(x), texts, qv)[:-1],
    }

    def run(name, fn):
        before = ctx.launch_count()
        try:
            out, rc = fn(), 0
        except ob.OcError as e:
            out, rc = (), e.code
        t = ctx.last_timing()
        print(f"{name} rc={rc} launches={ctx.launch_count() - before} h2d={t['h2d_bytes']} d2h={t['d2h_bytes']} "
              f"out={digest(out if isinstance(out, (tuple, list)) else [out])}", flush=True)

    for entry, mode, flt, extra in itertools.product(calls, MODES, ["none", "filter", "bits", "q_filters"],
                                                     ["plain", "items", "omc", "threshold"]):
        run(f"{entry} {mode} {flt} {extra}", lambda: calls[entry](params(mode, flt, extra), extra))

    # limit 0: groups and facets only
    for mode in MODES:
        run(f"oc_search_groups {mode} limit0", lambda: E.search_groups_arrays(tsc, gb, params(mode, "none", "plain", 0, 0), 3, texts, qv))
        run(f"oc_search_groups_pinned {mode} limit0",
            lambda: E.search_groups_arrays(tsc, gb, params(mode, "none", "plain", 0, 0), 2, texts, qv, promote=promote))
        run(f"oc_search_q_groups {mode} limit0",
            lambda: E.search_q_groups_arrays(tsc, params(mode, "filter", "plain", 0, 0), [(gb, 2)] * B, promote, texts, qv))
        run(f"oc_search_q_facets {mode} limit0",
            lambda: E.search_q_facets_arrays(tsc, store, params(mode, "q_filters", "plain", 0, 0), [{"color": {}}] * B,
                                             None, None, texts, qv)[:-1])

    # refusals
    big = [[(i, i) for i in range(1100)]] + [[]] * (B - 1)
    for mode in MODES:
        run(f"refuse {mode} limit0", lambda: tsc.execute_batch_arrays(params(mode, "none", "plain", 0, 0), texts, qv))
        run(f"refuse {mode} limit+offset", lambda: tsc.execute_batch_arrays(params(mode, "none", "plain", 1000, 100), texts, qv))
        run(f"refuse {mode} pins 2x", lambda: E.search_pinned_arrays(tsc, params(mode, "none", "plain", 600, 0), promote, texts, qv))
        run(f"refuse {mode} pins items", lambda: E.search_pinned_arrays(tsc, params(mode, "none", "plain"), big, texts, qv))
        run(f"refuse {mode} group stride",
            lambda: E.search_q_groups_arrays(tsc, params(mode, "none", "plain"), qgroups, promote, texts, qv, group_stride=2))
        run(f"refuse {mode} groups max_results", lambda: E.search_groups_arrays(tsc, gb, params(mode, "none", "plain"), 2000, texts, qv))
        run(f"refuse {mode} groups q_filters",
            lambda: E.search_groups_arrays(tsc, gb, params(mode, "q_filters", "plain"), 3, texts, qv))
        run(f"refuse {mode} q_facets limit0 flat",
            lambda: E.search_q_facets_arrays(tsc, store, params(mode, "none", "plain", 0, 0), facets, None, None, texts, qv)[:-1])

    # refusals that write nothing: the outputs keep their sentinel
    def raw_groups(n_queries, sort):
        sp, keep, _ = tsc._build_params(params("hybrid", "none", "plain"), texts, qv)
        sp.n_queries = n_queries
        d, s, n, c = np.full((B, 8), 7, np.uint64), np.full((B, 8), 7, np.float32), np.full(B, 7, np.uint32), np.full(B, 7, np.uint64)
        gd, gs, gn = np.full((B, 3, 2), 7, np.uint64), np.full((B, 3, 2), 7, np.float32), np.full((B, 3), 7, np.uint32)
        sv, gsv = np.full((B, 8), 7.0), np.full((B, 3, 2), 7.0)
        if sort:
            rc = _lib.lib().oc_search_groups_sorted(ctx._h, emb._h, strs._h, gb._h, C.byref(sp), 2, None, None, 2, E._p(d), E._p(s),
                                                    E._p(sv), E._p(n), E._p(c), E._p(gd), E._p(gs), E._p(gsv), E._p(gn))
        else:
            rc = _lib.lib().oc_search_groups(ctx._h, emb._h, strs._h, gb._h, C.byref(sp), 2, E._p(d), E._p(s), E._p(n), E._p(c),
                                             E._p(gd), E._p(gs), E._p(gn))
        return rc, d, s, n, c, gd, gs, gn, sv, gsv
    run("refuse groups n_queries", lambda: raw_groups(70000, False))
    run("refuse groups_sorted NULL sort", lambda: raw_groups(B, True))

    # oc_batcher: one round of B requests.  Per request: rc and output digest; per round: the launch delta, the last
    # call's h2d / d2h bytes and the stats delta.  A merged round starts its requests 30 ms apart from B threads into a
    # batcher that waits for all B, so each round is one merged call with the requests in index order.
    q_flt = [f_a, None, f_b, f_a, None, f_b]

    def bparams(mode, flt, i):
        kw = {"device_filter": f_a} if flt == "filter" else {"device_filter": q_flt[i]} if flt == "q_filters" else \
            {"filtered_doc_ids": host_bits, "filter_nbits": N} if flt == "bits" else {}
        return ob.TokenScoreParams(mode=MODES[mode], limit_hint=8, offset=1, similarity=0.0, **kw)

    bcalls = {
        "search": lambda bat, p, i: bat.search(p, texts[i], qv[i]),
        "search_sorted": lambda bat, p, i: bat.search_sorted(p, sorts[i], promote[i], texts[i], qv[i]),
        "search_groups": lambda bat, p, i: bat.search_groups(p, qgroups[i], promote[i], texts[i], qv[i]),
        "search_faceted": lambda bat, p, i: bat.search_faceted(store, p, facets[i], qgroups[i], promote[i], texts[i], qv[i]),
    }

    def batcher_round(name, max_batch, mode, flt, fns):
        bat = ob.SearchBatcher(tsc, max_batch=max_batch, max_wait_us=5_000_000)
        outs = [None] * B

        def one(i):
            if max_batch > 1 and flt != "bits":
                time.sleep(0.03 * i)
            try:
                outs[i] = (0, bcalls[fns[i]](bat, bparams(mode, flt, i), i))
            except ob.OcError as e:
                outs[i] = (e.code, ())

        before = ctx.launch_count()
        if max_batch == 1 or flt == "bits":   # every request runs directly: one at a time, so the last call is request B-1
            for i in range(B):
                one(i)
        else:
            th = [threading.Thread(target=one, args=(i,)) for i in range(B)]
            for t in th:
                t.start()
            for t in th:
                t.join()
        t, s = ctx.last_timing(), bat.stats()
        bat.close()
        for i, (rc, out) in enumerate(outs):
            print(f"batcher {name} req{i} {fns[i]} rc={rc} out={digest(out if isinstance(out, tuple) else [out])}", flush=True)
        print(f"batcher {name} launches={ctx.launch_count() - before} h2d={t['h2d_bytes']} d2h={t['d2h_bytes']} "
              f"queries={s['queries']} batches={s['batches']} direct={s['direct']}", flush=True)

    for fn, mode, (case, mb) in itertools.product(bcalls, MODES, [("direct", 1), ("merged", B)]):
        batcher_round(f"{fn} {mode} {case}", mb, mode, "none", [fn] * B)
    mixes = {"plain": ["search"] * B, "plain+sorted": ["search", "search_sorted"] * (B // 2), "grouped": ["search_groups"] * B}
    for mix, mode, flt in itertools.product(mixes, MODES, ["none", "filter", "bits", "q_filters"]):
        batcher_round(f"mix {mix} {mode} {flt}", B, mode, flt, mixes[mix])


if __name__ == "__main__":
    main()
