"""Per-query where-filters in one batch (oc_search_params.q_filters, TokenScoreParams.device_filters): every query of a
batch is scored exactly as if it were alone in an oc_search with p->filter = its own filter — same ids, same score bits,
same count — on the tensor-core sweep (B >= 8), the exact sweep (B < 8, limit > 128, re-runs of flagged queries) and
the BM25 kernels; checked against the CPU oracle, with where clauses of an IndexLoader corpus, through the batcher, and
for every refusal."""
import ctypes as C
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import _lib, synth
from oramacore_b200.engine import _p
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, TextQuery

pytestmark = pytest.mark.gpu

N, DIM, VOCAB = 60_000, 128, 3000
OC_ERR_INVALID, OC_ERR_UNSUPPORTED = -1, -4
MODES = {"fulltext": MODE_FULLTEXT, "vector": MODE_VECTOR, "hybrid": MODE_HYBRID}


def _filters(ctx, n, rng):
    """The mix of the issue: shared, distinct, empty, all-pass, ~0.05 %, nbits < corpus, ids >= nbits."""
    ids = np.arange(n, dtype=np.uint64)
    fs = {
        "share": ob.DeviceFilter.from_ids(ctx, ids[ids % 3 == 0], n),
        "d30": ob.DeviceFilter.from_ids(ctx, ids[rng.random(n) < 0.3], n),
        "d70": ob.DeviceFilter.from_ids(ctx, ids[rng.random(n) < 0.7], n),
        "empty": ob.DeviceFilter.from_ids(ctx, [], n),
        "all": ob.DeviceFilter.from_ids(ctx, ids, n),
        "sel": ob.DeviceFilter.from_ids(ctx, rng.choice(n, max(1, n // 2000), replace=False).astype(np.uint64), n),
        "half_nbits": ob.DeviceFilter.from_ids(ctx, ids[: n // 2][rng.random(n // 2) < 0.5], n // 2),
        "big_ids": ob.DeviceFilter.from_ids(ctx, np.concatenate([ids[rng.random(n) < 0.2], ids[-2000:] + np.uint64(5000)]), n - 3000),
    }
    return fs


def _assign(fs, B, seed):
    order = [None, "share", "d30", "share", "empty", "all", "sel", "half_nbits", "big_ids", "d70", None, "share"]
    rng = np.random.default_rng(seed)
    names = [order[i % len(order)] if i < len(order) else order[int(rng.integers(0, len(order)))] for i in range(B)]
    return [None if k is None else fs[k] for k in names]


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    rng = np.random.default_rng(2024)
    rows = synth.make_vectors(N, DIM, seed=61)
    data = synth.make_text_corpus(N, VOCAB, seed=63)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(N, dtype=np.uint64), rows)
    embh = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM, dtype="bf16")
    embh.insert_batch(np.arange(N, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    fs = _filters(gpu_ctx, N, rng)
    yield dict(ctx=gpu_ctx, rows=rows, data=data, emb=emb, embh=embh, strs=strs, fs=fs)
    for f in fs.values():
        f.close()
    emb.close(); embh.close(); strs.close()


def _inputs(B, seed, rows, multi=False):
    qv, _ = synth.make_vector_queries(rows, B, seed=seed)
    texts = synth.make_text_queries(VOCAB, B, seed=seed + 1)
    if multi:   # prefix / tolerance expansion: tokens that resolve to several index terms (K3)
        rng = np.random.default_rng(seed + 2)
        out = []
        for t in texts:
            ids = t.term_id.tolist()
            exp = [[x] + [int(v) for v in rng.integers(0, VOCAB, int(rng.integers(0, 3)))] for x in ids]
            off = np.cumsum([0] + [len(e) for e in exp]).astype(np.uint32)
            flat = np.asarray([v for e in exp for v in e], np.uint32)
            w = np.where(np.arange(flat.shape[0]) % 2 == 0, 2.0, 1.0).astype(np.float32)
            out.append(TextQuery(off, np.zeros(flat.shape[0], np.uint32), flat, w))
        texts = out
    return qv, texts


def _check_alone(tsc, mode, filters, texts, qv, **kw):
    """The batch with device_filters == every query alone with device_filter, byte for byte."""
    B = len(filters)
    got = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=mode, device_filters=filters, **kw), texts, qv)
    for b in range(B):
        one = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=mode, device_filter=filters[b], **kw),
                                       None if texts is None else [texts[b]], None if qv is None else qv[b:b + 1])
        for x, y, what in zip(got, one, ("docs", "scores", "n", "count")):
            assert x[b].tobytes() == y[0].tobytes(), (b, what, mode, kw)
    return got


@pytest.mark.parametrize("B", [1, 5, 48, 256])
@pytest.mark.parametrize("mode", list(MODES))
def test_batch_equals_each_query_alone(corpus, mode, B):
    c = corpus
    m = MODES[mode]
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"] if m != MODE_FULLTEXT else None, c["strs"] if m != MODE_VECTOR else None)
    qv, texts = _inputs(B, 100 + B, c["rows"])
    filters = _assign(c["fs"], B, B)
    if B == 1:
        filters = [c["fs"]["d30"]]
    _check_alone(tsc, m, filters, texts if m != MODE_VECTOR else None, qv if m != MODE_FULLTEXT else None, similarity=0.0)


@pytest.mark.parametrize("variant", ["threshold", "omc", "offset", "multi_term", "bf16", "limit200"])
def test_batch_equals_alone_variants(corpus, variant):
    c = corpus
    B = 48
    emb = c["embh"] if variant == "bf16" else c["emb"]
    tsc = ob.TokenScoreContext(c["ctx"], emb, c["strs"])
    qv, texts = _inputs(B, 300, c["rows"], multi=variant == "multi_term")
    filters = _assign(c["fs"], B, 7)
    kw = dict(similarity=0.0)
    if variant == "threshold":
        kw["threshold"] = 0.5
    elif variant == "omc":
        rng = np.random.default_rng(9)
        od = np.sort(rng.choice(N, 3000, replace=False)).astype(np.uint64)
        kw.update(omc_doc_ids=od, omc_mult=rng.uniform(0.5, 3.0, od.shape[0]).astype(np.float32))
    elif variant == "offset":
        kw.update(limit_hint=10, offset=5)
    elif variant == "limit200":
        kw["limit_hint"] = 200
    for mode in (MODE_FULLTEXT, MODE_HYBRID):
        _check_alone(tsc, mode, filters, texts, qv, **kw)
    if variant in ("bf16", "limit200", "offset"):
        _check_alone(tsc, MODE_VECTOR, filters, None, qv, **kw)


def test_uncommitted_deletes(gpu_ctx):
    n = 30_000
    rows = synth.make_vectors(n, DIM, seed=71)
    data = synth.make_text_corpus(n, VOCAB, seed=73)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    rng = np.random.default_rng(5)
    fs = _filters(gpu_ctx, n, rng)
    try:
        gone = rng.choice(n, 2000, replace=False).tolist()
        strs.delete(gone)
        emb.delete(gone)
        tsc = ob.TokenScoreContext(gpu_ctx, emb, strs)
        qv, texts = _inputs(40, 500, rows)
        filters = _assign(fs, 40, 3)
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            docs, _, n_hit, _ = _check_alone(tsc, mode, filters, texts, qv, similarity=0.0)
            assert not {int(d) for b in range(40) for d in docs[b, :n_hit[b]]} & set(gone)
    finally:
        for f in fs.values():
            f.close()
        emb.close(); strs.close()


def test_duplicate_rows_force_a_filtered_rerun(gpu_ctx):
    """3000 exact copies of one row within the query's filter: more than GEMM_MAX_RESCORE rows tie with the limit-th
    best, the tensor-core result is flagged and the query re-runs through the exact sweep under its own slot."""
    n = 40_000
    rows = synth.make_vectors(n, DIM, seed=81)
    rows[10_000:13_000] = rows[5]
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    ids = np.arange(n, dtype=np.uint64)
    f_dup = ob.DeviceFilter.from_ids(gpu_ctx, ids[(ids % 2 == 0)], n)           # half of the copies pass
    f_other = ob.DeviceFilter.from_ids(gpu_ctx, ids[(ids < 10_000) | (ids >= 13_000)], n)
    try:
        tsc = ob.TokenScoreContext(gpu_ctx, emb, None)
        B = 16
        qv = np.repeat(rows[5:6], B, axis=0).astype(np.float32)
        filters = [f_dup, f_other, None, f_dup] * 4
        tsc.execute_batch_arrays(ob.TokenScoreParams(mode=MODE_VECTOR, similarity=0.0, device_filters=filters), None, qv)
        t = gpu_ctx.last_timing()
        assert t["scan_tensor_core"] == 1 and t["scan_unproven"] > 0, t
        _check_alone(tsc, MODE_VECTOR, filters, None, qv, similarity=0.0)
    finally:
        f_dup.close(); f_other.close(); emb.close()


def test_oracle(corpus, orc):
    c = corpus
    B = 32
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    qv, texts = _inputs(B, 700, c["rows"])
    filters = _assign(c["fs"], B, 11)
    ix, st = orc.StrIndex(c["data"]), orc.EmbStore(c["rows"])
    for mode in (MODE_FULLTEXT, MODE_HYBRID):
        got = tsc.execute_batch(ob.TokenScoreParams(mode=mode, similarity=0.0, device_filters=filters), texts, qv)
        sb = orc.SearchBatch(ix, st)
        for i in range(B):
            f = filters[i]
            if f is None:
                sb.add(mode, limit=10, similarity=0.0, q_vec=qv[i], text=texts[i])
            else:
                sb.add(mode, limit=10, similarity=0.0, q_vec=qv[i], text=texts[i], filter_bits=f.read(), filter_nbits=f.nbits)
        od, os_, on, oc = sb.run(2)
        for i, h in enumerate(got):
            assert h.count == int(oc[i]), (mode, i)
            assert_topk_equal(h.doc_ids, h.scores, od[i, :on[i]], os_[i, :on[i]])


def test_where_clauses(gpu_ctx):
    rng = np.random.default_rng(13)
    n = 6000
    ld = IndexLoader(gpu_ctx, ["text"], embedding_dim=DIM, bool_fields=["b"], number_fields=["x"], string_filter_fields=["s"],
                     date_fields=["d"], geopoint_fields=["g"])
    words = [f"w{i}" for i in range(300)]
    vecs = synth.make_vectors(n, DIM, seed=91)
    try:
        for d in range(n):
            toks = [words[int(t)] for t in np.minimum(rng.zipf(1.3, int(rng.integers(3, 12))) - 1, 299)]
            terms = {}
            for i, t in enumerate(toks):
                terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
            vals = [{"type": "ScoreString2", "field": "text", "field_length": len(toks), "terms": terms},
                    {"type": "FilterBool2", "field": "b", "value": {"Plain": bool(rng.random() < 0.5)}},
                    {"type": "FilterNumber2", "field": "x", "value": {"I64": {"Plain": int(rng.integers(0, 100))}}},
                    {"type": "FilterString2", "field": "s", "value": {"Plain": f"k{int(rng.integers(0, 5))}"}},
                    {"type": "FilterDate2", "field": "d", "value": {"Plain": int(rng.integers(0, 10**12))}},
                    {"type": "FilterGeoPoint2", "field": "g",
                     "value": {"Plain": {"lat": float(rng.uniform(-50, 50)), "lon": float(rng.uniform(-90, 90))}}}]
            ld.apply({"type": "Index", "doc_id": d, "indexed_values": vals})
        ld.apply({"type": "IndexEmbedding", "data": [(d, [vecs[d].tolist()]) for d in range(n)]})
        ld.commit()
        ld.apply({"type": "DeleteDocuments", "doc_ids": [3, 77, 1000]})
        wheres = [{"b": True}, {"x": {"between": [10, 40]}}, {"s": "k2"}, {"d": {"gt": "1995-01-01T00:00:00Z"}},
                  {"g": {"radius": {"coordinates": {"lat": 0, "lon": 0}, "value": 2000, "unit": "km", "inside": True}}},
                  {"and": [{"b": False}, {"x": {"lt": 50}}]}, {"or": [{"s": "k0"}, {"s": "k4"}]}, {"not": {"x": {"gte": 90}}},
                  None]
        B = 27
        handles = [None if wheres[i % len(wheres)] is None else ld.where_filter(wheres[i % len(wheres)]) for i in range(B)]
        texts = ld.resolve([" ".join(words[int(t)] for t in rng.integers(0, 40, 2)) for _ in range(B)])
        qv = vecs[rng.integers(0, n, B)] + 0.01
        tsc = ld.context()
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            got = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=mode, similarity=0.0, device_filters=handles), texts, qv)
            for b in range(B):
                ref = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=mode, similarity=0.0, device_filter=handles[b]),
                                               _one_text(texts, b), qv[b:b + 1])
                for x, y in zip(got, ref):
                    assert x[b].tobytes() == y[0].tobytes(), (mode, b, wheres[b % len(wheres)])
        for h in handles:
            if h is not None:
                h.close()
    finally:
        ld.close()


def _one_text(batch, b):
    """Query b of a packed TextQueryBatch as a one-query TextQuery."""
    t0, t1 = int(batch.q_token_offsets[b]), int(batch.q_token_offsets[b + 1])
    e0, e1 = int(batch.token_term_offsets[t0]), int(batch.token_term_offsets[t1])
    off = (batch.token_term_offsets[t0:t1 + 1] - np.uint32(e0)).astype(np.uint32)
    return [TextQuery(off, batch.term_field[e0:e1].copy(), batch.term_id[e0:e1].copy(), batch.term_weight[e0:e1].copy())]


def test_batcher_coalesces_device_filtered_requests(corpus):
    c = corpus
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    T, Q = 8, 24
    qv, texts = _inputs(T * Q, 900, c["rows"])
    filters = _assign(c["fs"], T * Q, 21)
    expect = {}
    for i in range(T * Q):
        expect[i] = tsc.execute_batch(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i]),
                                      [texts[i]], qv[i:i + 1])[0]
    bat = ob.SearchBatcher(tsc, max_batch=64, max_wait_us=3000)
    bad = []
    n_filtered = sum(f is not None for f in filters)

    def worker(t):
        for i in range(t, T * Q, T):
            h = bat.search(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i]), texts[i], qv[i])
            e = expect[i]
            if not (h.count == e.count and h.doc_ids.tobytes() == e.doc_ids.tobytes() and h.scores.tobytes() == e.scores.tobytes()):
                bad.append(i)
    th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    st = bat.stats()
    assert not bad, bad[:10]
    assert n_filtered > 0 and st["direct"] == 0, st
    assert st["queries"] == T * Q and st["batches"] < st["queries"], st
    # a host bitmap still goes straight to oc_search
    bits = c["fs"]["share"].read()
    h = bat.search(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, filtered_doc_ids=bits, filter_nbits=N), texts[0], qv[0])
    e = tsc.execute_batch(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, filtered_doc_ids=bits, filter_nbits=N), [texts[0]], qv[0:1])[0]
    assert h.doc_ids.tobytes() == e.doc_ids.tobytes() and h.count == e.count
    assert bat.stats()["direct"] == 1
    bat.close()


def test_refusals(corpus, gpu_ctx):
    c = corpus
    L = _lib.lib()
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    B = 4
    qv, texts = _inputs(B, 950, c["rows"])
    fl = [c["fs"]["share"], None, c["fs"]["d30"], None]
    other = ob.Context(0)
    foreign = ob.DeviceFilter.from_ids(other, [1, 2, 3], N)
    try:
        def run(fn, **kw):
            sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filters=fl, **kw), texts, qv)
            docs = np.full((B, 10), 7, np.uint64); sc = np.full((B, 10), 7, np.float32)
            n = np.full(B, 7, np.uint32); cnt = np.full(B, 7, np.uint64)
            rc = fn(sp, docs, sc, n, cnt)
            assert (docs == 7).all() and (sc == 7).all() and (n == 7).all() and (cnt == 7).all()   # nothing written
            return rc

        P = _p
        srch = lambda sp, d, s, n, cnt: L.oc_search(c["ctx"]._h, c["emb"]._h, c["strs"]._h, C.byref(sp), P(d), P(s), P(n), P(cnt))  # noqa: E731
        # with filter / filter_bits
        def with_filter(sp, *a):
            sp.filter = c["fs"]["all"]._h
            return srch(sp, *a)

        def with_bits(sp, *a):
            bits = np.zeros((N + 63) // 64, np.uint64)
            sp.filter_bits, sp.filter_nbits = P(bits), N
            return srch(sp, *a)

        def sharded(sp, *a):
            sp.sharded = 1
            return srch(sp, *a)

        def foreign_handle(sp, *a):
            arr = (C.c_void_p * B)(fl[0]._h.value, None, foreign._h.value, None)
            sp.q_filters = C.cast(arr, C.c_void_p)
            return srch(sp, *a)

        assert run(with_filter) == OC_ERR_INVALID
        assert run(with_bits) == OC_ERR_INVALID
        assert run(foreign_handle) == OC_ERR_INVALID
        assert run(sharded) == OC_ERR_UNSUPPORTED
        # the other entry points refuse per-query filters
        st = ob.FacetStore(c["ctx"], N)
        st.add_bool_field("b", np.arange(0, N, 2), np.arange(1, N, 2))
        g = ob.GroupBy(st, ["b"])
        sf = ob.SortField(c["ctx"], N, np.arange(N, dtype=np.uint64), np.arange(N, dtype=np.float64), "number")
        try:
            def groups(sp, d, s, n, cnt):
                gd = np.zeros(B * 2 * 5, np.uint64); gs = np.zeros(B * 2 * 5, np.float32); gn = np.zeros(B * 2, np.uint32)
                return L.oc_search_groups(c["ctx"]._h, c["emb"]._h, c["strs"]._h, g._h, C.byref(sp), 5, P(d), P(s), P(n), P(cnt),
                                          P(gd), P(gs), P(gn))

            def pinned(sp, d, s, n, cnt):
                return L.oc_search_pinned(c["ctx"]._h, c["emb"]._h, c["strs"]._h, C.byref(sp), None, P(d), P(s), P(n), P(cnt), None, None)

            def sorted_(sp, d, s, n, cnt):
                so = _lib.Sort(sf._h, 0)
                return L.oc_search_sorted(c["ctx"]._h, c["emb"]._h, c["strs"]._h, C.byref(sp), C.byref(so), None, P(d), P(s), None,
                                          P(n), P(cnt), None, None)
            assert run(groups) == OC_ERR_UNSUPPORTED
            assert run(pinned) == OC_ERR_UNSUPPORTED
            assert run(sorted_) == OC_ERR_UNSUPPORTED
        finally:
            g.close(); sf.close(); st.close()
    finally:
        foreign.close()
        other.close()
