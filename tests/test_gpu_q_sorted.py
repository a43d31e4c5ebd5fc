"""One batch in which every query has its own sortBy, pin rules and where-filter (oc_search_q_sorted,
search_q_sorted_arrays) and the batcher's sorted requests (oc_batcher_search_sorted, SearchBatcher.search_sorted).

The rule: query b's outputs — hits, score bits, n, count, sort values, and its items' pin scores and present flags —
equal, byte for byte, what it gets alone with its own filter and items: oc_search_sorted with its sort, or
oc_search_pinned in score order (sort values NaN).  Checked over fulltext / vector / hybrid, B in {1, 5, 48, 256}, the
filter mix of test_gpu_query_filters, number fields with ties and multi-valued documents, a date and a bool field, the
threshold / OMC / multi-term / bf16 / limit 200 / offset variants, tombstones, a commit between calls and a tensor-core
re-run; plus the whole-batch equalities with oc_search_sorted and oc_search_pinned, promoted documents only another
query's filter admits, where clauses of an IndexLoader corpus, the oracle's score maps, every refusal, and many threads
through the batcher."""
import ctypes as C
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib, synth
from oramacore_b200.engine import _p
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from test_gpu_query_filters import DIM, MODES, N, OC_ERR_INVALID, OC_ERR_UNSUPPORTED, _assign, _filters, _inputs, _one_text
from test_gpu_query_filters import corpus  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fields(corpus):  # noqa: F811
    """Sort fields over the corpus: numbers with long runs of ties and multi-valued documents, a date, a bool."""
    ctx = corpus["ctx"]
    rng = np.random.default_rng(77)
    ids = np.arange(N, dtype=np.uint64)
    extra = rng.choice(N, N // 10, replace=False).astype(np.uint64)          # a second value for 10 % of the documents
    has = ids[rng.random(N) < 0.9]                                           # 10 % have no value
    raw = dict(num=(np.concatenate([has, extra]), np.concatenate([rng.integers(0, 40, has.shape[0]),
                                                                 rng.integers(0, 40, extra.shape[0])]).astype(np.float64), "number"),
               price=(ids, rng.uniform(0, 1000, N).round(2), "number"),
               date=(ids, (1_600_000_000_000 + rng.integers(0, 5000, N) * 86_400_000).astype(np.int64), "date"),
               flag=(ids[::2], rng.random(ids[::2].shape[0]) < 0.3, "bool"))
    fs = {}
    for k, (d, v, kind) in raw.items():
        fs[k] = ob.SortField(ctx, N, d, v, kind)
        fs[k].raw = (d, np.asarray(v, np.float64))   # (doc ids, values) for the restatement
    yield fs
    for f in fs.values():
        f.close()


def _sorts(fs, B, seed):
    """The mix of a shop's search page: none / number ASC / number DESC / date DESC, plus the other fields."""
    mix = [None, (fs["price"], "ASC"), (fs["price"], "DESC"), (fs["date"], "DESC"), (fs["num"], "ASC"), None,
           (fs["num"], "DESC"), (fs["flag"], "ASC"), (fs["flag"], "DESC"), (fs["date"], "ASC")]
    rng = np.random.default_rng(seed)
    return [mix[i] if i < len(mix) else mix[int(rng.integers(0, len(mix)))] for i in range(B)]


def _promote(B, seed, n=N, hits=None):
    """0-3 items per query at positions 0-12; some promote a document the query already lists."""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(B):
        k = int(rng.integers(0, 4))
        items = []
        for _ in range(k):
            d = int(rng.integers(0, n))
            if hits is not None and len(hits[b]) and rng.random() < 0.4:
                d = int(hits[b][int(rng.integers(0, len(hits[b])))])
            items.append((d, int(rng.integers(0, 13))))
        out.append(items)
    return out


def _alone(tsc, mode, flt, sort, items, text, qv, **kw):
    """(docs, scores, sort values, n, count, pin scores, pin present) of one query alone."""
    p = ob.TokenScoreParams(mode=mode, device_filter=flt, **kw)
    if sort is None:
        d, s, n, cnt, ps, pp = ob.search_pinned_arrays(tsc, p, [items], text, qv)
        L = d.shape[1]
        sv = np.where(np.arange(L)[None, :] < n[:, None], np.nan, 0.0)
        return d, s, sv, n, cnt, ps, pp
    return ob.search_sorted_arrays(tsc, p, sort[0], sort[1], [items], text, qv)


def _check(tsc, mode, filters, sorts, promote, texts, qv, **kw):
    """The batch equals every query alone, byte for byte."""
    B = len(sorts)
    got = ob.search_q_sorted_arrays(tsc, ob.TokenScoreParams(mode=mode, device_filters=filters, **kw), sorts, promote, texts, qv)
    off = np.cumsum([0] + [len(x) for x in promote])
    for b in range(B):
        one = _alone(tsc, mode, None if filters is None else filters[b], sorts[b], promote[b],
                     None if texts is None else _one(texts, b), None if qv is None else qv[b:b + 1], **kw)
        for what, x, y in zip(("docs", "scores", "sort values", "n", "count"), got[:5], one[:5]):
            assert x[b].tobytes() == y[0].tobytes(), (b, what, mode, sorts[b] and sorts[b][1], kw)
        for what, x, y in zip(("pin scores", "pin present"), got[5:], one[5:]):
            assert x[off[b]:off[b + 1]].tobytes() == y.tobytes(), (b, what, mode, kw)
    return got


def _one(texts, b):
    return _one_text(texts, b) if isinstance(texts, ob.TextQueryBatch) else [texts[b]]


def _tsc(c, m, emb=None):
    return ob.TokenScoreContext(c["ctx"], (emb or c["emb"]) if m != MODE_FULLTEXT else None, c["strs"] if m != MODE_VECTOR else None)


@pytest.mark.parametrize("B", [1, 5, 48, 256])
@pytest.mark.parametrize("mode", list(MODES))
def test_batch_equals_each_query_alone(corpus, fields, mode, B):  # noqa: F811
    c = corpus
    m = MODES[mode]
    qv, texts = _inputs(B, 1100 + B, c["rows"])
    filters = _assign(c["fs"], B, B + 3) if B > 1 else [c["fs"]["d30"]]
    sorts = _sorts(fields, B, B) if B > 1 else [(fields["price"], "DESC")]
    _check(_tsc(c, m), m, filters, sorts, _promote(B, B), texts if m != MODE_VECTOR else None,
           qv if m != MODE_FULLTEXT else None, similarity=0.0)


@pytest.mark.parametrize("variant", ["threshold", "omc", "offset", "multi_term", "bf16", "limit200", "no_filters"])
def test_batch_equals_alone_variants(corpus, fields, variant):  # noqa: F811
    c = corpus
    B = 48
    tsc = _tsc(c, MODE_HYBRID, c["embh"] if variant == "bf16" else None)
    qv, texts = _inputs(B, 1300, c["rows"], multi=variant == "multi_term")
    filters = None if variant == "no_filters" else _assign(c["fs"], B, 17)
    kw = dict(similarity=0.0)
    if variant == "threshold":
        kw["threshold"] = 0.5
    elif variant == "omc":
        rng = np.random.default_rng(19)
        od = np.sort(rng.choice(N, 3000, replace=False)).astype(np.uint64)
        kw.update(omc_doc_ids=od, omc_mult=rng.uniform(0.5, 3.0, od.shape[0]).astype(np.float32))
    elif variant == "offset":
        kw.update(limit_hint=10, offset=5)
    elif variant == "limit200":   # B = 48 at limit 200: the exact sweep
        kw["limit_hint"] = 200
    sorts, promote = _sorts(fields, B, 23), _promote(B, 29)
    for mode in (MODE_FULLTEXT, MODE_HYBRID):
        _check(tsc, mode, filters, sorts, promote, texts, qv, **kw)
    if variant in ("bf16", "limit200", "offset"):
        _check(tsc, MODE_VECTOR, filters, sorts, promote, None, qv, **kw)


def test_whole_batch_equalities(corpus, fields):  # noqa: F811
    """One sort for every query and no q_filters: oc_search_sorted; every entry NULL: oc_search_pinned."""
    c = corpus
    B = 64
    qv, texts = _inputs(B, 1500, c["rows"])
    promote = _promote(B, 31)
    for mode in (MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID):
        tsc = _tsc(c, mode)
        t, q = (texts if mode != MODE_VECTOR else None), (qv if mode != MODE_FULLTEXT else None)
        for kw in (dict(similarity=0.0), dict(similarity=0.0, device_filter=c["fs"]["d30"], offset=3)):
            p = ob.TokenScoreParams(mode=mode, **kw)
            got = ob.search_q_sorted_arrays(tsc, p, [(fields["price"], "DESC")] * B, promote, t, q)
            ref = ob.search_sorted_arrays(tsc, p, fields["price"], "DESC", promote, t, q)
            for x, y in zip(got, ref):
                assert x.tobytes() == y.tobytes(), (mode, kw)
            got = ob.search_q_sorted_arrays(tsc, p, [None] * B, promote, t, q)
            ref = ob.search_pinned_arrays(tsc, p, promote, t, q)
            for x, y in zip(got[:2] + got[3:], ref):
                assert x.tobytes() == y.tobytes(), (mode, kw)
            n = got[3]
            assert np.isnan(got[2][np.arange(p.limit_hint)[None, :] < n[:, None]]).all()


def test_promoted_document_only_another_filter_admits(corpus, fields):  # noqa: F811
    """Query 1 promotes a fulltext match its own filter rejects and slot 0 (query 0's filter) admits: 0.0, not present."""
    c = corpus
    qv, texts = _inputs(2, 1700, c["rows"])
    texts = [texts[1], texts[1]]   # d is a key of query 0's map: present there, rejected only by query 1's filter
    tsc = _tsc(c, MODE_FULLTEXT)
    hits = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=50), [texts[1]])
    cand = [int(d) for d in hits[0][0, :hits[2][0]] if int(d) % 3 == 0]
    assert cand
    d = cand[0]
    ids = np.arange(N, dtype=np.uint64)
    f1 = ob.DeviceFilter.from_ids(c["ctx"], ids[ids != d], N)
    try:
        filters = [c["fs"]["share"], f1]   # "share" = ids % 3 == 0 admits d
        for sorts in ([None, None], [(fields["price"], "ASC"), None], [None, (fields["price"], "ASC")]):
            for mode in (MODE_FULLTEXT, MODE_HYBRID):
                got = _check(_tsc(c, mode), mode, filters, sorts, [[(d, 0)], [(d, 0)]], texts, qv, similarity=0.0)
                ps, pp = got[5], got[6]
                assert pp[0] == 1 and pp[1] == 0 and ps[1] == 0.0, (sorts, mode, ps, pp)
    finally:
        f1.close()


def test_sorted_query_whose_best_documents_only_other_filters_admit(corpus, fields):  # noqa: F811
    c = corpus
    ids = np.arange(N, dtype=np.uint64)
    low = ids[ids < N // 10]                    # price ASC favours nothing in particular: use a field ranked by id
    rank = ob.SortField(c["ctx"], N, ids, ids.astype(np.float64), "number")
    f_low = ob.DeviceFilter.from_ids(c["ctx"], low, N)
    f_high = ob.DeviceFilter.from_ids(c["ctx"], ids[ids >= N // 10], N)
    try:
        B = 8
        qv, texts = _inputs(B, 1900, c["rows"])
        filters = [f_low, f_high] * (B // 2)
        sorts = [(rank, "ASC")] * B
        for mode in (MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID):
            got = _check(_tsc(c, mode), mode, filters, sorts, [[]] * B, texts if mode != MODE_VECTOR else None,
                         qv if mode != MODE_FULLTEXT else None, similarity=0.0)
            for b in range(1, B, 2):
                assert (got[0][b, :got[3][b]] >= N // 10).all(), (mode, b)
    finally:
        rank.close(); f_low.close(); f_high.close()


def test_tombstones_and_commit(gpu_ctx):
    """Uncommitted deletes, then an oc_str_commit between calls: the rank -> row maps of two fields are rebuilt."""
    n = 30_000
    rows = synth.make_vectors(n, DIM, seed=171)
    data = synth.make_text_corpus(n, 3000, seed=173)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    rng = np.random.default_rng(175)
    fs = _filters(gpu_ctx, n, rng)
    ids = np.arange(n + 10, dtype=np.uint64)
    a = ob.SortField(gpu_ctx, n + 10, ids, rng.integers(0, 30, n + 10).astype(np.float64), "number")
    b_ = ob.SortField(gpu_ctx, n + 10, ids, rng.integers(0, 10**6, n + 10).astype(np.int64) * 1000, "date")
    try:
        tsc = ob.TokenScoreContext(gpu_ctx, emb, strs)
        B = 40
        qv, texts = _inputs(B, 177, rows)
        filters = _assign(fs, B, 5)
        sorts = [[None, (a, "ASC"), (b_, "DESC"), (a, "DESC")][i % 4] for i in range(B)]
        promote = _promote(B, 179, n)
        gone = rng.choice(n, 2000, replace=False).tolist()
        strs.delete(gone)
        emb.delete(gone)
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            got = _check(tsc, mode, filters, sorts, promote, texts, qv, similarity=0.0)
            assert not {int(d) for q in range(B) for d in got[0][q, :got[3][q]]} & (set(gone) - {d for p in promote for d, _ in p})
        strs.commit()
        t0 = [int(x) for x in texts[0].term_id[:1]]
        for d in range(n, n + 10):   # new documents that match query 0
            strs.insert(d, 0, 3, {t0[0]: 2})
        strs.commit()
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            _check(tsc, mode, filters, sorts, promote, texts, qv, similarity=0.0)
    finally:
        for f in fs.values():
            f.close()
        a.close(); b_.close(); emb.close(); strs.close()


def test_duplicate_rows_force_a_rerun(gpu_ctx):
    """3000 exact copies of one row: the tensor-core result is flagged and re-run; the sorted tail runs again."""
    n = 40_000
    rows = synth.make_vectors(n, DIM, seed=181)
    rows[10_000:13_000] = rows[5]
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    ids = np.arange(n, dtype=np.uint64)
    f_dup = ob.DeviceFilter.from_ids(gpu_ctx, ids[(ids % 2 == 0)], n)
    f_other = ob.DeviceFilter.from_ids(gpu_ctx, ids[(ids < 10_000) | (ids >= 13_000)], n)
    srt = ob.SortField(gpu_ctx, n, ids, (ids % 97).astype(np.float64), "number")
    try:
        tsc = ob.TokenScoreContext(gpu_ctx, emb, None)
        B = 16
        qv = np.repeat(rows[5:6], B, axis=0).astype(np.float32)
        filters = [f_dup, f_other, None, f_dup] * 4
        sorts = [(srt, "ASC"), None, (srt, "DESC"), None] * 4
        promote = [[(11_000, 1)], [], [(12, 0), (10_002, 3)], [(5, 2)]] * 4
        ob.search_q_sorted_arrays(tsc, ob.TokenScoreParams(mode=MODE_VECTOR, similarity=0.0, device_filters=filters), sorts,
                                  promote, None, qv)
        t = gpu_ctx.last_timing()
        assert t["scan_tensor_core"] == 1 and t["scan_unproven"] > 0, t
        _check(tsc, MODE_VECTOR, filters, sorts, promote, None, qv, similarity=0.0)
    finally:
        f_dup.close(); f_other.close(); srt.close(); emb.close()


def test_where_clauses(gpu_ctx):
    """A different `where` per query through IndexLoader.where_filter, sorted by the loader's number and date fields."""
    rng = np.random.default_rng(191)
    n = 4000
    ld = IndexLoader(gpu_ctx, ["text"], embedding_dim=DIM, bool_fields=["b"], number_fields=["x"], date_fields=["d"])
    words = [f"w{i}" for i in range(200)]
    xs = rng.integers(0, 50, n)
    ds = rng.integers(0, 10**6, n) * 1000
    vecs = synth.make_vectors(n, DIM, seed=193)
    handles = []
    try:
        for d in range(n):
            toks = [words[int(t)] for t in np.minimum(rng.zipf(1.3, int(rng.integers(3, 10))) - 1, 199)]
            terms = {}
            for i, t in enumerate(toks):
                terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
            ld.apply({"type": "Index", "doc_id": d, "indexed_values": [
                {"type": "ScoreString2", "field": "text", "field_length": len(toks), "terms": terms},
                {"type": "FilterBool2", "field": "b", "value": {"Plain": bool(rng.random() < 0.5)}},
                {"type": "FilterNumber2", "field": "x", "value": {"I64": {"Plain": int(xs[d])}}},
                {"type": "FilterDate2", "field": "d", "value": {"Plain": int(ds[d])}}]})
        ld.apply({"type": "IndexEmbedding", "data": [(d, [vecs[d].tolist()]) for d in range(n)]})
        ld.commit()
        ld.apply({"type": "DeleteDocuments", "doc_ids": [3, 77, 1000]})
        ids = np.arange(n, dtype=np.uint64)
        fx = ob.SortField(gpu_ctx, n, ids, xs, "number")
        fd = ob.SortField(gpu_ctx, n, ids, ds.astype(np.int64), "date")
        wheres = [{"b": True}, {"x": {"between": [10, 40]}}, {"and": [{"b": False}, {"x": {"lt": 25}}]}, None,
                  {"not": {"x": {"gte": 45}}}, {"x": {"gt": 5}}]
        B = 24
        handles = [None if wheres[i % len(wheres)] is None else ld.where_filter(wheres[i % len(wheres)]) for i in range(B)]
        texts = ld.resolve([" ".join(words[int(t)] for t in rng.integers(0, 20, 2)) for _ in range(B)])
        texts = [_one_text(texts, b)[0] for b in range(B)]
        qv = (vecs[rng.integers(0, n, B)] + 0.01).astype(np.float32)
        sorts = [[(fx, "ASC"), (fx, "DESC"), (fd, "DESC"), None][i % 4] for i in range(B)]
        promote = [[(int(rng.integers(0, n)), int(rng.integers(0, 6))) for _ in range(i % 3)] for i in range(B)]
        tsc = ld.context()
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            _check(tsc, mode, handles, sorts, promote, texts, qv, similarity=0.0)
        fx.close(); fd.close()
    finally:
        for h in handles:
            if h is not None:
                h.close()
        ld.close()


def test_against_the_oracle(corpus, fields, orc):  # noqa: F811
    """sort.rs / pin_rules.rs restated with a different filter per query: each page is sort_token_scores with sort_by
    (or in score order) and pins over the oracle's filtered fulltext score map."""
    from test_gpu_sort import check, expect_flat, ranks
    from test_pins_host import apply_pin_rules
    c = corpus
    B, limit, offset = 24, 10, 2
    qv, texts = _inputs(B, 2500, c["rows"])
    filters = _assign(c["fs"], B, 51)
    sorts = _sorts(fields, B, 53)
    tsc = _tsc(c, MODE_FULLTEXT)
    ix = orc.StrIndex(c["data"])
    maps = []
    for b in range(B):
        f = filters[b]
        kw = {} if f is None else dict(filter_bits=f.read(), filter_nbits=f.nbits)
        d, s = orc.fulltext(ix, texts[b], **kw)
        maps.append(dict(zip(d.tolist(), s.tolist())))
    promote = _promote(B, 57, hits=[list(m)[:20] for m in maps])
    got = ob.search_q_sorted_arrays(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=limit, offset=offset,
                                                             device_filters=filters), sorts, promote, texts)
    for b in range(B):
        sm, items = maps[b], promote[b]
        if sorts[b] is None:
            keys = sorted(sm, key=lambda d: (-sm[d], d))[:(2 if items else 1) * (limit + offset)]
            page = apply_pin_rules(list(items), sm, [(d, sm[d]) for d in keys])[offset:offset + limit]
            exp = ([d for d, _ in page], [s for _, s in page], [np.nan] * len(page))
        else:
            field, order = sorts[b]
            exp = expect_flat(sm, ranks(*field.raw, order), limit, offset, items)
        k = int(got[3][b])
        check(got[0][b, :k], got[1][b, :k], got[2][b, :k], exp, exact=False)
        assert int(got[4][b]) == len(sm)


def test_refusals(corpus, fields, gpu_ctx):  # noqa: F811
    c = corpus
    L = _lib.lib()
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    B = 4
    qv, texts = _inputs(B, 2100, c["rows"])
    other = ob.Context(0)
    foreign = ob.DeviceFilter.from_ids(other, [1, 2, 3], N)
    foreign_sort = ob.SortField(other, N, [1, 2], [1.0, 2.0], "number")
    try:
        def run(sorts, promote=None, fl=(c["fs"]["share"], None, c["fs"]["d30"], None), q_sorts_null=False, edit=None, **kw):
            sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filters=fl, **kw), texts, qv)
            if edit:
                keep.append(edit(sp))
            arr = (_lib.Sort * B)(*[_lib.Sort(None, 0) if s is None else _lib.Sort(s[0], s[1]) for s in sorts])
            pins = None
            if promote is not None:
                off, doc, pos = promote
                pins = _lib.Pins(_p(off), _p(doc), _p(pos), 1)
            lim = kw.get("limit_hint", 10)
            d = np.full((B, lim), 7, np.uint64); s = np.full((B, lim), 7, np.float32); v = np.full((B, lim), 7, np.float64)
            n = np.full(B, 7, np.uint32); cnt = np.full(B, 7, np.uint64); ps = np.full(8, 7, np.float32); pp = np.full(8, 7, np.uint8)
            rc = L.oc_search_q_sorted(c["ctx"]._h, c["emb"]._h, c["strs"]._h, C.byref(sp), None if q_sorts_null else arr,
                                      None if pins is None else C.byref(pins), _p(d), _p(s), _p(v), _p(n), _p(cnt), _p(ps), _p(pp))
            for a in (d, s, v, n, cnt, ps, pp):
                assert (a == 7).all()   # nothing written
            return rc

        good = [(fields["price"]._h, 0), None, (fields["date"]._h, 1), None]
        items = (np.asarray([0, 1, 1, 2, 2], np.uint32), np.asarray([5, 6], np.uint64), np.asarray([0, 1], np.uint32))
        assert run(good, q_sorts_null=True) == OC_ERR_INVALID
        assert run([(fields["price"]._h, 2), None, None, None]) == OC_ERR_INVALID
        assert run([(foreign_sort._h, 0), None, None, None]) == OC_ERR_INVALID
        assert run(good, fl=(c["fs"]["share"], foreign, None, None)) == OC_ERR_INVALID
        assert run(good, edit=lambda sp: setattr(sp, "filter", c["fs"]["all"]._h)) == OC_ERR_INVALID
        bits = np.zeros((N + 63) // 64, np.uint64)

        def with_bits(sp):
            sp.filter_bits, sp.filter_nbits = _p(bits), N
        assert run(good, edit=with_bits) == OC_ERR_INVALID
        bad_off = (np.asarray([0, 2, 1, 2, 2], np.uint32), items[1], items[2])
        assert run(good, promote=bad_off) == OC_ERR_INVALID
        assert run(good, edit=lambda sp: setattr(sp, "sharded", 1)) == OC_ERR_UNSUPPORTED
        assert run(good, limit_hint=1000, offset=100) == OC_ERR_UNSUPPORTED            # limit + offset > OC_MAX_TOPK
        assert run(good, promote=items, limit_hint=500, offset=100) == OC_ERR_UNSUPPORTED   # active: 2 x (limit + offset)
        # the batcher refuses before joining: a foreign sort field, a bad order, malformed pins
        bat = ob.SearchBatcher(tsc, max_batch=8, max_wait_us=100)
        try:
            sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0), [texts[0]], qv[0:1])
            d = np.full(10, 7, np.uint64); s = np.full(10, 7, np.float32); v = np.full(10, 7, np.float64)
            n = np.full(1, 7, np.uint32); cnt = np.full(1, 7, np.uint64)
            for srt, pins in ((_lib.Sort(foreign_sort._h, 0), None), (_lib.Sort(fields["price"]._h, 5), None),
                              (None, _lib.Pins(_p(np.asarray([1, 0], np.uint32)), None, None, 1))):
                rc = L.oc_batcher_search_sorted(bat._h, C.byref(sp), None if srt is None else C.byref(srt),
                                                None if pins is None else C.byref(pins), _p(d), _p(s), _p(v), _p(n), _p(cnt), None, None)
                assert rc == OC_ERR_INVALID
                assert (d == 7).all() and (v == 7).all() and (n == 7).all() and (cnt == 7).all()
            assert bat.stats() == {"queries": 0, "batches": 0, "direct": 0}
            # out_sort_values may be NULL, as for oc_search_sorted
            srt = _lib.Sort(fields["price"]._h, 0)
            assert L.oc_batcher_search_sorted(bat._h, C.byref(sp), C.byref(srt), None, _p(d), _p(s), None, _p(n), _p(cnt),
                                              None, None) == 0
            ref = ob.search_sorted_arrays(tsc, ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0), fields["price"], "ASC",
                                          None, [texts[0]], qv[0:1])
            assert d.tobytes() == ref[0][0].tobytes() and n[0] == ref[3][0] and cnt[0] == ref[4][0]
        finally:
            bat.close()
    finally:
        foreign_sort.close()
        foreign.close()
        other.close()


def test_batcher_coalesces_sorted_and_pinned_requests(corpus, fields):  # noqa: F811
    c = corpus
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    T, Q = 12, 24
    qv, texts = _inputs(T * Q, 2300, c["rows"])
    filters = _assign(c["fs"], T * Q, 41)
    sorts = _sorts(fields, T * Q, 43)
    promote = _promote(T * Q, 47)
    plain = [i % 5 == 4 for i in range(T * Q)]   # every fifth request goes through search()
    expect = {}
    for i in range(T * Q):
        p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i])
        if plain[i]:
            expect[i] = tsc.execute_batch_arrays(p, [texts[i]], qv[i:i + 1])
        else:
            expect[i] = _alone(tsc, MODE_HYBRID, filters[i], sorts[i], promote[i], [texts[i]], qv[i:i + 1], similarity=0.0)
    bat = ob.SearchBatcher(tsc, max_batch=64, max_wait_us=3000)
    bad = []

    def worker(t):
        for i in range(t, T * Q, T):
            p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i])
            e = expect[i]
            if plain[i]:
                h = bat.search(p, texts[i], qv[i])
                k = int(e[2][0])
                ok = h.count == int(e[3][0]) and h.doc_ids.tobytes() == e[0][0, :k].tobytes() and h.scores.tobytes() == e[1][0, :k].tobytes()
            else:
                h, sv, ps, pp = bat.search_sorted(p, sorts[i], promote[i] if promote[i] else None, texts[i], qv[i])
                k = int(e[3][0])
                ok = (h.count == int(e[4][0]) and h.doc_ids.tobytes() == e[0][0, :k].tobytes()
                      and h.scores.tobytes() == e[1][0, :k].tobytes() and sv.tobytes() == e[2][0, :k].tobytes()
                      and ps.tobytes() == e[5].tobytes() and pp.tobytes() == e[6].tobytes())
            if not ok:
                bad.append(i)
    th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    st = bat.stats()
    bat.close()
    assert not bad, bad[:10]
    assert st["direct"] == 0 and st["queries"] == T * Q and st["batches"] < st["queries"], st
