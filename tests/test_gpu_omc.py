"""The OMC store on the device (oc_omc_*, OmcStore): commits against omc_spec.py byte for byte, and every search entry
point with p->omc = the store against the same call with the store's published version as omc_doc_ids / omc_mult,
byte for byte: ids, score bits, n, count, sort values, pin outputs, group rows and facet counts.  Covered: fulltext,
vector and hybrid on fp32 and bf16 stores, the scorer routes of the OC_BM25_* switches with plain, threshold and
multi-term queries, q_params / q_filters / q_where, pinned, sorted, grouped and faceted calls, tombstones, identity and
sparse document ids, an oc_str_commit and an oc_omc_commit_ex between searches (the row list is rebuilt), the oracle's
score maps with orc.apply_omc, a commit racing a thread of searches, both batchers, and the sharded search over 2 and
4 contexts of one GPU."""
import threading

import numpy as np
import pytest

import omc_spec as spec
import oramacore_b200 as ob
from oramacore_b200 import PromoteItem, synth
from oramacore_b200.engine import (FacetStore, GroupBy, OmcStore, QueryParams, SearchBatcher, SortField, TokenScoreContext,
                                   TokenScoreParams, search_facets, search_groups_arrays, search_pinned_arrays,
                                   search_q_facets_arrays, search_q_sorted_arrays, search_sorted_arrays)
from oramacore_b200.sharding import shard_range, shard_string_index
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, TextQuery
from oramacore_b200.where import compile_where, parse_where
from test_gpu_tile3 import _env
from test_gpu_topn_paths import SCORERS, _kind, _sorted, page

pytestmark = pytest.mark.gpu

MODES = {"fulltext": MODE_FULLTEXT, "vector": MODE_VECTOR, "hybrid": MODE_HYBRID}


def _same(a, b, ctx=""):
    """Two results (arrays, tuples / lists of them, dicts, SearchHits) equal byte for byte."""
    if isinstance(a, (tuple, list)):
        assert len(a) == len(b), ctx
        for x, y in zip(a, b):
            _same(x, y, ctx)
    elif isinstance(a, dict):
        assert a == b, ctx
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), (ctx, a.ravel()[:8], b.ravel()[:8])
    elif hasattr(a, "doc_ids"):
        _same((a.doc_ids, a.scores, np.asarray(a.count)), (b.doc_ids, b.scores, np.asarray(b.count)), ctx)
    else:
        assert a == b, (ctx, a, b)


def _arrays_of(store):
    d, m, _ = store.read()
    return dict(omc_doc_ids=d, omc_mult=m) if d.shape[0] else {}


def _both(store, call, ctx=""):
    """call(kw) with the store and with its read-back arrays: equal byte for byte.  Returns the store's result."""
    got = call(dict(omc_store=store))
    _same(got, call(_arrays_of(store)), ctx)
    return got


# ------------------------------------------------------------------ 1. the commit against the spec
def _check_read(store, want_doc, want_mult, version):
    d, m, v = store.read()
    assert v == version
    assert np.array_equal(d, want_doc) and m.tobytes() == want_mult.tobytes()


def test_commit_against_spec(gpu_ctx):
    st = OmcStore(gpu_ctx)
    try:
        doc, mult = spec.as_arrays({})
        _check_read(st, doc, mult, 0)                      # an empty store
        assert st.commit()["version"] == 1                 # a commit with no op
        _check_read(st, doc, mult, 1)
        rng = np.random.default_rng(7)
        ver = 1
        for rnd in range(24):
            n_docs = int(rng.choice([4, 60, 5000, 1 << 40]))
            ops = spec.random_ops(rng, int(rng.integers(0, 3000)), n_docs) if rnd % 6 != 5 else []
            # queue in several calls, sets and deletes interleaved as the ops come
            i = 0
            while i < len(ops):
                j = i
                while j < len(ops) and ops[j][0] == ops[i][0] and j - i < 97:
                    j += 1
                if ops[i][0] == "set":
                    st.set([o[1] for o in ops[i:j]], [o[2] for o in ops[i:j]])
                else:
                    st.delete([o[1] for o in ops[i:j]])
                i = j
            n_before = doc.shape[0]
            s = st.commit()
            ver += 1
            doc, mult = spec.commit(doc, mult, ops)
            _check_read(st, doc, mult, ver)
            assert s["version"] == ver
            assert s["rows_kept"] + s["rows_dropped"] == n_before and s["rows_kept"] + s["rows_added"] == doc.shape[0]
    finally:
        st.close()


def test_commit_one_million(gpu_ctx):
    rng = np.random.default_rng(11)
    st = OmcStore(gpu_ctx)
    try:
        d0 = rng.choice(4_000_000, size=1_000_000, replace=False).astype(np.uint64)
        m0 = rng.random(d0.shape[0]).astype(np.float32) * 4
        st.set(d0, m0)
        st.commit()
        doc, mult = spec.as_arrays(spec.replay([("set", int(a), float(b)) for a, b in zip(d0, m0)]))
        _check_read(st, doc, mult, 1)
        ops = [("set", int(x), float(np.float32(y))) for x, y in zip(rng.integers(0, 4_000_000, 300), rng.random(300))]
        ops += [("delete", int(x)) for x in rng.choice(doc, 30)]
        st.set([o[1] for o in ops[:300]], [o[2] for o in ops[:300]])
        st.delete([o[1] for o in ops[300:]])
        st.commit()
        doc, mult = spec.commit(doc, mult, ops)
        _check_read(st, doc, mult, 2)
    finally:
        st.close()


def test_store_refusals(gpu_ctx):
    st = OmcStore(gpu_ctx)
    other = ob.Context(0)
    st2 = OmcStore(other)
    try:
        st.set([1, 2], [2.0, 3.0])
        for bad in (np.nan, np.inf, -np.inf):
            with pytest.raises(ob.OcError) as e:
                st.set([5, 6], [1.0, bad])
            assert e.value.code == -1
        st.commit()
        d, m, v = st.read()
        assert d.tolist() == [1, 2] and m.tolist() == [2.0, 3.0] and v == 1
        st.set([3], [-1.5])                                # any finite value, zero and negatives included
        st.set([4], [0.0])
        st.commit()
        assert st.read()[0].tolist() == [1, 2, 3, 4]
        h = ob.StringFieldStorage(gpu_ctx, synth.make_text_corpus(500, 50, seed=1))
        tsc = TokenScoreContext(gpu_ctx, None, h)
        texts = synth.make_text_queries(50, 2, seed=2)
        with pytest.raises(ob.OcError) as e:               # the store together with arrays
            tsc.execute_batch_arrays(TokenScoreParams(mode=MODE_FULLTEXT, omc_store=st, omc_doc_ids=np.asarray([1], np.uint64),
                                                      omc_mult=np.asarray([2.0], np.float32)), texts)
        assert e.value.code == -1
        with pytest.raises(ob.OcError) as e:               # a store of another ctx
            tsc.execute_batch_arrays(TokenScoreParams(mode=MODE_FULLTEXT, omc_store=st2), texts)
        assert e.value.code == -1
        h.close()
    finally:
        st.close(); st2.close(); other.close()


# ------------------------------------------------------------------ 2. searches: store == arrays
N, DIM, VOCAB, B = 30000, 384, 2500, 8


@pytest.fixture(scope="module", params=[("identity", "f32"), ("sparse", "bf16")], ids=["identity_f32", "sparse_bf16"])
def corpus(request, gpu_ctx):
    sparse = request.param[0] == "sparse"
    rng = np.random.default_rng(41)
    rows = synth.make_vectors(N, DIM, seed=42)
    qv, _ = synth.make_vector_queries(rows, B, seed=43)
    data = synth.make_text_corpus(N, VOCAB, seed=44)
    texts = synth.make_text_queries(VOCAB, B - 2, seed=45)
    texts += [TextQuery.single_terms([0, 1, 2]),
              TextQuery.from_tokens([[(0, 3, 1.0), (0, 4, 2.0), (0, 9, 0.5)], [(0, 5, 1.0)]])]   # multi-term token
    ids = (np.arange(N, dtype=np.uint64) * 3 + 2) if sparse else np.arange(N, dtype=np.uint64)
    if sparse:
        data.row_doc_ids = ids
    nbits = int(ids.max()) + 1
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dtype=request.param[1])
    emb.insert_batch(ids, rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    gone = [5, 77, 4000, 12345]
    for d in ids[gone].tolist():
        strs.delete(d); emb.delete(d)
    deleted = np.zeros(N, np.uint8); deleted[gone] = 1
    cat = rng.integers(0, 5, size=N)
    fs = FacetStore(gpu_ctx, nbits)
    fs.add_string_field("cat", {f"c{k}": ids[cat == k] for k in range(5)})
    fs.add_number_field("price", ids, rng.integers(0, 50, size=N).astype(np.float64))
    store = OmcStore(gpu_ctx)
    od = rng.choice(ids, size=N // 3, replace=False)
    od = np.concatenate([od, np.asarray([nbits + 5, nbits + 900], np.uint64)])   # documents without a row
    store.set(od, rng.choice([0.0, 0.5, 2.0, 3.0, 1.25, -1.0], size=od.shape[0]).astype(np.float32))
    store.commit()
    c = dict(ids=ids, nbits=nbits, rows=rows, qv=qv, data=data, texts=texts, emb=emb, strs=strs, fs=fs, store=store,
             deleted=deleted, cat=cat, rng=rng, gone=ids[gone], dtype=request.param[1])
    yield c
    store.close(); fs.close(); emb.close(); strs.close()


def _tsc(c, mode):
    return TokenScoreContext(c["strs"].ctx, c["emb"] if mode != MODE_FULLTEXT else None, c["strs"] if mode != MODE_VECTOR else None)


def _inputs(c, mode):
    return (c["texts"] if mode != MODE_VECTOR else None), (c["qv"] if mode != MODE_FULLTEXT else None)


@pytest.mark.parametrize("mode", ["fulltext", "vector", "hybrid"])
def test_plain_threshold_pages(corpus, mode):
    c, m = corpus, MODES[mode]
    tsc = _tsc(c, m)
    texts, qv = _inputs(c, m)
    for thr in (None, 0.5, 1.0):
        for limit, offset in [(10, 0), (3, 5), (100, 412)]:
            for sim in (0.0, -2.0):
                p = lambda kw: TokenScoreParams(mode=m, limit_hint=limit, offset=offset, similarity=sim, threshold=thr, **kw)  # noqa: E731
                _both(c["store"], lambda kw: tsc.execute_batch_arrays(p(kw), texts, qv), (mode, thr, limit, offset, sim))


@pytest.mark.parametrize("route", list(SCORERS))
def test_scorer_routes(corpus, route):
    c = corpus
    tsc = _tsc(c, MODE_HYBRID)
    for mode in (MODE_FULLTEXT, MODE_HYBRID):
        with _env(**SCORERS[route]):
            for thr in (None, 0.5):
                p = lambda kw: TokenScoreParams(mode=mode, limit_hint=10, similarity=0.0, threshold=thr, **kw)  # noqa: E731
                _both(c["store"], lambda kw: tsc.execute_batch_arrays(p(kw), c["texts"], c["qv"]), (route, mode, thr))


def test_oracle_pages(corpus, orc):
    """The fulltext pages with the store equal the oracle's score maps with orc.apply_omc, exactly."""
    c = corpus
    tsc = _tsc(c, MODE_FULLTEXT)
    d, mult, _ = c["store"].read()
    alive = np.flatnonzero(c["deleted"] == 0)
    fb = orc.make_filter_bits(c["ids"][alive].tolist(), c["nbits"])
    ix = orc.StrIndex(c["data"])
    for limit, offset in [(10, 0), (7, 30)]:
        docs, scores, n, cnt = tsc.execute_batch_arrays(TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=limit, offset=offset,
                                                                         omc_store=c["store"]), c["texts"])
        for q in range(B):
            ref = _sorted(*orc.apply_omc(orc.fulltext(ix, c["texts"][q], filter_bits=fb, filter_nbits=c["nbits"]), d, mult))
            ed, es, ecnt = page(ref, limit, offset)
            assert int(cnt[q]) == ecnt and int(n[q]) == ed.shape[0]
            assert np.array_equal(docs[q, :n[q]], ed) and scores[q, :n[q]].tobytes() == es.tobytes(), (q, limit, offset)


def test_per_query_inputs(corpus):
    """q_params (mixed modes), q_filters and q_where."""
    c = corpus
    tsc = _tsc(c, MODE_HYBRID)
    qps = [QueryParams(mode=[MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID][b % 3], limit=[10, 4, 25][b % 3], offset=b,
                       similarity=0.0, threshold=0.5 if b == 4 else None) for b in range(B)]
    _both(c["store"], lambda kw: tsc.execute_batch_arrays(TokenScoreParams(mode=MODE_HYBRID, query_params=qps, **kw),
                                                          c["texts"], c["qv"]), "q_params")
    flts = [ob.DeviceFilter.from_ids(c["strs"].ctx, c["ids"][c["cat"] == k], c["nbits"]) for k in range(3)]
    try:
        dfl = [flts[b % 3] if b % 4 else None for b in range(B)]
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            _both(c["store"], lambda kw: tsc.execute_batch_arrays(TokenScoreParams(mode=mode, similarity=0.0, device_filters=dfl,
                                                                                   **kw), c["texts"], c["qv"]), ("q_filters", mode))
        progs = [compile_where(parse_where({"cat": f"c{b % 5}"}), c["fs"], {}, c["nbits"]) if b % 3 else None for b in range(B)]
        _both(c["store"], lambda kw: tsc.execute_batch_arrays(TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, where_programs=progs,
                                                                               **kw), c["texts"], c["qv"]), "q_where")
        _both(c["store"], lambda kw: tsc.execute_batch_arrays(TokenScoreParams(mode=MODE_HYBRID, query_params=qps, device_filters=dfl,
                                                                               **kw), c["texts"], c["qv"]), "q_params + q_filters")
    finally:
        for f in flts:
            f.close()


@pytest.mark.parametrize("mode", ["fulltext", "vector", "hybrid"])
def test_pinned_sorted_grouped_faceted(corpus, mode):
    c, m = corpus, MODES[mode]
    tsc = _tsc(c, m)
    texts, qv = _inputs(c, m)
    ids = c["ids"]
    promote = [[PromoteItem(int(ids[(7 * b + 1) % N]), b % 4), PromoteItem(int(c["gone"][0]), 2)] if b % 3 else [] for b in range(B)]
    st = c["store"]
    p = lambda kw, **x: TokenScoreParams(mode=m, limit_hint=x.get("limit", 10), similarity=0.0, **kw)  # noqa: E731
    _both(st, lambda kw: search_pinned_arrays(tsc, p(kw), promote, texts=texts, q_vecs=qv), "pinned")
    sf = SortField.from_facets(c["fs"], "price")
    gb = GroupBy(c["fs"], ["cat"])
    try:
        for order in ("ASC", "DESC"):
            _both(st, lambda kw: search_sorted_arrays(tsc, p(kw), sf, order, promote=promote, texts=texts, q_vecs=qv), ("sorted", order))
        sorts = [(sf, "DESC") if b % 2 else None for b in range(B)]
        _both(st, lambda kw: search_q_sorted_arrays(tsc, p(kw), sorts, promote=promote, texts=texts, q_vecs=qv), "q_sorted")
        _both(st, lambda kw: search_groups_arrays(tsc, gb, p(kw), max_results=3, texts=texts, q_vecs=qv), "groups")
        _both(st, lambda kw: search_groups_arrays(tsc, gb, p(kw), max_results=2, texts=texts, q_vecs=qv, promote=promote), "groups pinned")
        _both(st, lambda kw: search_groups_arrays(tsc, gb, p(kw), max_results=2, texts=texts, q_vecs=qv, sort_by=(sf, "ASC")), "groups sorted")
        facets = {"cat": {}, "price": {"ranges": [{"from": 0, "to": 20}, {"from": 10, "to": 49}]}}
        _both(st, lambda kw: search_facets(tsc, c["fs"], p(kw), facets, texts=texts, q_vecs=qv), "facets")
        qf = [facets if b % 2 else None for b in range(B)]
        qg = [(gb, 2) if b % 3 else None for b in range(B)]
        _both(st, lambda kw: search_q_facets_arrays(tsc, c["fs"], p(kw), qf, groups=qg, promote=promote, texts=texts, q_vecs=qv)[:-1],
              "q_facets")
    finally:
        gb.close(); sf.close()


def test_row_list_rebuilt(gpu_ctx):
    """An oc_str_commit and an oc_omc_commit_ex between searches: the store's row list follows both."""
    data = synth.make_text_corpus(6000, 300, seed=51)
    data.row_doc_ids = np.arange(6000, dtype=np.uint64) * 2
    strs = ob.StringFieldStorage(gpu_ctx, data)
    emb_rows = synth.make_vectors(6000, 64, seed=52)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "x", dim=64)
    emb.insert_batch(data.row_doc_ids, emb_rows)
    store = OmcStore(gpu_ctx)
    texts = synth.make_text_queries(300, 6, seed=53)
    qv, _ = synth.make_vector_queries(emb_rows, 6, seed=54)
    tsc = TokenScoreContext(gpu_ctx, emb, strs)
    rng = np.random.default_rng(55)
    try:
        def check(ctx):
            for mode in (MODE_FULLTEXT, MODE_HYBRID):
                _both(store, lambda kw: tsc.execute_batch_arrays(TokenScoreParams(mode=mode, limit_hint=20, similarity=-2.0, **kw),
                                                                 texts, qv), (ctx, mode))
        check("empty store")
        store.set(rng.choice(14000, 3000, replace=False), rng.choice([2.0, 0.5, 3.0], 3000))
        store.commit()
        check("first version")
        for k in range(3):
            for j in range(200):   # new documents, odd ids between the committed even ones, and beyond them
                d = int(rng.integers(0, 14000)) | 1
                strs.insert(d, 0, int(rng.integers(1, 30)), {int(t): 1 for t in rng.choice(300, 4, replace=False)})
            strs.delete(int(data.row_doc_ids[k * 7]))
            strs.commit()
            check(("str commit", k))
            store.set(rng.choice(14000, 100, replace=False), rng.choice([4.0, 0.25], 100))
            store.delete(rng.choice(14000, 50, replace=False))
            store.commit()
            check(("omc commit", k))
    finally:
        store.close(); emb.close(); strs.close()


# ------------------------------------------------------------------ 3. a commit racing searches
def test_commit_racing_searches(corpus):
    c = corpus
    tsc = _tsc(c, MODE_HYBRID)
    rng = np.random.default_rng(61)
    st = OmcStore(c["strs"].ctx)
    try:
        versions = []
        st.set(c["ids"][:5000], np.full(5000, 2.0, np.float32))
        st.commit()
        versions.append(_arrays_of(st))
        p = lambda kw: TokenScoreParams(mode=MODE_HYBRID, limit_hint=10, similarity=0.0, **kw)  # noqa: E731
        got, stop = [], threading.Event()

        def searcher():
            while not stop.is_set():
                got.append(tsc.execute_batch_arrays(p(dict(omc_store=st)), c["texts"], c["qv"]))
        th = threading.Thread(target=searcher)
        th.start()
        try:
            for _ in range(6):
                st.set(rng.choice(c["ids"], 4000, replace=False), rng.choice([0.5, 3.0, 5.0], 4000))
                st.delete(rng.choice(c["ids"], 500, replace=False))
                st.commit()
                versions.append(_arrays_of(st))
        finally:
            stop.set()
            th.join()
        expect = [tsc.execute_batch_arrays(p(v), c["texts"], c["qv"]) for v in versions]
        assert got
        for r in got:
            assert any(all(x.tobytes() == y.tobytes() for x, y in zip(r, e)) for e in expect)
    finally:
        st.close()


# ------------------------------------------------------------------ 4. the batchers
@pytest.mark.parametrize("mixed", [False, True], ids=["default", "mixed"])
def test_batcher(corpus, mixed):
    c = corpus
    tsc = _tsc(c, MODE_HYBRID)
    rng = np.random.default_rng(71)
    other = OmcStore(c["strs"].ctx)
    other.set(c["ids"][::2], np.full(N // 2, 3.0, np.float32))
    other.commit()
    bat = SearchBatcher(tsc, max_batch=64, max_wait_us=20000, mixed=mixed)
    try:
        jobs = []
        for i in range(48):
            mode = [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR][i % 3] if mixed else MODE_HYBRID
            st = c["store"] if i % 4 else other
            jobs.append((TokenScoreParams(mode=mode, limit_hint=10 if not mixed else 5 + i % 7, similarity=0.0, omc_store=st),
                         c["texts"][i % B], c["qv"][i % B]))
        out = [None] * len(jobs)

        def run(i):
            p, t, v = jobs[i]
            out[i] = bat.search(p, text=t if p.mode != MODE_VECTOR else None, q_vec=v if p.mode != MODE_FULLTEXT else None)
        th = [threading.Thread(target=run, args=(i,)) for i in range(len(jobs))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        s = bat.stats()
        assert s["queries"] == len(jobs) and s["direct"] == 0
        assert 2 <= s["batches"] < len(jobs)   # two handles: never one batch; same-handle requests share batches
        for i, (p, t, v) in enumerate(jobs):
            alone = tsc.execute_batch(p, None if p.mode == MODE_VECTOR else [t], None if p.mode == MODE_FULLTEXT else v[None])[0]
            _same(out[i], alone, i)
    finally:
        bat.close(); other.close()


# ------------------------------------------------------------------ 5. sharded over contexts of one GPU
@pytest.mark.parametrize("W", [2, 4])
def test_sharded_local(gpu_ctx, W):
    """Each rank holds the whole map in its own store (the caller contract); rank results equal the unsharded search
    with the same map, byte for byte."""
    from test_gpu_topn_paths import N_ZIPF, V_ZIPF
    data = synth.make_text_corpus(N_ZIPF, V_ZIPF, seed=4242)
    texts, skw, _, _ = _kind("omc")
    ctxs = [ob.Context(0) for _ in range(W)]
    handles = []
    try:
        ob.Context.comm_init_local(ctxs)
        docs = np.arange(data.n_rows, dtype=np.uint64)
        emb_rows = synth.make_vectors(data.n_rows, 64, seed=81)
        qv, _ = synth.make_vector_queries(emb_rows, len(texts), seed=82)
        ranks = []
        for r, ctx in enumerate(ctxs):
            lo, hi = shard_range(data.n_rows, r, W)
            sd, gdf = shard_string_index(data, lo, hi)
            s = ob.StringFieldStorage(ctx, sd, global_df=gdf)
            e = ob.EmbeddingFieldStorage(ctx, "x", dim=64)
            e.insert_batch(docs[lo:hi], emb_rows[lo:hi])
            o = OmcStore(ctx)
            o.set(skw["omc_doc_ids"], skw["omc_mult"])
            o.commit()
            handles += [s, e, o]
            ranks.append((TokenScoreContext(ctx, e, s), o))
        s1 = ob.StringFieldStorage(gpu_ctx, data)
        e1 = ob.EmbeddingFieldStorage(gpu_ctx, "x", dim=64)
        e1.insert_batch(docs, emb_rows)
        o1 = OmcStore(gpu_ctx)
        o1.set(skw["omc_doc_ids"], skw["omc_mult"])
        o1.commit()
        handles += [s1, e1, o1]
        single = TokenScoreContext(gpu_ctx, e1, s1)
        for mode, sim in (("fulltext", 0.0), ("hybrid", 0.0), ("hybrid", -2.0), ("vector", 0.0)):
            m = MODES[mode]
            for limit, offset in [(10, 0), (7, 23)]:
                out, errs = [None] * W, [None] * W

                def go(r):
                    try:
                        t, o = ranks[r]
                        out[r] = t.execute_batch_arrays(TokenScoreParams(mode=m, limit_hint=limit, offset=offset, similarity=sim,
                                                                         sharded=True, omc_store=o), texts, qv)
                    except ob.OcError as ex:
                        errs[r] = ex
                th = [threading.Thread(target=go, args=(r,)) for r in range(W)]
                for t in th:
                    t.start()
                for t in th:
                    t.join()
                assert errs == [None] * W, errs
                ctx_ = (W, mode, sim, limit, offset)
                for r in range(1, W):
                    _same(out[r], out[0], ctx_)
                _both(o1, lambda kw: single.execute_batch_arrays(TokenScoreParams(mode=m, limit_hint=limit, offset=offset,
                                                                                  similarity=sim, **kw), texts, qv), ctx_)
                _same(out[0], single.execute_batch_arrays(TokenScoreParams(mode=m, limit_hint=limit, offset=offset, similarity=sim,
                                                                           omc_store=o1), texts, qv), ctx_)
    finally:
        for h in handles:
            h.close()
        for c in ctxs:
            c.close()
