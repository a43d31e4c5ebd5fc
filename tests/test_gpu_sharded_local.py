"""The document-sharded search on one GPU: W contexts on device 0 joined by the in-process transport
(Context.comm_init_local), each holding one shard, run the real pack / exchange / merge kernels (shard.cuh), the df
all-reduce and the lock-step re-runs, one thread per rank.  Every search asserts:
  (a) every rank's result is byte-identical to rank 0's (doc ids, score bits, hit counts, match counts);
  (b) rank 0's result is byte-identical to the unsharded search of the whole corpus on one context;
  (c) it equals the oracle's page of the whole score map, sorted by (-score, doc id) (ref_map / page of
      test_gpu_topn_paths): exactly for fulltext and signed-unit-axis embeddings, within 1e-5 for random embeddings.
Shards are doc-id ranges (every row of a document on one shard, DESIGN.md §6); the unsharded store holds the embedding
rows in shard order, so both sides see the same global rows."""
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import _lib, synth
from oramacore_b200.engine import (FacetStore, GroupBy, QueryParams, SortField, TokenScoreContext, TokenScoreParams,
                                   from_bf16, search_facets, search_groups_arrays, search_pinned_arrays,
                                   search_sorted_arrays, to_bf16)
from oramacore_b200.sharding import shard_range, shard_string_index
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, TextQuery
from oramacore_b200.where import WhereProgram
from test_gpu_topn_paths import DIM, KINDS, N_ZIPF, V_ZIPF, _kind, _sorted, axis_query, axis_rows, page, postings

gpu = pytest.mark.gpu
MODES = {"fulltext": MODE_FULLTEXT, "vector": MODE_VECTOR, "hybrid": MODE_HYBRID}
WORLDS = (2, 3, 4, 8, 16)
PAGES = [(1, 0), (10, 0), (10, 23), (100, 0), (7, 500)]
N_VEC, V_VEC, B_VEC = 20011, 2000, 12   # the corpus with random embeddings: 20011 rows, divisible by no world size
OC_ERR_INVALID, OC_ERR_UNSUPPORTED = -1, -4   # include/oramacore_b200.h


@pytest.fixture(scope="module")
def pool():
    """16 contexts on device 0; a test joins the first W of them into one group."""
    ctxs = [ob.Context(0) for _ in range(16)]
    yield ctxs
    for c in ctxs:
        c.close()


@pytest.fixture(scope="module")
def zipf():
    return synth.make_text_corpus(N_ZIPF, V_ZIPF, seed=4242)


def _join(pool, W):
    ctxs = pool[:W]
    ob.Context.comm_init_local(ctxs)
    return ctxs


class Sharded:
    """One corpus split over the ranks of a group, the same corpus unsharded on `single`, and the oracle's view of it.
    data: the string rows (ascending doc ids); emb_docs / emb_rows: the embedding rows (any order, several per doc).
    bounds: each rank's string-row range (default shard_range); cuts: each rank's doc-id range (default: from bounds,
    or from the embedded doc ids when there is no string data)."""

    def __init__(self, ctxs, single, orc, data=None, emb_docs=None, emb_rows=None, bounds=None, cuts=None,
                 model="BGESmall", dim=None, dtype="f32", global_df=True):
        W = len(ctxs)
        self.ctxs, self.W, self.single, self.orc = ctxs, W, single, orc
        if cuts is None:
            if data is not None:
                docs = np.arange(data.n_rows, dtype=np.uint64) if data.row_doc_ids is None else data.row_doc_ids
                bounds = bounds or [shard_range(data.n_rows, r, W) for r in range(W)]
                cuts = [0] + [int(docs[lo]) if lo < data.n_rows else 2 ** 63 for lo, _ in bounds[1:]] + [2 ** 64 - 1]
            else:
                u = np.unique(emb_docs)
                cuts = [0] + [int(u[shard_range(len(u), r, W)[0]]) for r in range(1, W)] + [2 ** 64 - 1]
        cuts = np.asarray(cuts, np.uint64)
        self.ix = self.st = None
        self.strs, self.embs, self.strs1, self.emb1 = [None] * W, [None] * W, None, None
        if data is not None:
            docs = np.arange(data.n_rows, dtype=np.uint64) if data.row_doc_ids is None else data.row_doc_ids
            for r, ctx in enumerate(ctxs):
                lo, hi = np.searchsorted(docs, cuts[r]), np.searchsorted(docs, cuts[r + 1])
                sd, gdf = shard_string_index(data, int(lo), int(hi))
                self.strs[r] = ob.StringFieldStorage(ctx, sd, global_df=gdf if global_df else None)
                if not global_df:
                    self.strs[r].set_global(data.document_count, [f.avg_field_len for f in data.fields])
            self.strs1 = ob.StringFieldStorage(single, data)
            self.ix = orc.StrIndex(data)
        if emb_docs is not None:
            emb_docs = np.asarray(emb_docs, np.uint64)
            rank_of = np.searchsorted(cuts, emb_docs, side="right") - 1
            o = np.argsort(rank_of, kind="stable")   # the global row order of the sharded store: shard by shard
            emb_docs, emb_rows, rank_of = emb_docs[o], np.asarray(emb_rows, np.float32)[o], rank_of[o]
            kw = dict(dim=dim, dtype=dtype)
            for r, ctx in enumerate(ctxs):
                self.embs[r] = ob.EmbeddingFieldStorage(ctx, model, **kw)
                if (rank_of == r).any():
                    self.embs[r].insert_batch(emb_docs[rank_of == r], emb_rows[rank_of == r])
            self.emb1 = ob.EmbeddingFieldStorage(single, model, **kw)
            self.emb1.insert_batch(emb_docs, emb_rows)
            rows = from_bf16(to_bf16(emb_rows)) if dtype == "bf16" else emb_rows
            self.st = orc.EmbStore(rows, row_doc_ids=emb_docs, is_e5=model.startswith("MultilingualE5"))
        self.n_rows = [0 if s is None else s.info()["total_documents"] for s in self.strs]

    def close(self):
        for h in self.strs + self.embs + [self.strs1, self.emb1]:
            if h is not None:
                h.close()

    def _tscs(self, mode):
        ft, v = mode != MODE_VECTOR, mode != MODE_FULLTEXT
        return [TokenScoreContext(c, self.embs[r] if v else None, self.strs[r] if ft else None) for r, c in enumerate(self.ctxs)]

    def on_ranks(self, fn):
        """fn(rank) on one thread per rank; returns the results, or the OcError of every rank that raised"""
        out, errs = [None] * self.W, [None] * self.W

        def go(r):
            try:
                out[r] = fn(r)
            except ob.OcError as e:
                errs[r] = e
        th = [threading.Thread(target=go, args=(r,)) for r in range(self.W)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        return out, errs

    def sharded(self, mode, texts=None, qv=None, **kw):
        m = MODES[mode]
        tscs = self._tscs(m)
        out, errs = self.on_ranks(lambda r: (tscs[r].execute_batch_arrays(TokenScoreParams(mode=m, sharded=True, **kw),
                                                                           texts, qv), self.ctxs[r].last_timing()))
        assert errs == [None] * self.W, errs
        return [o[0] for o in out], [o[1] for o in out]

    def unsharded(self, mode, texts=None, qv=None, **kw):
        m = MODES[mode]
        tsc = TokenScoreContext(self.single, self.emb1 if m != MODE_FULLTEXT else None, self.strs1 if m != MODE_VECTOR else None)
        return tsc.execute_batch_arrays(TokenScoreParams(mode=m, **kw), texts, qv)

    def ref(self, mode, text, qv, limit, similarity=0.0, threshold=None, omc_doc_ids=None, omc_mult=None,
            filtered_doc_ids=None, filter_nbits=0):
        """The oracle's whole score map of one query, sorted (the vector stage's depth is `limit`)."""
        orc, fb, nb = self.orc, filtered_doc_ids, filter_nbits
        if mode == "vector":
            m = orc.vector(self.st, qv, limit, similarity, fb, nb)
        else:
            m = orc.fulltext(self.ix, text, threshold=threshold, filter_bits=fb, filter_nbits=nb)
            if mode == "hybrid":
                m = orc.hybrid_combine(orc.vector(self.st, qv, limit, similarity, fb, nb), m)
        if omc_doc_ids is not None:
            m = orc.apply_omc(m, omc_doc_ids, omc_mult)
        return _sorted(*m)

    def check(self, mode, texts=None, qv=None, oracle="exact", refs=None, ctx="", **kw):
        """(a), (b) and — oracle = "exact" | "near" | None — (c).  refs: the sorted maps, when the caller has them.
        Returns the ranks' timings."""
        res, tim = self.sharded(mode, texts, qv, **kw)
        d0, s0, n0, c0 = res[0]
        for r in range(1, self.W):   # (a)
            d, s, n, c = res[r]
            assert np.array_equal(n, n0) and np.array_equal(c, c0), (ctx, "rank", r, n, n0, c, c0)
            assert np.array_equal(d, d0) and np.array_equal(s.view(np.uint32), s0.view(np.uint32)), (ctx, "rank", r)
        d1, s1, n1, c1 = self.unsharded(mode, texts, qv, **kw)   # (b)
        assert np.array_equal(n0, n1) and np.array_equal(c0, c1), (ctx, "unsharded", n0, n1, c0, c1)
        for i in range(d0.shape[0]):
            assert np.array_equal(d0[i], d1[i]), (ctx, "unsharded", i, d0[i, :n0[i]][:12], d1[i, :n1[i]][:12])
            assert np.array_equal(s0[i].view(np.uint32), s1[i].view(np.uint32)), (ctx, "unsharded", i, s0[i, :12], s1[i, :12])
        if oracle is None:
            return tim
        limit, offset = kw.get("limit_hint", 10), kw.get("offset", 0)
        okw = {k: kw[k] for k in ("similarity", "threshold", "omc_doc_ids", "omc_mult", "filtered_doc_ids", "filter_nbits")
               if k in kw}
        B = d0.shape[0]
        for i in range(B):   # (c)
            ref = refs[i] if refs is not None else self.ref(mode, None if texts is None else texts[i],
                                                           None if qv is None else qv[i], limit, **okw)
            d, s, cnt = page(ref, limit, offset)
            n = int(n0[i])
            assert int(c0[i]) == cnt and n == d.shape[0], (ctx, "oracle", i, int(c0[i]), cnt, n, d.shape[0])
            if oracle == "exact":
                assert np.array_equal(d0[i, :n], d) and np.array_equal(s0[i, :n], s), (ctx, "oracle", i, d0[i, :n][:12], d[:12])
            else:
                assert_topk_equal(d0[i, :n], s0[i, :n], d, s, atol=1e-5)
        return tim


def _page_kw(limit, offset, **kw):
    return dict(limit_hint=limit, offset=offset, **kw)


# ------------------------------------------------------------------ 1. fulltext: every query kind, world and page
@gpu
@pytest.mark.parametrize("W", WORLDS)
def test_fulltext_kinds(pool, gpu_ctx, orc, zipf, W):
    """The Zipf corpus (70000 rows: 9 tiles unsharded, 1 to 5 per shard) with the query kinds of test_gpu_topn_paths:
    plain, threshold 0.5 and 1.0, OMC multipliers 0 / 0.5 / 2 / 3 on 6000 docs, multi-term tokens (df counted on
    the device and summed across the ranks).  Exact against the oracle, tie order included."""
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=zipf)
    try:
        for kind in KINDS:
            texts, skw, okw, _ = _kind(kind)
            refs = [sh.ref("fulltext", t, None, 10, **skw) for t in texts]
            for limit, offset in PAGES:
                sh.check("fulltext", texts, refs=refs, ctx=(W, kind, limit, offset), **_page_kw(limit, offset, **skw))
    finally:
        sh.close()


# ------------------------------------------------------------------ 2. vector and hybrid with random embeddings
def _vec_corpus(n=N_VEC, dim=384, seed=41):
    """n string rows, an embedding per doc and 2 more chunks for every 5th doc (all near the doc's first one)."""
    data = synth.make_text_corpus(n, V_VEC, seed=seed + 2)
    rows = synth.make_vectors(n, dim, seed=seed)
    rng = np.random.default_rng(seed)
    extra = np.arange(0, n, 5)
    chunks = np.concatenate([rows[extra] + 0.05 * rng.standard_normal((extra.size, dim)).astype(np.float32),
                             rows[extra] + 0.05 * rng.standard_normal((extra.size, dim)).astype(np.float32)])
    docs = np.concatenate([np.arange(n), extra, extra]).astype(np.uint64)
    perm = rng.permutation(docs.size)   # chunks of one document far apart in the store
    return data, docs[perm], np.concatenate([rows, chunks])[perm], rows


@pytest.fixture(scope="module")
def vec_corpus():
    return _vec_corpus()


@gpu
@pytest.mark.parametrize("W", WORLDS)
def test_vector_hybrid_pages(pool, gpu_ctx, orc, vec_corpus, W):
    """Vector and hybrid mode, random BGE-small embeddings, documents of 1 and 3 chunks, at every page."""
    data, docs, erows, rows = vec_corpus
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=data, emb_docs=docs, emb_rows=erows)
    qv, _ = synth.make_vector_queries(rows, B_VEC, seed=42)
    texts = synth.make_text_queries(V_VEC, B_VEC, seed=44)
    try:
        for limit, offset in PAGES:
            for mode in ("vector", "hybrid"):
                sh.check(mode, texts if mode == "hybrid" else None, qv, "near", ctx=(W, mode, limit, offset),
                         **_page_kw(limit, offset, similarity=0.0))
    finally:
        sh.close()


@gpu
@pytest.mark.parametrize("store", ["bge", "e5", "bf16", "sim0.7"])
def test_vector_stores(pool, gpu_ctx, orc, store):
    """BGE and E5 stores (E5 rescales the score, so the raw key order is not the score order), a bf16 store, and
    similarity 0.7, which drops hits (the rank with the best rows holds all of them)."""
    data, docs, erows, rows = _vec_corpus(6007, 384, seed=7)
    model = "MultilingualE5Small" if store == "e5" else "BGESmall"
    sim = 0.7 if store == "sim0.7" else 0.0
    for W in (3, 16):
        sh = Sharded(_join(pool, W), gpu_ctx, orc, data=data, emb_docs=docs, emb_rows=erows, model=model,
                     dtype="bf16" if store == "bf16" else "f32")
        qv, _ = synth.make_vector_queries(rows, B_VEC, seed=43)
        texts = synth.make_text_queries(V_VEC, B_VEC, seed=45)
        try:
            for limit, offset in ((10, 0), (100, 0), (10, 23)):
                for mode in ("vector", "hybrid"):
                    sh.check(mode, texts if mode == "hybrid" else None, qv, "near", ctx=(store, W, mode, limit, offset),
                             **_page_kw(limit, offset, similarity=sim))
        finally:
            sh.close()


@gpu
def test_tensor_core_rerun_every_rank(pool, gpu_ctx, orc):
    """6000 duplicate rows on rank 0 only and a query on them: rank 0's tensor-core scan flags the query, and every
    rank re-runs pack, exchange and merge in lock step (rerun_ms > 0 on each)."""
    n, dim, B = N_VEC, 384, 12
    rows = synth.make_vectors(n, dim, seed=41)
    rows[1000:7000] = rows[5]
    qv, _ = synth.make_vector_queries(rows, B, seed=42)
    qv[3] = rows[5] * 2.0
    data = synth.make_text_corpus(n, V_VEC, seed=43)
    texts = synth.make_text_queries(V_VEC, B, seed=44)
    sh = Sharded(_join(pool, 2), gpu_ctx, orc, data=data, emb_docs=np.arange(n), emb_rows=rows)
    try:
        for mode in ("vector", "hybrid"):
            tim = sh.check(mode, texts if mode == "hybrid" else None, qv, "near", ctx=mode, **_page_kw(10, 0, similarity=0.0))
            assert tim[0]["scan_tensor_core"] == 1 and tim[0]["scan_unproven"] >= 1, tim[0]
            for r, t in enumerate(tim):
                assert t["rerun_ms"] > 0.0, (mode, r, t)
    finally:
        sh.close()


# ------------------------------------------------------------------ 3. ties
@gpu
@pytest.mark.parametrize("W", WORLDS)
def test_vector_ties_doc_order(pool, gpu_ctx, orc, W):
    """Signed unit axes (every score is -1, 0 or 1) with doc ids that descend along the rows, and docs of two and
    three chunks: equal scores must come out in doc-id order, as top_n breaks ties, not in store-row order."""
    rng = np.random.default_rng(W)
    n = 3001
    docs = (np.arange(n, 0, -1) * 7).astype(np.uint64)
    docs = np.concatenate([docs, docs[::97], docs[::211]])
    rows = axis_rows(rng.integers(0, 3, docs.size), rng.choice([-1.0, 1.0], docs.size))
    sh = Sharded(_join(pool, W), gpu_ctx, orc, emb_docs=docs, emb_rows=rows, model="BGEBase", dim=DIM)
    try:
        qv = np.concatenate([axis_query(2, 0), axis_query(2, 1, -1.0)])
        for limit, offset in PAGES + [(200, 0), (1024, 0), (30, 994)]:
            sh.check("vector", None, qv, "exact", ctx=(W, limit, offset), **_page_kw(limit, offset, similarity=-2.0))
    finally:
        sh.close()


@gpu
@pytest.mark.parametrize("W", [2, 3, 4])
def test_hybrid_vector_only_ties(pool, gpu_ctx, orc, W):
    """Hybrid mode with tied vector hits whose documents have no string row, spread over the shards (string rows
    hold the multiples of 10, the vector-only docs end in 5): among themselves they must keep doc-id order.  Compared
    with the unsharded search only: a vector-only hit tying a string-row doc diverges from the oracle (DESIGN.md §4)."""
    sdocs = np.arange(0, 640, 10, dtype=np.uint64)
    data = postings(64, [([3, 20, 40, 60], [1, 2, 1, 3], 10)], row_doc_ids=sdocs)
    vdocs = np.asarray([605, 45, 305, 125, 5, 15, 455, 30, 200, 415, 25, 535], np.uint64)
    axes = np.asarray([0, 0, 0, 0, 0, 0, 0, 1, 1, 0, 2, 0])
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=data, emb_docs=vdocs, emb_rows=axis_rows(axes, np.ones(len(axes))),
                 model="BGEBase", dim=DIM)
    try:
        for limit, offset in ((3, 0), (8, 0), (12, 0), (4, 3)):
            sh.check("hybrid", [TextQuery.single_terms([0])] * 2, axis_query(2), None, ctx=(W, limit, offset),
                     **_page_kw(limit, offset, similarity=0.0))
    finally:
        sh.close()


# ------------------------------------------------------------------ 4. rank-proxy re-run
@gpu
@pytest.mark.parametrize("W", [2, 3])
def test_rank_proxy_rerun_deterministic(pool, gpu_ctx, orc, W):
    """test_gpu_topn_paths.test_rank_proxy_rerun_deterministic sharded: docs A (0, multiplier 0.5) and B (1) on rank 0,
    the vector hit at cosine -1 (doc 2) on rank 1.  The tiles rank by (ft - 0) * m and keep A at limit 1; the true
    order (ft - min) * m with min = -1 puts B first, so the re-run must happen on every rank."""
    data = postings(4, [([0, 1], [1000, 1], 10)])
    rows = axis_rows([0], [-1.0])
    bounds = [(0, 2), (2, 4)] if W == 2 else [(0, 2), (2, 3), (3, 4)]
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=data, emb_docs=[2], emb_rows=rows, bounds=bounds, model="BGEBase", dim=DIM)
    od, om = np.asarray([0, 1], np.uint64), np.asarray([0.5, 1.0], np.float32)
    texts, q = [TextQuery.single_terms([0])], axis_query(1)
    try:
        assert sh.ref("hybrid", texts[0], q[0], 1, -2.0, omc_doc_ids=od, omc_mult=om)[0][0] == 1   # the premise
        for limit in (1, 3):
            sh.check("hybrid", texts, q, "exact", ctx=(W, limit), **_page_kw(limit, 0, similarity=-2.0, omc_doc_ids=od, omc_mult=om))
    finally:
        sh.close()


@gpu
@pytest.mark.parametrize("W", [2, 3])
def test_rank_proxy_rerun_zipf(pool, gpu_ctx, orc, zipf, W):
    """The Zipf version: OMC multipliers (0, 0.5, 2, 3) on the docs of rank 0 only, 300 embedded docs of which 297 sit
    at cosine -1 to the query, so every query's global min is -1."""
    rng = np.random.default_rng(9)
    texts, skw, _, _ = _kind("omc")
    hi0 = shard_range(N_ZIPF, 1, W)[0]
    keep = skw["omc_doc_ids"] < hi0
    od, om = skw["omc_doc_ids"][keep], skw["omc_mult"][keep]
    docs = np.sort(rng.choice(N_ZIPF, 300, replace=False)).astype(np.uint64)
    rows = axis_rows(np.where(np.arange(300) < 297, 0, 1), np.full(300, -1.0))[rng.permutation(300)]
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=zipf, emb_docs=docs, emb_rows=rows, model="BGEBase", dim=DIM)
    q = axis_query(len(texts))
    try:
        for limit, offset in ((1, 0), (10, 0), (10, 23), (100, 0)):
            sh.check("hybrid", texts, q, "exact", ctx=(W, limit, offset),
                     **_page_kw(limit, offset, similarity=-2.0, omc_doc_ids=od, omc_mult=om))
    finally:
        sh.close()


# ------------------------------------------------------------------ 5. merge-buffer regimes
@gpu
def test_world16_streaming_merge(pool, gpu_ctx, orc, zipf):
    """W = 16 at limit 200: W * n_keep + v_stride = 3400 keys exceed the merge's 2048-key buffer, so shard_fuse_kernel
    selects with block_topn_stream.  Fulltext exact; hybrid on signed axes, exact."""
    rng = np.random.default_rng(3)
    docs = np.sort(rng.choice(N_ZIPF, 5000, replace=False)).astype(np.uint64)
    rows = axis_rows(rng.integers(0, 3, 5000), rng.choice([-1.0, 1.0], 5000))
    sh = Sharded(_join(pool, 16), gpu_ctx, orc, data=zipf, emb_docs=docs, emb_rows=rows, model="BGEBase", dim=DIM)
    texts, _, _, _ = _kind("plain")
    try:
        for limit, offset in ((200, 0), (200, 300), (150, 850)):
            sh.check("fulltext", texts, None, "exact", ctx=("ft", limit, offset), **_page_kw(limit, offset))
            sh.check("hybrid", texts, axis_query(len(texts)), "exact", ctx=("hy", limit, offset),
                     **_page_kw(limit, offset, similarity=-2.0))
    finally:
        sh.close()


@gpu
def test_cold_wide_pack_overflow(pool, gpu_ctx, orc):
    """34 tiles over 2 ranks (17 each), one term in every row, OC_BM25_SEED=0 (the threshold starts cold) and
    n_keep = 1024: each shard's 17 x 1024 tile candidates exceed the pack kernel's 16384-key buffer, so
    shard_pack_kernel takes its streaming branch."""
    from test_gpu_tile3 import _env
    n = 34 * 8192
    rng = np.random.default_rng(11)
    rows = np.arange(n)
    data = postings(n, [(rows, rng.integers(1, 6, n), rng.integers(5, 80, n)), (rows[::3], 1, rng.integers(5, 80, rows[::3].size))])
    sh = Sharded(_join(pool, 2), gpu_ctx, orc, data=data)
    try:
        for texts in ([TextQuery.single_terms([0])] * 2, [TextQuery.single_terms([0, 1])] * 2):
            refs = [sh.ref("fulltext", t, None, 10) for t in texts]
            with _env(OC_BM25_SEED="0"):
                for limit, offset in ((1024, 0), (24, 1000), (10, 0)):
                    sh.check("fulltext", texts, None, "exact", refs=refs, ctx=(limit, offset), **_page_kw(limit, offset))
    finally:
        sh.close()


# ------------------------------------------------------------------ 6. empty shard, df all-reduce, tombstones
@gpu
@pytest.mark.parametrize("W", [3, 8])
def test_empty_rank_and_df_allreduce(pool, gpu_ctx, orc, W):
    """Rank 1 holds no string row and no embedding row (n_tiles == 0) and still enters every collective: fulltext,
    vector and hybrid, a filter (df counted and all-reduced), multi-term tokens."""
    n = 9001
    data = synth.make_text_corpus(n, 800, seed=W)
    rng = np.random.default_rng(W)
    bounds = [shard_range(n, r, W) for r in range(W)]
    bounds[1] = (bounds[1][0], bounds[1][0])
    bounds[2] = (bounds[1][0], bounds[2][1])
    rows = axis_rows(rng.integers(0, 4, n), rng.choice([-1.0, 1.0], n))
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=data, emb_docs=np.arange(n), emb_rows=rows, bounds=bounds,
                 model="BGEBase", dim=DIM)
    assert sh.n_rows[1] == 0
    texts = synth.make_text_queries(800, 8, seed=W + 1)
    multi = [TextQuery.from_tokens([[(0, int(a), 1.0), (0, int(b), 0.5)], [(0, int(c), 2.0)]])
             for a, b, c in rng.integers(0, 300, (8, 3))]
    fb = orc.make_filter_bits(np.sort(rng.choice(n, n // 3, replace=False)).tolist(), n)
    q = axis_query(8)
    try:
        for limit, offset in ((10, 0), (100, 0), (7, 50)):
            pk = _page_kw(limit, offset, similarity=-2.0)
            sh.check("fulltext", texts, None, ctx=("ft", limit), **pk)
            sh.check("fulltext", multi, None, ctx=("multi", limit), **pk)
            sh.check("vector", None, q, ctx=("v", limit), **pk)
            sh.check("hybrid", texts, q, ctx=("hy", limit), **pk)
            sh.check("fulltext", texts, None, ctx=("ft+filter", limit), filtered_doc_ids=fb, filter_nbits=n, **pk)
            sh.check("hybrid", texts, q, ctx=("hy+filter", limit), filtered_doc_ids=fb, filter_nbits=n, **pk)
    finally:
        sh.close()


@gpu
@pytest.mark.parametrize("W", [3, 16])
def test_tombstones_and_counted_df(pool, gpu_ctx, orc, zipf, W):
    """Deletes on one shard only with OC_SHARD_TOMBSTONES on every rank (df counted under the alive rows and
    all-reduced), then shards without the corpus-wide df tables (N and avg length from set_global) with
    OC_SHARD_COUNT_DF: both equal the oracle over the alive documents."""
    texts, _, _, _ = _kind("plain")
    lo, hi = shard_range(N_ZIPF, 1, W)
    rng = np.random.default_rng(W)
    gone = np.sort(rng.choice(np.arange(lo, hi), 300, replace=False)).astype(np.uint64)
    alive = orc.make_filter_bits(np.setdiff1d(np.arange(N_ZIPF), gone).tolist(), N_ZIPF)
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=zipf)
    try:
        sh.strs[1].delete(gone)
        sh.strs1.delete(gone)
        refs = [sh.ref("fulltext", t, None, 10, filtered_doc_ids=alive, filter_nbits=N_ZIPF) for t in texts]
        for limit, offset in PAGES:
            sh.check("fulltext", texts, None, refs=refs, ctx=("tomb", limit, offset), shard_tombstones=True,
                     **_page_kw(limit, offset))
    finally:
        sh.close()
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=zipf, global_df=False)
    try:
        for kind in ("plain", "thr0.5", "multi"):
            texts, skw, _, _ = _kind(kind)
            for limit, offset in ((10, 0), (100, 0)):
                sh.check("fulltext", texts, None, ctx=("count_df", kind, limit), shard_count_df=True, **_page_kw(limit, offset, **skw))
    finally:
        sh.close()


# ------------------------------------------------------------------ 7. refusals
@gpu
def test_refusals_enter_no_collective(pool, gpu_ctx, orc):
    """Per-query where programs, filters and parameters, facets, groups, pins and sortBy are refused with `sharded`
    set, on every rank with the same code, before any collective: the next sharded search on the group succeeds."""
    W, n = 3, 3001
    data = synth.make_text_corpus(n, 500, seed=5)
    texts = synth.make_text_queries(500, 4, seed=6)
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=data)
    handles = []
    try:
        def call(kind):
            def fn(r):
                ctx, tsc = sh.ctxs[r], sh._tscs(MODE_FULLTEXT)[r]
                p = TokenScoreParams(mode=MODE_FULLTEXT, sharded=True)
                if kind == "q_params":
                    p.query_params = [QueryParams(MODE_FULLTEXT, 10)] * 4
                elif kind in ("q_filters", "q_where"):
                    f = ob.DeviceFilter.from_ids(ctx, np.arange(0, n, 2), n)
                    handles.append(f)
                    if kind == "q_filters":
                        p.device_filters = [f, None, f, None]
                    else:
                        p.where_programs = [WhereProgram(n, [(_lib.OC_WHERE_FILTER, 0, 0, 0.0, 0.0, 0.0, f._h.value, None)])] * 4
                elif kind in ("facets", "groups"):
                    st = FacetStore(ctx, n)
                    st.add_bool_field("b", np.arange(0, n, 2), np.arange(1, n, 2))
                    handles.append(st)
                    if kind == "facets":
                        return search_facets(tsc, st, p, {"b": {}}, texts=texts)
                    g = GroupBy(st, ["b"])
                    handles.append(g)
                    return search_groups_arrays(tsc, g, p, 1, texts=texts)
                elif kind == "pins":
                    return search_pinned_arrays(tsc, p, [[(5, 0)]] * 4, texts)
                elif kind == "sorted":
                    f = SortField(ctx, n, np.arange(n), np.arange(n) % 17, "number")
                    handles.append(f)
                    return search_sorted_arrays(tsc, p, f, "ASC", None, texts)
                return tsc.execute_batch_arrays(p, texts)
            return fn
        for kind in ("q_params", "q_filters", "q_where", "facets", "groups", "pins", "sorted"):
            out, errs = sh.on_ranks(call(kind))
            assert all(e is not None for e in errs), (kind, out, errs)
            assert {e.code for e in errs} == {OC_ERR_UNSUPPORTED}, (kind, errs)
            sh.check("fulltext", texts, None, ctx=("after", kind), **_page_kw(10, 0))
    finally:
        for h in handles:
            h.close()
        sh.close()


@gpu
def test_comm_init_local_arguments(pool):
    """oc_comm_init_local refuses an empty or oversized group and a context listed twice; a local group refuses the
    NVLink window export."""
    L = _lib.lib()
    import ctypes as C
    arr = (C.c_void_p * 17)(*[c._h for c in pool] + [pool[0]._h])
    assert L.oc_comm_init_local(None, 2) == OC_ERR_INVALID
    assert L.oc_comm_init_local(arr, 0) == OC_ERR_INVALID
    assert L.oc_comm_init_local(arr, 17) == OC_ERR_INVALID
    dup = (C.c_void_p * 2)(pool[0]._h, pool[0]._h)
    assert L.oc_comm_init_local(dup, 2) == OC_ERR_INVALID
    _join(pool, 2)
    with pytest.raises(ob.OcError) as e:
        pool[0].comm_enable_p2p(lambda b: [b, b])
    assert e.value.code == OC_ERR_INVALID
