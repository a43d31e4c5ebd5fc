"""Top-n selection of the fulltext and hybrid paths against the oracle's whole score map, at every limit / offset,
scorer route and candidate-buffer regime the kernels branch on.

The expected page is built from the oracle's full score map (`orc.fulltext` + `orc.apply_omc`, or `orc.vector` +
`orc.hybrid_combine`), sorted by (-score, doc id) and cut at [offset, offset + limit); the count is the map's size.
The order is fully determined: the GPU key is (score, ~row) (oc_common.cuh:33), rows are in ascending doc order, and
top_n breaks ties by doc id (oracle.c:274-279, 468).  So fulltext pages must equal it exactly: doc ids, scores and
count, tie order included.  Hybrid pages use signed unit-axis embeddings (every cosine is -1, 0 or 1 in any summation
order and precision), so they are compared exactly as well.

Every plain case runs through all four scorers, chosen by the per-launch environment switches: K3d
(bm25_warp_kernel, the default at n_keep <= 32), K3c (bm25_tile3_kernel, OC_BM25_WARP=0 or n_keep > 32), K3b
(bm25_tile2_kernel, OC_BM25_TILE3=0) and K3 (bm25_tile_kernel, OC_BM25_TILE2=0), each crossed with OC_BM25_SEED=0,
OC_BM25_SHARE=force|off and OC_BM25_DENSE=0.  Threshold and OMC queries route to K3b (or K3); multi-term tokens to K3."""
import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import synth
from oramacore_b200.types import FieldPostings, StringIndexData, TextQuery
from test_gpu_tile3 import _env, _queries

gpu = pytest.mark.gpu

SCORERS = {"K3d": {}, "K3c": {"OC_BM25_WARP": "0"}, "K3b": {"OC_BM25_TILE3": "0"}, "K3": {"OC_BM25_TILE2": "0"}}
MODS = {"": {}, "seed0": {"OC_BM25_SEED": "0"}, "share_force": {"OC_BM25_SHARE": "force"},
        "share_off": {"OC_BM25_SHARE": "off"}, "dense0": {"OC_BM25_DENSE": "0"}}
ALL, THR = ("K3d", "K3c", "K3b", "K3"), ("K3b", "K3")
PAGES = [(1, 0), (32, 0), (10, 22), (10, 23), (33, 0), (100, 0), (7, 500), (1024, 0), (1, 1023), (24, 1000)]
DIM = 64


# ------------------------------------------------------------------ reference pages
def _sorted(docs, scores):
    """A score map in result order: NaN dropped (sort.rs:264-267), then (-score, doc id); count = the map's size."""
    docs, scores = np.asarray(docs, np.uint64), np.asarray(scores, np.float32)
    keep = scores == scores
    d, s = docs[keep], scores[keep]
    o = np.lexsort((d, -s.astype(np.float64)))
    return d[o], s[o], int(docs.shape[0])


def ref_map(orc, ix, q, mode="fulltext", st=None, qv=None, limit=10, similarity=0.0, threshold=None,
            omc_doc=None, omc_mult=None, **ft_kw):
    """The whole score map of one request, sorted; `limit` is the vector stage's depth (search.rs:330-336).
    ft_kw goes to orc.fulltext: filter_bits / filter_nbits, b, k."""
    if mode == "vector":
        m = orc.vector(st, qv, limit, similarity)
    else:
        m = orc.fulltext(ix, q, threshold=threshold, **ft_kw)
        if mode == "hybrid":
            m = orc.hybrid_combine(orc.vector(st, qv, limit, similarity), m)
    if omc_doc is not None:
        m = orc.apply_omc(m, omc_doc, omc_mult)
    return _sorted(*m)


def page(sorted_map, limit, offset):
    d, s, count = sorted_map
    return d[offset:offset + limit], s[offset:offset + limit], count


def _eq(h, ref, ctx=""):
    d, s, count = ref
    assert h.count == count, (ctx, h.count, count)
    assert np.array_equal(h.doc_ids, d), (ctx, h.doc_ids[:16], d[:16])
    assert np.array_equal(h.scores, s), (ctx, h.scores[:16], s[:16])


def _routes(scorers):
    for sn in scorers:
        for mn, mod in MODS.items():
            yield f"{sn}{'+' + mn if mn else ''}", {**SCORERS[sn], **mod}


def check_routes(ctx, strs, texts, refs, limit, offset, scorers=ALL, emb=None, qv=None, mode="fulltext", **kw):
    """Every route's result equals the reference page of every query (refs: sorted maps)."""
    for name, env in _routes(scorers):
        with _env(**env):
            hits = ob.search(ctx, emb, strs, mode, texts=texts, q_vecs=qv, limit=limit, offset=offset, **kw)
        for i, h in enumerate(hits):
            _eq(h, page(refs[i], limit, offset), (name, limit, offset, i))


def postings(n_rows, lists, document_count=None, avg=None, row_doc_ids=None):
    """One string field from explicit posting lists: lists[t] = (rows, tf, len) (tf / len scalars or arrays)."""
    offs, rows, tfs, lens = [0], [], [], []
    for r, tf, ln in lists:
        r = np.asarray(r, np.uint32)
        rows.append(r)
        tfs.append(np.broadcast_to(np.asarray(tf, np.uint16), r.shape))
        lens.append(np.broadcast_to(np.asarray(ln, np.uint16), r.shape))
        offs.append(offs[-1] + r.shape[0])
    cat = lambda a, t: np.concatenate(a).astype(t) if a else np.zeros(0, t)  # noqa: E731
    pl = cat(lens, np.uint16)
    f = FieldPostings(float(pl.mean()) if avg is None and pl.size else float(avg or 0.0), np.asarray(offs, np.uint64),
                      cat(rows, np.uint32), cat(tfs, np.uint16), pl)
    return StringIndexData([f], n_rows, n_rows if document_count is None else document_count, row_doc_ids)


def axis_rows(axes, signs):
    """Signed unit axes: every cosine against another signed axis is exactly -1, 0 or 1."""
    rows = np.zeros((len(axes), DIM), np.float32)
    rows[np.arange(len(axes)), np.asarray(axes)] = np.asarray(signs, np.float32)
    return rows


def axis_query(b, axis=0, sign=1.0):
    q = np.zeros((b, DIM), np.float32)
    q[:, axis] = sign
    return q


# ------------------------------------------------------------------ the Zipf corpus and its query kinds
N_ZIPF, V_ZIPF, B_ZIPF = 70000, 3000, 16


@pytest.fixture(scope="module")
def zipf():
    return synth.make_text_corpus(N_ZIPF, V_ZIPF, seed=4242)


def _kind(kind):
    """(texts, search kwargs, oracle kwargs, scorers) of one query kind on the Zipf corpus."""
    rng = np.random.default_rng(KINDS.index(kind))
    if kind == "multi":   # tokens expanding to several terms with different weights (prefix / fuzzy shape)
        texts = []
        for _ in range(B_ZIPF):
            toks = []
            for _t in range(int(rng.integers(1, 4))):
                k = int(rng.integers(2, 5))
                ids = rng.choice(V_ZIPF // 3, size=k, replace=False)
                toks.append([(0, int(t), float(w)) for t, w in zip(ids, rng.choice([1.0, 2.0, 0.5], size=k))])
            texts.append(TextQuery.from_tokens(toks))
        return texts, {}, {}, ("K3",)
    texts = _queries(V_ZIPF, rng, B_ZIPF, 3)
    if kind.startswith("thr"):
        t = float(kind[3:])
        return texts, dict(threshold=t), dict(threshold=t), THR
    if kind == "omc":
        od = np.sort(rng.choice(N_ZIPF, size=6000, replace=False)).astype(np.uint64)
        om = rng.choice([0.0, 0.5, 2.0, 3.0], size=od.shape[0]).astype(np.float32)
        return texts, dict(omc_doc_ids=od, omc_mult=om), dict(omc_doc=od, omc_mult=om), THR
    return texts, {}, {}, ALL


KINDS = ["plain", "thr0.5", "thr1.0", "omc", "multi"]


def test_reference_page_equals_oracle_search(orc, zipf):
    """The page builder above equals the oracle's own search (heap top-(limit+offset), skip, take) at every
    (limit, offset) of the n_keep sweep, for each query kind, tie order included — fulltext and hybrid.  No GPU."""
    ix = orc.StrIndex(zipf)
    st = orc.EmbStore(axis_rows(np.arange(N_ZIPF) % 4, np.where(np.arange(N_ZIPF) % 3 == 0, -1.0, 1.0)))
    qv = axis_query(1, 1)[0]
    for kind in KINDS:
        texts, _, okw, _ = _kind(kind)
        texts = texts[:6]
        refs = [ref_map(orc, ix, t, **okw) for t in texts]
        for limit, offset in PAGES:
            sb = orc.SearchBatch(ix, None)
            for t in texts:
                sb.add(0, limit=limit, offset=offset, text=t, **okw)
            od, os_, on, oc = sb.run(8)
            for i in range(len(texts)):
                d, s, c = page(refs[i], limit, offset)
                assert int(oc[i]) == c and int(on[i]) == d.shape[0], (kind, limit, offset, i)
                assert np.array_equal(od[i, :on[i]], d) and np.array_equal(os_[i, :on[i]], s), (kind, limit, offset, i)
        for limit, offset in ((10, 0), (33, 0), (7, 500)):
            sb = orc.SearchBatch(ix, st)
            for t in texts:
                sb.add(2, limit=limit, offset=offset, similarity=-2.0, q_vec=qv, text=t, **okw)
            od, os_, on, oc = sb.run(8)
            for i, t in enumerate(texts):
                d, s, c = page(ref_map(orc, ix, t, "hybrid", st, qv, limit, -2.0, **okw), limit, offset)
                assert int(oc[i]) == c and np.array_equal(od[i, :on[i]], d) and np.array_equal(os_[i, :on[i]], s)


# ------------------------------------------------------------------ 1. n_keep sweep
@gpu
@pytest.mark.parametrize("kind", KINDS)
def test_nkeep_sweep(gpu_ctx, orc, zipf, kind):
    """n_keep = limit + offset over {1, 32, 33, 100, 507, 1024}: arg-max selection and the bitonic keep of
    block_keep_top (bm25.cuh:279, the n > 32 branch at :283) in K3 / K3b, K3c's keep at n_keep > 32, K3d at <= 32,
    and K4's bitonic vs radix-select branches (fuse.cuh:227).  (10, 22) / (10, 23) straddle n_keep = 32, the switch
    between K3d and K3c and between the seeded and unseeded runs; (1024, 0), (1, 1023) and (24, 1000) fill the
    candidate buffer of every tile to cap = 2048 (capi.cu:2379).  The Zipf corpus has 9 tiles, its hot terms match
    thousands of rows per tile, so every kernel's overflow and keep paths run."""
    texts, skw, okw, scorers = _kind(kind)
    strs = ob.StringFieldStorage(gpu_ctx, zipf)
    ix = orc.StrIndex(zipf)
    refs = [ref_map(orc, ix, t, **okw) for t in texts]
    for limit, offset in PAGES:
        check_routes(gpu_ctx, strs, texts, refs, limit, offset, scorers, **skw)
    strs.close()


# ------------------------------------------------------------------ 2. overflow redo
def _one_tile(tie, n=8000, seed=0):
    rng = np.random.default_rng(seed)
    rows = np.arange(n)
    if tie:
        return postings(n, [(rows, 1, 20), (rows[::5], 1, 20)])
    return postings(n, [(rows, rng.integers(1, 6, n), rng.integers(5, 80, n)),
                        (rows[::5], rng.integers(1, 4, n // 5), rng.integers(5, 80, n // 5))])


@gpu
@pytest.mark.parametrize("tie", [False, True])
def test_cold_threshold_overflow_redo(gpu_ctx, orc, tie):
    """B = 1, one tile of 8000 rows, OC_BM25_SEED=0 and a term in every row: the threshold starts cold, so every matched
    row pushes — more than cap = 2048 keys in K3 / K3b / K3c and more than the 256-key warp buffer of K3d — and each
    kernel redoes its pass with a tighter threshold (K3 bm25.cuh:577-584, K3b :999-1006, K3c :1317-1321, K3d
    :1499-1502).  With `tie` every row has the same score, so the tighter threshold lands inside a run of equal keys.
    n_keep = 1024 with 8000 matches fills the buffer to exactly cap = 2048 before the compress step."""
    data = _one_tile(tie)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    for texts in ([TextQuery.single_terms([0])], [TextQuery.single_terms([0, 1])]):
        refs = [ref_map(orc, ix, t) for t in texts]
        for limit, offset in ((1, 0), (10, 0), (32, 0), (10, 30), (100, 0), (1024, 0), (24, 1000)):
            for name, env in _routes(ALL):
                with _env(**{**env, "OC_BM25_SEED": "0"}):
                    h = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=limit, offset=offset)
                _eq(h[0], page(refs[0], limit, offset), (name, limit, offset))
        for thr in (0.5, 1.0):   # threshold: K3b / K3 with the same cold start
            refs = [ref_map(orc, ix, t, threshold=thr) for t in texts]
            check_routes(gpu_ctx, strs, texts, refs, 10, 0, THR, threshold=thr)
            check_routes(gpu_ctx, strs, texts, refs, 1000, 24, THR, threshold=thr)
    strs.close()


# ------------------------------------------------------------------ 3. K4's selection branches
def _k4_corpus(per_tile, n_tiles=20, seed=1):
    """Term t matches per_tile[t] rows of each of n_tiles tiles; tf / len vary so scores tie in small runs."""
    rng = np.random.default_rng(seed)
    lists = []
    for c in per_tile:
        r = np.concatenate([np.sort(rng.choice(8192, size=c, replace=False)) + 8192 * t for t in range(n_tiles)])
        lists.append((r, rng.integers(1, 4, r.shape[0]), rng.integers(5, 40, r.shape[0])))
    return postings(8192 * n_tiles, lists)


@gpu
@pytest.mark.parametrize("mode", ["fulltext", "hybrid"])
def test_k4_selection_branches(gpu_ctx, orc, mode):
    """Every tile holds fewer matches than n_keep, so no tile ever raises the shared threshold (each emit site raises it
    only when its count reaches n_keep: K3 bm25.cuh:602, K3b :1013, K3c :1329; the seed is off at n_keep > 32) and
    every tile emits all its matches.  K4 then sees exactly (tiles x matches per tile) valid candidates
    (fuse.cuh:217-246):
      - term 0, 1000 per tile x 20 tiles = 20000 > 16384 at n_keep = 1024: the streaming block_topn_stream;
      - term 1, 600 per tile = 12000 at n_keep = 1024 (np2 16384 > 2 x 1024): radix select;
      - term 2, 50 per tile = 1000 at n_keep = 100 (np2 1024 > 2 x 128): radix select;
      - term 3, 40 per tile = 800 at n_keep = 1024, and term 4, 5 per tile = 100 at n_keep = 100: bitonic sort.
    In hybrid mode the `limit` vector hits (cosine 1 rows, most of them not fulltext matches) join the stream."""
    data = _k4_corpus([1000, 600, 50, 40, 5])
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    emb = st = qv = None
    n = data.n_rows
    if mode == "hybrid":
        rng = np.random.default_rng(2)
        rows = axis_rows(rng.integers(0, 8, n), rng.choice([-1.0, 1.0], n))
        emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
        emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
        st = orc.EmbStore(rows)
    for term, n_keep in ((0, 1024), (1, 1024), (2, 100), (3, 1024), (4, 100)):
        texts = [TextQuery.single_terms([term])]
        for limit, offset in ((n_keep, 0), (10, n_keep - 10)):
            q = None if emb is None else axis_query(1)
            refs = [ref_map(orc, ix, texts[0], mode, st, None if q is None else q[0], limit, 0.0)]
            check_routes(gpu_ctx, strs, texts, refs, limit, offset, ALL, emb, q, mode, similarity=0.0)
    strs.close()
    if emb is not None:
        emb.close()


# ------------------------------------------------------------------ 4. paging over ties
@gpu
def test_paging_over_ties(gpu_ctx, orc):
    """30000 documents of equal length, tf = 1, sparse ascending doc ids: every match of a term has the same score, so
    each page must be exactly the next run of ascending doc ids.  Term 0 matches 20000 rows (every tile's buffer
    overflows inside one run of equal keys), term 1 matches 700 (offset = count - 1, = count, > count), term 2 exactly
    1024 (limit + offset = 1024 = count).  Queries [0, 1] have two score levels, so a page cuts through the boundary."""
    rng = np.random.default_rng(4)
    n = 30000
    data = postings(n, [(np.sort(rng.choice(n, 20000, replace=False)), 1, 12),
                        (np.sort(rng.choice(n, 700, replace=False)), 1, 12),
                        (np.sort(rng.choice(n, 1024, replace=False)), 1, 12)],
                    row_doc_ids=np.arange(n, dtype=np.uint64) * 3 + 7)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    for terms in ([0], [1], [2], [0, 1]):
        texts = [TextQuery.single_terms(terms)]
        refs = [ref_map(orc, ix, texts[0])]
        cnt = refs[0][2]
        pages = [(10, 0), (1, 0), (32, 0), (33, 0), (100, 0), (1024, 0), (24, 1000), (7, 500)]
        if cnt <= 1024:   # the last document, the first offset past the end, past it by one, to n_keep = 1024
            pages += [(1, cnt - 1), (1, cnt), (5, cnt + 1), (1025 - cnt, cnt - 1), (10, cnt - 5)]
        for limit, offset in [pg for pg in pages if sum(pg) <= 1024]:
            check_routes(gpu_ctx, strs, texts, refs, limit, offset)
    strs.close()


# ------------------------------------------------------------------ 5. rank-proxy re-run
@gpu
def test_rank_proxy_rerun_deterministic(gpu_ctx, orc):
    """capi.cu:2764-2783.  Hybrid with OMC: the tiles rank candidates by (ft - 0) * m, the real ranking is
    (ft - min) * m.  Doc A (row 0) and doc B (row 1) share a tile; A has multiplier
    0.5, B 1.  One term: A has tf 1000 (score ~2.2 idf), B tf 1 (1.0 idf).  With min = 0, A ranks first
    (ftA * 0.5 > ftB); with min = -1 (the one vector hit, doc 2, is at cosine -1, similarity -2) B does.  At limit 1 each tile keeps one candidate, so without the re-run K4 only ever
    sees A and returns it."""
    data = postings(4, [([0, 1], [1000, 1], 10)])
    ix = orc.StrIndex(data)
    ft = dict(zip(*[a.tolist() for a in orc.fulltext(ix, TextQuery.single_terms([0]))]))
    assert ft[0] * np.float32(0.5) > ft[1] and (ft[0] + 1) * 0.5 < ft[1] + 1, ft   # the premise
    rows = axis_rows([0, 0, 0, 0], [1.0, 1.0, -1.0, 1.0])
    od, om = np.asarray([0, 1], np.uint64), np.asarray([0.5, 1.0], np.float32)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
    emb.insert_batch(np.asarray([2], np.uint64), rows[2:3])
    st = orc.EmbStore(rows[2:3], row_doc_ids=np.asarray([2], np.uint64))
    texts, q = [TextQuery.single_terms([0])], axis_query(1)
    ref = ref_map(orc, ix, texts[0], "hybrid", st, q[0], 1, -2.0, omc_doc=od, omc_mult=om)
    assert ref[0][0] == 1
    check_routes(gpu_ctx, strs, texts, [ref], 1, 0, THR, emb, q, "hybrid", similarity=-2.0, omc_doc_ids=od, omc_mult=om)
    ref = ref_map(orc, ix, texts[0], "hybrid", st, q[0], 3, -2.0, omc_doc=od, omc_mult=om)
    check_routes(gpu_ctx, strs, texts, [ref], 3, 0, THR, emb, q, "hybrid", similarity=-2.0, omc_doc_ids=od, omc_mult=om)
    strs.close(); emb.close()


@gpu
def test_rank_proxy_rerun_zipf(gpu_ctx, orc, zipf):
    """The same three conditions on the Zipf corpus: hybrid, OMC multipliers (0, 0.5, 2, 3) on 6000 docs, and 300
    embedded docs of which 297 sit at cosine -1 to the query (3 at 0), so at limit >= 4 every query's vector hits
    include a negative score and its global min is -1 (similarity -2)."""
    rng = np.random.default_rng(9)
    texts, skw, okw, _ = _kind("omc")
    docs = np.sort(rng.choice(N_ZIPF, 300, replace=False)).astype(np.uint64)
    rows = axis_rows(np.where(np.arange(300) < 297, 0, 1), np.full(300, -1.0))[rng.permutation(300)]
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
    emb.insert_batch(docs, rows)
    st = orc.EmbStore(rows, row_doc_ids=docs)
    strs = ob.StringFieldStorage(gpu_ctx, zipf)
    ix = orc.StrIndex(zipf)
    q = axis_query(len(texts))
    for limit, offset in ((1, 0), (10, 0), (10, 23), (100, 0)):
        refs = [ref_map(orc, ix, t, "hybrid", st, q[0], limit, -2.0, **okw) for t in texts]
        check_routes(gpu_ctx, strs, texts, refs, limit, offset, THR, emb, q, "hybrid", similarity=-2.0, **skw)
    strs.close(); emb.close()


# ------------------------------------------------------------------ 6. token shapes
@gpu
@pytest.mark.parametrize("variant", ["plain", "thr0.5", "thr1.0", "omc"])
def test_token_shapes(gpu_ctx, orc, zipf, variant):
    """Query shapes, in two batches because a batch is routed by its longest query.
    Batch 1 has 5-, 8- and 32-token queries, the same term repeated in one query, and tokens that match no term
    (unknown id, empty expansion).  Its longest query has more than BM25_FLAT_TOK = 4 tokens, so the flat scorers
    (K3c / K3d) are skipped and every route but OC_BM25_TILE2=0 (K3) runs K3b, which builds its token table in the
    kernel (bm25.cuh:745); the 32-token query fills that BM25_MAX_TOK-entry table exactly.
    Batch 2 has 33- and 40-token queries: more than BM25_MAX_TOK, so the batch goes to K3 on every route
    (capi.cu:2156).  The token bit wraps at 32 (capi.cu:2121), and floor(n * threshold) exceeds 32 at threshold 1.0,
    so nothing passes there."""
    rng = np.random.default_rng(6)
    short, long_ = [], []
    for n in (5, 8, 32):
        short.append(TextQuery.single_terms(rng.choice(400, n, replace=False)))
    for n in (33, 40):
        long_.append(TextQuery.single_terms(rng.choice(400, n, replace=False)))
    short.append(TextQuery.single_terms([3, 3, 50]))
    short.append(TextQuery.single_terms([3, 50, 3, 50, 3]))
    short.append(TextQuery.single_terms([7, V_ZIPF + 5, 90]))
    short.append(TextQuery.from_tokens([[(0, 7, 1.0)], [], [(0, 90, 1.0)]]))
    short.append(TextQuery.single_terms([V_ZIPF + 1, V_ZIPF + 2]))
    skw, okw, scorers = {}, {}, ALL
    if variant.startswith("thr"):
        skw = okw = dict(threshold=float(variant[3:]))
        scorers = THR
    elif variant == "omc":
        od = np.sort(rng.choice(N_ZIPF, 8000, replace=False)).astype(np.uint64)
        om = rng.choice([0.0, 0.5, 2.0], size=od.shape[0]).astype(np.float32)
        skw, okw, scorers = dict(omc_doc_ids=od, omc_mult=om), dict(omc_doc=od, omc_mult=om), THR
    strs = ob.StringFieldStorage(gpu_ctx, zipf)
    ix = orc.StrIndex(zipf)
    for texts, routes in ((short, scorers), (long_, ("K3",))):
        refs = [ref_map(orc, ix, t, **okw) for t in texts]
        for limit, offset in ((10, 0), (33, 0), (24, 1000)):
            check_routes(gpu_ctx, strs, texts, refs, limit, offset, routes, **skw)
    strs.close()


# ------------------------------------------------------------------ 7. tile edges
@gpu
@pytest.mark.parametrize("n_rows", [1, 2, 31, 255, 256, 8191, 8192, 8193, 16383, 24577])
def test_tile_edges(gpu_ctx, orc, n_rows):
    """Stores that end just before, at and just after a tile boundary (BM25_TILE = 8192 rows), with a term only in row
    0, one only in the last row, one only in the last (partial) tile and one in every row."""
    rng = np.random.default_rng(n_rows)
    last0 = (n_rows - 1) // 8192 * 8192
    tail = np.arange(last0, n_rows)[::3]
    every = np.arange(n_rows)
    data = postings(n_rows, [([0], 2, 9), ([n_rows - 1], 1, 9), (tail, rng.integers(1, 4, tail.shape[0]), 11),
                             (every, rng.integers(1, 5, n_rows), rng.integers(3, 30, n_rows))])
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    texts = [TextQuery.single_terms(t) for t in ([0], [1], [2], [3], [0, 1], [2, 3], [0, 1, 2, 3])]
    refs = [ref_map(orc, ix, t) for t in texts]
    for limit, offset in ((1, 0), (10, 0), (40, 0), (5, 30)):
        check_routes(gpu_ctx, strs, texts, refs, limit, offset)
    refs = [ref_map(orc, ix, t, threshold=0.5) for t in texts]
    check_routes(gpu_ctx, strs, texts, refs, 10, 0, THR, threshold=0.5)
    strs.close()


# ------------------------------------------------------------------ 8. degenerate postings
def _degenerate(case):
    n = 64
    rows = np.arange(n)
    if case == "tf_len":      # tf 0 / 65535 and field length 0 / 65535 next to ordinary postings
        tf = np.where(rows % 4 == 0, 0, np.where(rows % 4 == 1, 65535, 1 + rows % 3))
        ln = np.where(rows % 5 == 0, 0, np.where(rows % 5 == 1, 65535, 10 + rows % 7))
        return postings(n, [(rows, tf, ln), (rows[::2], 1, ln[::2]), (rows[1::3], tf[1::3], 20)])
    if case == "avg0":        # avg_field_len 0: the length normalisation divides by zero
        return postings(n, [(rows, 1 + rows % 3, rows % 3), (rows[::2], 1, 0)], avg=0.0)
    if case == "neg_idf":     # document_count < df: negative idf, negative scores, negative fold minima
        return postings(n, [(rows, 1 + rows % 3, 10 + rows % 7), (rows[::2], 2, 12), (rows[:5], 1, 10)],
                        document_count=8)
    raise ValueError(case)


@gpu
@pytest.mark.parametrize("mode", ["fulltext", "hybrid"])
@pytest.mark.parametrize("case", ["tf_len", "avg0", "neg_idf"])
def test_degenerate_postings(gpu_ctx, orc, case, mode):
    """Postings whose contribution is zero, subnormal, huge, infinite or NaN, and term weights 0, 1e-40 (subnormal)
    and 1e30: each scorer skips a non-normal folded tf on its own (bm25.rs:387: precompute bm25.cuh:222, K3 :422/:450,
    K3b :843, K3c :1101, point lookup :1601/:1611, seed :1683), and negative idf gives negative scores and minima."""
    data = _degenerate(case)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    texts = []
    for w in (1.0, 0.0, 1e-40, 1e30):
        texts.append(TextQuery.from_tokens([[(0, 0, w)], [(0, 1, 1.0)]]))
        texts.append(TextQuery.from_tokens([[(0, 2, w)]]))
    texts.append(TextQuery.from_tokens([[(0, 0, 1e-40), (0, 1, 1.0)], [(0, 2, 1e30)]]))   # multi-term token: K3
    emb = st = q = None
    if mode == "hybrid":
        rows = axis_rows(np.arange(data.n_rows) % 3, np.where(np.arange(data.n_rows) % 2, 1.0, -1.0))
        emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
        emb.insert_batch(np.arange(data.n_rows, dtype=np.uint64), rows)
        st = orc.EmbStore(rows)
        q = axis_query(len(texts))
    for limit, offset in ((10, 0), (40, 3)):
        refs = [ref_map(orc, ix, t, mode, st, None if q is None else q[0], limit, -2.0) for t in texts]
        check_routes(gpu_ctx, strs, texts[:-1], refs[:-1], limit, offset, ALL, emb, q if q is None else q[:-1], mode,
                     similarity=-2.0)
        check_routes(gpu_ctx, strs, texts[-1:], refs[-1:], limit, offset, ("K3",), emb, q if q is None else q[-1:], mode,
                     similarity=-2.0)
    strs.close()
    if emb is not None:
        emb.close()


# ------------------------------------------------------------------ 9. seed edges
@gpu
def test_seed_edges(gpu_ctx, orc):
    """bm25_seed_kernel (bm25.cuh:1638) runs for plain queries at n_keep <= 32 on stores of more than one tile.  It
    samples the first 64 postings of the rarest list token with at least n_keep postings (:1650); tokens here have
    exactly n_keep and n_keep - 1 postings, so the choice flips between them, and with only hot or too-rare tokens it
    falls back to the first 256 rows.  The rare token's first postings all score alike and low (the k-th seed key sits
    in a run of ties) and its best postings lie after the 64-row sample.  (The fallback's n_rows < 256 exit cannot be
    reached: a store of fewer than 8193 rows has one tile, and the seed is only launched for more; the 255 / 256-row
    stores are covered by test_tile_edges.)  OC_BM25_SHARE=force puts term 4 (300 postings) in precomputed form
    (TD_PRE); terms 0-3 stay lists under every route, since sharing skips lists shorter than 64 postings (capi.cu:2176)
    and n_keep <= 32."""
    rng = np.random.default_rng(12)
    n = 3 * 8192
    lists = []
    for k in (10, 9, 32, 31):   # terms 0-3: exactly n_keep / n_keep - 1 postings for n_keep in {10, 32}
        lists.append((np.sort(rng.choice(n, k, replace=False)), rng.integers(1, 4, k), rng.integers(5, 30, k)))
    r = np.sort(rng.choice(n, 300, replace=False))   # term 4: low tied scores first, the best after the sample
    lists.append((r, np.where(np.arange(300) < 100, 1, rng.integers(2, 9, 300)), np.where(np.arange(300) < 100, 60, 8)))
    hot = np.arange(0, n, 3)   # term 5: hot (dense form under the default routing)
    lists.append((hot, rng.integers(1, 4, hot.shape[0]), rng.integers(5, 40, hot.shape[0])))
    data = postings(n, lists)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    texts = [TextQuery.single_terms(t) for t in ([0, 5], [1, 5], [2, 5], [3, 5], [0, 1], [2, 3], [4], [4, 5], [5],
                                                 [0, 1, 2, 3], [4, 0])]
    refs = [ref_map(orc, ix, t) for t in texts]
    for limit, offset in ((10, 0), (9, 0), (1, 9), (32, 0), (31, 0), (1, 31), (5, 5)):
        check_routes(gpu_ctx, strs, texts, refs, limit, offset)
    strs.close()


# ------------------------------------------------------------------ 10. tie order of vector hits
def _dup_store(gpu_ctx, orc, docs, axes):
    rows = axis_rows(axes, np.ones(len(axes)))
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
    emb.insert_batch(np.asarray(docs, np.uint64), rows)
    return emb, orc.EmbStore(rows, row_doc_ids=np.asarray(docs, np.uint64))


@gpu
def test_vector_ties_order_by_doc_id(gpu_ctx, orc):
    """Duplicate embeddings inserted with descending doc ids (plus a doc of two chunks): the vector list is in
    (score, store row) order, the result must be in (score, doc id) order as top_n breaks ties.  Vector mode, and
    hybrid mode where every hit has a string row (rows hold every doc id) or none has one (two vector-only docs tie)."""
    docs = [50, 40, 30, 20, 10, 7, 7, 60, 45]
    axes = [0, 0, 0, 0, 0, 0, 0, 1, 0]
    emb, st = _dup_store(gpu_ctx, orc, docs, axes)
    q = axis_query(1)
    for limit, offset in ((3, 0), (9, 0), (2, 2), (9, 4)):
        ref = ref_map(orc, None, None, "vector", st, q[0], limit, 0.0)
        _eq(ob.search(gpu_ctx, emb, None, "vector", q_vecs=q, limit=limit, offset=offset, similarity=0.0)[0],
            page(ref, limit, offset), ("vector", limit, offset))
    # hybrid: the string store's rows cover docs 0..63, the query term matches only docs 60 and 61
    data = postings(64, [([60, 61], [1, 2], 10)])
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    texts = [TextQuery.single_terms([0])]
    for limit in (3, 9):
        ref = ref_map(orc, ix, texts[0], "hybrid", st, q[0], limit, 0.0)
        check_routes(gpu_ctx, strs, texts, [ref], limit, 0, ALL, emb, q, "hybrid", similarity=0.0)
    strs.close(); emb.close()
    # hybrid, vector-only hits: docs 25 and 15 have no string row (rows hold docs 100..163), in both insert orders
    data = postings(64, [([1, 2], 1, 10)], row_doc_ids=np.arange(100, 164, dtype=np.uint64))
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    for vdocs in ([25, 15, 120], [15, 25, 120]):
        emb, st = _dup_store(gpu_ctx, orc, vdocs, [0, 0, 1])
        for limit in (3, 4):
            ref = ref_map(orc, ix, texts[0], "hybrid", st, q[0], limit, 0.0)
            check_routes(gpu_ctx, strs, texts, [ref], limit, 0, ALL, emb, q, "hybrid", similarity=0.0)
        emb.close()
    strs.close()


@gpu
@pytest.mark.xfail(strict=True, reason="a hybrid vector hit without a string row has no row index, so its key index "
                                       "sorts after every row on equal scores, whatever its doc id (DESIGN.md, K4)")
def test_hybrid_vector_only_hit_ties_string_doc(gpu_ctx, orc):
    """Doc 15 is a vector hit with no string row; doc 20 has a string row but does not match the query.  Both sit at
    cosine 1, so both score (1 - min) / (max - min): the oracle puts doc 15 first, K4 (fuse.cuh) puts doc 20 first."""
    emb, st = _dup_store(gpu_ctx, orc, [15, 20], [0, 0])
    data = postings(3, [([2], 1, 10)], row_doc_ids=np.asarray([10, 20, 30], np.uint64))
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ix = orc.StrIndex(data)
    texts, q = [TextQuery.single_terms([0])], axis_query(1)
    ref = ref_map(orc, ix, texts[0], "hybrid", st, q[0], 2, 0.0)
    try:
        _eq(ob.search(gpu_ctx, emb, strs, "hybrid", texts=texts, q_vecs=q, limit=2, similarity=0.0)[0], page(ref, 2, 0))
    finally:
        strs.close(); emb.close()
