"""Multi-field BM25F queries and large term expansions against the oracle, bit for bit.

In an index with several string fields every query token resolves to one term per searched field, and a prefix or typo
expansion to many more (csrc/dict.h plan_one).  One such token sends its whole batch to the accumulator scorer K3
(bm25_tile_kernel<MULTI=true>) with the dense arrays off, its df to the device pre-pass (bm25_df_kernel: the union of
the token's rows over all its terms and fields), and the hybrid lookups of its vector hits to bm25_point_kernel's
multi-term branch.  This file runs those shapes on a corpus of four string fields over 150 K documents (19 tiles) —
a title (mean 5 tokens), tags (mean 2, 30 % of documents without), a description (mean 40) and a body (mean 200), each
with its own Zipf order over one sorted list of 20 K pseudo-words — whose term ids come from a TermDictionary fed in a
shuffled order, so an expansion arrives in string order with non-monotone ids, as in production:

  - K3 loads a query's terms in passes of TERM_PASS = 96 and re-reads a token's earlier-pass terms when it finalizes
    the token (bm25.cuh:435-460): tokens of 95, 96, 97, 192 and 193 terms, a token straddling a pass boundary, a token
    whose only term with postings in a tile lies in the earlier pass, a (field, term) twice in one token;
  - the empty query "", which expands to every term of every searched field in one token (the reference's browse
    search), over all fields and over a `properties` subset;
  - dictionary-resolved queries: exact, prefixes of 1 to 3 letters, tolerance 1 and 2 expanded on the device, the
    English stemmer, field boosts 0 / 0.5 / 3, `properties` subsets and exact_match_boost 2 and 3.5;
  - 33 to 40 tokens mixing single- and multi-term tokens (the token bit wraps at 32);
  - pages, thresholds, OMC (multiplier 0 included), a host and a device filter, per-query filters, deletes before and
    after a commit, sparse document ids, hybrid mode with and without the side stream, groups and facet counts;
  - bm25 k and b other than the defaults, alternated on one store so every field's postings are re-derived;
  - the sharing routes (OC_BM25_SHARE=force puts the single-term tokens of a K3 batch in precomputed form) and
    OC_BM25_TILE2=0, and each query of a mixed batch against the same query alone.

Every comparison is exact: doc ids, score bits and count, tie order included (the page builder of
test_gpu_topn_paths).  The CPU tests at the end check the shapes the GPU tests rely on, so that a change of the
generator cannot quietly drop the coverage."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oramacore_b200 as ob
import oramacore_b200.engine as engine
from oramacore_b200.types import FieldPostings, StringIndexData, TextQuery
from test_gpu_dict_resolve import _typo
from test_gpu_facets import _oracle_counts
from test_gpu_groups import _check_groups, _oracle_groups
from test_gpu_tile3 import _env
from test_gpu_topn_paths import DIM, _eq, _sorted, axis_query, axis_rows, page, ref_map

gpu = pytest.mark.gpu

N_DOCS, TILE, TERM_PASS = 150_000, 8192, 96
N_WORDS = 20_000
MEAN_LEN = (5.0, 2.0, 40.0, 200.0)         # title, tags, description, body
VOCAB = (20_000, 3_000, 20_000, 20_000)    # words in each field's dictionary (and term ids of its postings)
ROUTES = {"default": {}, "share_force": {"OC_BM25_SHARE": "force"}, "share_off": {"OC_BM25_SHARE": "off"},
          "K3": {"OC_BM25_TILE2": "0"}}
PAGES = [(1, 0), (10, 0), (33, 0), (7, 500), (1024, 0), (24, 1000)]
KB = [(1.2, 0.75), (0.9, 0.3), (2.0, 1.0), (1.2, 0.0), (0.9, 0.3), (2.0, 1.0), (1.2, 0.75)]   # (k, b), alternated


# ------------------------------------------------------------------ the word list, the dictionary, the corpus
def make_words(n=N_WORDS, seed=31):
    """n distinct pseudo-words, sorted.  The first letter is one of 8 and the others of 12, so each first letter starts
    ~n / 8 words and each two-letter prefix ~n / 96; one word in six ends in "ing", "s" or "ed" (the stemmer's food)."""
    rng = np.random.default_rng(seed)
    out = set()
    while len(out) < n:
        lens = rng.integers(3, 9, size=n)
        first = rng.integers(0, 8, size=n)
        rest = rng.integers(0, 12, size=(n, 8))
        suf = rng.integers(0, 18, size=n)
        for i in range(n):
            w = chr(97 + first[i]) + "".join(chr(97 + c) for c in rest[i, :lens[i] - 1])
            out.add(w + (("ing", "s", "ed")[suf[i]] if suf[i] < 3 else ""))
            if len(out) == n:
                break
    return sorted(out)


class World:
    """The words, the dictionary of the four fields and, per field, term_of_rank: the term id of each Zipf rank."""

    def __init__(self):
        rng = np.random.default_rng(32)
        self.words = make_words()
        self.dict = ob.TermDictionary(len(VOCAB))
        self.term_of_rank = []
        for f, v in enumerate(VOCAB):
            order = rng.permutation(N_WORDS)[:v]          # this field's Zipf order: rank r is word order[r]
            feed = rng.permutation(v)                      # dictionary ids in a shuffled order of the words
            ids = self.dict.add_terms(f, [self.words[order[j]] for j in feed])
            assert ids.tolist() == list(range(v))
            tor = np.zeros(v, np.uint32)
            tor[feed] = ids
            self.term_of_rank.append(tor)

    def close(self):
        self.dict.close()


def _lengths(rng, f, n):
    if f == 0:
        return 1 + rng.poisson(MEAN_LEN[0] - 1, n)
    if f == 1:
        return np.where(rng.random(n) < 0.3, 0, 1 + rng.poisson(MEAN_LEN[1] - 1, n))
    sigma = 0.5
    return np.clip(np.rint(np.exp(rng.normal(np.log(MEAN_LEN[f]) - sigma * sigma / 2, sigma, n))), 1, 65535).astype(np.int64)


def _field(rng, lens, tor):
    """One field's postings: document d holds lens[d] tokens, Zipf(1) ranks mapped to term ids by `tor`.  The average
    length is the mean over the documents that hold the field, as a commit computes it (oc_str_commit)."""
    v = tor.shape[0]
    cdf = np.cumsum(1.0 / np.arange(1, v + 1))
    cdf /= cdf[-1]
    ntok = int(lens.sum())
    terms = tor[np.minimum(np.searchsorted(cdf, rng.random(ntok), side="right"), v - 1)].astype(np.uint64)
    docs = np.repeat(np.arange(lens.shape[0], dtype=np.uint64), lens)
    uk, tf = np.unique((terms << np.uint64(32)) | docs, return_counts=True)
    pt = (uk >> np.uint64(32)).astype(np.int64)
    rows = (uk & np.uint64(0xffffffff)).astype(np.uint32)
    offs = np.zeros(v + 1, np.uint64)
    offs[1:] = np.cumsum(np.bincount(pt, minlength=v)).astype(np.uint64)
    held = lens > 0
    avg = float(np.float32(int(lens[held].sum()) / int(held.sum())))
    return FieldPostings(avg, offs, rows, np.minimum(tf, 65535).astype(np.uint16), lens[rows].astype(np.uint16))


def make_corpus(world, seed=33):
    rng = np.random.default_rng(seed)
    fields = [_field(rng, _lengths(rng, f, N_DOCS), world.term_of_rank[f]) for f in range(len(VOCAB))]
    return StringIndexData(fields, N_DOCS, N_DOCS, None)


def drop_rows(data, dead):
    """The store a commit leaves after deleting the documents of rows `dead`: rows renumbered over the survivors,
    document_count = survivors, each field's average length recomputed over the documents that hold it."""
    alive = np.ones(data.n_rows, bool)
    alive[dead] = False
    new_row = np.cumsum(alive) - 1
    docs = np.arange(data.n_rows, dtype=np.uint64) if data.row_doc_ids is None else np.asarray(data.row_doc_ids, np.uint64)
    fields = []
    for f in data.fields:
        keep = alive[f.post_row]
        counts = np.diff(f.term_offsets.astype(np.int64))
        term = np.repeat(np.arange(f.n_terms), counts)[keep]
        offs = np.zeros(f.n_terms + 1, np.uint64)
        offs[1:] = np.cumsum(np.bincount(term, minlength=f.n_terms)).astype(np.uint64)
        rows = f.post_row[keep]
        ln = f.post_len[keep]
        ur, first = np.unique(rows, return_index=True)
        avg = float(np.float32(int(ln[first].astype(np.int64).sum()) / ur.shape[0]))
        fields.append(FieldPostings(avg, offs, new_row[rows].astype(np.uint32), f.post_tf[keep], ln))
    n = int(alive.sum())
    return StringIndexData(fields, n, n, docs[alive])


# ------------------------------------------------------------------ the queries
def dict_queries(world, ctx=None):
    """[(name, TextQuery)] resolved through the dictionary; with a ctx the typo expansions run on its device."""
    rng = np.random.default_rng(34)
    w = world.words
    pick = lambda k: " ".join(w[int(i)] for i in rng.integers(0, len(w), size=k))   # noqa: E731
    out = []

    def add(kind, texts, **kw):
        b = world.dict.resolve_batch(texts, ctx=ctx, **kw)
        out.extend((f"{kind}:{t}", b.query(i)) for i, t in enumerate(texts))

    add("exact", [pick(1), pick(2), pick(3)], exact=True)
    add("prefix", ["b", "ca", "dak", "e ga", pick(1) + " f", pick(2)])
    long_words = [x for x in w if len(x) >= 5]
    add("tol1", [" ".join(_typo(rng, long_words[int(i)]) for i in rng.integers(0, len(long_words), 2)) for _ in range(3)],
        tolerance=1)
    add("tol2", [_typo(rng, long_words[int(i)]) for i in rng.integers(0, len(long_words), 3)], tolerance=2)
    add("boost", [pick(2), "h " + pick(1)], boost=[1.0, 0.0, 0.5, 3.0])
    add("props", [pick(2), "g", pick(1), "ab " + pick(1)], properties=[[0, 2], [1], [3], [1, 2, 3]])
    add("emb3.5", [pick(2), pick(1) + " c"], exact_match_boost=3.5)
    suffixed = [[x for x in w if x.endswith(s)] for s in ("ing", "s", "ed")]
    world.dict.use_english_stemmer()
    try:
        add("stem", [" ".join(ws[int(i)] for i in rng.integers(0, len(ws), 2)) for ws in suffixed])
    finally:
        world.dict.set_stemmer(None)
    add("browse", ["", ""], properties=[None, [0, 1]])
    return out


def _term_pool(world, data, rng, f, n, lo=0):
    """n distinct term ids of field f, ranks log-uniform from `lo` (hot, mid and rare terms), each with postings."""
    v = VOCAB[f]
    out = []
    while len(out) < n:
        r = min(int(np.exp(rng.uniform(np.log(lo + 1), np.log(v)))) - 1, v - 1)
        t = int(world.term_of_rank[f][max(r, lo)])
        if t not in out and data.fields[f].term_offsets[t + 1] > data.fields[f].term_offsets[t]:
            out.append(t)
    return out


def _token(world, data, rng, n):
    """n distinct (field, term) pairs over all four fields, weights 0.5 / 1 / 2 / 3."""
    fs = rng.integers(0, len(VOCAB), size=n)
    pairs = []
    for f in range(len(VOCAB)):
        pairs += [(f, t) for t in _term_pool(world, data, rng, f, int((fs == f).sum()))]
    rng.shuffle(pairs)
    return [(int(f), int(t), float(x)) for (f, t), x in zip(pairs, rng.choice([0.5, 1.0, 2.0, 3.0], size=n))]


def _tiles_of(data, f, t):
    fp = data.fields[f]
    return set((fp.post_row[int(fp.term_offsets[t]):int(fp.term_offsets[t + 1])] // TILE).tolist())


def early_pass_token(world, data):
    """A 100-term title token: term 0 is the only one with postings in tile `tile`, the finalize step (term 99, pass
    1) has to re-read it from the descriptors.  Returns (token, tile)."""
    rng = np.random.default_rng(35)
    fp = data.fields[0]
    lens = np.diff(fp.term_offsets.astype(np.int64))
    first = int(world.term_of_rank[0][300])          # a mid-frequency title term
    tile = min(_tiles_of(data, 0, first))
    pad = []
    for t in rng.permutation(np.flatnonzero((lens >= 1) & (lens <= 6))).tolist():
        if t != first and tile not in _tiles_of(data, 0, t):
            pad.append(t)
            if len(pad) == 99:
                break
    return [(0, first, 1.0)] + [(0, t, 1.0) for t in pad], tile


def shape_queries(world, data):
    """[(name, TextQuery)] of exact token shapes around TERM_PASS and beyond BM25_MAX_TOK."""
    rng = np.random.default_rng(36)
    tok = lambda n: _token(world, data, rng, n)   # noqa: E731
    out = [(f"tok{n}", TextQuery.from_tokens([tok(n)])) for n in (95, 96, 97, 192, 193)]
    out.append(("97+96", TextQuery.from_tokens([tok(97), tok(96)])))
    out.append(("90|10", TextQuery.from_tokens([tok(30), tok(30), tok(30), tok(10)])))
    out.append(("early_pass", TextQuery.from_tokens([early_pass_token(world, data)[0]])))
    (f0, t0, _), (f1, t1, _) = tok(2)[:2]
    out.append(("dup", TextQuery.from_tokens([[(f0, t0, 1.0), (f1, t1, 0.5), (f0, t0, 2.0)], [(f1, t1, 3.0)]])))
    for n in (33, 36, 40):
        out.append((f"{n}tok", TextQuery.from_tokens([tok(1 if rng.random() < 0.5 else int(rng.integers(2, 6)))
                                                       for _ in range(n)])))
    return out


def single_term_queries(world, data, n=8):
    """Plain queries of 3 single-term body tokens (hot to rare): alone they run on K3d / K3c."""
    rng = np.random.default_rng(37)
    return [(f"plain{i}", TextQuery.single_terms(_term_pool(world, data, rng, 3, 3), field=3)) for i in range(n)]


# ------------------------------------------------------------------ oracle maps and checks
def refs(orc, ix, queries, **kw):
    """The sorted score map of each query (ref_map), on all cores: the oracle releases the GIL."""
    with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
        return list(ex.map(lambda q: ref_map(orc, ix, q[1], **kw), queries))


def run(ctx, strs, queries, limit, offset, env=None, emb=None, qv=None, mode="fulltext", **kw):
    with _env(**(env or {})):
        return ob.search(ctx, emb, strs, mode, texts=[q for _, q in queries], q_vecs=qv, limit=limit, offset=offset, **kw)


def check(ctx, strs, queries, maps, pages=PAGES, routes=ROUTES, **kw):
    for rn, env in routes.items():
        for limit, offset in pages:
            hits = run(ctx, strs, queries, limit, offset, env, **kw)
            for (name, _), h, m in zip(queries, hits, maps):
                _eq(h, page(m, limit, offset), (rn, limit, offset, name))


def _bytes(h):
    return h.doc_ids.tobytes() + h.scores.tobytes() + int(h.count).to_bytes(8, "little")


@pytest.fixture(scope="module")
def world():
    w = World()
    yield w
    w.close()


@pytest.fixture(scope="module")
def corpus(world):
    return make_corpus(world)


@pytest.fixture(scope="module")
def store(gpu_ctx, orc, world, corpus):
    """The device store, the oracle's view and the query sets (typo expansions on the device), with the oracle's maps
    of the default parameters."""
    strs = ob.StringFieldStorage(gpu_ctx, corpus)
    ix = orc.StrIndex(corpus)
    dq = dict_queries(world, gpu_ctx)
    sq = shape_queries(world, corpus)
    s = dict(strs=strs, ix=ix, data=corpus, dict=dq, shape=sq, plain=single_term_queries(world, corpus))
    s["maps"] = {k: refs(orc, ix, s[k]) for k in ("dict", "shape", "plain")}
    yield s
    strs.close()


# ------------------------------------------------------------------ 1. pages on every route
@gpu
@pytest.mark.parametrize("kind", ["dict", "shape"])
def test_pages_on_every_route(gpu_ctx, world, store, kind):
    """Dictionary-resolved and shaped queries at every page, on the default route, OC_BM25_SHARE=force|off and
    OC_BM25_TILE2=0; the device-resolved typo expansions equal the host's."""
    if kind == "dict":
        host = dict_queries(world)
        for (n, a), (_, b) in zip(store["dict"], host):
            for x in ("token_term_offsets", "term_field", "term_id"):
                assert np.array_equal(getattr(a, x), getattr(b, x)), (n, x)
            assert np.array_equal(a.term_weight.view(np.uint32), b.term_weight.view(np.uint32)), n
    check(gpu_ctx, store["strs"], store[kind], store["maps"][kind])


# ------------------------------------------------------------------ 2. thresholds, OMC, filters
@gpu
@pytest.mark.parametrize("thr", [0.34, 0.5, 1.0])
def test_thresholds(gpu_ctx, orc, store, thr):
    qs = store["dict"] + store["shape"]
    check(gpu_ctx, store["strs"], qs, refs(orc, store["ix"], qs, threshold=thr), [(10, 0), (33, 0), (24, 1000)],
          threshold=thr)


@gpu
def test_omc(gpu_ctx, orc, store):
    rng = np.random.default_rng(40)
    od = np.sort(rng.choice(N_DOCS, 20000, replace=False)).astype(np.uint64)
    om = rng.choice([0.0, 0.5, 2.0, 3.0], size=od.shape[0]).astype(np.float32)
    qs = store["dict"] + store["shape"]
    check(gpu_ctx, store["strs"], qs, refs(orc, store["ix"], qs, omc_doc=od, omc_mult=om), [(10, 0), (33, 0), (7, 500)],
          omc_doc_ids=od, omc_mult=om)


@gpu
def test_host_and_device_filter(gpu_ctx, orc, store):
    """df of a multi-term token is the union of its rows that pass the filter, over all its terms and fields."""
    rng = np.random.default_rng(41)
    allowed = np.flatnonzero(rng.random(N_DOCS) < 0.4).astype(np.uint64)
    bits = orc.make_filter_bits(allowed, N_DOCS)
    qs = store["dict"] + store["shape"]
    maps = refs(orc, store["ix"], qs, filter_bits=bits, filter_nbits=N_DOCS)
    pages = [(10, 0), (33, 0), (7, 500)]
    check(gpu_ctx, store["strs"], qs, maps, pages, filtered_doc_ids=bits, filter_nbits=N_DOCS)
    flt = ob.DeviceFilter.from_ids(gpu_ctx, allowed, N_DOCS)
    try:
        check(gpu_ctx, store["strs"], qs, maps, pages, device_filter=flt)
    finally:
        flt.close()


@gpu
def test_per_query_filters(gpu_ctx, orc, store):
    rng = np.random.default_rng(42)
    qs = store["dict"] + store["shape"] + store["plain"][:3]
    sets = [np.flatnonzero(rng.random(N_DOCS) < p).astype(np.uint64) for p in (0.2, 0.6)]
    flts = [ob.DeviceFilter.from_ids(gpu_ctx, s, N_DOCS) for s in sets]
    try:
        which = [i % 3 for i in range(len(qs))]    # 0, 1: a filter; 2: none
        maps = []
        for (name, q), k in zip(qs, which):
            kw = {} if k == 2 else dict(filter_bits=orc.make_filter_bits(sets[k], N_DOCS), filter_nbits=N_DOCS)
            maps.append(ref_map(orc, store["ix"], q, **kw))
        check(gpu_ctx, store["strs"], qs, maps, [(10, 0), (33, 0), (7, 500)],
              device_filters=[None if k == 2 else flts[k] for k in which])
    finally:
        for f in flts:
            f.close()


# ------------------------------------------------------------------ 3. deletes, commit, sparse document ids
@gpu
def test_deletes_before_and_after_commit(gpu_ctx, orc, store):
    """Tombstones: the deleted documents leave the df union and the score map (the oracle filters them out).  After the
    commit the rows are renumbered, N and every field's average length change (the oracle gets the rebuilt store)."""
    data = store["data"]
    qs = store["dict"] + store["shape"]
    strs = ob.StringFieldStorage(gpu_ctx, data)
    try:
        rng = np.random.default_rng(43)
        top = [int(m[0][0]) for m in store["maps"]["dict"] if m[0].shape[0]]
        dead = np.unique(np.concatenate([np.asarray(top, np.int64), rng.choice(N_DOCS, 15000, replace=False)]))
        strs.delete(dead.astype(np.uint64))
        alive = np.setdiff1d(np.arange(N_DOCS), dead)
        bits = orc.make_filter_bits(alive.astype(np.uint64), N_DOCS)
        check(gpu_ctx, strs, qs, refs(orc, store["ix"], qs, filter_bits=bits, filter_nbits=N_DOCS),
              [(10, 0), (33, 0), (7, 500)])
        strs.commit()
        after = drop_rows(data, dead)
        assert strs.info()["total_documents"] == after.n_rows
        check(gpu_ctx, strs, qs, refs(orc, orc.StrIndex(after), qs), [(10, 0), (33, 0), (7, 500), (1024, 0)])
    finally:
        strs.close()


@gpu
def test_sparse_doc_ids(gpu_ctx, orc, store):
    data = store["data"]
    sparse = StringIndexData(data.fields, N_DOCS, N_DOCS, np.arange(N_DOCS, dtype=np.uint64) * 3 + 5)
    qs = store["dict"] + store["shape"]
    strs = ob.StringFieldStorage(gpu_ctx, sparse)
    try:
        ix = orc.StrIndex(sparse)
        check(gpu_ctx, strs, qs, refs(orc, ix, qs), [(1, 0), (10, 0), (33, 0), (24, 1000)])
        nb = 3 * N_DOCS + 5
        bits = orc.make_filter_bits(np.arange(5, nb, 6, dtype=np.uint64), nb)   # every other document
        check(gpu_ctx, strs, qs, refs(orc, ix, qs, filter_bits=bits, filter_nbits=nb), [(10, 0), (7, 500)],
              {"default": {}}, filtered_doc_ids=bits, filter_nbits=nb)
    finally:
        strs.close()


# ------------------------------------------------------------------ 4. bm25 k and b
@gpu
def test_k_and_b_alternated_on_one_store(gpu_ctx, orc, store, monkeypatch):
    """Each b change re-derives the streamed postings of every field with that field's own average length
    (capi.cu ft_descriptors); the sequence comes back to each (k, b) so every field is re-derived more than once."""
    qs = store["dict"] + store["shape"] + store["plain"]
    for k, b in KB:
        monkeypatch.setattr(engine, "BM25_K", k)
        monkeypatch.setattr(engine, "BM25_B", b)
        maps = refs(orc, store["ix"], qs, k=k, b=b)
        check(gpu_ctx, store["strs"], qs, maps, [(10, 0), (33, 0)], {"default": {}, "K3": ROUTES["K3"]})
        check(gpu_ctx, store["strs"], store["plain"], maps[-len(store["plain"]):], [(10, 0), (1024, 0)], {"default": {}})


# ------------------------------------------------------------------ 5. hybrid
@gpu
def test_hybrid_with_and_without_the_side_stream(gpu_ctx, orc, store):
    """Axis embeddings (every cosine is -1, 0 or 1, exactly): the vector hits' fulltext scores come from the point
    lookups, the multi-term branch for the dictionary batch.  OC_SIDE_STREAM=0 gives the same bytes; the plain batch
    (single-term tokens, no device df) is the one that runs the fulltext prologue on the side stream by default."""
    rng = np.random.default_rng(44)
    rows = axis_rows(rng.integers(0, 4, N_DOCS), rng.choice([-1.0, 1.0], N_DOCS))
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
    try:
        emb.insert_batch(np.arange(N_DOCS, dtype=np.uint64), rows)
        st = orc.EmbStore(rows)
        for kind in ("dict", "plain"):
            qs = store[kind]
            qv = axis_query(len(qs), 1)
            run(gpu_ctx, store["strs"], qs, 10, 0, emb=emb, qv=qv, mode="hybrid", similarity=0.0)   # b derived, warm
            for limit, offset in ((10, 0), (33, 0), (7, 500), (100, 0)):
                vec = orc.vector(st, qv[0], limit, 0.0)
                a = run(gpu_ctx, store["strs"], qs, limit, offset, emb=emb, qv=qv, mode="hybrid", similarity=0.0)
                z = run(gpu_ctx, store["strs"], qs, limit, offset, {"OC_SIDE_STREAM": "0"}, emb=emb, qv=qv, mode="hybrid",
                        similarity=0.0)
                for (name, _), x, y, m in zip(qs, a, z, store["maps"][kind]):
                    assert _bytes(x) == _bytes(y), (kind, limit, offset, name)
                    d, s, _ = m
                    ref = _sorted(*orc.hybrid_combine(vec, (np.sort(d), s[np.argsort(d)])))
                    _eq(x, page(ref, limit, offset), (kind, limit, offset, name))
    finally:
        emb.close()


# ------------------------------------------------------------------ 6. groups and facet counts
@gpu
def test_groups_and_facets(gpu_ctx, orc, store):
    """groupBy (the raw-score export of the tile scorer) and facet counts (its matched-row bitmap) of the K3 batch,
    against the oracle's score maps."""
    rng = np.random.default_rng(45)
    ids = np.arange(N_DOCS, dtype=np.uint64)
    flag = rng.random(N_DOCS) < 0.3
    cat = rng.integers(0, 5, N_DOCS)
    cat_docs = {f"c{k}": ids[cat == k] for k in range(5)}
    fs = ob.FacetStore(gpu_ctx, N_DOCS)
    gb = None
    try:
        fs.add_bool_field("in_stock", ids[flag], ids[~flag])
        fs.add_string_field("category", cat_docs)
        gb = ob.GroupBy(fs, ["in_stock", "category"])
        members = [(None, set(ids[(flag == b) & (cat == k)].tolist())) for b in (True, False) for k in range(5)]
        assert gb.values == [[b, f"c{k}"] for b in (True, False) for k in range(5)]
        qs = store["dict"] + store["shape"]
        tsc = ob.TokenScoreContext(gpu_ctx, None, store["strs"])
        texts = [q for _, q in qs]
        for thr in (None, 0.5):
            maps = refs(orc, store["ix"], qs, threshold=thr)
            res = ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=ob.MODE_FULLTEXT, limit_hint=10, threshold=thr),
                                   max_results=3, texts=texts)
            for (name, _), (hits, groups), m in zip(qs, res, maps):
                _eq(hits, page(m, 10, 0), (thr, name))
                _check_groups(groups, _oracle_groups((m[0], m[1]), members, 3), exact=True)
        facets = {"in_stock": {"true": True, "false": True}, "category": {}}
        variants = {"in_stock": {"true": ids[flag], "false": ids[~flag]}, "category": cat_docs}
        got = ob.search_facets(tsc, fs, ob.TokenScoreParams(mode=ob.MODE_FULLTEXT), facets, texts=texts)
        for (name, _), g, m in zip(qs, got, store["maps"]["dict"] + store["maps"]["shape"]):
            for f in facets:
                assert g[f]["values"] == _oracle_counts(m[0], variants[f]), (name, f)
    finally:
        if gb is not None:
            gb.close()
        fs.close()


# ------------------------------------------------------------------ 7. batch against alone
@gpu
def test_each_query_in_a_mixed_batch_equals_it_alone(gpu_ctx, store):
    """Plain queries ride K3 in a batch with multi-term neighbours and K3d / K3c alone; every query's bytes in the mixed
    batch equal its bytes alone, on every route and with a threshold (K3b alone)."""
    qs = store["plain"][:4] + store["dict"] + store["plain"][4:] + store["shape"]
    for rn, env in ROUTES.items():
        for limit, offset, thr in ((10, 0, None), (33, 0, None), (10, 0, 0.5)):
            batch = run(gpu_ctx, store["strs"], qs, limit, offset, env, threshold=thr)
            for q, h in zip(qs, batch):
                alone = run(gpu_ctx, store["strs"], [q], limit, offset, env, threshold=thr)[0]
                assert _bytes(h) == _bytes(alone), (rn, limit, offset, thr, q[0])
    maps = store["maps"]["plain"]
    for (name, _), h, m in zip(store["plain"], run(gpu_ctx, store["strs"], store["plain"] + store["dict"], 10, 0), maps):
        _eq(h, page(m, 10, 0), name)


# ------------------------------------------------------------------ CPU: the shapes the GPU tests rely on
def _n_terms(q):
    return np.diff(q.token_term_offsets.astype(np.int64))


def test_shape_queries_cross_the_term_passes(world, corpus):
    sq = dict(shape_queries(world, corpus))
    for n in (95, 96, 97, 192, 193):
        assert _n_terms(sq[f"tok{n}"]).tolist() == [n]
        assert len(set(sq[f"tok{n}"].term_field.tolist())) == 4
    assert _n_terms(sq["97+96"]).tolist() == [97, 96]
    ends = np.cumsum(_n_terms(sq["90|10"]))
    assert ends.tolist() == [30, 60, 90, 100] and ends[2] < TERM_PASS < ends[3]
    tok, tile = early_pass_token(world, corpus)
    q = sq["early_pass"]
    assert _n_terms(q).tolist() == [100] and q.term_id.tolist() == [t for _, t, _ in tok]
    with_postings = [i for i, (f, t, _) in enumerate(tok) if tile in _tiles_of(corpus, f, t)]
    assert with_postings == [0]
    d = sq["dup"]
    assert (int(d.term_field[0]), int(d.term_id[0])) == (int(d.term_field[2]), int(d.term_id[2]))
    assert d.term_weight[0] != d.term_weight[2]
    for n in (33, 36, 40):
        nt = _n_terms(sq[f"{n}tok"])
        assert nt.shape[0] == n and (nt == 1).any() and (nt > 1).any()
    assert corpus.n_rows == N_DOCS and (N_DOCS + TILE - 1) // TILE == 19


def test_dictionary_queries_span_fields_and_passes(world):
    dq = dict_queries(world)
    longest = max(int(_n_terms(q).max()) for _, q in dq)
    assert longest > 2 * TERM_PASS
    assert sum(int((_n_terms(q) > TERM_PASS).sum()) for _, q in dq) >= 5
    multi_field = 0
    for _, q in dq:
        offs = q.token_term_offsets
        for t in range(q.n_tokens):
            multi_field += len(set(q.term_field[offs[t]:offs[t + 1]].tolist())) > 1
    assert multi_field >= 10
    of = lambda kind: [(n.split(":", 1)[1], q) for n, q in dq if n.split(":", 1)[0] == kind]   # noqa: E731
    for kind in ("exact", "prefix", "tol1", "tol2", "boost", "props", "emb3.5", "stem", "browse"):
        assert of(kind) and all(q.term_id.size for _, q in of(kind)), kind
    ws = {f: set() for f in range(len(VOCAB))}   # boost 0 on the tags, 0.5 on the description, 3 on the body (x2 exact)
    for _, q in of("boost"):
        for f in ws:
            ws[f] |= set(q.term_weight[q.term_field == f].tolist())
    assert ws[1] == {0.0} and 0.5 in ws[2] <= {0.5, 1.0} and 3.0 in ws[3] <= {3.0, 6.0}
    assert all(q.n_tokens > len(t.split()) for t, q in of("stem"))   # the stems are tokens of their own
    assert all((q.term_weight == np.float32(3.5)).any() for _, q in of("emb3.5"))
    assert all(int(_n_terms(q).max()) > 1 for _, q in of("tol1") + of("tol2"))
    # the first letters and two-letter prefixes each cover hundreds of words
    w = world.words
    assert all(sum(x.startswith(p) for x in w) >= 2000 for p in "abcdefgh")
    assert min(sum(x.startswith(p) for x in w) for p in ("ca", "ga", "ab", "hl")) >= 100


def test_browse_query_expands_to_every_term(world):
    """The empty query is one token holding every term of every searched field, field by field in string order."""
    dq = [q for n, q in dict_queries(world) if n.startswith("browse")]
    assert len(dq) == 2 and all(q.n_tokens == 1 for q in dq)
    assert dq[0].term_id.shape[0] == sum(world.dict.size(f) for f in range(len(VOCAB))) == sum(VOCAB)
    assert dq[1].term_id.shape[0] == VOCAB[0] + VOCAB[1]
    for f in range(len(VOCAB)):
        ids = dq[0].term_id[dq[0].term_field == f]
        assert ids.shape[0] == VOCAB[f] and not np.all(np.diff(ids.astype(np.int64)) > 0)   # non-monotone ids


def test_oracle_takes_k_and_b(orc):
    rng = np.random.default_rng(46)
    n = 2000
    offs, rows, tfs, lens = [0], [], [], []
    for t in range(20):
        r = np.sort(rng.choice(n, int(rng.integers(20, 400)), replace=False)).astype(np.uint32)
        rows.append(r); tfs.append(rng.integers(1, 5, r.shape[0]).astype(np.uint16))
        lens.append(rng.integers(3, 60, r.shape[0]).astype(np.uint16))
        offs.append(offs[-1] + r.shape[0])
    f = FieldPostings(27.5, np.asarray(offs, np.uint64), np.concatenate(rows), np.concatenate(tfs), np.concatenate(lens))
    ix = orc.StrIndex(StringIndexData([f], n, n, None))
    q = TextQuery.from_tokens([[(0, 1, 1.0), (0, 2, 0.5)], [(0, 3, 2.0)]])
    base = orc.fulltext(ix, q)
    same = orc.fulltext(ix, q, b=0.75, k=1.2)
    assert np.array_equal(base[0], same[0]) and np.array_equal(base[1].view(np.uint32), same[1].view(np.uint32))
    for k, b in KB[1:4]:
        other = orc.fulltext(ix, q, b=b, k=k)
        assert np.array_equal(other[0], base[0]) and not np.array_equal(other[1], base[1]), (k, b)
    sb = orc.SearchBatch(ix, None)
    sb.add(0, limit=5, text=q, b=0.3, k=0.9)
    od, os_, on, oc = sb.run(1)
    ref = page(_sorted(*orc.fulltext(ix, q, b=0.3, k=0.9)), 5, 0)
    assert np.array_equal(od[0, :on[0]], ref[0]) and np.array_equal(os_[0, :on[0]], ref[1])
