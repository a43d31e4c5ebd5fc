"""oc_search_indexes: every index of a collection in one call, merged on the device, byte for byte against the
per-index recipe (oc_search_q_sorted per index with limit' = limit + offset, 2 x that for an active pinned query,
offset' = 0, vector_limit = limit, pins with apply = 0) merged by oc_merge_results / oc_merge_pinned / oc_merge_sorted."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import _lib, synth
from oramacore_b200 import engine as E
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, FieldPostings, StringIndexData

pytestmark = pytest.mark.gpu

N, DIM, VOCAB, B = 6000, 384, 800, 16


def _split(data, owner, i):
    """the documents with owner[d] == i as one index: own row space, own average length and document count."""
    f = data.fields[0]
    df = np.diff(f.term_offsets.astype(np.int64))
    term_of = np.repeat(np.arange(f.n_terms, dtype=np.int64), df)
    docs = np.nonzero(owner == i)[0].astype(np.uint64)
    loc = np.zeros(data.n_rows, np.int64)
    loc[docs.astype(np.int64)] = np.arange(docs.shape[0])
    sel = owner[f.post_row.astype(np.int64)] == i
    offs = np.zeros(f.n_terms + 1, np.uint64)
    offs[1:] = np.cumsum(np.bincount(term_of[sel], minlength=f.n_terms)).astype(np.uint64)
    lens = np.zeros(data.n_rows, np.int64)
    lens[f.post_row[sel]] = f.post_len[sel]
    avg = float(lens[docs.astype(np.int64)].mean())
    fp = FieldPostings(avg, offs, loc[f.post_row[sel].astype(np.int64)].astype(np.uint32), f.post_tf[sel].copy(), f.post_len[sel].copy())
    return StringIndexData([fp], docs.shape[0], docs.shape[0], docs)


@pytest.fixture(scope="module")
def corpus():
    rows = synth.make_vectors(N, DIM, seed=71)
    qv, _ = synth.make_vector_queries(rows, B, seed=72)
    data = synth.make_text_corpus(N, VOCAB, seed=73)
    texts = synth.make_text_queries(VOCAB, B, seed=74)
    return rows, qv, data, texts


class Collection:
    """n indexes over one corpus, split by doc id mod n or by contiguous ranges; with `empty`, one more empty index."""

    def __init__(self, ctx, corpus, n, how, empty=False, emb=True, bf16=True):
        rows, self.qv, data, self.texts = corpus
        owner = np.arange(N) % n if how == "mod" else np.arange(N) * n // N
        self.parts, self.stores = [], []
        for i in range(n):
            sd = _split(data, owner, i)
            docs = sd.row_doc_ids
            e = None
            if emb:
                e = ob.EmbeddingFieldStorage(ctx, "BGESmall", dtype="bf16" if bf16 and i % 2 else "f32")
                e.insert_batch(docs, rows[docs.astype(np.int64)])
            s = ob.StringFieldStorage(ctx, sd)
            self.stores.append((e, s, docs))
            self.parts.append(E.IndexPart(ob.TokenScoreContext(ctx, e, s), self.texts, self.qv))
        if empty:
            e = ob.EmbeddingFieldStorage(ctx, "BGESmall") if emb else None
            s = ob.StringFieldStorage.empty(ctx, 1)
            self.stores.append((e, s, np.zeros(0, np.uint64)))
            self.parts.append(E.IndexPart(ob.TokenScoreContext(ctx, e, s), self.texts, self.qv))

    def close(self):
        for e, s, _ in self.stores:
            if e is not None:
                e.close()
            s.close()


_COLLECTIONS = {}


@pytest.fixture(scope="module")
def collections(gpu_ctx, corpus):
    def get(n, how, empty=False, emb=True, bf16=True):
        key = (n, how, empty, emb, bf16)
        if key not in _COLLECTIONS:
            _COLLECTIONS[key] = Collection(gpu_ctx, corpus, n, how, empty, emb, bf16)
        return _COLLECTIONS[key]
    yield get
    for c in _COLLECTIONS.values():
        c.close()
    _COLLECTIONS.clear()


def _one_index(part, params, sorts, promote, Bq):
    """oc_search_q_sorted on one index with pins apply = 0: (docs, scores, sort values, n, count, pin scores, present)."""
    sp, keep, _ = part.tsc._build_params(dataclasses.replace(params, **dict(part.fields or {})), part.texts, part.q_vecs)
    srt = E._q_sorts(sorts if sorts is not None else [None] * Bq, Bq)
    pins = None if promote is None else E._pins(promote, Bq, False)[0]
    n_items = 0 if pins is None else int(pins._keep[0][-1])
    L = E._stride(params)
    docs, scores, sv = np.zeros((Bq, L), np.uint64), np.zeros((Bq, L), np.float32), np.zeros((Bq, L), np.float64)
    n, cnt = np.zeros(Bq, np.uint32), np.zeros(Bq, np.uint64)
    ps, pp = np.zeros(max(n_items, 1), np.float32), np.zeros(max(n_items, 1), np.uint8)
    t = part.tsc
    _lib.check(_lib.lib().oc_search_q_sorted(t.ctx._h, t.emb._h if t.emb else None, t.str._h if t.str else None, C.byref(sp),
                                             srt, None if pins is None else C.byref(pins), E._p(docs), E._p(scores), E._p(sv),
                                             E._p(n), E._p(cnt), E._p(ps), E._p(pp)))
    return docs, scores, sv, n, cnt, ps[:n_items], pp[:n_items]


def _slice_part(part, b):
    f = dict(part.fields or {})
    for k in ("device_filters", "where_programs"):
        if f.get(k) is not None:
            f[k] = [f[k][b]]
    return E.IndexPart(part.tsc, None if part.texts is None else part.texts[b:b + 1],
                       None if part.q_vecs is None else part.q_vecs[b:b + 1], f)


def _recipe(parts, params, sorts, promote):
    """The documented per-index recipe, query by query (B = 1 merges), in the layout of oc_search_indexes."""
    Bq = len(parts[0].texts) if parts[0].texts is not None else parts[0].q_vecs.shape[0]
    stride = E._stride(params)
    od, os_, ov = np.zeros((Bq, stride), np.uint64), np.zeros((Bq, stride), np.float32), np.zeros((Bq, stride), np.float64)
    on, oc = np.zeros(Bq, np.uint32), np.zeros(Bq, np.uint64)
    ps_all, pp_all = [], []
    for b in range(Bq):
        if params.query_params is not None:
            e = params.query_params[b]
            pb = dataclasses.replace(params, query_params=None, mode=e.mode, limit_hint=e.limit, offset=e.offset,
                                     similarity=e.similarity, threshold=e.threshold)
        else:
            pb = params
        L, O = pb.limit_hint, pb.offset
        prom = None if promote is None else [promote[b]]
        active = prom is not None and len(prom[0]) > 0
        depth = (L + O) * (2 if active else 1)
        srt_b = [None if sorts is None or sorts[i] is None else [sorts[i][b]] for i in range(len(parts))]
        field_order = srt_b[0] is not None and srt_b[0][0] is not None
        per = [_one_index(_slice_part(p, b), dataclasses.replace(pb, limit_hint=depth, offset=0, vector_limit=L), srt_b[i], prom, 1)
               for i, p in enumerate(parts)]
        if field_order:
            hits, sv = E.merge_index_results_sorted(per if prom is not None else [r[:5] for r in per], srt_b[0][0][1], L, O, prom)
            ov[b, :L] = sv[0]
        elif prom is not None:
            hits = E.merge_index_results_pinned([(r[0], r[1], r[3], r[4], r[5], r[6]) for r in per], prom, L, O)
        else:
            hits = E.merge_index_results([(r[0], r[1], r[3], r[4]) for r in per], L, O)
        h = hits[0]
        k = len(h.doc_ids)
        od[b, :k], os_[b, :k], on[b], oc[b] = h.doc_ids, h.scores, k, h.count
        if not field_order:
            ov[b, :k] = np.nan
        if prom is not None:   # each item: the first index whose map holds it
            for j in range(len(prom[0])):
                s, pr = np.float32(0), 0
                for r in per:
                    if r[6][j]:
                        s, pr = r[5][j], 1
                        break
                ps_all.append(s); pp_all.append(pr)
    return od, os_, ov, on, oc, np.asarray(ps_all, np.float32), np.asarray(pp_all, np.uint8)


def _same(got, exp):
    d, s, v, n, c, ps, pp = got
    ed, es, ev, en, ec, eps, epp = exp
    assert np.array_equal(n, en)
    assert np.array_equal(c, ec)
    assert np.array_equal(d, ed)
    assert np.array_equal(s.view(np.uint32), es.view(np.uint32))
    assert np.array_equal(v.view(np.uint64), ev.view(np.uint64))
    assert np.array_equal(ps.view(np.uint32), eps.view(np.uint32))
    assert np.array_equal(pp, epp)


def _check(ctx, parts, params, sorts=None, promote=None):
    got = E.search_indexes_arrays(ctx, parts, params, sorts, promote)
    _same(got, _recipe(parts, params, sorts, promote))
    return got


@pytest.mark.parametrize("how", ["mod", "range"])
@pytest.mark.parametrize("n", [1, 2, 3, 5])
@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID])
def test_union_matches_the_recipe(gpu_ctx, collections, how, n, mode):
    col = collections(n - 1 if n == 5 else n, how, empty=n == 5)
    for limit, offset in ((10, 0), (7, 13), (1000, 24)):
        got = _check(gpu_ctx, col.parts, ob.TokenScoreParams(mode=mode, limit_hint=limit, offset=offset, similarity=0.0))
        assert got[4].max() > 0   # (a vector-only page past the vector depth is empty, as in the reference)
    t = gpu_ctx.last_timing()
    assert t["kernel_launches"] > 0 and t["d2h_bytes"] > 0


def test_index_without_embedding_store(gpu_ctx, collections):
    col = collections(3, "mod", emb=False)
    _check(gpu_ctx, col.parts, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=20, offset=5))


def _promote(rng, Bq, items_max, skip_every=3):
    out = []
    for b in range(Bq):
        if b % skip_every == 0:
            out.append([])
            continue
        k = int(rng.integers(1, items_max + 1))
        out.append([(int(d), int(p)) for d, p in zip(rng.integers(0, N + 50, k), rng.integers(0, 40, k))])
    return out


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID])
@pytest.mark.parametrize("limit,offset", [(10, 0), (5, 7), (500, 12)])
def test_pins(gpu_ctx, collections, mode, limit, offset):
    col = collections(3, "range")
    rng = np.random.default_rng(limit + offset)
    prom = _promote(rng, B, 6)
    prom[1] = [(3, 0), (3, 2), (N - 1, 1)]   # a document promoted twice, equal positions
    p = ob.TokenScoreParams(mode=mode, limit_hint=limit, offset=offset, similarity=0.0)
    _check(gpu_ctx, col.parts, p, promote=prom)
    _check(gpu_ctx, col.parts, p, promote=[[] for _ in range(B)])   # pins given, no query active


@pytest.fixture(scope="module")
def sort_fields(gpu_ctx, collections):
    col = collections(3, "mod")
    fields = []
    for _, _, docs in col.stores:
        vals = (docs % 7).astype(np.float64)   # values tied across indexes
        keep = docs % 11 != 0                  # and documents without a value
        fields.append(ob.SortField(gpu_ctx, N, docs[keep], vals[keep], "number"))
    yield col, fields
    for f in fields:
        f.close()


@pytest.mark.parametrize("order", ["ASC", "DESC"])
@pytest.mark.parametrize("limit,offset", [(10, 0), (9, 30), (400, 100)])
def test_sorted(gpu_ctx, sort_fields, order, limit, offset):
    col, fields = sort_fields
    p = ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=limit, offset=offset, similarity=0.0)
    sorts = [[(f, order)] * B for f in fields]
    _check(gpu_ctx, col.parts, p, sorts)
    rng = np.random.default_rng(3)
    _check(gpu_ctx, col.parts, p, sorts, _promote(rng, B, 4))
    # mixed batch: every other query in score order, the rest in either order
    mixed = [[None if b % 2 else (f, "ASC" if b % 4 == 0 else "DESC") for b in range(B)] for f in fields]
    _check(gpu_ctx, col.parts, p, mixed, _promote(rng, B, 3))


def test_q_params(gpu_ctx, sort_fields):
    col, fields = sort_fields
    rng = np.random.default_rng(5)
    modes = [MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID]
    qps = [E.QueryParams(mode=modes[b % 3], limit=int(rng.integers(1, 60)), offset=int(rng.integers(0, 40)), similarity=0.0,
                         threshold=None) for b in range(B)]
    p = ob.TokenScoreParams(mode=MODE_HYBRID, query_params=qps)
    _check(gpu_ctx, col.parts, p)
    sorts = [[None if b % 3 == 0 else (f, "DESC" if b % 2 else "ASC") for b in range(B)] for f in fields]
    _check(gpu_ctx, col.parts, p, sorts, _promote(rng, B, 5))


def test_where_omc_and_tombstones(gpu_ctx, corpus):
    col = Collection(gpu_ctx, corpus, 3, "mod")
    omcs, flts = [], []
    try:
        rng = np.random.default_rng(9)
        for i, (e, s, docs) in enumerate(col.stores):
            o = ob.OmcStore(gpu_ctx)
            pick = np.sort(rng.choice(docs, size=200, replace=False))
            o.set(pick, rng.uniform(0.5, 3.0, pick.shape[0]).astype(np.float32))
            o.commit()
            omcs.append(o)
            qf = [None if b % 2 else ob.DeviceFilter.from_ids(gpu_ctx, docs[(docs + b) % (i + 2) == 0], N) for b in range(B)]
            flts += [f for f in qf if f is not None]
            col.parts[i].fields = {"omc_store": o, "device_filters": qf}
        p = ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=25, offset=5, similarity=0.0)
        _check(gpu_ctx, col.parts, p)
        for e, s, docs in col.stores:   # uncommitted deletes, then the commit
            dead = docs[::17]
            for d in dead.tolist():
                s.delete(int(d)); e.delete(int(d))
        _check(gpu_ctx, col.parts, p, promote=_promote(rng, B, 4))
        for e, s, docs in col.stores:
            s.commit()
        _check(gpu_ctx, col.parts, p, promote=_promote(rng, B, 4))
    finally:
        for f in flts:
            f.close()
        for o in omcs:
            o.close()
        col.close()


def test_union_matches_the_oracle(gpu_ctx, orc, corpus, collections):
    rows, qv, data, texts = corpus
    col = collections(3, "mod", bf16=False)   # the oracle scores fp32 rows
    limit, offset = 10, 4
    hits = E.search_indexes(gpu_ctx, col.parts, ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=limit, offset=offset, similarity=0.0))
    owner = np.arange(N) % 3
    union, counts = [dict() for _ in range(B)], np.zeros(B, np.int64)
    for i in range(3):
        sd = _split(data, owner, i)
        docs = sd.row_doc_ids
        ix, st = orc.StrIndex(sd), orc.EmbStore(rows[docs.astype(np.int64)], row_doc_ids=docs)
        for q in range(B):
            m = orc.hybrid_combine(orc.vector(st, qv[q], limit, 0.0), orc.fulltext(ix, texts[q]))
            counts[q] += len(m[0])
            for d, s in zip(*m):
                if s == s:
                    union[q][int(d)] = np.float32(s)
    for q in range(B):
        exp = sorted(union[q].items(), key=lambda kv: (-kv[1], kv[0]))[offset:offset + limit]
        assert hits[q].count == int(counts[q])
        assert_topk_equal(hits[q].doc_ids, hits[q].scores, np.asarray([d for d, _ in exp], np.uint64),
                          np.asarray([s for _, s in exp], np.float32))


def _raw(ctx, parts, params, sorts=None, n_indexes=None, pins=None):
    """oc_search_indexes with sentinel-filled outputs: (code, outputs untouched)."""
    keep, ixs = [], (_lib.IndexQuery * max(len(parts), 1))()
    Bq = B
    for i, part in enumerate(parts):
        sp, k, Bq = part.tsc._build_params(part.fields.get("params", params) if part.fields else params, part.texts, part.q_vecs)
        keep += [sp, k]
        srt = None if sorts is None or sorts[i] is None else E._q_sorts(sorts[i], Bq)
        keep.append(srt)
        ixs[i] = _lib.IndexQuery(part.tsc.emb._h if part.tsc.emb else None, part.tsc.str._h if part.tsc.str else None,
                                 C.pointer(sp), None if srt is None else C.cast(srt, C.c_void_p))
    L = max(params.limit_hint, 1)
    outs = [np.full((Bq, L), 7, np.uint64), np.full((Bq, L), 7, np.float32), np.full((Bq, L), 7, np.float64),
            np.full(Bq, 7, np.uint32), np.full(Bq, 7, np.uint64), np.full(64, 7, np.float32), np.full(64, 7, np.uint8)]
    code = _lib.lib().oc_search_indexes(ctx._h, len(parts) if n_indexes is None else n_indexes, ixs,
                                        None if pins is None else C.byref(pins), *[E._p(o) for o in outs])
    untouched = all((o == 7).all() for o in outs)
    return code, untouched


def test_refusals_write_nothing(gpu_ctx, collections, sort_fields, corpus):
    col = collections(2, "mod")
    p = ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=10, similarity=0.0)
    INVALID, UNSUPPORTED = -1, -4
    assert _raw(gpu_ctx, col.parts, p, n_indexes=0) == (INVALID, True)
    assert _raw(gpu_ctx, col.parts * 17, p) == (INVALID, True)   # 34 > OC_MAX_INDEXES
    other = [col.parts[0], E.IndexPart(col.parts[1].tsc, col.texts, col.qv, {"params": dataclasses.replace(p, limit_hint=11)})]
    assert _raw(gpu_ctx, other, p) == (INVALID, True)            # request fields differ
    assert _raw(gpu_ctx, col.parts, dataclasses.replace(p, vector_limit=5)) == (INVALID, True)
    assert _raw(gpu_ctx, col.parts, dataclasses.replace(p, limit_hint=1000, offset=100)) == (UNSUPPORTED, True)
    assert _raw(gpu_ctx, col.parts, dataclasses.replace(p, sharded=True)) == (UNSUPPORTED, True)
    pins, _ = E._pins([[(1, 0)]] + [[]] * (B - 1), B)
    assert _raw(gpu_ctx, col.parts, dataclasses.replace(p, limit_hint=500, offset=20), pins=pins) == (UNSUPPORTED, True)
    scol, fields = sort_fields
    half = [[(fields[0], "ASC")] * B, None, None]
    assert _raw(gpu_ctx, scol.parts, p, half) == (INVALID, True)   # a sort on some indexes only
    two = [[(fields[0], "ASC")] * B, [(fields[1], "DESC")] * B, [(fields[2], "ASC")] * B]
    assert _raw(gpu_ctx, scol.parts, p, two) == (INVALID, True)    # orders that differ
    ctx2 = ob.Context(0)   # a store of another ctx
    try:
        e2 = ob.StringFieldStorage(ctx2, _split(corpus[2], np.arange(N) % 2, 0))
        mixed = [col.parts[0], E.IndexPart(ob.TokenScoreContext(gpu_ctx, None, e2), col.texts, col.qv)]
        assert _raw(gpu_ctx, mixed, dataclasses.replace(p, mode=MODE_FULLTEXT)) == (INVALID, True)
        e2.close()
    finally:
        ctx2.close()
