"""oc_search_indexes_ex: groupBy and facets across the indexes of a collection in one call, byte for byte against the
per-index recipe — each index alone through oc_search_q_groups (limit' = limit + offset, 2 x that for an active pinned
query, offset' = 0, vector_limit = limit, pins with apply = 0, group depth max_results, 2 x max_results for an active
query), its group rows scattered to the collection's keys and merged on the host (score order: score desc, ties by
ascending doc; field order: by value, the lower index first; an active query spliced by apply_pin_rules_to_group, not
truncated).  Active pins are also checked independently: on small corpora each index's whole score map comes back from
oc_search, and the groups are compared with sort_groups + apply_pin_rules_to_group (read/sort.rs:129-230, 377-391)
restated over the union of those maps.  Hits, counts and pin outputs are oc_search_indexes'.  Also every refusal of
the call, which writes nothing and reports its own check.  The facets are in test_gpu_multi_index_facets.py."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib, synth
from oramacore_b200 import engine as E
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from oramacore_b200.where import compile_where, parse_where
from test_gpu_multi_index import DIM, N, VOCAB, _split

pytestmark = pytest.mark.gpu

B = 12
CATS = ["c0", "c1", "c2", "c3"]


@pytest.fixture(scope="module")
def corpus():
    rows = synth.make_vectors(N, DIM, seed=81)
    qv, _ = synth.make_vector_queries(rows, B, seed=82)
    data = synth.make_text_corpus(N, VOCAB, seed=83)
    texts = synth.make_text_queries(VOCAB, B, seed=84)
    return rows, qv, data, texts


class Collection:
    """n indexes split by doc id mod n or by range; each has a FacetStore with cat (4 keys, registered in another
    order on odd indexes), num (8 values), flag (bool) and, from index 1 on, a field `only1`; `empty` adds an empty
    index, which has no filter fields."""

    def __init__(self, ctx, corpus, n, how, empty=False):
        rows, self.qv, data, self.texts = corpus
        nd = self.n_docs = data.n_rows
        owner = np.arange(nd) % n if how == "mod" else np.arange(nd) * n // nd
        self.owner = owner
        self.parts, self.own = [], []
        for i in range(n):
            sd = _split(data, owner, i)
            docs = sd.row_doc_ids.astype(np.int64)
            e = ob.EmbeddingFieldStorage(ctx, "BGESmall")
            e.insert_batch(sd.row_doc_ids, rows[docs])
            s = ob.StringFieldStorage(ctx, sd)
            st = ob.FacetStore(ctx, nd)
            order = CATS if i % 2 == 0 else CATS[::-1]
            st.add_string_field("cat", {c: docs[docs % 4 == CATS.index(c)] for c in order})
            st.add_number_field("num", docs, (docs % 8).astype(np.float64) - 3.0)
            st.add_bool_field("flag", docs[docs % 3 == 0], docs[docs % 3 != 0])
            if i >= 1:
                st.add_bool_field("only1", docs[docs % 5 == 0], docs[docs % 5 != 0])
            self.parts.append(E.IndexPart(ob.TokenScoreContext(ctx, e, s), self.texts, self.qv, None, st))
            self.own.append((e, s, st))
        if empty:
            e = ob.EmbeddingFieldStorage(ctx, "BGESmall")
            s = ob.StringFieldStorage.empty(ctx, 1)
            self.parts.append(E.IndexPart(ob.TokenScoreContext(ctx, e, s), self.texts, self.qv, None, None))
            self.own.append((e, s, None))
        self.gbs = {}

    def group_by(self, props):
        key = tuple(props)
        if key not in self.gbs:
            self.gbs[key] = [ob.GroupBy(p.store, props) if p.store is not None and all(x in p.store.fields for x in props) else None
                             for p in self.parts]
        return self.gbs[key]

    def close(self):
        for gbs in self.gbs.values():
            for g in gbs:
                if g is not None:
                    g.close()
        for e, s, st in self.own:
            e.close(); s.close()
            if st is not None:
                st.close()


_COLS = {}


@pytest.fixture(scope="module")
def cols(gpu_ctx, corpus):
    def get(n, how, empty=False):
        if (n, how, empty) not in _COLS:
            _COLS[(n, how, empty)] = Collection(gpu_ctx, corpus, n, how, empty)
        return _COLS[(n, how, empty)]
    yield get
    for c in _COLS.values():
        c.close()
    _COLS.clear()


def _part_b(part, b):
    f = dict(part.fields or {})
    for k in ("device_filters", "where_programs"):
        if f.get(k) is not None:
            f[k] = [f[k][b]]
    return E.IndexPart(part.tsc, None if part.texts is None else part.texts[b:b + 1],
                       None if part.q_vecs is None else part.q_vecs[b:b + 1], f, part.store)


def _index_groups(part, params, gb, depth, sort, promote):
    """oc_search_q_groups on one index (B = 1, pins apply = 0): group docs, scores, sort values, n [G, depth]."""
    sp, keep, _ = part.tsc._build_params(dataclasses.replace(params, **dict(part.fields or {})), part.texts, part.q_vecs)
    req, rows = E._group_reqs([(gb, depth, sort)], 1)
    pins = None if promote is None else E._pins(promote, 1, False)[0]
    n_items = 0 if pins is None else int(pins._keep[0][-1])
    L, R, S = E._stride(params), int(rows[-1]), max(depth, 1)
    d, s, v, n, c, ps, pp, gd, gs, gsv, gn = E._q_outputs(1, L, n_items, R, S)
    t = part.tsc
    _lib.check(_lib.lib().oc_search_q_groups(t.ctx._h, t.emb._h if t.emb else None, t.str._h if t.str else None, C.byref(sp), req,
                                             None if pins is None else C.byref(pins), S, E._p(d), E._p(s), E._p(v), E._p(n),
                                             E._p(c), E._p(ps), E._p(pp), E._p(gd), E._p(gs), E._p(gsv), E._p(gn)))
    return gd, gs, gsv, gn, ps[:n_items], pp[:n_items]


def _splice(lst, items, member):
    """apply_pin_rules_internal over lst [(doc, score, value)]: items [(doc, position, score)] that are members."""
    its = [(pos, j, d, sc) for j, (d, pos, sc) in enumerate(items) if member(d)]
    if not its:
        return lst
    drop = {d for _, _, d, _ in its}
    out = [e for e in lst if e[0] not in drop]
    for pos, _, d, sc in sorted(its, key=lambda x: (x[0], x[1])):
        out.insert(min(pos, len(out)), (d, sc, np.nan))
    return out


_VALUE = {"cat": lambda d: CATS[d % 4], "num": lambda d: float(d % 8) - 3.0, "flag": lambda d: d % 3 == 0, "only1": lambda d: d % 5 == 0}


def _member(col, i, props, vals, d):
    """d is a document of index i whose values are vals"""
    return d < col.n_docs and col.owner[d] == i and all(_VALUE[p](d) == v for p, v in zip(props, vals))


def _recipe_groups(col, params, groups, sorts, promote):
    """The collection rows of the recipe: docs, scores, values [R, S], n [R]."""
    rows, S = [], 0
    for b, g in enumerate(groups):
        if g is None:
            continue
        gbs, m = g
        keys, maps = E.collection_group_keys(gbs)
        prom = None if promote is None else [promote[b]]
        active = prom is not None and len(prom[0]) > 0
        if params.query_params is not None:
            e = params.query_params[b]
            pb = dataclasses.replace(params, query_params=None, mode=e.mode, limit_hint=e.limit, offset=e.offset,
                                     similarity=e.similarity, threshold=e.threshold)
        else:
            pb = params
        L, O = pb.limit_hint, pb.offset
        pi = dataclasses.replace(pb, limit_hint=(L + O) * (2 if active else 1), offset=0, vector_limit=L)
        srt = None if sorts is None else sorts[0][b]
        depth = m * (2 if active else 1)
        lists = [[] for _ in keys]
        members = [[] for _ in keys]
        item_sc = None
        for i, part in enumerate(col.parts):
            if gbs[i] is None:
                per = None
                if prom is not None:   # the index's item lookups still count for the item scores
                    per = _index_groups(_part_b(part, b), pi, None, 0, None if sorts is None else sorts[i][b], prom)
            else:
                per = _index_groups(_part_b(part, b), pi, gbs[i], depth, None if sorts is None else sorts[i][b], prom)
                gd, gs, gsv, gn = per[:4]
                for lg in range(gbs[i].n_groups):
                    k = int(maps[i][lg])
                    lists[k].append([(int(gd[lg, j]), gs[lg, j], gsv[lg, j]) for j in range(int(gn[lg]))])
                    members[k].append((i, gbs[i].properties, gbs[i].values[lg]))
            if prom is not None and item_sc is None:
                item_sc = [None] * len(prom[0])
            if prom is not None:
                for j in range(len(prom[0])):
                    if item_sc[j] is None and per[5][j]:
                        item_sc[j] = per[4][j]
        for k in range(len(keys)):
            if srt is None:
                merged = sorted([e for l in lists[k] for e in l], key=lambda e: (-float(e[1]), e[0]))
            else:
                desc = srt[1] == "DESC"
                tagged = [(e, i, j) for i, l in enumerate(lists[k]) for j, e in enumerate(l)]
                merged = [t[0] for t in sorted(tagged, key=lambda t: ((-t[0][2]) if desc else t[0][2], t[1], t[2]))]
            merged = merged[:depth]
            if active:
                items = [(d, pos, np.float32(0) if item_sc[j] is None else item_sc[j]) for j, (d, pos) in enumerate(prom[0])]
                merged = _splice(merged, items, lambda d, k=k: any(_member(col, i, props, vals, d) for i, props, vals in members[k]))
            if srt is None:
                merged = [(d, s, np.nan) for d, s, _ in merged]
            rows.append(merged)
            S = max(S, len(merged))
    return rows


def _same_groups(got, rows):
    gd, gs, gsv, gn = got[7], got[8], got[9], got[10]
    assert gn.tolist() == [len(r) for r in rows]
    for r, exp in enumerate(rows):
        k = len(exp)
        assert gd[r, :k].tolist() == [e[0] for e in exp]
        assert np.array_equal(gs[r, :k].view(np.uint32), np.asarray([e[1] for e in exp], np.float32).view(np.uint32))
        assert np.array_equal(gsv[r, :k].view(np.uint64), np.asarray([e[2] for e in exp], np.float64).view(np.uint64))
        assert not gd[r, k:].any() and not gs[r, k:].any() and not gsv[r, k:].any()


def _plain(ctx, col, params, sorts=None, promote=None):
    return E.search_indexes_arrays(ctx, col.parts, params, sorts, promote)


def _check(ctx, col, params, groups, sorts=None, promote=None):
    got = E.search_indexes_arrays(ctx, col.parts, params, sorts, promote, groups=groups)
    plain = _plain(ctx, col, params, sorts, promote)
    for a, b in zip(got[:7], plain):   # the hits, counts and pin outputs do not change
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    _same_groups(got, _recipe_groups(col, params, groups, sorts, promote))
    return got


@pytest.mark.parametrize("how", ["mod", "range"])
@pytest.mark.parametrize("n", [1, 2, 3, 5])
@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID])
def test_groups_score_order(gpu_ctx, cols, how, n, mode):
    col = cols(n - 1 if n == 5 else n, how, empty=n == 5)
    p = ob.TokenScoreParams(mode=mode, limit_hint=10, offset=3, similarity=0.0)
    for props, m in ((["cat"], 7), (["num", "flag"], 1), (["cat"], 0)):
        _check(gpu_ctx, col, p, [(col.group_by(props), m)] * B)


def test_groups_max_results_512(gpu_ctx, cols):
    col = cols(3, "mod")
    _check(gpu_ctx, col, ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=20, similarity=0.0), [(col.group_by(["cat"]), 512)] * B)


@pytest.mark.parametrize("order", ["ASC", "DESC"])
def test_groups_field_order(gpu_ctx, cols, order):
    col = cols(3, "range")
    fields = [ob.SortField.from_facets(p.store, "num") for p in col.parts]
    try:
        sorts = [[(f, order)] * B for f in fields]
        p = ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=8, similarity=0.0)
        _check(gpu_ctx, col, p, [(col.group_by(["cat"]), 7)] * B, sorts)
        rng = np.random.default_rng(5)
        promote = [[(int(rng.integers(N)), int(rng.integers(6))) for _ in range(b % 4)] for b in range(B)]
        _check(gpu_ctx, col, p, [(col.group_by(["cat"]), 5)] * B, sorts, promote)
    finally:
        for f in fields:
            f.close()


def test_groups_active_pins(gpu_ctx, cols):
    col = cols(2, "mod")
    rng = np.random.default_rng(9)
    hits = _plain(gpu_ctx, col, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=30))[0]
    promote = []
    for b in range(B):   # items that are hits, others that match nothing, one promoted twice
        it = [(int(hits[b, j]), int(rng.integers(8))) for j in range(0, 6, 2) if hits[b, j]]
        it += [(int(rng.integers(N)), int(rng.integers(8))) for _ in range(b % 3)]
        if b % 4 == 1 and it:
            it.append((it[0][0], 0))
        promote.append(it)
    for mode in (MODE_FULLTEXT, MODE_HYBRID):
        p = ob.TokenScoreParams(mode=mode, limit_hint=10, offset=2, similarity=0.0)
        _check(gpu_ctx, col, p, [(col.group_by(["cat"]), 4)] * B, promote=promote)
        _check(gpu_ctx, col, p, [(col.group_by(["num"]), 1)] * B, promote=promote)


def test_groups_mixed_batch_and_missing_property(gpu_ctx, cols):
    col = cols(2, "range", empty=True)
    g1, g2, g3 = col.group_by(["cat"]), col.group_by(["flag", "num"]), col.group_by(["only1"])
    groups = [None if b % 4 == 0 else (g1, 3) if b % 4 == 1 else (g2, 6) if b % 4 == 2 else (g3, 2) for b in range(B)]
    qp = [ob.QueryParams(mode=[MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID][b % 3], limit=5 + b % 4, offset=b % 3, similarity=0.0)
          for b in range(B)]
    p = ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=10, similarity=0.0, query_params=qp)
    got = _check(gpu_ctx, col, p, groups)
    assert got[11].tolist()[-1] == sum(0 if g is None else len(E.collection_group_keys(g[0])[0]) for g in groups)


def where_programs(part, where):
    """per query b: `where[b]` (a where clause, or None) compiled over the index's filter fields"""
    return [None if w is None else compile_where(parse_where(w), part.store, {}, part.store.nbits) for w in where]


@pytest.mark.parametrize("kind", ["q_filters", "where_programs"])
def test_groups_filters_and_omc(gpu_ctx, cols, kind):
    col = cols(3, "mod")
    base = list(col.parts)
    try:
        for i, part in enumerate(col.parts):
            docs = np.arange(N, dtype=np.uint64)[np.arange(N) % 3 == i]
            fields = {"omc_doc_ids": docs[::7].copy(), "omc_mult": np.full(docs[::7].shape[0], 1.5, np.float32)}
            if kind == "q_filters":
                flt = ob.DeviceFilter.from_ids(gpu_ctx, docs[docs % 2 == 0], N)
                fields["device_filters"] = [flt if b % 2 else None for b in range(B)]
            else:
                fields["where_programs"] = where_programs(part, [None if b % 2 == 0 else {"flag": True} if b % 4 == 1 else
                                                                 {"num": {"gte": 0}} for b in range(B)])
            col.parts[i] = dataclasses.replace(part, fields=fields)
        _check(gpu_ctx, col, ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=10, similarity=0.0), [(col.group_by(["cat"]), 5)] * B)
    finally:
        col.parts[:] = base


# ---------------------------------------------------------------- active pins against the reference's rule
N_SMALL, B_SMALL = 600, 8


@pytest.fixture(scope="module")
def small_corpus():
    rows = synth.make_vectors(N_SMALL, DIM, seed=91)
    qv, _ = synth.make_vector_queries(rows, B_SMALL, seed=92)
    data = synth.make_text_corpus(N_SMALL, 120, seed=93)
    texts = synth.make_text_queries(120, B_SMALL, seed=94)
    return rows, qv, data, texts


def _union_map(col, mode, L):
    """per query the union of the indexes' whole score maps {doc: score}: each index through oc_search at limit
    OC_MAX_TOPK, vector_limit = L (the collection's vector depth); the map must fit (count <= OC_MAX_TOPK)"""
    maps = [dict() for _ in range(B_SMALL)]
    for part in col.parts:
        d, s, n, c = part.tsc.execute_batch_arrays(ob.TokenScoreParams(mode=mode, limit_hint=1024, vector_limit=L, similarity=0.0),
                                                   part.texts, part.q_vecs)
        for b in range(B_SMALL):
            assert int(n[b]) == int(c[b]) <= 1024   # the whole map came back
            for j in range(int(n[b])):
                maps[b][int(d[b, j])] = s[b, j]
    return maps


def _reference_groups(score_map, vals, m, items):
    """sort_groups (the top 2 x m members of the map, score desc, ties by doc, NaN dropped; read/sort.rs:129-230) and
    apply_pin_rules_to_group (the items whose document is a member, with its map value or 0.0; read/sort.rs:377-391),
    for the group of documents whose category is vals[0]"""
    member = lambda d: d < N_SMALL and CATS[d % 4] == vals[0]   # noqa: E731
    top = sorted((d for d, sc in score_map.items() if member(d) and sc == sc), key=lambda d: (-float(score_map[d]), d))
    top = [(d, score_map[d]) for d in top[:2 * m if items else m]]
    its = [(pos, j, d) for j, (d, pos) in enumerate(items) if member(d)]
    if not its:
        return top
    drop = {d for _, _, d in its}
    out = [e for e in top if e[0] not in drop]
    for pos, _, d in sorted(its):
        out.insert(min(pos, len(out)), (d, score_map.get(d, np.float32(0.0))))
    return out


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID])
@pytest.mark.parametrize("n", [2, 3])
def test_groups_active_pins_against_the_reference_rule(gpu_ctx, small_corpus, mode, n):
    col = Collection(gpu_ctx, small_corpus, n, "mod")
    try:
        L, m = 10, 4
        maps = _union_map(col, mode, L)
        rng = np.random.default_rng(17 + n)
        promote = []
        for b in range(B_SMALL):   # keys of the map, documents outside it, a promoted document listed twice; b = 0: none
            keys = sorted(maps[b])
            it = [(int(keys[int(rng.integers(len(keys)))]), int(rng.integers(6))) for _ in range(3 if keys else 0)]
            it += [(int(rng.integers(N_SMALL)), int(rng.integers(6))) for _ in range(2)]
            if b % 3 == 1:
                it.append((it[0][0], 0))
            promote.append(it if b else [])
        groups = [(col.group_by(["cat"]), m)] * B_SMALL
        p = ob.TokenScoreParams(mode=mode, limit_hint=L, similarity=0.0)
        got = E.search_indexes_arrays(gpu_ctx, col.parts, p, promote=promote, groups=groups)
        gd, gs, gn, rows, keys = got[7], got[8], got[10], got[11], got[12]
        for b in range(B_SMALL):
            assert len(keys[b]) == len(CATS)
            for k, vals in enumerate(keys[b]):
                r = int(rows[b]) + k
                exp = _reference_groups(maps[b], vals, m, promote[b])
                assert gd[r, :gn[r]].tolist() == [d for d, _ in exp]
                es = np.asarray([sc for _, sc in exp], np.float32)
                assert np.array_equal(gs[r, :gn[r]].view(np.uint32), es.view(np.uint32))
    finally:
        col.close()


def test_groups_around_a_commit(gpu_ctx, corpus):
    col = Collection(gpu_ctx, corpus, 2, "mod")
    try:
        gb = col.group_by(["cat"])
        p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10)
        _check(gpu_ctx, col, p, [(gb, 5)] * B)
        for i, part in enumerate(col.parts):
            part.tsc.str.delete(np.arange(i, N, 2 * 7, dtype=np.uint64))   # tombstones before the commit
        _check(gpu_ctx, col, p, [(gb, 5)] * B)
        for part in col.parts:
            part.tsc.str.commit()
        _check(gpu_ctx, col, p, [(gb, 5)] * B)
    finally:
        col.close()


# ---------------------------------------------------------------- refusals
def _raw(ctx, col, p, n_keys, max_res, keymaps, gbs, stride, foff=None, freqs=None, fslots=None, fstore=None):
    """oc_search_indexes_ex with hand-made key maps; returns (code, outputs)"""
    keep, ixs = [], (_lib.IndexQuery * len(col.parts))()
    for i, part in enumerate(col.parts):
        sp, k, _ = part.tsc._build_params(p, part.texts, part.q_vecs)
        keep += [sp, k]
        ixs[i] = _lib.IndexQuery(part.tsc.emb._h, part.tsc.str._h, C.pointer(sp), None)
    ex = (_lib.IndexExtras * len(col.parts))()
    for i in range(len(col.parts)):
        if gbs[i] is not None:
            a = (C.c_void_p * B)(*([gbs[i]._h] * B))
            km = (C.c_void_p * B)(*([keymaps[i].ctypes.data] * B))
            keep += [a, km]
            ex[i].q_groups, ex[i].q_group_keys = C.cast(a, C.c_void_p), C.cast(km, C.c_void_p)
        if freqs is not None and i == 0:
            arr = (_lib.FacetReq * len(freqs))(*[_lib.FacetReq(*r) for r in freqs])
            sl = np.asarray(fslots, np.uint32)
            keep += [arr, sl]
            ex[i].facets, ex[i].n_facet_reqs, ex[i].facet_reqs, ex[i].facet_slots = fstore._h, len(freqs), C.cast(arr, C.c_void_p), sl.ctypes.data
    L, R = p.limit_hint, int(np.sum(n_keys))
    sentinel = 0xAB
    outs = [np.full((B, L), sentinel, np.uint64), np.zeros((B, L), np.float32),
            np.zeros((B, L)), np.zeros(B, np.uint32), np.zeros(B, np.uint64), np.zeros(1, np.float32), np.zeros(1, np.uint8),
            np.full((max(R, 1), max(stride, 1)), sentinel, np.uint64), np.zeros((max(R, 1), max(stride, 1)), np.float32),
            np.zeros((max(R, 1), max(stride, 1))), np.full(max(R, 1), sentinel, np.uint32), np.full(64, sentinel, np.uint64)]
    nk, mr = np.asarray(n_keys, np.uint32), np.asarray(max_res, np.uint32)
    fo = None if foff is None else np.asarray(foff, np.uint32)
    code = _lib.lib().oc_search_indexes_ex(ctx._h, len(col.parts), ixs, ex, None, E._p(nk), E._p(mr), stride, E._p(fo),
                                           *[E._p(o) for o in outs])
    return code, outs


def test_refusals_write_nothing(gpu_ctx, cols):
    col = cols(2, "mod")
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=5)
    gbs = col.group_by(["cat"])
    good = [np.arange(4, dtype=np.uint32), np.arange(4, dtype=np.uint32)[::-1].copy()]
    code, outs = _raw(gpu_ctx, col, p, [4] * B, [3] * B, good, gbs, 3)
    assert code == 0 and outs[10].max() <= 3

    INVALID, UNSUPPORTED = -1, -4

    def refused(code_expected, text, *a, **kw):   # each case fails its own check: its code and its message
        code, outs = _raw(gpu_ctx, col, *a, **kw)
        assert code == code_expected
        assert text in _lib.lib().oc_last_error().decode()
        assert (outs[0] == 0xAB).all() and (outs[7] == 0xAB).all() and (outs[10] == 0xAB).all() and (outs[11] == 0xAB).all()

    refused(INVALID, ">= q_n_keys", p, [4] * B, [3] * B, [good[0], np.array([0, 1, 2, 4], np.uint32)], gbs, 3)
    refused(INVALID, "have one key", p, [4] * B, [3] * B, [good[0], np.array([0, 1, 1, 2], np.uint32)], gbs, 3)
    refused(INVALID, "group_stride 2 <", p, [4] * B, [3] * B, good, gbs, 2)
    refused(UNSUPPORTED, "max_results 2000 >", p, [4] * B, [2000] * B, good, gbs, 2000)
    refused(INVALID, "limit must be >= 1", dataclasses.replace(p, limit_hint=0), [4] * B, [3] * B, good, gbs, 3)
    st = col.parts[0].store
    fid = st.fields["cat"]["id"]
    foff = [2 * b for b in range(B + 1)]
    refused(INVALID, f"slot {2 * B} outside", p, [4] * B, [3] * B, good, gbs, 3, foff, [(fid, 0, 0, 0)], [2 * B], st)
    refused(INVALID, "two facet requests on slot 1", p, [4] * B, [3] * B, good, gbs, 3, foff, [(fid, 0, 0, 0), (fid, 1, 0, 0)], [1, 1], st)
    refused(INVALID, "unknown variant 99", p, [4] * B, [3] * B, good, gbs, 3, foff, [(fid, 99, 0, 0)], [1], st)
    other = ob.Context(0)
    try:
        ost = ob.FacetStore(other, N)
        ost.add_bool_field("b", [0], [1])
        refused(INVALID, "facets belong to another ctx", p, [4] * B, [3] * B, good, gbs, 3, foff, [(0, 0, 0, 0)], [1], ost)
        ogb = ob.GroupBy(ost, ["b"])
        refused(INVALID, "group_by of query 0 belongs to another ctx", p, [2] * B, [3] * B,
                [np.arange(2, dtype=np.uint32), good[1]], [ogb, gbs[1]], 3)
        ogb.close(); ost.close()
    finally:
        other.close()


def test_over_deep_pinned_groups_refused_alike(gpu_ctx, cols):
    """An active pinned query whose group lists would be 2 x max_results > OC_MAX_TOPK deep: oc_search_indexes_ex refuses
    it with the code and message oc_search_q_groups gives for one of its indexes."""
    col = cols(2, "mod")
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=5)
    gbs = col.group_by(["cat"])
    promote, part = [[(1, 0)]] * B, col.parts[0]
    calls = (lambda: E.search_indexes_arrays(gpu_ctx, col.parts, p, promote=promote, groups=[(gbs, 600)] * B, group_stride=2000),
             lambda: E.search_q_groups_arrays(part.tsc, dataclasses.replace(p, **dict(part.fields or {})), [(gbs[0], 600)] * B,
                                              promote, part.texts, part.q_vecs, group_stride=2000))
    for call in calls:
        with pytest.raises(ob.OcError) as e:
            call()
        assert e.value.code == -4   # OC_ERR_UNSUPPORTED
        assert "query 0: pins: 2 x max_results 1200 > 1024" in _lib.lib().oc_last_error().decode()
