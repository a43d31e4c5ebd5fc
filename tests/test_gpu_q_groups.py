"""One batch in which every query has its own groupBy, sortBy, pin rules and where-filter (oc_search_q_groups,
search_q_groups_arrays) and the batcher's grouped requests (oc_batcher_search_groups, SearchBatcher.search_groups).

The rule: query b's outputs — hits, score bits, sort values, n, count, its items' pin scores and present flags, and its
group rows (ids, score bits, sort values, n) — equal, byte for byte, what it gets alone with its own filter and items:
oc_search_q_sorted without groups, oc_search_groups in score order without items, oc_search_groups_pinned in score
order with items, oc_search_groups_sorted with a sort.  Checked over fulltext / vector / hybrid, B in {1, 5, 48, 256},
limit 0, max_results in {0, 1, 3, 10}, handles of 1, 10, 20 and 1000 groups and queries without groups, the filter mix of
test_gpu_query_filters, tombstones and a commit between calls; plus the whole-batch equalities with the three grouped
calls, the oracle's score maps, every refusal, and many threads through the batcher."""
import ctypes as C
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib, synth
from oramacore_b200.engine import _p
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from test_gpu_q_sorted import _alone, _one, _promote, _sorts, _tsc
from test_gpu_q_sorted import fields  # noqa: F401  (fixture)
from test_gpu_query_filters import DIM, MODES, N, OC_ERR_INVALID, OC_ERR_UNSUPPORTED, _assign, _filters, _inputs
from test_gpu_query_filters import corpus  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def _facets(ctx, n, seed):
    """Handles of 1, 10, 20 (bool x string_filter) and 1000 groups over documents [0, n); `members` restates them."""
    rng = np.random.default_rng(seed)
    ids = np.arange(n)
    st = ob.FacetStore(ctx, n)
    st.add_string_field("one", {"all": ids})
    cat = rng.integers(0, 10, n)
    st.add_string_field("cat", {f"c{k}": ids[cat == k] for k in range(10)})
    flag = rng.random(n) < 0.4
    st.add_bool_field("flag", ids[flag], ids[~flag])
    num = (ids * 7919) % 1000
    st.add_number_field("num", ids, num.astype(np.float64))
    gbs = {1: ob.GroupBy(st, ["one"]), 10: ob.GroupBy(st, ["cat"]), 20: ob.GroupBy(st, ["flag", "cat"]),
           1000: ob.GroupBy(st, ["num"])}
    members = {1: [set(ids.tolist())], 10: [set(ids[cat == k].tolist()) for k in range(10)],
               20: [set(ids[(flag == f) & (cat == k)].tolist()) for f in (True, False) for k in range(10)],
               1000: [set(ids[num == v].tolist()) for v in range(1000)]}
    for k, gb in gbs.items():
        assert gb.n_groups == k
    return st, gbs, members


@pytest.fixture(scope="module")
def grouping(corpus):  # noqa: F811
    st, gbs, members = _facets(corpus["ctx"], N, 5)
    yield dict(gbs=gbs, members=members)
    for gb in gbs.values():
        gb.close()
    st.close()


def _requests(gbs, fs, B, seed, with_1000=True):
    """Per query None, or (GroupBy or None, max_results, sort): the handles, max_results 0 / 1 / 3 / 10 and the sort mix."""
    rng = np.random.default_rng(seed)
    sorts = _sorts(fs, B, seed)
    kinds = [10, 20, None, 1, 10, 1000 if with_1000 else 20, 20, None]
    out = []
    for b in range(B):
        k = kinds[b % len(kinds)] if b < len(kinds) else kinds[int(rng.integers(0, len(kinds)))]
        m = [1, 3, 10, 0, 3, 1][b % 6]
        out.append((None if k is None else gbs[k], m, sorts[b]))
    return out


def _single(tsc, mode, flt, req, items, text, qv, **kw):
    """One query alone, by the call the rule names: (docs, scores, sort values, n, count, pin scores, pin present,
    group docs [G, s], group scores, group sort values, group n [G]); no group arrays without groups."""
    gb, m, sort = req if req is not None else (None, 0, None)
    if gb is None:
        return _alone(tsc, mode, flt, sort, items, text, qv, **kw) + (None,) * 4
    p = ob.TokenScoreParams(mode=mode, device_filter=flt, **kw)
    if sort is None:
        d, s, n, cnt, gd, gs, gn = ob.search_groups_arrays(tsc, gb, p, m, text, qv, promote=[items] if items else None)
        sv = np.where(np.arange(d.shape[1])[None, :] < n[:, None], np.nan, 0.0)
        gsv = np.where(np.arange(gd.shape[2])[None, None, :] < gn[:, :, None], np.nan, 0.0)
    else:
        d, s, n, cnt, gd, gs, gn, sv, gsv = ob.search_groups_arrays(tsc, gb, p, m, text, qv, promote=[items], sort_by=sort)
    ps = pp = None
    if p.limit_hint:   # the items' values come from the same score map: the flat single call's
        ps, pp = _alone(tsc, mode, flt, sort, items, text, qv, **kw)[5:]
    return d, s, sv, n, cnt, ps, pp, gd[0], gs[0], gsv[0], gn[0]


def _check(tsc, mode, filters, reqs, promote, texts, qv, **kw):
    """The batch equals every query alone, byte for byte."""
    B = len(reqs)
    got = ob.search_q_groups_arrays(tsc, ob.TokenScoreParams(mode=mode, device_filters=filters, **kw), reqs, promote, texts, qv)
    d, s, sv, n, cnt, ps, pp, gd, gs, gsv, gn, rows = got
    off = np.cumsum([0] + [len(x) for x in promote])
    S = gd.shape[1]
    for b in range(B):
        one = _single(tsc, mode, None if filters is None else filters[b], reqs[b], promote[b],
                      None if texts is None else _one(texts, b), None if qv is None else qv[b:b + 1], **kw)
        r = reqs[b] or (None, 0, None)
        ctx = (b, mode, r[1], r[0] is not None and r[0].n_groups, r[2] and r[2][1], kw)
        for what, x, y in zip(("docs", "scores", "sort values", "n", "count"), (d, s.view(np.uint32), sv, n, cnt), one[:5]):
            y = y.view(np.uint32) if what == "scores" else y
            assert x[b].tobytes() == y[0].tobytes(), (what,) + ctx
        if one[5] is not None:
            assert ps[off[b]:off[b + 1]].tobytes() == one[5].tobytes(), ("pin scores",) + ctx
            assert pp[off[b]:off[b + 1]].tobytes() == one[6].tobytes(), ("pin present",) + ctx
        r0, r1 = int(rows[b]), int(rows[b + 1])
        if one[7] is None:
            assert r0 == r1
            continue
        w = one[7].shape[1]
        assert r1 - r0 == one[7].shape[0] and w <= S, ctx
        assert gn[r0:r1].tobytes() == one[10].tobytes(), ("group n",) + ctx
        for what, x, y in zip(("group docs", "group scores", "group sort values"), (gd, gs.view(np.uint32), gsv),
                              (one[7], one[8].view(np.uint32), one[9])):
            assert x[r0:r1, :w].tobytes() == np.ascontiguousarray(y).tobytes(), (what,) + ctx
            assert not x[r0:r1, w:].any(), (what + " past the single call's stride",) + ctx
    return got


@pytest.mark.parametrize("B", [1, 5, 48, 256])
@pytest.mark.parametrize("mode", list(MODES))
def test_batch_equals_each_query_alone(corpus, fields, grouping, mode, B):  # noqa: F811
    c = corpus
    m = MODES[mode]
    qv, texts = _inputs(B, 3100 + B, c["rows"])
    filters = _assign(c["fs"], B, B + 7) if B > 1 else [c["fs"]["d30"]]
    reqs = _requests(grouping["gbs"], fields, B, B) if B > 1 else [(grouping["gbs"][10], 3, (fields["price"], "DESC"))]
    _check(_tsc(c, m), m, filters, reqs, _promote(B, B + 1), texts if m != MODE_VECTOR else None,
           qv if m != MODE_FULLTEXT else None, similarity=0.0)


@pytest.mark.parametrize("mode", list(MODES))
def test_limit_zero(corpus, fields, grouping, mode):  # noqa: F811
    """limit 0 (every query grouped): no hits, no vector depth, the groups of each query alone."""
    c = corpus
    m = MODES[mode]
    B = 24
    qv, texts = _inputs(B, 3300, c["rows"])
    reqs = [r if r[0] is not None else (grouping["gbs"][20], r[1], r[2]) for r in _requests(grouping["gbs"], fields, B, 61)]
    _check(_tsc(c, m), m, _assign(c["fs"], B, 63), reqs, _promote(B, 65), texts if m != MODE_VECTOR else None,
           qv if m != MODE_FULLTEXT else None, similarity=0.0, limit_hint=0)


def test_whole_batch_equalities(corpus, fields, grouping):  # noqa: F811
    """Uniform requests without q_filters: oc_search_groups, oc_search_groups_pinned and oc_search_groups_sorted."""
    c = corpus
    B = 32
    qv, texts = _inputs(B, 3500, c["rows"])
    promote = _promote(B, 67)
    gb = grouping["gbs"][20]
    k = max(len(x) for x in promote)
    for mode in (MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID):
        tsc = _tsc(c, mode)
        t, q = (texts if mode != MODE_VECTOR else None), (qv if mode != MODE_FULLTEXT else None)
        for kw in (dict(similarity=0.0), dict(similarity=0.0, device_filter=c["fs"]["d30"], offset=2)):
            p = ob.TokenScoreParams(mode=mode, **kw)
            got = ob.search_q_groups_arrays(tsc, p, [(gb, 3)] * B, [[]] * B, t, q)
            ref = ob.search_groups_arrays(tsc, gb, p, 3, t, q)
            for x, y in zip((got[0], got[1], got[3], got[4], got[7], got[8], got[10]), ref):
                assert x.tobytes() == y.reshape(x.shape).tobytes(), (mode, kw)
            got = ob.search_q_groups_arrays(tsc, p, [(gb, 3)] * B, promote, t, q, group_stride=6 + k)
            ref = ob.search_groups_arrays(tsc, gb, p, 3, t, q, promote=promote)
            for x, y in zip((got[0], got[1], got[3], got[4], got[7], got[8], got[10]), ref):
                assert x.tobytes() == y.reshape(x.shape).tobytes(), (mode, kw)
            srt = (fields["date"], "DESC")
            got = ob.search_q_groups_arrays(tsc, p, [(gb, 3, srt)] * B, promote, t, q, group_stride=6 + k)
            ref = ob.search_groups_arrays(tsc, gb, p, 3, t, q, promote=promote, sort_by=srt)
            for x, y in zip((got[0], got[1], got[3], got[4], got[7], got[8], got[10], got[2], got[9]),
                            (ref[0], ref[1], ref[2], ref[3], ref[4], ref[5], ref[6], ref[7], ref[8])):
                assert x.tobytes() == y.reshape(x.shape).tobytes(), (mode, kw)


def test_against_the_oracle(corpus, grouping, orc):  # noqa: F811
    """sort_groups restated over the oracle's fulltext score map of each query's own filter: per group the top
    max_results members that are keys, by score descending, ties by ascending id (test_gpu_groups' restatement)."""
    c = corpus
    B = 16
    qv, texts = _inputs(B, 3700, c["rows"])
    filters = _assign(c["fs"], B, 71)
    ks = [10, 20, 1, 10, 20, 1000, 10, 20] * 2
    ms = [1, 3, 10, 0] * 4
    reqs = [(grouping["gbs"][k], m) for k, m in zip(ks, ms)]
    got = ob.search_q_groups_arrays(_tsc(c, MODE_FULLTEXT), ob.TokenScoreParams(mode=MODE_FULLTEXT, device_filters=filters),
                                    reqs, None, texts)
    gd, gs, gn, rows = got[7], got[8], got[10], got[11]
    ix = orc.StrIndex(c["data"])
    for b in range(B):
        f = filters[b]
        kw = {} if f is None else dict(filter_bits=f.read(), filter_nbits=f.nbits)
        d, s = orc.fulltext(ix, texts[b], **kw)
        sm = dict(zip(d.tolist(), s.tolist()))
        for g, mem in enumerate(grouping["members"][ks[b]]):
            cand = sorted(((x, sm[x]) for x in mem if x in sm), key=lambda t: (-np.float32(t[1]), t[0]))[:ms[b]]
            r = int(rows[b]) + g
            k = int(gn[r])
            assert gd[r, :k].tolist() == [x for x, _ in cand], (b, g)
            assert np.allclose(gs[r, :k], [y for _, y in cand], rtol=0, atol=1e-5), (b, g)


def test_tombstones_and_commit(gpu_ctx):
    """Uncommitted deletes, then an oc_str_commit between calls: every handle's rows are mapped again."""
    n = 30_000
    rows = synth.make_vectors(n, DIM, seed=271)
    data = synth.make_text_corpus(n, 3000, seed=273)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    rng = np.random.default_rng(275)
    fs = _filters(gpu_ctx, n, rng)
    st, gbs, _ = _facets(gpu_ctx, n + 10, 277)
    ids = np.arange(n + 10, dtype=np.uint64)
    a = ob.SortField(gpu_ctx, n + 10, ids, rng.integers(0, 30, n + 10).astype(np.float64), "number")
    try:
        tsc = ob.TokenScoreContext(gpu_ctx, emb, strs)
        B = 40
        qv, texts = _inputs(B, 279, rows)
        filters = _assign(fs, B, 5)
        reqs = [[(gbs[10], 3, None), (gbs[20], 1, (a, "ASC")), None, (gbs[1000], 2, (a, "DESC")), (None, 0, (a, "ASC"))][i % 5]
                for i in range(B)]
        promote = _promote(B, 281, n)
        gone = rng.choice(n, 2000, replace=False).tolist()
        strs.delete(gone)
        emb.delete(gone)
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            _check(tsc, mode, filters, reqs, promote, texts, qv, similarity=0.0)
        strs.commit()
        t0 = [int(x) for x in texts[0].term_id[:1]]
        for d in range(n, n + 10):   # new documents that match query 0
            strs.insert(d, 0, 3, {t0[0]: 2})
        strs.commit()
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            _check(tsc, mode, filters, reqs, promote, texts, qv, similarity=0.0)
    finally:
        for f in fs.values():
            f.close()
        for gb in gbs.values():
            gb.close()
        st.close(); a.close(); emb.close(); strs.close()


def test_refusals(corpus, fields, grouping, gpu_ctx):  # noqa: F811
    c = corpus
    L = _lib.lib()
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    B = 4
    qv, texts = _inputs(B, 3900, c["rows"])
    other = ob.Context(0)
    foreign = ob.DeviceFilter.from_ids(other, [1, 2, 3], N)
    foreign_sort = ob.SortField(other, N, [1, 2], [1.0, 2.0], "number")
    ost, ogbs, _ = _facets(other, 2000, 3)
    g10, g20 = grouping["gbs"][10]._h, grouping["gbs"][20]._h
    items = (np.asarray([0, 1, 1, 2, 2], np.uint32), np.asarray([5, 6], np.uint64), np.asarray([0, 1], np.uint32))
    try:
        def run(reqs, promote=None, stride=16, fl=(c["fs"]["share"], None, c["fs"]["d30"], None), null_reqs=False, edit=None, **kw):
            sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filters=fl, **kw), texts, qv)
            if edit:
                keep.append(edit(sp))
            arr = (_lib.GroupReq * B)()
            for i, r in enumerate(reqs):
                if r is not None:
                    arr[i].groups, arr[i].max_results = r[0], r[1]
                    if len(r) > 2:
                        arr[i].sort = _lib.Sort(*r[2])
            pins = None
            if promote is not None:
                pins = _lib.Pins(_p(promote[0]), _p(promote[1]), _p(promote[2]), 1)
            lim = kw.get("limit_hint", 10)
            d = np.full((B, max(lim, 1)), 7, np.uint64); s = np.full((B, max(lim, 1)), 7, np.float32)
            v = np.full((B, max(lim, 1)), 7, np.float64)
            n = np.full(B, 7, np.uint32); cnt = np.full(B, 7, np.uint64); ps = np.full(8, 7, np.float32); pp = np.full(8, 7, np.uint8)
            gd = np.full(4 * 20 * stride + 1, 7, np.uint64); gs = np.full(gd.shape, 7, np.float32)
            gv = np.full(gd.shape, 7, np.float64); gn = np.full(4 * 20, 7, np.uint32)
            rc = L.oc_search_q_groups(c["ctx"]._h, c["emb"]._h, c["strs"]._h, C.byref(sp), None if null_reqs else arr,
                                      None if pins is None else C.byref(pins), stride, _p(d), _p(s), _p(v), _p(n), _p(cnt),
                                      _p(ps), _p(pp), _p(gd), _p(gs), _p(gv), _p(gn))
            for a in (d, s, v, n, cnt, ps, pp, gd, gs, gv, gn):
                assert (a == 7).all()   # nothing written
            return rc

        good = [(g10, 3, (fields["price"]._h, 0)), None, (g20, 1), (g10, 0, (fields["date"]._h, 1))]
        assert run(good, null_reqs=True) == OC_ERR_INVALID
        assert run([(g10, 3, (fields["price"]._h, 2)), None, None, None]) == OC_ERR_INVALID          # bad order
        assert run([(g10, 3, (foreign_sort._h, 0)), None, None, None]) == OC_ERR_INVALID            # sort field of another ctx
        assert run([(ogbs[10]._h, 3), None, None, None]) == OC_ERR_INVALID                          # group_by of another ctx
        assert run(good, fl=(c["fs"]["share"], foreign, None, None)) == OC_ERR_INVALID              # filter of another ctx
        assert run(good, edit=lambda sp: setattr(sp, "filter", c["fs"]["all"]._h)) == OC_ERR_INVALID
        bits = np.zeros((N + 63) // 64, np.uint64)

        def with_bits(sp):
            sp.filter_bits, sp.filter_nbits = _p(bits), N
        assert run(good, edit=with_bits) == OC_ERR_INVALID
        assert run(good, promote=(np.asarray([0, 2, 1, 2, 2], np.uint32), items[1], items[2])) == OC_ERR_INVALID   # not monotone
        assert run(good, stride=2) == OC_ERR_INVALID                                                 # below max_results 3
        assert run([(g10, 5), None, None, None], promote=items, stride=10) == OC_ERR_INVALID         # active: 2 x 5 + 1
        assert run(good, limit_hint=0) == OC_ERR_INVALID                                             # a query without groups
        assert run(good, edit=lambda sp: setattr(sp, "sharded", 1)) == OC_ERR_UNSUPPORTED
        assert run([(g10, 1025), None, None, None], stride=1025) == OC_ERR_UNSUPPORTED               # max_results > OC_MAX_TOPK
        assert run([(g10, 600), None, None, None], promote=items, stride=1201) == OC_ERR_UNSUPPORTED  # active: 2 x 600
        assert run(good, limit_hint=1000, offset=100) == OC_ERR_UNSUPPORTED                          # limit + offset
        assert run(good, promote=items, limit_hint=500, offset=100) == OC_ERR_UNSUPPORTED            # active: 2 x (limit + offset)
        # the batcher refuses before joining: a stride below the need, a bad order, malformed pins, foreign handles
        bat = ob.SearchBatcher(tsc, max_batch=8, max_wait_us=100)
        try:
            sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0), [texts[0]], qv[0:1])
            for req, pins, stride in (((g10, 3), None, 2), ((g10, 3, (fields["price"]._h, 5)), None, 3),
                                      ((g10, 3), _lib.Pins(_p(np.asarray([1, 0], np.uint32)), None, None, 1), 8),
                                      ((ogbs[10]._h, 3), None, 3), ((g10, 3, (foreign_sort._h, 0)), None, 3)):
                r = _lib.GroupReq(req[0], req[1], _lib.Sort(*req[2]) if len(req) > 2 else _lib.Sort(None, 0))
                d = np.full(10, 7, np.uint64); s = np.full(10, 7, np.float32); n = np.full(1, 7, np.uint32)
                cnt = np.full(1, 7, np.uint64); gd = np.full(10 * 8, 7, np.uint64); gs = np.full(10 * 8, 7, np.float32)
                gn = np.full(10, 7, np.uint32)
                rc = L.oc_batcher_search_groups(bat._h, C.byref(sp), C.byref(r), None if pins is None else C.byref(pins), stride,
                                                _p(d), _p(s), None, _p(n), _p(cnt), None, None, _p(gd), _p(gs), None, _p(gn))
                assert rc == OC_ERR_INVALID
                assert (d == 7).all() and (n == 7).all() and (cnt == 7).all() and (gd == 7).all() and (gn == 7).all()
            assert bat.stats() == {"queries": 0, "batches": 0, "direct": 0}
            # a request the merged call would refuse runs alone and gets the library's error
            p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0)
            with pytest.raises(ob.OcError) as e:
                bat.search_groups(p, (grouping["gbs"][10], 1025), None, texts[0], qv[0])
            assert e.value.code == OC_ERR_UNSUPPORTED
            assert bat.stats()["direct"] == 1
        finally:
            bat.close()
    finally:
        for gb in ogbs.values():
            gb.close()
        ost.close()
        foreign_sort.close()
        foreign.close()
        other.close()


def test_batcher_coalesces_grouped_requests(corpus, fields, grouping):  # noqa: F811
    """Threads mix grouped (search_groups), sorted (search_sorted) and plain (search) requests; each answer equals the
    direct B = 1 call, grouped requests use strides above their need, and the batcher coalesces."""
    c = corpus
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    T, Q = 12, 24
    qv, texts = _inputs(T * Q, 4100, c["rows"])
    filters = _assign(c["fs"], T * Q, 81)
    reqs = _requests(grouping["gbs"], fields, T * Q, 83, with_1000=False)
    promote = _promote(T * Q, 85)
    kind = [("plain", "sorted", "grouped", "grouped", "grouped")[i % 5] for i in range(T * Q)]
    expect = {}
    for i in range(T * Q):
        p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i])
        if kind[i] == "plain":
            expect[i] = tsc.execute_batch_arrays(p, [texts[i]], qv[i:i + 1])
        elif kind[i] == "sorted":
            expect[i] = _alone(tsc, MODE_HYBRID, filters[i], reqs[i][2], promote[i], [texts[i]], qv[i:i + 1], similarity=0.0)
        else:
            pd = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filters=[filters[i]])
            expect[i] = ob.search_q_groups_arrays(tsc, pd, [reqs[i]], [promote[i]], [texts[i]], qv[i:i + 1])
    bat = ob.SearchBatcher(tsc, max_batch=64, max_wait_us=3000)
    bad = []

    def worker(t):
        for i in range(t, T * Q, T):
            p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i])
            e = expect[i]
            if kind[i] == "plain":
                h = bat.search(p, texts[i], qv[i])
                k = int(e[2][0])
                ok = h.count == int(e[3][0]) and h.doc_ids.tobytes() == e[0][0, :k].tobytes() and h.scores.tobytes() == e[1][0, :k].tobytes()
            elif kind[i] == "sorted":
                h, sv, ps, pp = bat.search_sorted(p, reqs[i][2], promote[i] if promote[i] else None, texts[i], qv[i])
                k = int(e[3][0])
                ok = (h.count == int(e[4][0]) and h.doc_ids.tobytes() == e[0][0, :k].tobytes()
                      and h.scores.tobytes() == e[1][0, :k].tobytes() and sv.tobytes() == e[2][0, :k].tobytes())
            else:
                own = e[7].shape[1] + i % 3   # a stride above the need: the rows come back at it, padded with 0
                r = bat.search_groups(p, reqs[i], promote[i] if promote[i] else None, texts[i], qv[i], group_stride=own)
                ok = all(x.tobytes() == y[0].tobytes() for x, y in zip(r[:3], e[:3]))
                ok = ok and r[3] == e[3][0] and r[4] == e[4][0] and r[5].tobytes() == e[5].tobytes() and r[6].tobytes() == e[6].tobytes()
                w = e[7].shape[1]
                for x, y in zip(r[7:10], e[7:10]):
                    ok = ok and x[:, :w].tobytes() == np.ascontiguousarray(y).tobytes() and not x[:, w:].any()
                ok = ok and r[10].tobytes() == e[10].tobytes()
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
