"""Per-query facets in the batched grouped call (oc_search_q_facets, search_q_facets_arrays) and the batcher's faceted
requests (oc_batcher_search_faceted, SearchBatcher.search_faceted).

The rule: query b's hits, scores, sort values, n, count, pin outputs and group rows equal, byte for byte, what
oc_search_q_groups gives the same batch without facets; query b's facet counts equal what oc_search_facets gives it
alone (B = 1, its own requests, its where-filter ignored).  Checked over fulltext / vector / hybrid, identity and sparse
document ids, B up to 64, a mix of queries without facets, bool, string_filter and number-range facets, repeated and
overlapping requests, an empty range and from > to, each with and without a filter, groups, a sort and pins; against a
numpy count over the oracle's unfiltered score maps (OMC, a threshold, tombstones, a commit); the reference's pinned
facet answers inside a mixed batch; limit 0; every refusal; and many threads through the batcher."""
import ctypes as C
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import build_index
from oramacore_b200 import _lib, synth
from oramacore_b200.engine import _p
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from test_gpu_q_groups import _facets, _requests
from test_gpu_q_sorted import _one, _promote, _tsc
from test_gpu_q_sorted import fields  # noqa: F401  (fixture)
from test_gpu_query_filters import DIM, MODES, N, OC_ERR_INVALID, OC_ERR_UNSUPPORTED, _assign, _filters, _inputs
from test_gpu_query_filters import corpus  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

_RANGES = [{"from": 0, "to": 100}, {"from": 50, "to": 500}, {"from": 0, "to": 100}]   # overlapping and repeated
_MIX = [None,
        {"flag": {"true": True, "false": True}},
        {"cat": {}},
        {"num": {"ranges": _RANGES}},
        {"num": {"ranges": [{"from": 2000, "to": 3000}, {"from": 10, "to": 5}]}},   # an empty range and from > to
        {"flag": {"true": True}, "cat": {}, "num": {"ranges": [{"from": 900, "to": 999}]}},
        {"cat": {}, "flag": {"false": True}},
        {"cat": {}}]


def _mix(B, seed):
    rng = np.random.default_rng(seed)
    return [_MIX[b] if b < len(_MIX) else _MIX[int(rng.integers(0, len(_MIX)))] for b in range(B)]


@pytest.fixture(scope="module")
def faceting(corpus):  # noqa: F811
    st, gbs, members = _facets(corpus["ctx"], N, 5)
    yield dict(st=st, gbs=gbs)
    for gb in gbs.values():
        gb.close()
    st.close()


def _facets_alone(tsc, st, mode, flt, facets, text, qv, **kw):
    """oc_search_facets of one query alone: its counts in request order."""
    reqs, _ = ob.facet_requests(st, facets)
    sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=mode, device_filter=flt, **kw), text, qv)
    arr = (_lib.FacetReq * max(len(reqs), 1))(*[_lib.FacetReq(*r) for r in reqs])
    out = np.zeros(max(len(reqs), 1), np.uint64)
    rc = _lib.lib().oc_search_facets(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, st._h,
                                     C.byref(sp), arr, len(reqs), _p(out))
    assert rc == 0, _lib.lib().oc_last_error()
    return out[:len(reqs)]


def _check(tsc, st, mode, filters, groups, promote, facets, texts, qv, alone_kw=None, **kw):
    """Hits and groups equal oc_search_q_groups of the same batch; counts equal oc_search_facets of each query alone."""
    B = len(facets)
    p = ob.TokenScoreParams(mode=mode, device_filters=filters, **kw)
    got = ob.search_q_facets_arrays(tsc, st, p, facets, groups, promote, texts, qv)
    ref = ob.search_q_groups_arrays(tsc, p, groups if groups is not None else [None] * B, promote, texts, qv)
    names = ("docs", "scores", "sort values", "n", "count", "pin scores", "pin present", "group docs", "group scores",
             "group sort values", "group n", "rows")
    for what, x, y in zip(names, got[:12], ref):
        assert x.tobytes() == y.tobytes(), (what, mode, B, kw)
    fc, foff = got[12], got[13]
    for b in range(B):
        if not facets[b]:
            assert foff[b + 1] == foff[b]
            continue
        one = _facets_alone(tsc, st, mode, None if filters is None else filters[b], facets[b],
                            None if texts is None else _one(texts, b), None if qv is None else qv[b:b + 1], **(alone_kw or kw))
        assert fc[foff[b]:foff[b + 1]].tolist() == one.tolist(), (b, mode, facets[b], filters is not None and filters[b] is not None)
    return got


@pytest.mark.parametrize("B", [1, 7, 64])
@pytest.mark.parametrize("mode", list(MODES))
def test_batch_equals_each_query_alone(corpus, fields, faceting, mode, B):  # noqa: F811
    c = corpus
    m = MODES[mode]
    qv, texts = _inputs(B, 5100 + B, c["rows"])
    filters = _assign(c["fs"], B, B + 17) if B > 1 else [c["fs"]["d30"]]
    groups = _requests(faceting["gbs"], fields, B, B + 3, with_1000=False) if B > 1 else [(faceting["gbs"][10], 3, None)]
    facets = _mix(B, B) if B > 1 else [_MIX[5]]
    t, q = (texts if m != MODE_VECTOR else None), (qv if m != MODE_FULLTEXT else None)
    _check(_tsc(c, m), faceting["st"], m, filters, groups, _promote(B, B + 1), facets, t, q, similarity=0.0)
    # no groups, no filters, no pins: every count comes from the main pass
    _check(_tsc(c, m), faceting["st"], m, None, None, None, facets, t, q, similarity=0.0)


def test_whole_batch_filter_and_offsets(corpus, faceting):  # noqa: F811
    """p->filter (every query filtered: all counted on the unfiltered re-score) and q_facet_offsets[0] > 0."""
    c = corpus
    B = 9
    qv, texts = _inputs(B, 5300, c["rows"])
    tsc = _tsc(c, MODE_HYBRID)
    st = faceting["st"]
    facets = _mix(B, 3)
    p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=c["fs"]["d30"], offset=1)
    got = ob.search_q_facets_arrays(tsc, st, p, facets, None, None, texts, qv)
    ref = ob.search_q_groups_arrays(tsc, p, [None] * B, None, texts, qv)
    for x, y in zip(got[:12], ref):
        assert x.tobytes() == y.tobytes()
    for b in range(B):
        if facets[b]:
            one = _facets_alone(tsc, st, MODE_HYBRID, c["fs"]["d30"], facets[b], [texts[b]], qv[b:b + 1], similarity=0.0, offset=1)
            assert got[12][got[13][b]:got[13][b + 1]].tolist() == one.tolist(), b
    # the requests may start past index 0 of the caller's arrays: entries before q_facet_offsets[0] are not touched
    sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0), texts[:2], qv[:2])
    reqs = [(0, 0, 0.0, 0.0)] * 3 + ob.facet_requests(st, _MIX[5])[0]
    arr = (_lib.FacetReq * len(reqs))(*[_lib.FacetReq(*r) for r in reqs])
    off = np.asarray([3, 3, len(reqs)], np.uint32)
    L = 10
    d, s, sv = np.zeros((2, L), np.uint64), np.zeros((2, L), np.float32), np.zeros((2, L), np.float64)
    n, cnt = np.zeros(2, np.uint32), np.zeros(2, np.uint64)
    fc = np.full(len(reqs), 7, np.uint64)
    rc = _lib.lib().oc_search_q_facets(c["ctx"]._h, c["emb"]._h, c["strs"]._h, C.byref(sp), None, None, 0, st._h, _p(off), arr,
                                       _p(d), _p(s), _p(sv), _p(n), _p(cnt), None, None, None, None, None, None, _p(fc))
    assert rc == 0
    assert fc[:3].tolist() == [7, 7, 7]
    one = _facets_alone(tsc, st, MODE_HYBRID, None, _MIX[5], [texts[1]], qv[1:2], similarity=0.0)
    assert fc[3:].tolist() == one.tolist()


@pytest.mark.parametrize("mode", list(MODES))
def test_limit_zero(corpus, fields, faceting, mode):  # noqa: F811
    """limit 0 with every query grouped or faceted: no hits, vector depth 0 in both passes.  The counts are those of the
    fulltext map alone (fulltext and hybrid) or empty (vector)."""
    c = corpus
    m = MODES[mode]
    B = 24
    qv, texts = _inputs(B, 5500, c["rows"])
    filters = _assign(c["fs"], B, 91)
    groups = _requests(faceting["gbs"], fields, B, 93, with_1000=False)
    facets = [f if f or g is not None and g[0] is not None else {"cat": {}} for f, g in zip(_mix(B, 95), groups)]
    tsc, st = _tsc(c, m), faceting["st"]
    t, q = (texts if m != MODE_VECTOR else None), (qv if m != MODE_FULLTEXT else None)
    p = ob.TokenScoreParams(mode=m, device_filters=filters, similarity=0.0, limit_hint=0)
    promote = _promote(B, 97)
    got = ob.search_q_facets_arrays(tsc, st, p, facets, groups, promote, t, q)
    assert not got[3].any()
    ft = _tsc(c, MODE_FULLTEXT)
    rows, S = got[11], got[7].shape[1]
    for b in range(B):
        if groups[b] is not None and groups[b][0] is not None:   # oc_search_q_groups refuses the facet-only queries at limit 0
            pb = ob.TokenScoreParams(mode=m, device_filters=[filters[b]], similarity=0.0, limit_hint=0)
            one = ob.search_q_groups_arrays(tsc, pb, [groups[b]], [promote[b]], None if t is None else [t[b]],
                                            None if q is None else q[b:b + 1], group_stride=S)
            assert got[4][b] == one[4][0], (b, mode)
            r0, r1 = int(rows[b]), int(rows[b + 1])
            for x, y in zip((got[7], got[8], got[9], got[10]), one[7:11]):
                assert x[r0:r1].tobytes() == y.tobytes(), (b, mode)
        if not facets[b]:
            continue
        want = (np.zeros(got[13][b + 1] - got[13][b], np.uint64) if m == MODE_VECTOR
                else _facets_alone(ft, st, MODE_FULLTEXT, None, facets[b], [texts[b]], None))
        assert got[12][got[13][b]:got[13][b + 1]].tolist() == want.tolist(), (b, mode)
    # and without any group: every query has facets
    facets = [f or {"flag": {"true": True}} for f in _mix(B, 99)]
    got = ob.search_q_facets_arrays(tsc, st, p, facets, None, None, t, q)
    assert got[3].shape == (B,) and not got[3].any()


@pytest.mark.parametrize("mode,sparse_ids", [(MODE_FULLTEXT, False), (MODE_FULLTEXT, True), (MODE_HYBRID, False),
                                              (MODE_HYBRID, True), (MODE_VECTOR, True)])
def test_against_the_oracle_score_maps(gpu_ctx, orc, mode, sparse_ids):
    """Counts equal a numpy count over the oracle's score-map keys: a query's own map without a filter, the unfiltered map
    with one.  OMC multipliers, a threshold, uncommitted deletes, then a commit."""
    n, dim, vocab, B = 30000, 64, 2000, 16
    rng = np.random.default_rng(31)
    rows = synth.make_vectors(n, dim, seed=33)
    qv, _ = synth.make_vector_queries(rows, B, seed=34)
    data = synth.make_text_corpus(n, vocab, seed=35)
    texts = synth.make_text_queries(vocab, B, seed=36)
    ids = (np.arange(n, dtype=np.uint64) * 3 + 2) if sparse_ids else np.arange(n, dtype=np.uint64)
    if sparse_ids:
        data.row_doc_ids = ids
    nbits = int(ids.max()) + 1
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=dim)
    emb.insert_batch(ids, rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    gone = rng.choice(n, 300, replace=False)
    for d in ids[gone].tolist():
        strs.delete(d); emb.delete(d)
    deleted = np.zeros(n, np.uint8); deleted[gone] = 1
    tsc = ob.TokenScoreContext(gpu_ctx, emb if mode != MODE_FULLTEXT else None, strs if mode != MODE_VECTOR else None)
    flag = rng.random(n) < 0.3
    cat = rng.integers(0, 10, size=n)
    price = np.round(rng.gamma(2.0, 30.0, size=n), 2)
    st = ob.FacetStore(gpu_ctx, nbits)
    st.add_bool_field("flag", ids[flag], ids[~flag])
    cat_docs = {f"c{k}": np.concatenate([ids[cat == k], ids[(cat == (k + 1) % 10) & (rng.random(n) < 0.1)]]) for k in range(10)}
    st.add_string_field("cat", cat_docs)
    st.add_number_field("price", ids, price)
    ranges = [(0, 20), (20, 50.5), (50.5, 1e9), (-5, -1), (30, 10)]
    variants = {"flag": {"true": ids[flag], "false": ids[~flag]}, "cat": cat_docs,
                "price": [ids[(price >= a) & (price <= b)] for a, b in ranges]}
    mix = [{"flag": {"true": True, "false": True}}, {"cat": {}}, {"price": {"ranges": [{"from": a, "to": b} for a, b in ranges]}},
           None, {"cat": {}, "price": {"ranges": [{"from": 0, "to": 20}]}}]
    facets = [mix[b % len(mix)] for b in range(B)]
    flt = ob.DeviceFilter.from_ids(gpu_ctx, ids[::2], nbits)
    filters = [flt if b % 3 == 0 else None for b in range(B)]
    omc = (ids[:50:7], np.full(len(ids[:50:7]), 1.5, np.float32))
    try:
        for thr, commit in ((None, False), (0.5, False), (None, True)):
            if commit:
                strs.commit()
            kw = dict(similarity=0.0, threshold=thr, omc_doc_ids=omc[0], omc_mult=omc[1])
            t, q = (texts if mode != MODE_VECTOR else None), (qv if mode != MODE_FULLTEXT else None)
            got = ob.search_q_facets_arrays(tsc, st, ob.TokenScoreParams(mode=mode, device_filters=filters, **kw), facets,
                                            None, None, t, q)
            alive = orc.make_filter_bits(ids[deleted == 0].tolist(), nbits)
            ix = orc.StrIndex(data)   # after the commit too: its key set under `alive` is the committed store's
            est = orc.EmbStore(rows, row_doc_ids=ids, deleted=deleted)
            for b in range(B):
                if not facets[b]:
                    continue
                if mode == MODE_VECTOR:
                    keys = orc.vector(est, qv[b], 10, 0.0)[0]
                else:
                    ft = orc.fulltext(ix, texts[b], threshold=thr, filter_bits=alive, filter_nbits=nbits)
                    keys = ft[0] if mode == MODE_FULLTEXT else orc.hybrid_combine(orc.vector(est, qv[b], 10, 0.0), ft)[0]
                ks = np.asarray(keys, np.uint64)
                want = []
                for name, d in facets[b].items():
                    if name == "flag":
                        want += [int(np.isin(variants["flag"][k], ks).sum()) for k in ("true", "false") if d.get(k)]
                    elif name == "cat":
                        want += [int(np.isin(v, ks).sum()) for v in cat_docs.values()]
                    else:
                        want += [int(np.isin(ids[(price >= r["from"]) & (price <= r["to"])], ks).sum()) for r in d["ranges"]]
                assert got[12][got[13][b]:got[13][b + 1]].tolist() == want, (b, mode, thr, commit)
    finally:
        flt.close(); st.close(); emb.close(); strs.close()


def test_reference_pins_in_a_mixed_batch(gpu_ctx):
    """facets.rs:10-98, 253-342, 408-460 restated through oc_search_q_facets, each pinned query inside a batch with
    queries of other facets and filters."""
    # :10-98 and a neighbour without facets and one with a filter
    h = build_index([(i, {"text": "text " * (i + 1)}) for i in range(100)])
    tsc = ob.TokenScoreContext(gpu_ctx, None, ob.StringFieldStorage(gpu_ctx, h.data))
    st = ob.FacetStore(gpu_ctx, 100)
    st.add_number_field("number", np.arange(100), np.arange(100, dtype=np.float64))
    ranges = [(0, 10), (0.5, 10.5), (-10, 10), (-10, -1), (1, 100), (99, 105), (102, 105)]
    fa = {"number": {"ranges": [{"from": a, "to": b} for a, b in ranges]}}
    odd = ob.DeviceFilter.from_ids(gpu_ctx, range(1, 100, 2), 100)
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, device_filters=[None, odd, odd])
    res = ob.search_q_facets(tsc, st, p, [fa, None, fa], texts=[h.resolve("text")] * 3)
    want = {"-10--1": 0, "-10-10": 11, "0-10": 11, "0.5-10.5": 10, "1-100": 99, "102-105": 0, "99-105": 1}
    assert res[0][2]["number"] == {"count": 7, "values": want}
    assert res[1][2] is None and res[1][0].count == 50
    assert res[2][2]["number"]["values"] == want                     # the filter does not reach the counts
    odd.close(); st.close(); tsc.str.close()
    # :253-342: the document that does not match the term is not counted
    h = build_index([(1, {"text": "text"}), (2, {"text": "text text"}), (3, {"text": "another"})])
    tsc = ob.TokenScoreContext(gpu_ctx, None, ob.StringFieldStorage(gpu_ctx, h.data))
    st = ob.FacetStore(gpu_ctx, 4)
    st.add_bool_field("bool", [1, 3], [2])
    st.add_number_field("number", [1, 2, 3], [1.0, 2.0, 1.0])
    fb = {"bool": {"true": True, "false": True}, "number": {"ranges": [{"from": 0, "to": 10}]}}
    res = ob.search_q_facets(tsc, st, ob.TokenScoreParams(mode=MODE_FULLTEXT), [{"bool": {"true": True}}, fb],
                             texts=[h.resolve("another"), h.resolve("text")])
    assert res[0][2] == {"bool": {"count": 1, "values": {"true": 1}}}
    assert res[1][2]["bool"] == {"count": 2, "values": {"true": 1, "false": 1}}
    assert res[1][2]["number"] == {"count": 1, "values": {"0-10": 2}}
    st.close(); tsc.str.close()
    # :408-460: term "", where category = A -> the hits are filtered, the facets still report A: 5, B: 5
    h = build_index([(i, {"title": f"title {i}"}) for i in range(10)], fields=("title",))
    tsc = ob.TokenScoreContext(gpu_ctx, None, ob.StringFieldStorage(gpu_ctx, h.data))
    st = ob.FacetStore(gpu_ctx, 10)
    st.add_string_field("category", {"A": range(0, 10, 2), "B": range(1, 10, 2)})
    a = st.leaf("category", "A")
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, device_filters=[a, None])
    res = ob.search_q_facets(tsc, st, p, [{"category": {}}, {"category": {}}], texts=[h.resolve("")] * 2)
    assert res[0][0].count == 5 and res[1][0].count == 10
    assert res[0][2] == res[1][2] == {"category": {"count": 2, "values": {"A": 5, "B": 5}}}
    a.close(); st.close(); tsc.str.close()


def test_refusals(corpus, fields, faceting):  # noqa: F811
    c = corpus
    L = _lib.lib()
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    st = faceting["st"]
    B = 4
    qv, texts = _inputs(B, 5900, c["rows"])
    other = ob.Context(0)
    ost = ob.FacetStore(other, N)
    ost.add_bool_field("flag", [1], [2])
    g10 = faceting["gbs"][10]._h
    flag, num = st.fields["flag"]["id"], st.fields["num"]["id"]
    good = [(flag, 0, 0.0, 0.0), (num, 0, 0.0, 10.0), (flag, 1, 0.0, 0.0)]
    try:
        def run(reqs=good, off=(0, 1, 1, 2, 3), store=None, groups=((g10, 3), None, None, None), null_off=False, edit=None, **kw):
            sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0,
                                                                device_filters=(c["fs"]["share"], None, None, None), **kw), texts, qv)
            if edit:
                keep.append(edit(sp))
            arr = (_lib.GroupReq * B)()
            for i, r in enumerate(groups):
                if r is not None:
                    arr[i].groups, arr[i].max_results = r[0], r[1]
            fr = (_lib.FacetReq * len(reqs))(*[_lib.FacetReq(*r) for r in reqs])
            o = np.asarray(off, np.uint32)
            lim = kw.get("limit_hint", 10)
            d = np.full((B, max(lim, 1)), 7, np.uint64); s = np.full((B, max(lim, 1)), 7, np.float32)
            v = np.full((B, max(lim, 1)), 7, np.float64)
            n = np.full(B, 7, np.uint32); cnt = np.full(B, 7, np.uint64)
            gd = np.full(10 * 16, 7, np.uint64); gs = np.full(gd.shape, 7, np.float32); gv = np.full(gd.shape, 7, np.float64)
            gn = np.full(10, 7, np.uint32); fc = np.full(8, 7, np.uint64)
            rc = L.oc_search_q_facets(c["ctx"]._h, c["emb"]._h, c["strs"]._h, C.byref(sp), arr, None, 16, (store or st)._h,
                                      None if null_off else _p(o), fr, _p(d), _p(s), _p(v), _p(n), _p(cnt), None, None, _p(gd),
                                      _p(gs), _p(gv), _p(gn), _p(fc))
            for a in (d, s, v, n, cnt, gd, gs, gv, gn, fc):
                assert (a == 7).all()   # nothing written
            return rc

        assert run(store=ost) == OC_ERR_INVALID                                                   # facets of another ctx
        assert run(null_off=True) == OC_ERR_INVALID
        assert run(off=(0, 2, 1, 2, 3)) == OC_ERR_INVALID                                          # not monotone
        assert run(reqs=[(99, 0, 0.0, 0.0)] + good[1:]) == OC_ERR_INVALID                          # unknown field
        assert run(reqs=[(flag, 2, 0.0, 0.0)] + good[1:]) == OC_ERR_INVALID                        # unknown variant
        assert run(reqs=good[:1] + [(num, 0, float("nan"), 10.0)] + good[2:]) == OC_ERR_INVALID     # NaN bound
        assert run(reqs=good[:1] + [(num, 0, 0.0, float("nan"))] + good[2:]) == OC_ERR_INVALID
        assert run(edit=lambda sp: setattr(sp, "sharded", 1)) == OC_ERR_UNSUPPORTED
        assert run(limit_hint=0, off=(0, 1, 1, 2, 3)) == OC_ERR_INVALID                            # query 2: no groups, no facets
        assert run(groups=((g10, 1025), None, None, None)) == OC_ERR_UNSUPPORTED                   # what oc_search_q_groups refuses
        assert run(limit_hint=1000, offset=100) == OC_ERR_UNSUPPORTED
        assert run(edit=lambda sp: setattr(sp, "filter", c["fs"]["all"]._h)) == OC_ERR_INVALID     # q_filters with filter
        assert run(limit_hint=0, off=(0, 1, 1, 2, 3), groups=((g10, 3), None, (g10, 3), None)) == OC_ERR_INVALID
        # the Python helper refuses what has no oc_facet_req: date fields, ranges on a variant field, a number field without ranges
        st.add_date_field("when", [1, 2], [10, 20])
        for bad in ({"when": {}}, {"flag": {"ranges": []}}, {"num": {}}):
            with pytest.raises(ValueError):
                ob.facet_requests(st, bad)
        # the batcher refuses before joining: a foreign store, a request oc_facets_check refuses
        bat = ob.SearchBatcher(tsc, max_batch=8, max_wait_us=100)
        try:
            sp, keep, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0), [texts[0]], qv[0:1])
            for store, reqs in ((ost, good[:1]), (st, [(99, 0, 0.0, 0.0)]), (st, [(num, 0, float("nan"), 1.0)])):
                fr = (_lib.FacetReq * len(reqs))(*[_lib.FacetReq(*r) for r in reqs])
                d = np.full(10, 7, np.uint64); s = np.full(10, 7, np.float32); n = np.full(1, 7, np.uint32)
                cnt = np.full(1, 7, np.uint64); fc = np.full(2, 7, np.uint64)
                rc = L.oc_batcher_search_faceted(bat._h, C.byref(sp), store._h, fr, len(reqs), None, None, 0, _p(d), _p(s), None,
                                                 _p(n), _p(cnt), None, None, None, None, None, None, _p(fc))
                assert rc == OC_ERR_INVALID
                assert (d == 7).all() and (n == 7).all() and (cnt == 7).all() and (fc == 7).all()
            assert bat.stats() == {"queries": 0, "batches": 0, "direct": 0}
        finally:
            bat.close()
    finally:
        ost.close()
        other.close()


def test_batcher_coalesces_faceted_requests(corpus, fields, faceting):  # noqa: F811
    """Threads send faceted requests with differing facets, groups, filters and pins, plus plain ones; each answer equals
    the query alone through search_q_facets_arrays, the batcher coalesces, and a malformed request fails alone."""
    c = corpus
    tsc = ob.TokenScoreContext(c["ctx"], c["emb"], c["strs"])
    st = faceting["st"]
    T, Q = 12, 16
    qv, texts = _inputs(T * Q, 6100, c["rows"])
    filters = _assign(c["fs"], T * Q, 101)
    groups = _requests(faceting["gbs"], fields, T * Q, 103, with_1000=False)
    promote = _promote(T * Q, 105)
    facets = _mix(T * Q, 107)
    kind = [("plain", "faceted", "faceted", "faceted", "faceted", "faceted", "faceted", "bad")[i % 8] for i in range(T * Q)]
    expect = {}
    for i in range(T * Q):
        p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i])
        if kind[i] == "plain":
            expect[i] = tsc.execute_batch_arrays(p, [texts[i]], qv[i:i + 1])
        elif kind[i] == "faceted":
            pd = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filters=[filters[i]])
            expect[i] = ob.search_q_facets_arrays(tsc, st, pd, [facets[i]], [groups[i]], [promote[i]], [texts[i]], qv[i:i + 1])
    bat = ob.SearchBatcher(tsc, max_batch=64, max_wait_us=3000)
    bad = []

    def worker(t):
        for i in range(t, T * Q, T):
            p = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, device_filter=filters[i])
            e = expect.get(i)
            if kind[i] == "plain":
                h = bat.search(p, texts[i], qv[i])
                k = int(e[2][0])
                ok = h.count == int(e[3][0]) and h.doc_ids.tobytes() == e[0][0, :k].tobytes()
            elif kind[i] == "bad":   # a NaN bound: oc_facets_check refuses it before it joins a batch
                try:
                    bat.search_faceted(st, p, {"cat": {}, "num": {"ranges": [{"from": np.nan, "to": 1}]}}, None, None, texts[i], qv[i])
                    ok = False
                except ob.OcError as x:
                    ok = x.code == OC_ERR_INVALID
            else:
                g = groups[i]
                r = bat.search_faceted(st, p, facets[i], g, promote[i] if promote[i] else None, texts[i], qv[i])
                ok = all(x.tobytes() == y[0].tobytes() for x, y in zip(r[:3], e[:3]))
                ok = ok and r[3] == e[3][0] and r[4] == e[4][0] and r[5].tobytes() == e[5].tobytes() and r[6].tobytes() == e[6].tobytes()
                ok = ok and all(x.tobytes() == y.tobytes() for x, y in zip(r[7:11], e[7:11]))
                ok = ok and r[11].tobytes() == e[12].tobytes()
            if not ok:
                bad.append(i)
    th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    s = bat.stats()
    bat.close()
    assert not bad, bad[:10]
    n_ok = sum(k != "bad" for k in kind)
    assert s["queries"] == n_ok and s["direct"] == 0 and s["batches"] < s["queries"], s


def test_tombstones_and_commit(gpu_ctx):
    """Uncommitted deletes, then a commit between calls, with the filtered queries' re-score."""
    n = 30_000
    rows = synth.make_vectors(n, DIM, seed=371)
    data = synth.make_text_corpus(n, 3000, seed=373)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    rng = np.random.default_rng(375)
    fs = _filters(gpu_ctx, n, rng)
    st, gbs, _ = _facets(gpu_ctx, n + 10, 377)
    try:
        tsc = ob.TokenScoreContext(gpu_ctx, emb, strs)
        B = 30
        qv, texts = _inputs(B, 379, rows)
        filters = _assign(fs, B, 5)
        groups = [[(gbs[10], 3, None), None, (gbs[20], 1, None)][i % 3] for i in range(B)]
        facets = _mix(B, 381)
        gone = rng.choice(n, 2000, replace=False).tolist()
        strs.delete(gone)
        emb.delete(gone)
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            _check(tsc, st, mode, filters, groups, _promote(B, 383, n), facets, texts, qv, similarity=0.0)
        strs.commit()
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            _check(tsc, st, mode, filters, groups, _promote(B, 383, n), facets, texts, qv, similarity=0.0)
    finally:
        for f in fs.values():
            f.close()
        for gb in gbs.values():
            gb.close()
        st.close(); emb.close(); strs.close()
