"""Pin rules on the GPU (oc_search_pinned, oc_search_groups_pinned) against (1) the reference's own answers
(src/tests/pin_rules.rs, src/tests/groupby.rs:984-1062) and (2) a restatement of apply_pin_rules_internal
(read/sort.rs:285-391) over sort_token_scores / sort_groups (:17-46, 129-230) on the oracle's score maps: fulltext,
vector and hybrid mode, identity and sparse document ids, a where-filter, uncommitted deletes, OMC, a threshold, and
promoted documents that are vector-only hits, fulltext-only, both, filtered out, deleted or unknown.  Also: queries
without items, empty pins and apply = 0 are byte-identical to oc_search / oc_search_groups, the multi-index union
through oc_merge_pinned, and every refused call."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal, build_index
from oramacore_b200 import PromoteItem, _lib
from oramacore_b200 import filters as F
from oramacore_b200 import synth
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, TextQuery
from test_pins_host import apply_pin_rules, top_n

pytestmark = pytest.mark.gpu

ATOL = 1e-5   # test_gpu_parity's tolerance for vector / hybrid scores


def _ft(ctx, h):
    return ob.TokenScoreContext(ctx, None, ob.StringFieldStorage(ctx, h.data))


def _ids(hits):
    return hits.doc_ids.tolist()


# ---------------------------------------------------------------- reference answers
@pytest.fixture(scope="module")
def twenty(gpu_ctx):
    # pin_rules.rs: 20 documents {"c": "c-<i>"}; every one of them scores the same for "c"
    h = build_index([(i, {"c": f"c n{i}"}) for i in range(20)], fields=("c",))
    tsc = _ft(gpu_ctx, h)
    yield h, tsc
    tsc.str.close()


def _pinned(tsc, h, items, limit=10, offset=0, term="c"):
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=limit, offset=offset)
    return ob.search_pinned(tsc, p, [items], texts=[h.resolve(term)])[0]


def test_reference_simple(twenty):
    h, tsc = twenty
    hits = _pinned(tsc, h, [PromoteItem(5, 1), PromoteItem(7, 2)])   # :9-106, :371-435
    assert _ids(hits) == [0, 5, 7, 1, 2, 3, 4, 6, 8, 9] and hits.count == 20


def test_reference_already_returned_and_far_position(twenty):
    h, tsc = twenty
    assert _ids(_pinned(tsc, h, [PromoteItem(0, 3)])) == [1, 2, 3, 0, 4, 5, 6, 7, 8, 9]           # :242-302
    assert _ids(_pinned(tsc, h, [PromoteItem(0, 3000)])) == [1, 2, 3, 4, 5, 6, 7, 8, 9, 10]       # :305-365


def test_reference_pagination(twenty):
    h, tsc = twenty   # :368-508
    assert _ids(_pinned(tsc, h, [PromoteItem(0, 3)])) == [1, 2, 3, 0, 4, 5, 6, 7, 8, 9]
    for offset, exp in [(0, [1, 2]), (1, [2, 3]), (2, [3, 0]), (3, [0, 4]), (4, [4, 5])]:
        assert _ids(_pinned(tsc, h, [PromoteItem(0, 3)], limit=2, offset=offset)) == exp


def test_reference_promote_non_matching(gpu_ctx):
    # :671-753 only document 1 matches "blue jeans"; document 2 is promoted to position 1
    h = build_index([(0, {"text": "red shirt"}), (1, {"text": "blue jeans"}), (2, {"text": "green hat"})])
    tsc = _ft(gpu_ctx, h)
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10)
    docs, scores, n, cnt, ps, pp = ob.search_pinned_arrays(tsc, p, [[PromoteItem(2, 1)]], texts=[h.resolve("blue jeans")])
    assert docs[0, :n[0]].tolist() == [1, 2] and int(cnt[0]) == 1
    assert scores[0, 1] == 0.0 and scores[0, 0] > 0.0
    assert ps.tolist() == [0.0] and pp.tolist() == [0]
    tsc.str.close()


def test_reference_group_by_with_pins(gpu_ctx):
    # groupby.rs:984-1062: doc3 (food, no match) promoted to 1 in every group: food -> [doc1, doc3], tech -> [doc2, doc5]
    docs = [("apple fruit", "food"), ("apple phone", "tech"), ("banana fruit", "food"), ("orange tech", "tech"), ("apple laptop", "tech")]
    h = build_index([(i, {"title": t}) for i, (t, _) in enumerate(docs)], fields=("title",))
    tsc = _ft(gpu_ctx, h)
    st = ob.FacetStore(gpu_ctx, len(docs))
    st.add_string_field("category", {c: [i for i, (_, cc) in enumerate(docs) if cc == c] for c in ("food", "tech")})
    gb = ob.GroupBy(st, ["category"])
    hits, groups = ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10), max_results=3,
                                    texts=[h.resolve("apple")], promote=[[PromoteItem(2, 1)]])[0]
    g = {tuple(x["values"]): x["result"] for x in groups}
    assert [d for d, _ in g[("food",)]] == [0, 2] and [d for d, _ in g[("tech",)]] == [1, 4]
    assert g[("food",)][1][1] == 0.0
    assert _ids(hits) == [0, 2, 1, 4] and hits.count == 3
    gb.close(); st.close(); tsc.str.close()


# ---------------------------------------------------------------- random corpus against the oracle's score maps
N, DIM, VOCAB, B = 40000, 384, 3000, 12


@pytest.fixture(scope="module", params=[False, True], ids=["identity_ids", "sparse_ids"])
def corpus(request, gpu_ctx):
    sparse = request.param
    rng = np.random.default_rng(29)
    rows = synth.make_vectors(N, DIM, seed=61)
    qv, _ = synth.make_vector_queries(rows, B, seed=62)
    data = synth.make_text_corpus(N, VOCAB, seed=63)
    texts = synth.make_text_queries(VOCAB, B - 1, seed=64) + [TextQuery.single_terms([0, 1, 2])]
    ids = (np.arange(N, dtype=np.uint64) * 3 + 2) if sparse else np.arange(N, dtype=np.uint64)
    if sparse:
        data.row_doc_ids = ids
    nbits = int(ids.max()) + 1
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(ids, rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    gone = [5, 77, 4000, 12345]
    for d in ids[gone].tolist():
        strs.delete(d); emb.delete(d)
    deleted = np.zeros(N, np.uint8); deleted[gone] = 1
    cat = rng.integers(0, 5, size=N)
    st = ob.FacetStore(gpu_ctx, nbits)
    st.add_string_field("category", {f"c{k}": ids[cat == k] for k in range(5)})
    omc_doc = np.sort(rng.choice(ids, size=3000, replace=False)).astype(np.uint64)
    omc_mult = rng.choice([2.0, 3.0, 0.5], size=3000).astype(np.float32)
    c = dict(ids=ids, nbits=nbits, rows=rows, qv=qv, data=data, texts=texts, emb=emb, strs=strs, st=st, deleted=deleted,
             cat=cat, omc=(omc_doc, omc_mult), rng=rng, alive=np.flatnonzero(deleted == 0), gone=ids[gone], sparse=sparse)
    yield c
    st.close(); emb.close(); strs.close()


def _oracle_maps(orc, c, mode, q, vlimit, where=None, threshold=None, omc=None):
    """(score map, vector map, fulltext map) as {doc: score}; the last two before fusion and OMC."""
    nbits = c["nbits"]
    allowed = c["alive"] if where is None else np.intersect1d(c["alive"], where)
    fbits = orc.make_filter_bits(c["ids"][allowed].tolist(), nbits)
    est = orc.EmbStore(c["rows"], row_doc_ids=c["ids"], deleted=c["deleted"])
    vec = ft = (np.zeros(0, np.uint64), np.zeros(0, np.float32))
    if mode != MODE_FULLTEXT:
        vec = orc.vector(est, c["qv"][q], vlimit, 0.0, None if where is None else orc.make_filter_bits(c["ids"][where].tolist(), nbits),
                         0 if where is None else nbits)
    if mode != MODE_VECTOR:
        ft = orc.fulltext(orc.StrIndex(c["data"]), c["texts"][q], threshold=threshold, filter_bits=fbits, filter_nbits=nbits)
    m = vec if mode == MODE_VECTOR else ft if mode == MODE_FULLTEXT else orc.hybrid_combine(vec, ft)
    if omc is not None:
        m = orc.apply_omc(m, *omc)
    as_dict = lambda x: dict(zip(x[0].tolist(), x[1].tolist()))  # noqa: E731
    return as_dict(m), as_dict(vec), as_dict(ft)


def _promote_for(c, rng, sm, vm, fm, where):
    """Items covering every kind of promoted document, at assorted positions (equal ones included)."""
    kinds = {
        "vector_only": [d for d in vm if d not in fm],
        "fulltext_only": [d for d in fm if d not in vm],
        "both": [d for d in vm if d in fm],
        "filtered": [] if where is None else [int(d) for d in c["ids"][np.setdiff1d(np.arange(N), where)][:200] if int(d) not in sm],
        "deleted": [int(d) for d in c["gone"]],
        "unknown": [c["nbits"] + 7, 1 if c["sparse"] else c["nbits"] + 100],
        "ranked": list(sm)[:20],
    }
    items = []
    for name, pool in kinds.items():
        if pool:
            for _ in range(2):
                items.append((int(pool[int(rng.integers(0, len(pool)))]), int(rng.choice([0, 1, 3, 3, 9, 40, 5000]))))
    rng.shuffle(items)
    return items


def _expect_flat(sm, items, limit, offset):
    active = len(items) > 0
    top = top_n(sm, 2 * (limit + offset) if active else limit + offset)
    if active:
        top = apply_pin_rules(items, sm, top)
    return top[offset:offset + limit]


def _compare(got_docs, got_scores, exp, items, exact):
    ed = [d for d, _ in exp]
    es = np.asarray([s for _, s in exp], np.float32)
    if exact:
        assert list(got_docs) == ed, (list(got_docs), ed)
        assert np.asarray(got_scores, np.float32).view(np.uint32).tolist() == es.view(np.uint32).tolist()
        return
    assert len(got_docs) == len(ed)
    promoted = {d for d, _ in items}
    pin_slots = [i for i, d in enumerate(ed) if d in promoted]
    for i in pin_slots:   # the promoted documents sit in their slots ...
        assert got_docs[i] == ed[i], (i, list(got_docs), ed)
    rest = [i for i in range(len(ed)) if i not in pin_slots]   # ... around the ranking, equal up to boundary ties
    assert_topk_equal(np.asarray(got_docs)[rest], np.asarray(got_scores)[rest], np.asarray(ed, np.uint64)[rest], es[rest], atol=ATOL)
    assert np.allclose(np.asarray(got_scores, np.float64), es.astype(np.float64), rtol=0, atol=ATOL, equal_nan=True)


def _tsc(c, mode):
    return ob.TokenScoreContext(c["strs"].ctx, c["emb"] if mode != MODE_FULLTEXT else None, c["strs"] if mode != MODE_VECTOR else None)


def _inputs(c, mode):
    return (c["texts"] if mode != MODE_VECTOR else None), (c["qv"] if mode != MODE_FULLTEXT else None)


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
@pytest.mark.parametrize("filtered", [False, True], ids=["plain", "filter_omc_threshold"])
def test_hits_against_the_restatement(corpus, orc, mode, filtered):
    c = corpus
    rng = np.random.default_rng(100 + mode + 10 * filtered)
    where = np.flatnonzero(c["rng"].random(N) < 0.5) if filtered else None
    thr = 0.5 if filtered and mode != MODE_VECTOR else None
    omc = c["omc"] if filtered else None
    kw = {}
    if filtered:
        kw = dict(filtered_doc_ids=F.to_bitmap(F.Ids(c["ids"][where]), c["nbits"]), filter_nbits=c["nbits"],
                  omc_doc_ids=omc[0], omc_mult=omc[1], threshold=thr)
    tsc = _tsc(c, mode)
    texts, qv = _inputs(c, mode)
    for limit, offset in [(10, 0), (3, 5), (100, 412)]:
        p = ob.TokenScoreParams(mode=mode, limit_hint=limit, offset=offset, similarity=0.0, **kw)
        maps = [_oracle_maps(orc, c, mode, q, limit, where=where, threshold=thr, omc=omc) for q in range(B)]
        promote = [_promote_for(c, rng, *maps[q], where) if q % 4 != 3 else [] for q in range(B)]
        docs, scores, n, cnt, ps, pp = ob.search_pinned_arrays(tsc, p, promote, texts=texts, q_vecs=qv)
        plain = tsc.execute_batch_arrays(p, texts, qv)
        i = 0
        for q in range(B):
            sm = maps[q][0]
            assert int(cnt[q]) == int(plain[3][q])   # count is the map size: promoted documents are not counted
            _compare(docs[q, :n[q]].tolist(), scores[q, :n[q]], _expect_flat(sm, promote[q], limit, offset), promote[q],
                     exact=mode == MODE_FULLTEXT)
            for d, _ in promote[q]:
                assert pp[i] == (1 if d in sm else 0), (q, d)
                exp = np.float32(sm.get(d, 0.0))
                if mode == MODE_FULLTEXT:
                    assert np.float32(ps[i]).view(np.uint32) == exp.view(np.uint32), (q, d)
                else:
                    assert abs(float(ps[i]) - float(exp)) <= ATOL, (q, d, ps[i], exp)
                i += 1
            if not promote[q]:   # a query without items: oc_search's bytes
                assert docs[q].tolist() == plain[0][q].tolist() and scores[q].view(np.uint32).tolist() == plain[1][q].view(np.uint32).tolist()
                assert n[q] == plain[2][q]


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
def test_inactive_empty_and_apply_zero_are_oc_search(corpus, mode):
    c = corpus
    tsc = _tsc(c, mode)
    texts, qv = _inputs(c, mode)
    rng = np.random.default_rng(3)
    for limit, offset in [(10, 0), (7, 30), (64, 448)]:
        p = ob.TokenScoreParams(mode=mode, limit_hint=limit, offset=offset, similarity=0.0)
        plain = tsc.execute_batch_arrays(p, texts, qv)
        mixed = [[(int(rng.choice(c["ids"])), int(rng.integers(0, 20))) for _ in range(3)] if q % 2 else [] for q in range(B)]
        for promote, apply in [(mixed, True), ([[] for _ in range(B)], True), (mixed, False)]:
            got = ob.search_pinned_arrays(tsc, p, promote, texts=texts, q_vecs=qv, apply=apply)
            for q in range(B):
                if apply and promote[q]:
                    continue
                assert got[0][q].tolist() == plain[0][q].tolist()
                assert got[1][q].view(np.uint32).tolist() == plain[1][q].view(np.uint32).tolist()
                assert got[2][q] == plain[2][q] and got[3][q] == plain[3][q]


def _expect_groups(sm, members, m, items):
    out = []
    for mem in members:
        cand = top_n({d: sm[d] for d in mem if d in sm}, m * 2 if items else m)
        if items:
            cand = apply_pin_rules([(d, pos) for d, pos in items if d in mem], sm, cand)
        out.append(cand)
    return out


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
@pytest.mark.parametrize("m", [0, 2, 5])
def test_groups_against_the_restatement(corpus, orc, mode, m):
    c = corpus
    rng = np.random.default_rng(200 + m + mode)
    gb = ob.GroupBy(c["st"], ["category"])
    members = [set(c["ids"][c["cat"] == k].tolist()) for k in range(5)]
    tsc = _tsc(c, mode)
    texts, qv = _inputs(c, mode)
    p = ob.TokenScoreParams(mode=mode, limit_hint=10, similarity=0.0)
    maps = [_oracle_maps(orc, c, mode, q, 10) for q in range(B)]
    promote = [_promote_for(c, rng, *maps[q], None) if q % 3 else [] for q in range(B)]
    docs, scores, n, cnt, gd, gs, gn = ob.search_groups_arrays(tsc, gb, p, m, texts=texts, q_vecs=qv, promote=promote)
    plain = ob.search_groups_arrays(tsc, gb, p, m, texts=texts, q_vecs=qv)
    assert gd.shape[2] == 2 * m + max(len(x) for x in promote)
    longer = False
    for q in range(B):
        sm = maps[q][0]
        _compare(docs[q, :n[q]].tolist(), scores[q, :n[q]], _expect_flat(sm, promote[q], 10, 0), promote[q], exact=mode == MODE_FULLTEXT)
        exp = _expect_groups(sm, members, m, promote[q])
        for g in range(5):
            k = int(gn[q, g])
            _compare(gd[q, g, :k].tolist(), gs[q, g, :k], exp[g], promote[q], exact=mode == MODE_FULLTEXT)
            longer = longer or k > m
            if not promote[q]:   # a query without items: oc_search_groups' bytes
                assert k == plain[6][q, g]
                assert gd[q, g, :m].tolist() == plain[4][q, g].tolist()
                assert gs[q, g, :m].view(np.uint32).tolist() == plain[5][q, g].view(np.uint32).tolist()
    assert longer   # active queries keep their lists untruncated
    gb.close()


def test_multi_index_merge(gpu_ctx, orc):
    n, vocab, limit, offset = 20000, 800, 10, 2
    texts = synth.make_text_queries(vocab, 6, seed=91)
    parts = []
    for i in range(2):   # disjoint document ids
        data = synth.make_text_corpus(n, vocab, seed=95 + i)
        ids = np.arange(n, dtype=np.uint64) * 2 + i
        data.row_doc_ids = ids
        parts.append(dict(data=data, ids=ids, strs=ob.StringFieldStorage(gpu_ctx, data)))
    maps = []
    for q in range(len(texts)):
        um = {}
        for pt in parts:
            d, s = orc.fulltext(orc.StrIndex(pt["data"]), texts[q])
            um.update(zip(d.tolist(), s.tolist()))
        maps.append(um)
    rng = np.random.default_rng(4)
    promote = []
    for q in range(len(texts)):
        ranked = list(maps[q])
        promote.append([] if q == 0 else [(int(rng.choice(ranked)), 1), (int(rng.choice(parts[1]["ids"])), 0), (10 ** 7, 4)])
    per = []
    for pt in parts:
        tsc = ob.TokenScoreContext(gpu_ctx, None, pt["strs"])
        p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=2 * (limit + offset), vector_limit=limit)
        per.append(ob.search_pinned_arrays(tsc, p, promote, texts=texts, apply=False))
    hits = ob.merge_index_results_pinned(per, promote, limit, offset)
    for q in range(len(texts)):
        exp = _expect_flat(maps[q], promote[q], limit, offset)
        _compare(hits[q].doc_ids.tolist(), hits[q].scores, exp, promote[q], exact=True)
        assert hits[q].count == len(maps[q])
    for pt in parts:
        pt["strs"].close()


def test_rejections(gpu_ctx, twenty):
    h, tsc = twenty
    txt = [h.resolve("c")]
    item = [[PromoteItem(1, 0)]]

    def code(fn):
        with pytest.raises(ob.OcError) as e:
            fn()
        return e.value.code
    assert code(lambda: ob.search_pinned(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT, sharded=True), item, texts=txt)) == -4
    assert code(lambda: ob.search_pinned(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=500, offset=13), item, texts=txt)) == -4
    ob.search_pinned(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=500, offset=12), item, texts=txt)
    ob.search_pinned(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=1000), [[]], texts=txt)   # inactive: no doubling
    many = [[PromoteItem(i, i) for i in range(1025)]]
    assert code(lambda: ob.search_pinned(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT), many, texts=txt)) == -4
    ob.search_pinned(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT), [many[0][:1024]], texts=txt)
    # q_pin_offsets not monotone: nothing is written
    sp, keep, B = tsc._build_params(ob.TokenScoreParams(mode=MODE_FULLTEXT), txt, None)
    off, doc, pos = np.asarray([2, 1], np.uint32), np.zeros(2, np.uint64), np.zeros(2, np.uint32)
    pins = _lib.Pins(off.ctypes.data, doc.ctypes.data, pos.ctypes.data, 1)
    out = [np.full(10, 7, np.uint64), np.zeros(10, np.float32), np.full(1, 7, np.uint32), np.full(1, 7, np.uint64)]
    rc = _lib.lib().oc_search_pinned(tsc.ctx._h, None, tsc.str._h, C.byref(sp), C.byref(pins), *[o.ctypes.data for o in out], None, None)
    assert rc == -1 and out[2][0] == 7 and out[3][0] == 7 and out[0][0] == 7
    # groups: 2 x max_results, group_stride, a handle of another ctx
    st = ob.FacetStore(gpu_ctx, 20)
    st.add_string_field("k", {"a": list(range(10)), "b": list(range(10, 20))})
    gb = ob.GroupBy(st, ["k"])
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT)
    assert code(lambda: ob.search_groups(tsc, gb, p, max_results=513, texts=txt, promote=item)) == -4
    ob.search_groups(tsc, gb, p, max_results=512, texts=txt, promote=item)
    ob.search_groups(tsc, gb, p, max_results=1024, texts=txt, promote=[[]])
    assert code(lambda: ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT, sharded=True), texts=txt, promote=item)) == -4
    sp, keep, B = tsc._build_params(p, txt, None)
    pins, most = ob.engine._pins(item, 1)
    G, m = gb.n_groups, 3
    gd, gs, gn = np.zeros(G * 16, np.uint64), np.zeros(G * 16, np.float32), np.full(G, 9, np.uint32)
    hd, hs, hn, hc = np.zeros(10, np.uint64), np.zeros(10, np.float32), np.zeros(1, np.uint32), np.full(1, 9, np.uint64)
    args = lambda stride: (tsc.ctx._h, None, tsc.str._h, gb._h, C.byref(sp), m, C.byref(pins), stride,  # noqa: E731
                           hd.ctypes.data, hs.ctypes.data, hn.ctypes.data, hc.ctypes.data, gd.ctypes.data, gs.ctypes.data, gn.ctypes.data)
    assert _lib.lib().oc_search_groups_pinned(*args(2 * m)) == -1 and hc[0] == 9 and gn[0] == 9   # needs 2 * m + 1
    assert _lib.lib().oc_search_groups_pinned(*args(2 * m + 1)) == 0
    other = ob.Context(0)
    try:
        st2 = ob.FacetStore(other, 2)
        st2.add_string_field("k", {"a": [0]})
        gb2 = ob.GroupBy(st2, ["k"])
        assert code(lambda: ob.search_groups(tsc, gb2, p, texts=txt, promote=item)) == -1
        h2 = build_index([(0, {"c": "c"})], fields=("c",))
        tsc2 = _ft(other, h2)
        assert code(lambda: ob.search_pinned(ob.TokenScoreContext(gpu_ctx, None, tsc2.str), p, item, texts=[h2.resolve("c")])) == -1
        tsc2.str.close(); gb2.close(); st2.close()
    finally:
        other.close()
    gb.close(); st.close()
