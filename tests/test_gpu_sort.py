"""sortBy on the GPU (oc_search_sorted, oc_search_groups_sorted) against (1) the reference's own answers
(src/tests/sort.rs, groupby.rs:469-575, 1065-1144, pin_rules.rs:578-668, multi_index.rs:406-508) and (2) a restatement
of sort_token_scores / sort_groups with sort_by (read/sort.rs:17-46, 48-126, 147-201) over the oracle's score maps:
fulltext, vector and hybrid mode, identity and sparse ids, a where-filter, deletes, a threshold, OMC, documents with no
value, multi-valued documents, long runs of equal values, vector hits without a string row, pins, zero keys and
offsets past the keys.
Also: count equals oc_search's, the rank -> row map is rebuilt after a commit, and every refused call."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import build_index
from oramacore_b200 import PromoteItem, _lib
from oramacore_b200 import filters as F
from oramacore_b200 import synth
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, TextQuery
from test_gpu_pins import B, N, _inputs, _oracle_maps, _promote_for, _tsc, corpus  # noqa: F401  (corpus: fixture)
from test_pins_host import apply_pin_rules

pytestmark = pytest.mark.gpu

ATOL = 1e-5


def ranks(doc_ids, values, order):
    """The field's order: value, then ascending id; a document once, at its first value in that order.
    Returns {doc: (rank, value)}."""
    e = sorted(zip(values.tolist(), doc_ids.tolist()), key=lambda x: ((x[0] if order == "ASC" else -x[0]), x[1]))
    out = {}
    for v, d in e:
        if d not in out:
            out[d] = (len(out), v)
    return out


def expect_flat(sm, rk, limit, offset, items=()):
    """(docs, scores, sort values) of sort_token_scores with sort_by, pins and skip/take."""
    active = len(items) > 0
    keys = sorted((d for d in sm if d in rk), key=lambda d: rk[d][0])[:(2 if active else 1) * (limit + offset)]
    page = apply_pin_rules(list(items), sm, [(d, sm[d]) for d in keys])[offset:offset + limit]
    promoted = {d for d, _ in items} if active else set()
    return [d for d, _ in page], [s for _, s in page], [np.nan if d in promoted else rk[d][1] for d, _ in page]


def expect_groups(sm, rk, members, m, items):
    out = []
    for mem in members:
        keys = sorted((d for d in mem if d in sm and d in rk), key=lambda d: rk[d][0])[:(2 if items else 1) * m]
        top = [(d, sm[d]) for d in keys]
        if items:
            top = apply_pin_rules([(d, p) for d, p in items if d in mem], sm, top)
        out.append(top)
    return out


def check(got_d, got_s, got_v, exp, exact):
    ed, es, ev = exp
    assert list(got_d) == ed, (list(got_d), ed)
    es = np.asarray(es, np.float32)
    if exact:
        assert np.asarray(got_s, np.float32).view(np.uint32).tolist() == es.view(np.uint32).tolist()
    else:
        assert np.allclose(np.asarray(got_s, np.float64), es.astype(np.float64), rtol=0, atol=ATOL, equal_nan=True), (got_s, es)
    if got_v is not None:
        np.testing.assert_array_equal(np.asarray(got_v), np.asarray(ev, np.float64))


# ---------------------------------------------------------------- reference answers
def _ft(ctx, h):
    return ob.TokenScoreContext(ctx, None, ob.StringFieldStorage(ctx, h.data))


def _two(gpu_ctx, values, kind):
    # sort.rs: {"id": "1", "name": "Tommaso", ...}, {"id": "2", "name": "Michele", ...}; term "" is every document
    h = build_index([(1, {"name": "all tommaso"}), (2, {"name": "all michele"})], fields=("name",))
    tsc = _ft(gpu_ctx, h)
    f = ob.SortField(gpu_ctx, 3, [1, 2], values, kind)
    return h, tsc, f


@pytest.mark.parametrize("kind,values", [("number", [1990, 1994]),
                                         ("date", np.asarray(["2020-01-01T00:00:00", "2021-06-01T12:00:00"], "datetime64[ms]")),
                                         ("bool", [False, True])])
def test_reference_number_date_bool(gpu_ctx, kind, values):
    # sort.rs:8-111, 113-218, 220-322: the default order is ASC; document 1 holds the smaller value
    h, tsc, f = _two(gpu_ctx, values, kind)
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10)
    for order, exp in [(None, [1, 2]), ("ASC", [1, 2]), ("DESC", [2, 1])]:
        field, o = ob.resolve_sort_by({"v": f, "name": "string"}, ob.SortBy("v") if order is None else ob.SortBy("v", order))
        hits = ob.search_sorted(tsc, p, field, o, texts=[h.resolve("all")])[0]
        assert hits.doc_ids.tolist() == exp and hits.count == 2
    f.close(); tsc.str.close()


def test_reference_groups_ascending_descending(gpu_ctx):
    # groupby.rs:469-522, 524-575
    for order, docs, exp in [
        ("ASC", [("apple", "food", 30), ("banana", "food", 10), ("cherry", "food", 20), ("phone", "tech", 200), ("laptop", "tech", 100)],
         {"food": [1, 2, 0], "tech": [4, 3]}),
        ("DESC", [("apple", "food", 30), ("banana", "food", 10), ("phone", "tech", 200), ("laptop", "tech", 100)],
         {"food": [0, 1], "tech": [2, 3]})]:
        h = build_index([(i, {"title": "all " + t}) for i, (t, _, _) in enumerate(docs)], fields=("title",))
        tsc = _ft(gpu_ctx, h)
        st = ob.FacetStore(gpu_ctx, len(docs))
        st.add_string_field("category", {c: [i for i, d in enumerate(docs) if d[1] == c] for c in ("food", "tech")})
        gb = ob.GroupBy(st, ["category"])
        f = ob.SortField(gpu_ctx, len(docs), range(len(docs)), [d[2] for d in docs], "number")
        _, groups = ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10), max_results=10,
                                     texts=[h.resolve("all")], sort_by=(f, order))[0]
        assert {x["values"][0]: [d for d, _ in x["result"]] for x in groups} == exp
        f.close(); gb.close(); st.close(); tsc.str.close()


def test_reference_groups_with_pins(gpu_ctx):
    # groupby.rs:1065-1144: doc5 ("baz", tech, no match) promoted to 0: food -> [doc1], tech -> [doc5, doc2, doc4]
    docs = [("apple fruit", "food", 30), ("apple phone", "tech", 100), ("banana fruit", "food", 10), ("apple laptop", "tech", 200),
            ("baz", "tech", 200)]
    h = build_index([(i, {"title": t}) for i, (t, _, _) in enumerate(docs)], fields=("title",))
    tsc = _ft(gpu_ctx, h)
    st = ob.FacetStore(gpu_ctx, len(docs))
    st.add_string_field("category", {c: [i for i, d in enumerate(docs) if d[1] == c] for c in ("food", "tech")})
    gb = ob.GroupBy(st, ["category"])
    f = ob.SortField(gpu_ctx, len(docs), range(len(docs)), [d[2] for d in docs], "number")
    _, groups = ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10), max_results=3,
                                 texts=[h.resolve("apple")], promote=[[PromoteItem(4, 0)]], sort_by=(f, "ASC"))[0]
    assert {x["values"][0]: [d for d, _ in x["result"]] for x in groups} == {"food": [0], "tech": [4, 1, 3]}
    f.close(); gb.close(); st.close(); tsc.str.close()


def test_reference_pins_with_sort(gpu_ctx):
    # pin_rules.rs:578-668: 20 documents {"c": "c-<i>", "n": i}; 5 -> position 1, 7 -> position 2
    h = build_index([(i, {"c": f"c n{i}"}) for i in range(20)], fields=("c",))
    tsc = _ft(gpu_ctx, h)
    f = ob.SortField(gpu_ctx, 20, range(20), range(20), "number")
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10)
    pr = [[PromoteItem(5, 1), PromoteItem(7, 2)]]
    asc = ob.search_sorted(tsc, p, f, "ASC", promote=pr, texts=[h.resolve("c")])[0]
    assert asc.doc_ids.tolist() == [0, 5, 7, 1, 2, 3, 4, 6, 8, 9]
    desc = ob.search_sorted(tsc, p, f, "DESC", promote=pr, texts=[h.resolve("c")])[0]
    assert desc.doc_ids.tolist() == [19, 5, 7, 18, 17, 16, 15, 14, 13, 12]
    f.close(); tsc.str.close()


def test_reference_multi_index(gpu_ctx):
    # multi_index.rs:406-508: index 1 {doc1: 1, doc2: 3}, index 2 {doc3: 2, doc4: 4}, merged by oc_merge_sorted
    parts = []
    for docs in ([(1, 1), (2, 3)], [(3, 2), (4, 4)]):
        h = build_index([(d, {"text": "item"}) for d, _ in docs])
        tsc = _ft(gpu_ctx, h)
        parts.append((h, tsc, ob.SortField(gpu_ctx, 5, [d for d, _ in docs], [v for _, v in docs], "number")))
    for order, exp in [("ASC", [1, 3, 2, 4]), ("DESC", [4, 2, 3, 1])]:
        per = []
        for h, tsc, f in parts:
            r = ob.search_sorted_arrays(tsc, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, vector_limit=10), f, order,
                                        texts=[h.resolve("item")])
            per.append(r[:5])
        hits, _ = ob.merge_index_results_sorted(per, order, 10)
        assert hits[0].doc_ids.tolist() == exp and hits[0].count == 4
    for _, tsc, f in parts:
        f.close(); tsc.str.close()


# ---------------------------------------------------------------- random corpus against the oracle's score maps
@pytest.fixture(scope="module")
def field_values(corpus):
    """A number field over the corpus: ~1/5 of the documents without a value, ~1/10 with two or three values, values
    from a small set (long runs of equal values), ids past nbits ignored."""
    c = corpus
    rng = np.random.default_rng(5)
    has = np.flatnonzero(rng.random(N) >= 0.2)
    d = [c["ids"][has]]
    v = [rng.integers(0, 40, size=has.shape[0]).astype(np.float64)]
    multi = has[rng.random(has.shape[0]) < 0.1]
    for _ in range(2):
        d.append(c["ids"][multi]); v.append(rng.normal(20, 15, size=multi.shape[0]).round(1))
    d.append(np.asarray([c["nbits"] + 3], np.uint64)); v.append(np.asarray([-1e9]))
    doc_ids, values = np.concatenate(d).astype(np.uint64), np.concatenate(v)
    f = ob.SortField(c["strs"].ctx, c["nbits"], doc_ids, values, "number")
    yield f, {o: ranks(doc_ids[doc_ids < c["nbits"]], values[doc_ids < c["nbits"]], o) for o in ("ASC", "DESC")}
    f.close()


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
@pytest.mark.parametrize("filtered", [False, True], ids=["plain", "filter_omc_threshold"])
@pytest.mark.parametrize("order", ["ASC", "DESC"])
def test_hits_against_the_restatement(corpus, field_values, orc, mode, filtered, order):
    c = corpus
    f, rk = field_values[0], field_values[1][order]
    rng = np.random.default_rng(300 + mode + 10 * filtered)
    where = np.flatnonzero(c["rng"].random(N) < 0.5) if filtered else None
    thr = 0.5 if filtered and mode != MODE_VECTOR else None
    omc = c["omc"] if filtered else None
    kw = {}
    if filtered:
        kw = dict(filtered_doc_ids=F.to_bitmap(F.Ids(c["ids"][where]), c["nbits"]), filter_nbits=c["nbits"],
                  omc_doc_ids=omc[0], omc_mult=omc[1], threshold=thr)
    tsc = _tsc(c, mode)
    texts, qv = _inputs(c, mode)
    for limit, offset, pinned in [(10, 0, False), (3, 5, True), (100, 412, True), (1024, 0, False), (500, 12, True)]:
        p = ob.TokenScoreParams(mode=mode, limit_hint=limit, offset=offset, similarity=0.0, **kw)
        maps = [_oracle_maps(orc, c, mode, q, limit, where=where, threshold=thr, omc=omc) for q in range(B)]
        promote = [_promote_for(c, rng, *maps[q], where) if (pinned and q % 4 != 3) else [] for q in range(B)]
        docs, scores, sv, n, cnt, ps, pp = ob.search_sorted_arrays(tsc, p, f, order, promote=promote, texts=texts, q_vecs=qv)
        plain = tsc.execute_batch_arrays(p, texts, qv)
        for q in range(B):
            assert int(cnt[q]) == int(plain[3][q])   # count: oc_search's
            check(docs[q, :n[q]], scores[q, :n[q]], sv[q, :n[q]], expect_flat(maps[q][0], rk, limit, offset, promote[q]),
                  exact=mode == MODE_FULLTEXT)
            assert not docs[q, n[q]:].any() and not sv[q, n[q]:].any()


def test_vector_hit_without_row(gpu_ctx):
    # hybrid over documents 0..99 with a string row and documents 100..199 with only a vector
    n, dim = 200, 384
    rows = synth.make_vectors(n, dim, seed=8)
    h = build_index([(i, {"text": ("needle " if i == 17 else "") + f"w{i}"}) for i in range(100)])
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(np.arange(100, n, dtype=np.uint64), rows[100:])
    strs = ob.StringFieldStorage(gpu_ctx, h.data)
    vals = (n - 1 - np.arange(n)).astype(np.float64)
    vals[17] = -1.0   # the fulltext match sorts first
    f = ob.SortField(gpu_ctx, n, np.arange(n), vals, "number")
    tsc = ob.TokenScoreContext(gpu_ctx, emb, strs)
    needle = h.resolve("needle")
    # vector hits with no string row are keys: they follow the fulltext match in field order
    qv = np.ascontiguousarray(rows[[150, 120]])
    p = ob.TokenScoreParams(mode=MODE_HYBRID, limit_hint=5, similarity=0.0)
    docs, scores, sv, nn, cnt, _, _ = ob.search_sorted_arrays(tsc, p, f, "ASC", texts=[needle] * 2, q_vecs=qv)
    plain = tsc.execute_batch_arrays(p, [needle] * 2, qv)
    for q in range(2):
        assert int(cnt[q]) == int(plain[3][q])
        got = docs[q, :nn[q]].tolist()
        assert got[0] == 17 and len(got) == 5 and all(d >= 100 for d in got[1:])
        assert got == sorted(got, key=lambda d: vals[d]) and sv[q, :nn[q]].tolist() == [vals[d] for d in got]
    f.close(); emb.close(); strs.close()


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
@pytest.mark.parametrize("m", [0, 3])
def test_groups_against_the_restatement(corpus, field_values, orc, mode, m):
    c = corpus
    f, rk = field_values[0], field_values[1]["DESC"]
    rng = np.random.default_rng(400 + m + mode)
    gb = ob.GroupBy(c["st"], ["category"])
    members = [set(c["ids"][c["cat"] == k].tolist()) for k in range(5)]
    tsc = _tsc(c, mode)
    texts, qv = _inputs(c, mode)
    p = ob.TokenScoreParams(mode=mode, limit_hint=10, similarity=0.0)
    maps = [_oracle_maps(orc, c, mode, q, 10) for q in range(B)]
    promote = [_promote_for(c, rng, *maps[q], None) if q % 3 else [] for q in range(B)]
    docs, scores, n, cnt, gd, gs, gn, sv, gsv = ob.search_groups_arrays(tsc, gb, p, m, texts=texts, q_vecs=qv, promote=promote,
                                                                      sort_by=(f, "DESC"))
    plain = ob.search_groups_arrays(tsc, gb, p, m, texts=texts, q_vecs=qv)
    for q in range(B):
        sm = maps[q][0]
        assert cnt[q] == plain[3][q]
        check(docs[q, :n[q]], scores[q, :n[q]], sv[q, :n[q]], expect_flat(sm, rk, 10, 0, promote[q]), exact=mode == MODE_FULLTEXT)
        exp = expect_groups(sm, rk, members, m, promote[q])
        promoted = {d for d, _ in promote[q]}
        for g in range(5):
            k = int(gn[q, g])
            ev = [np.nan if d in promoted else rk[d][1] for d, _ in exp[g]]
            check(gd[q, g, :k], gs[q, g, :k], gsv[q, g, :k], ([d for d, _ in exp[g]], [s for _, s in exp[g]], ev),
                  exact=mode == MODE_FULLTEXT)
    gb.close()


def test_thousand_groups_and_batch_sizes(gpu_ctx, orc):
    # 1000 groups over a number field; B = 1 and 256 against the restatement (fulltext, bit-exact scores)
    n, vocab = 30000, 2000
    data = synth.make_text_corpus(n, vocab, seed=81)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    tsc = ob.TokenScoreContext(gpu_ctx, None, strs)
    rng = np.random.default_rng(82)
    grp = rng.integers(0, 1000, size=n)
    st = ob.FacetStore(gpu_ctx, n)
    st.add_number_field("g", np.arange(n), grp.astype(np.float64))
    gb = ob.GroupBy(st, ["g"])
    vals = rng.integers(0, 50, size=n).astype(np.float64)
    f = ob.SortField(gpu_ctx, n, np.arange(n), vals, "number")
    rk = ranks(np.arange(n), vals, "ASC")
    members = [set(np.flatnonzero(grp == k).tolist()) for k in range(1000)]
    for Bq in (1, 256):
        texts = synth.make_text_queries(vocab, Bq, seed=83 + Bq)
        p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, offset=3)
        docs, scores, nn, cnt, gd, gs, gn, sv, gsv = ob.search_groups_arrays(tsc, gb, p, 2, texts=texts, sort_by=(f, "ASC"))
        for q in range(0, Bq, 37 if Bq > 1 else 1):
            d, s = orc.fulltext(orc.StrIndex(data), texts[q])
            sm = dict(zip(d.tolist(), s.tolist()))
            assert int(cnt[q]) == len(sm)
            check(docs[q, :nn[q]], scores[q, :nn[q]], sv[q, :nn[q]], expect_flat(sm, rk, 10, 3), exact=True)
            exp = expect_groups(sm, rk, members, 2, [])
            for g in range(1000):
                k = int(gn[q, g])
                check(gd[q, g, :k], gs[q, g, :k], None, ([d for d, _ in exp[g]], [x for _, x in exp[g]], None), exact=True)
    f.close(); gb.close(); st.close(); strs.close()


def test_zero_keys_and_offset_past_keys(corpus, field_values, orc):
    c = corpus
    f, rk = field_values[0], field_values[1]["ASC"]
    tsc = _tsc(c, MODE_FULLTEXT)
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, offset=0)
    none = [TextQuery.single_terms([VOCAB_UNKNOWN])] * 3
    docs, scores, sv, n, cnt, _, _ = ob.search_sorted_arrays(tsc, p, f, "ASC", texts=none)
    assert n.tolist() == [0, 0, 0] and cnt.tolist() == [0, 0, 0] and not docs.any()
    rare = [TextQuery.single_terms([t]) for t in (2990, 2999)]   # few matches: the offset lies past them
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, offset=1014)
    docs, scores, sv, n, cnt, _, _ = ob.search_sorted_arrays(tsc, p, f, "ASC", texts=rare)
    for q in range(2):
        d, s = orc.fulltext(orc.StrIndex(c["data"]), rare[q])
        sm = dict(zip(d.tolist(), s.tolist()))
        assert int(cnt[q]) == len(sm)
        check(docs[q, :n[q]], scores[q, :n[q]], sv[q, :n[q]], expect_flat(sm, rk, 10, 1014), exact=True)


VOCAB_UNKNOWN = 10 ** 6


def test_commit_rebuilds_the_row_map(gpu_ctx):
    # the same handle before and after a commit that deletes documents (rows shift): equal to a fresh handle's answer
    n = 3000
    h = build_index([(i, {"text": "all " + ("odd" if i % 2 else "even")}) for i in range(n)])
    strs = ob.StringFieldStorage(gpu_ctx, h.data)
    tsc = ob.TokenScoreContext(gpu_ctx, None, strs)
    vals = (np.arange(n) * 7919 % 1000).astype(np.float64)
    f = ob.SortField(gpu_ctx, n, np.arange(n), vals, "number")
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=50)
    txt = [h.resolve("odd")]
    before = ob.search_sorted(tsc, p, f, "ASC", texts=txt)[0]
    assert all(d % 2 for d in before.doc_ids.tolist())
    strs.delete(np.arange(0, 1500, dtype=np.uint64))
    strs.commit()
    after = ob.search_sorted(tsc, p, f, "ASC", texts=txt)[0]
    fresh = ob.SortField(gpu_ctx, n, np.arange(n), vals, "number")
    exp = ob.search_sorted(tsc, p, fresh, "ASC", texts=txt)[0]
    assert after.doc_ids.tolist() == exp.doc_ids.tolist() and after.scores.tobytes() == exp.scores.tobytes()
    assert all(d % 2 and d >= 1500 for d in after.doc_ids.tolist())
    assert [vals[d] for d in after.doc_ids.tolist()] == sorted(vals[d] for d in after.doc_ids.tolist())
    fresh.close(); f.close(); strs.close()


def test_rejections(gpu_ctx):
    h = build_index([(i, {"c": f"c n{i}"}) for i in range(20)], fields=("c",))
    tsc = _ft(gpu_ctx, h)
    f = ob.SortField(gpu_ctx, 20, range(20), range(20), "number")
    txt = [h.resolve("c")]
    item = [[PromoteItem(1, 0)]]

    def code(fn):
        with pytest.raises(ob.OcError) as e:
            fn()
        return e.value.code
    P = lambda **k: ob.TokenScoreParams(mode=MODE_FULLTEXT, **k)  # noqa: E731
    assert code(lambda: ob.search_sorted(tsc, P(sharded=True), f, texts=txt)) == -4
    assert code(lambda: ob.search_sorted(tsc, P(limit_hint=1000, offset=25), f, texts=txt)) == -4
    ob.search_sorted(tsc, P(limit_hint=1000, offset=24), f, texts=txt)
    assert code(lambda: ob.search_sorted(tsc, P(limit_hint=500, offset=13), f, promote=item, texts=txt)) == -4
    ob.search_sorted(tsc, P(limit_hint=500, offset=12), f, promote=item, texts=txt)
    ob.search_sorted(tsc, P(limit_hint=1000), f, promote=[[]], texts=txt)   # inactive: no doubling
    # a bad order and a NULL field: nothing is written
    sp, keep, _ = tsc._build_params(P(), txt, None)
    out = [np.full(10, 7, np.uint64), np.zeros(10, np.float32), np.zeros(10, np.float64), np.full(1, 7, np.uint32), np.full(1, 7, np.uint64)]
    for srt in (_lib.Sort(f._h, 2), _lib.Sort(None, 0)):
        rc = _lib.lib().oc_search_sorted(tsc.ctx._h, None, tsc.str._h, C.byref(sp), C.byref(srt), None, *[o.ctypes.data for o in out],
                                         None, None)
        assert rc == -1 and out[0][0] == 7 and out[3][0] == 7 and out[4][0] == 7
    # groups: 2 x max_results with pins, sharded, group_stride
    st = ob.FacetStore(gpu_ctx, 20)
    st.add_string_field("k", {"a": list(range(10)), "b": list(range(10, 20))})
    gb = ob.GroupBy(st, ["k"])
    assert code(lambda: ob.search_groups(tsc, gb, P(), max_results=513, texts=txt, promote=item, sort_by=(f, "ASC"))) == -4
    ob.search_groups(tsc, gb, P(), max_results=512, texts=txt, promote=item, sort_by=(f, "ASC"))
    assert code(lambda: ob.search_groups(tsc, gb, P(sharded=True), texts=txt, sort_by=(f, "ASC"))) == -4
    G = gb.n_groups
    gd, gs, gv, gn = np.zeros(G * 16, np.uint64), np.zeros(G * 16, np.float32), np.zeros(G * 16), np.full(G, 9, np.uint32)
    srt = _lib.Sort(f._h, 0)
    assert _lib.lib().oc_search_groups_sorted(tsc.ctx._h, None, tsc.str._h, gb._h, C.byref(sp), 3, C.byref(srt), None, 2,
                                              *[o.ctypes.data for o in out], gd.ctypes.data, gs.ctypes.data, gv.ctypes.data,
                                              gn.ctypes.data) == -1
    assert gn[0] == 9 and out[4][0] == 7
    # a sort field of another ctx
    other = ob.Context(0)
    try:
        f2 = ob.SortField(other, 20, range(20), range(20), "number")
        assert code(lambda: ob.search_sorted(tsc, P(), f2, texts=txt)) == -1
        assert code(lambda: ob.search_groups(tsc, gb, P(), texts=txt, sort_by=(f2, "ASC"))) == -1
        f2.close()
    finally:
        other.close()
    assert code(lambda: ob.SortField(gpu_ctx, 2 ** 32, [1], [1.0], "number")) == -1
    gb.close(); st.close(); f.close(); tsc.str.close()
