"""groupBy on the GPU (oc_search_groups) against (1) the reference's own pinned answers (src/tests/groupby.rs) and
(2) a numpy restatement of sort_groups' capped-heap branch (read/sort.rs:129-230: per group, the top max_results
documents of the group that are keys of the score map, by score descending, ties by ascending document id, NaN
dropped) over the oracle's score maps: fulltext, vector and hybrid mode, identity and sparse document ids, a
where-filter, uncommitted deletes, OMC, a threshold, multi-term tokens, several group fields, and max_results up to
OC_MAX_TOPK.  Also: hits / count byte-identical to oc_search, a one-group grouping reproducing oc_search's top-limit,
the multi-index merge, and the rejected calls."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal, build_index
from oramacore_b200 import _lib
from oramacore_b200 import filters as F
from oramacore_b200 import synth
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, TextQuery

pytestmark = pytest.mark.gpu

ATOL = 1e-5   # test_gpu_parity's tolerance for vector / hybrid scores


def _ft(ctx, h):
    return ob.TokenScoreContext(ctx, None, ob.StringFieldStorage(ctx, h.data))


def _by_value(groups):
    return {tuple(g["values"]): g["result"] for g in groups}


# ---------------------------------------------------------------- reference pins (src/tests/groupby.rs)
def test_reference_pin_simple(gpu_ctx):
    # groupby.rs:9-175: 100 docs "text " x (i+1), number i % 5, bool i % 2 == 0, string_filter s{i % 3}; limit 0
    h = build_index([(i, {"text": "text " * (i + 1)}) for i in range(100)])
    tsc = _ft(gpu_ctx, h)
    st = ob.FacetStore(gpu_ctx, 100)
    ids = np.arange(100)
    st.add_number_field("number", ids, (ids % 5).astype(np.float64))
    st.add_bool_field("bool", ids[ids % 2 == 0], ids[ids % 2 == 1])
    st.add_string_field("string_filter", {f"s{k}": ids[ids % 3 == k] for k in range(3)})
    p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=0)
    for props, expect in [(["number"], {(float(v),) for v in range(5)}),
                          (["number", "bool"], {(float(v), b) for v in range(5) for b in (True, False)}),
                          (["number", "bool", "string_filter"], {(float(v), b, f"s{k}") for v in range(5) for b in (True, False) for k in range(3)})]:
        gb = ob.GroupBy(st, props)
        hits, groups = ob.search_groups(tsc, gb, p, max_results=5, texts=[h.resolve("text")])[0]
        assert hits.count == 100 and len(hits.doc_ids) == 0
        assert {tuple(g["values"]) for g in groups} == expect and len(groups) == len(expect)
        for g in groups:
            assert len(g["result"]) <= 5
            # every returned document really holds the group's values
            for d, _ in g["result"]:
                assert float(d % 5) == g["values"][0]
                if len(props) > 1:
                    assert (d % 2 == 0) == g["values"][1]
        gb.close()
    st.close(); tsc.str.close()


def _category_index(gpu_ctx, docs, extra=None):
    """docs: list of (title, category); ids 0..n-1."""
    h = build_index([(i, {"title": t}) for i, (t, _) in enumerate(docs)], fields=("title",))
    tsc = _ft(gpu_ctx, h)
    st = ob.FacetStore(gpu_ctx, len(docs))
    cats = list(dict.fromkeys(c for _, c in docs))
    st.add_string_field("category", {c: [i for i, (_, cc) in enumerate(docs) if cc == c] for c in cats})
    if extra:
        for name, vals in extra.items():
            st.add_number_field(name, np.arange(len(docs)), np.asarray(vals, np.float64))
    return h, tsc, st


def _run(tsc, st, h, props, term, max_results=1, limit=10):
    gb = ob.GroupBy(st, props)
    try:
        return ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=limit), max_results=max_results,
                                texts=[h.resolve(term)])[0]
    finally:
        gb.close()


def test_reference_pins_max_results(gpu_ctx):
    # :580-622 the default max_results is 1
    h, tsc, st = _category_index(gpu_ctx, [("apple fruit sweet", "food"), ("apple fruit red", "food"), ("apple fruit green", "food"),
                                           ("apple phone tech", "tech"), ("apple watch tech", "tech")])
    _, groups = _run(tsc, st, h, ["category"], "apple")
    assert len(groups) == 2 and all(len(g["result"]) == 1 for g in groups)
    st.close(); tsc.str.close()
    # :624-660 max_results 0 -> the group is there, empty;  :665-702 more than available -> all of them
    h, tsc, st = _category_index(gpu_ctx, [("apple", "food"), ("banana", "food")])
    _, groups = _run(tsc, st, h, ["category"], "", max_results=0)
    assert groups == [{"values": ["food"], "result": []}]
    _, groups = _run(tsc, st, h, ["category"], "", max_results=10)
    assert len(groups) == 1 and sorted(d for d, _ in groups[0]["result"]) == [0, 1]
    # :815-856 a search without hits still yields the (empty) group
    hits, groups = _run(tsc, st, h, ["category"], "nonexistent", max_results=5)
    assert hits.count == 0 and groups == [{"values": ["food"], "result": []}]
    st.close(); tsc.str.close()


def test_reference_pins_group_sizes(gpu_ctx):
    # :704-754 A:2, B:2, C:1 with max_results 2
    h, tsc, st = _category_index(gpu_ctx, [("test", "A"), ("test", "A"), ("test", "A"), ("test", "B"), ("test", "B"), ("test", "C")])
    _, groups = _run(tsc, st, h, ["category"], "test", max_results=2)
    assert {g["values"][0]: len(g["result"]) for g in groups} == {"A": 2, "B": 2, "C": 1}
    st.close(); tsc.str.close()
    # :902-948 food 2, tech 1 with max_results 5
    h, tsc, st = _category_index(gpu_ctx, [("test", "food"), ("test", "food"), ("test", "tech")])
    _, groups = _run(tsc, st, h, ["category"], "test", max_results=5)
    assert {g["values"][0]: len(g["result"]) for g in groups} == {"food": 2, "tech": 1}
    st.close(); tsc.str.close()
    # :756-813 three float groups (4.5, 3.2, 2.8)
    h, tsc, st = _category_index(gpu_ctx, [("test", "A"), ("test", "B"), ("test", "A"), ("test", "B"), ("test", "A")],
                                 extra={"rating": [4.5, 4.5, 3.2, 3.2, 2.8]})
    _, groups = _run(tsc, st, h, ["rating"], "test", max_results=3)
    assert [g["values"] for g in groups] == [[2.8], [3.2], [4.5]]
    assert [sorted(d for d, _ in g["result"]) for g in groups] == [[4], [2, 3], [0, 1]]
    st.close(); tsc.str.close()


def test_reference_pin_sort_by_score_default(gpu_ctx):
    # :416-467 "apple": hits doc1, doc2; group food -> [doc1], tech -> [doc2]
    h, tsc, st = _category_index(gpu_ctx, [("apple fruit", "food"), ("apple phone", "tech"), ("banana fruit", "food"), ("orange tech", "tech")])
    hits, groups = _run(tsc, st, h, ["category"], "apple", max_results=10)
    assert sorted(hits.doc_ids.tolist()) == [0, 1]
    g = _by_value(groups)
    assert [d for d, _ in g[("food",)]] == [0] and [d for d, _ in g[("tech",)]] == [1]
    st.close(); tsc.str.close()


# ---------------------------------------------------------------- random corpus against the oracle's score maps
N, DIM, VOCAB, B = 40000, 384, 3000, 12


@pytest.fixture(scope="module", params=[False, True], ids=["identity_ids", "sparse_ids"])
def corpus(request, gpu_ctx):
    sparse = request.param
    rng = np.random.default_rng(19)
    rows = synth.make_vectors(N, DIM, seed=71)
    qv, _ = synth.make_vector_queries(rows, B, seed=72)
    data = synth.make_text_corpus(N, VOCAB, seed=73)
    texts = synth.make_text_queries(VOCAB, B - 1, seed=74) + [TextQuery.single_terms([0, 1, 2])]   # the last one matches most docs
    ids = (np.arange(N, dtype=np.uint64) * 3 + 2) if sparse else np.arange(N, dtype=np.uint64)
    if sparse:
        data.row_doc_ids = ids
    nbits = int(ids.max()) + 1
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(ids, rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    gone = [5, 77, 4000, 12345]
    for d in ids[gone].tolist():   # uncommitted deletes stay excluded from the score map
        strs.delete(d); emb.delete(d)
    deleted = np.zeros(N, np.uint8); deleted[gone] = 1
    flag = rng.random(N) < 0.3
    cat = rng.integers(0, 6, size=N)
    st = ob.FacetStore(gpu_ctx, nbits)
    st.add_bool_field("in_stock", ids[flag], ids[~flag])
    # a doc may hold 2 keys; "none" holds no document, so its combinations are empty
    cat_docs = {f"c{k}": np.concatenate([ids[cat == k], ids[(cat == (k + 1) % 6) & (rng.random(N) < 0.1)]]) for k in range(6)}
    cat_docs["none"] = np.zeros(0, np.uint64)
    st.add_string_field("category", cat_docs)
    price = (rng.integers(0, 7, size=N) * 2.5).astype(np.float64)          # repeated values
    st.add_number_field("price", ids, price)
    st.add_string_field("all", {"all": ids})
    omc_doc = np.sort(rng.choice(ids, size=3000, replace=False)).astype(np.uint64)
    omc_mult = rng.choice([2.0, 3.0, 0.5], size=3000).astype(np.float32)
    c = dict(ids=ids, nbits=nbits, rows=rows, qv=qv, data=data, texts=texts, emb=emb, strs=strs, st=st, deleted=deleted,
             flag=flag, cat_docs=cat_docs, price=price, omc=(omc_doc, omc_mult), rng=rng,
             alive=np.flatnonzero(deleted == 0))
    yield c
    st.close(); emb.close(); strs.close()


def _members(c, props):
    """Group g's documents (set) and values, mixed radix over props, last fastest."""
    ids = c["ids"]
    per = []
    for p in props:
        if p == "in_stock":
            per.append([(True, set(ids[c["flag"]].tolist())), (False, set(ids[~c["flag"]].tolist()))])
        elif p == "category":
            per.append([(k, set(v.tolist())) for k, v in c["cat_docs"].items()])
        elif p == "price":
            per.append([(float(v), set(ids[c["price"] == v].tolist())) for v in np.unique(c["price"])])
        else:
            per.append([("all", set(ids.tolist()))])
    out = [([], None)]
    for vs in per:
        out = [(v + [x], s if m is None else (m & s)) for v, m in out for x, s in vs]
    return out


def _oracle_map(orc, c, mode, q, vlimit, similarity=0.0, where=None, threshold=None, omc=None):
    nbits = c["nbits"]
    allowed = c["alive"] if where is None else np.intersect1d(c["alive"], where)
    fbits = orc.make_filter_bits(c["ids"][allowed].tolist(), nbits)
    est = orc.EmbStore(c["rows"], row_doc_ids=c["ids"], deleted=c["deleted"])
    empty = (np.zeros(0, np.uint64), np.zeros(0, np.float32))
    vec = lambda: orc.vector(est, c["qv"][q], vlimit, similarity, None if where is None else orc.make_filter_bits(c["ids"][where].tolist(), nbits),
                             0 if where is None else nbits) if vlimit else empty
    if mode == MODE_VECTOR:
        m = vec()
    else:
        ft = orc.fulltext(orc.StrIndex(c["data"]), c["texts"][q], threshold=threshold, filter_bits=fbits, filter_nbits=nbits)
        m = ft if mode == MODE_FULLTEXT else orc.hybrid_combine(vec(), ft)
    if omc is not None:
        m = orc.apply_omc(m, *omc)
    return m


def _oracle_groups(score_map, members, m):
    docs, scores = score_map
    sc = dict(zip(docs.tolist(), scores.tolist()))
    out = []
    for _, mem in members:
        cand = [(d, sc[d]) for d in mem if d in sc and sc[d] == sc[d]]
        cand.sort(key=lambda t: (-np.float32(t[1]), t[0]))
        out.append(cand[:m])
    return out


def _check_groups(got, exp, exact):
    for g, (gg, ee) in enumerate(zip(got, exp)):
        gd = np.asarray([d for d, _ in gg["result"]], np.uint64)
        gs = np.asarray([s for _, s in gg["result"]], np.float32)
        ed = np.asarray([d for d, _ in ee], np.uint64)
        es = np.asarray([s for _, s in ee], np.float32)
        if exact:
            assert gd.tolist() == ed.tolist(), (g, gd, ed)
            assert gs.view(np.uint32).tolist() == es.view(np.uint32).tolist(), (g, gs, es)
        else:
            assert_topk_equal(gd, gs, ed, es, atol=ATOL)


def _search(c, mode, gb, m, limit=10, **kw):
    emb = c["emb"] if mode != MODE_FULLTEXT else None
    strs = c["strs"] if mode != MODE_VECTOR else None
    tsc = ob.TokenScoreContext(c["strs"].ctx, emb, strs)
    p = ob.TokenScoreParams(mode=mode, limit_hint=limit, similarity=0.0, **kw)
    texts = c["texts"] if mode != MODE_VECTOR else None
    qv = c["qv"] if mode != MODE_FULLTEXT else None
    return tsc, p, texts, qv, ob.search_groups(tsc, gb, p, max_results=m, texts=texts, q_vecs=qv)


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
@pytest.mark.parametrize("m", [0, 1, 3, 1024])
def test_groups_against_the_oracle(corpus, orc, mode, m):
    c = corpus
    props = ["in_stock", "category"]
    gb = ob.GroupBy(c["st"], props)
    members = _members(c, props)
    assert gb.n_groups == 14 and [v for v, _ in members] == gb.values
    tsc, p, texts, qv, res = _search(c, mode, gb, m)
    hits_ref = tsc.execute_batch(p, texts, qv)
    for q in range(B):
        hits, groups = res[q]
        assert hits.doc_ids.tolist() == hits_ref[q].doc_ids.tolist() and hits.count == hits_ref[q].count
        assert hits.scores.view(np.uint32).tolist() == hits_ref[q].scores.view(np.uint32).tolist()
        exp = _oracle_groups(_oracle_map(orc, c, mode, q, 10), members, m)
        _check_groups(groups, exp, exact=mode == MODE_FULLTEXT)
        assert all(len(g["result"]) == 0 for g, (v, _) in zip(groups, members) if v[1] == "none")
    if m == 1024 and mode == MODE_FULLTEXT:   # the busiest groups hold more matches than max_results
        big = max(len(_oracle_groups(_oracle_map(orc, c, mode, B - 1, 10), members, 10 ** 9)[g]) for g in range(gb.n_groups))
        assert big > 1024
    gb.close()


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
def test_groups_where_filter_omc_threshold(corpus, orc, mode):
    c = corpus
    props = ["price"]
    gb = ob.GroupBy(c["st"], props)
    members = _members(c, props)
    assert gb.values == [[v] for v in np.unique(c["price"]).tolist()]
    where = np.flatnonzero(c["rng"].random(N) < 0.5)
    kw = dict(filtered_doc_ids=F.to_bitmap(F.Ids(c["ids"][where]), c["nbits"]), filter_nbits=c["nbits"],
              omc_doc_ids=c["omc"][0], omc_mult=c["omc"][1])
    thr = 0.5 if mode != MODE_VECTOR else None
    _, _, _, _, res = _search(c, mode, gb, 5, threshold=thr, **kw)
    _, _, _, _, unfiltered = _search(c, mode, gb, 5)
    changed = False
    for q in range(B):
        exp = _oracle_groups(_oracle_map(orc, c, mode, q, 10, where=where, threshold=thr, omc=c["omc"]), members, 5)
        _check_groups(res[q][1], exp, exact=mode == MODE_FULLTEXT)
        changed = changed or res[q][1] != unfiltered[q][1]
        for g in res[q][1]:   # the where-filter IS applied to the groups (search.rs:415-429)
            assert set(d for d, _ in g["result"]) <= set(c["ids"][where].tolist())
    assert changed
    gb.close()


def test_groups_multi_term_tokens_use_the_k3_path(corpus, orc):
    c = corpus
    rng = np.random.default_rng(5)
    texts = []
    for _ in range(B):   # tokens expanding to several index terms (prefix expansion shape)
        k = int(rng.integers(2, 5))
        t = rng.choice(VOCAB // 4, size=k, replace=False)
        texts.append(TextQuery.from_tokens([[(0, int(x), float(w)) for x, w in zip(t, rng.choice([1.0, 2.0, 0.5], size=k))]]))
    gb = ob.GroupBy(c["st"], ["category", "in_stock"])
    members = _members(c, ["category", "in_stock"])
    tsc = ob.TokenScoreContext(c["strs"].ctx, None, c["strs"])
    for thr in (None, 0.5):
        p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, threshold=thr)
        res = ob.search_groups(tsc, gb, p, max_results=3, texts=texts)
        cc = dict(c, texts=texts)
        for q in range(B):
            _check_groups(res[q][1], _oracle_groups(_oracle_map(orc, cc, MODE_FULLTEXT, q, 10, threshold=thr), members, 3), exact=True)
    gb.close()


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
def test_groups_bit_identity_with_oc_search(corpus, mode):
    c = corpus
    gb = ob.GroupBy(c["st"], ["all"])
    assert gb.n_groups == 1
    for limit in (10, 100):
        tsc, p, texts, qv, res = _search(c, mode, gb, limit, limit=limit)
        hits = tsc.execute_batch(p, texts, qv)
        for q in range(B):   # one group holding every document, max_results = limit: oc_search's top-limit
            g = res[q][1][0]["result"]
            assert [d for d, _ in g] == hits[q].doc_ids.tolist()
            assert np.asarray([s for _, s in g], np.float32).view(np.uint32).tolist() == hits[q].scores.view(np.uint32).tolist()
    gb.close()
    gb = ob.GroupBy(c["st"], ["category", "price"])
    tsc, p, texts, qv, res = _search(c, mode, gb, 50, limit=10)
    deep = tsc.execute_batch(ob.TokenScoreParams(mode=mode, limit_hint=1024, vector_limit=10, similarity=0.0), texts, qv)
    n_seen = 0
    for q in range(B):   # every group hit also in oc_search's top 1024 carries the same score bits
        ref = dict(zip(deep[q].doc_ids.tolist(), deep[q].scores.view(np.uint32).tolist()))
        for g in res[q][1]:
            for d, s in g["result"]:
                if d in ref:
                    n_seen += 1
                    assert np.float32(s).view(np.uint32) == ref[d], (q, d)
    assert n_seen > 0
    gb.close()


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
def test_groups_limit_zero(corpus, orc, mode):
    c = corpus
    gb = ob.GroupBy(c["st"], ["category"])
    members = _members(c, ["category"])
    tsc, p, texts, qv, res = _search(c, mode, gb, 4, limit=0)
    for q in range(B):
        hits, groups = res[q]
        assert len(hits.doc_ids) == 0
        exp = _oracle_groups(_oracle_map(orc, c, mode, q, 0), members, 4)   # vector depth 0: no vector hit at all
        _check_groups(groups, exp, exact=mode != MODE_HYBRID)
        if mode == MODE_VECTOR:
            assert hits.count == 0 and all(not g["result"] for g in groups)
        else:
            assert hits.count == len(orc.fulltext(orc.StrIndex(c["data"]), c["texts"][q],
                                                  filter_bits=orc.make_filter_bits(c["ids"][c["alive"]].tolist(), c["nbits"]),
                                                  filter_nbits=c["nbits"])[0])
    gb.close()


def test_groups_multi_index_merge(gpu_ctx, orc):
    n, vocab = 20000, 800
    rng = np.random.default_rng(23)
    texts = synth.make_text_queries(vocab, 6, seed=81)
    parts = []
    for i in range(2):   # disjoint document ids, the same category keys
        data = synth.make_text_corpus(n, vocab, seed=90 + i)
        ids = np.arange(n, dtype=np.uint64) * 2 + i
        data.row_doc_ids = ids
        strs = ob.StringFieldStorage(gpu_ctx, data)
        st = ob.FacetStore(gpu_ctx, 2 * n)
        cat = rng.integers(0, 4, size=n)
        st.add_string_field("category", {f"k{k}": ids[cat == k] for k in range(4)})
        parts.append(dict(data=data, ids=ids, strs=strs, st=st, cat=cat))
    m, B2 = 7, len(texts)
    per = []
    for pt in parts:
        gb = ob.GroupBy(pt["st"], ["category"])
        tsc = ob.TokenScoreContext(gpu_ctx, None, pt["strs"])
        _, _, _, _, gd, gs, gn = ob.search_groups_arrays(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10), m, texts=texts)
        G = gb.n_groups
        per.append((gd.reshape(B2 * G, m), gs.reshape(B2 * G, m), gn.reshape(B2 * G), gn.reshape(B2 * G).astype(np.uint64)))
        gb.close()
    merged = ob.merge_index_results(per, limit=m)
    for q in range(B2):
        maps = [orc.fulltext(orc.StrIndex(pt["data"]), texts[q]) for pt in parts]
        um = (np.concatenate([x[0] for x in maps]), np.concatenate([x[1] for x in maps]))
        members = [(None, set(np.concatenate([pt["ids"][pt["cat"] == k] for pt in parts]).tolist())) for k in range(4)]
        exp = _oracle_groups(um, members, m)
        for g in range(4):
            r = merged[q * 4 + g]
            _check_groups([{"result": list(zip(r.doc_ids.tolist(), r.scores.tolist()))}], [exp[g]], exact=True)
    for pt in parts:
        pt["st"].close(); pt["strs"].close()


def test_groups_rejections(gpu_ctx):
    h, tsc, st = _category_index(gpu_ctx, [("apple", "food"), ("banana", "tech")])
    gb = ob.GroupBy(st, ["category"])
    txt = [h.resolve("apple")]
    with pytest.raises(ob.OcError) as e:
        ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT, sharded=True), texts=txt)
    assert e.value.code == -4
    with pytest.raises(ob.OcError) as e:
        ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT), max_results=1025, texts=txt)
    assert e.value.code == -4
    ob.search_groups(tsc, gb, ob.TokenScoreParams(mode=MODE_FULLTEXT), max_results=1024, texts=txt)
    # an unknown field id
    out, n = C.c_void_p(), C.c_uint64()
    bad = np.asarray([0, 7], np.uint32)
    assert _lib.lib().oc_group_by_create(st._h, bad.ctypes.data_as(C.c_void_p), 2, C.byref(out), C.byref(n)) == -1
    # a handle from another ctx
    other = ob.Context(0)
    try:
        st2 = ob.FacetStore(other, 2)
        st2.add_string_field("category", {"food": [0]})
        gb2 = ob.GroupBy(st2, ["category"])
        with pytest.raises(ob.OcError) as e:
            ob.search_groups(tsc, gb2, ob.TokenScoreParams(mode=MODE_FULLTEXT), texts=txt)
        assert e.value.code == -1
        gb2.close(); st2.close()
    finally:
        other.close()
    # more than 2^20 groups: 1025 x 1025 combinations
    st.add_string_field("wide", {f"w{i}": [] for i in range(1025)})
    with pytest.raises(ob.OcError) as e:
        ob.GroupBy(st, ["wide", "wide"])
    assert e.value.code == -4
    gb.close(); st.close(); tsc.str.close()
