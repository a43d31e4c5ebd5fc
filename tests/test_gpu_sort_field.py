"""The device build of a sort field: oc_sort_field_create and oc_sort_field_from_facets against sort_field_spec.py and
against each other, byte for byte in the read-back (oc_sort_field_read) and in every sorted search; IndexLoader's
sort_by over seeded op streams; and a from_facets build racing a commit of its store."""
import ctypes as C
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from index_model import IndexModel
from oramacore_b200 import PromoteItem, synth
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from sort_field_spec import random_entries, rank_order, variant_entries
from test_gpu_index_lifecycle import FILTERS, STRING_FIELDS, Expect, Stream, _as_dict
from test_gpu_sort import check, expect_flat, ranks

pytestmark = pytest.mark.gpu

ORDERS = ("ASC", "DESC")


def _bits(x):
    return np.asarray(x, np.float64).view(np.uint64).tolist()


def assert_matches_spec(f, doc_ids, values, nbits, tag):
    for order in ORDERS:
        r = f.read(order)
        ed, ev = rank_order(doc_ids, values, nbits, order)
        assert r["nbits"] == nbits, tag
        assert r["rank_doc"].tolist() == ed.tolist(), (tag, order)
        assert _bits(r["rank_value"]) == _bits(ev), (tag, order)


def assert_same_build(a, b, tag):
    for order in ORDERS:
        ra, rb = a.read(order), b.read(order)
        assert ra["nbits"] == rb["nbits"], tag
        assert ra["rank_doc"].tobytes() == rb["rank_doc"].tobytes(), (tag, order)
        assert ra["rank_value"].tobytes() == rb["rank_value"].tobytes(), (tag, order)


# ---------------------------------------------------------------- 1. oc_sort_field_create = the spec
@pytest.mark.parametrize("n,nbits", [(0, 1), (1, 1), (9, 4), (1000, 300), (65537, 70000), (300000, 20000), (1 << 20, 1 << 20)])
def test_create_equals_the_spec(gpu_ctx, n, nbits):
    rng = np.random.default_rng(n + nbits)
    d, v = random_entries(rng, n, nbits)
    f = ob.SortField(gpu_ctx, nbits, d, v, "number")
    try:
        assert f.read()["facets_version"] == 0
        assert_matches_spec(f, d, v, nbits, (n, nbits))
    finally:
        f.close()


def test_create_is_deterministic_and_refuses(gpu_ctx):
    rng = np.random.default_rng(1)
    d, v = random_entries(rng, 200000, 50000)
    a, b = ob.SortField(gpu_ctx, 50000, d, v, "number"), ob.SortField(gpu_ctx, 50000, d, v, "number")
    assert_same_build(a, b, "twice")
    n = C.c_uint64(1)
    out = np.zeros(1, np.uint64)
    assert ob._lib.lib().oc_sort_field_read(a._h, 0, None, C.byref(n), out.ctypes.data, None, None) == -1   # capacity
    assert ob._lib.lib().oc_sort_field_read(a._h, 2, None, C.byref(n), None, None, None) == -1              # order
    a.close(); b.close()
    with pytest.raises(ValueError):
        ob.SortField(gpu_ctx, 4, [1], [np.nan], "number")
    h = C.c_void_p()
    x, dd = np.asarray([np.nan]), np.asarray([1], np.uint64)
    assert ob._lib.lib().oc_sort_field_create(gpu_ctx._h, 4, 1, dd.ctypes.data, x.ctypes.data, C.byref(h)) == -1 and not h.value


# ---------------------------------------------------------------- 2. from_facets = create over read_field
def _created(ctx, store, name, variant_values=None):
    lay = store.read_field(name)
    if "values" in lay:
        d, v = lay["doc_ids"], lay["values"]
    else:
        d, v = variant_entries(lay, variant_values)
    return ob.SortField(ctx, store.nbits, d, v, "number"), d, v


def _from_facets_raw(store, name, variant_values):
    vv = np.ascontiguousarray(variant_values, np.float64)
    f = ob.SortField.__new__(ob.SortField)
    f.ctx, f.kind, f._h = store.ctx, "number", C.c_void_p()
    ob.engine.check(ob._lib.lib().oc_sort_field_from_facets(store._h, store.fields[name]["id"], vv.ctypes.data, C.byref(f._h)))
    return f


def compare_store(ctx, store, version, tag):
    for name, fd in store.fields.items():
        kind = fd["kind"]
        if kind == "string":
            vv = np.linspace(-3.0, 3.0, len(fd["keys"]))[::-1].copy()
            vv[::3] = 0.0                               # ties between keys
            got = _from_facets_raw(store, name, vv)
        else:
            vv = [1.0 if k == "true" else 0.0 for k in fd["keys"]] if kind == "bool" else None
            got = ob.SortField.from_facets(store, name)
        exp, d, v = _created(ctx, store, name, vv)
        try:
            assert got.read()["facets_version"] == version, tag
            assert_same_build(got, exp, (tag, name))
            assert_matches_spec(got, d, v, store.nbits, (tag, name))
        finally:
            got.close(); exp.close()


def _store(ctx, rng, n_docs, nbits):
    st = ob.FacetStore(ctx, nbits)
    d = rng.integers(0, n_docs, size=n_docs + n_docs // 3).astype(np.uint64)          # repeats: multi-valued documents
    x = rng.choice([-0.0, 0.0, 1.5, -2.0, np.inf, -np.inf], size=d.shape[0])
    ints = rng.random(d.shape[0]) < 0.5
    x[ints] = rng.integers(-20, 20, size=int(ints.sum()))
    st.add_number_field("price", d, x)
    ms = rng.integers(2 ** 53 - 10 ** 6, 2 ** 53, size=n_docs // 2)
    st.add_date_field("when", rng.integers(0, n_docs, size=n_docs // 2), ms)
    t = rng.random(n_docs) < 0.4
    both = rng.random(n_docs) < 0.1
    st.add_bool_field("flag", np.flatnonzero(t | both), np.flatnonzero(~t | both))
    cat = rng.integers(0, 6, size=n_docs)
    st.add_string_field("cat", {f"k{k}": np.flatnonzero(cat == k) for k in range(6)})
    return st


@pytest.mark.parametrize("n_docs", [1, 500, 60000])
def test_from_facets_equals_create(gpu_ctx, n_docs):
    rng = np.random.default_rng(7 + n_docs)
    nbits = n_docs + 5
    st = _store(gpu_ctx, rng, n_docs, nbits)
    try:
        compare_store(gpu_ctx, st, 0, "add_*")
        for c in range(4):
            m = max(n_docs // 4, 3)
            grow = nbits + int(rng.integers(0, 50))
            docs = rng.integers(0, grow, size=m)
            st.insert_numbers("price", docs, rng.choice([-0.0, 0.0, 3.0, -1e300, np.inf], size=m))
            st.insert_numbers("when", docs[: m // 2], rng.integers(-2 ** 53, 2 ** 53, size=m // 2))
            st.insert_variants("flag", docs, rng.random(m) < 0.5)
            st.insert_variants("cat", docs, [f"k{int(k)}" for k in rng.integers(0, 9, size=m)])   # new keys too
            st.clear("price", rng.integers(0, grow, size=m // 5))
            st.clear("flag", rng.integers(0, grow, size=m // 5))
            st.delete(rng.integers(0, grow, size=m // 7))
            stats = st.commit(grow)
            nbits = grow
            compare_store(gpu_ctx, st, stats["version"], f"commit {c}")
            assert stats["version"] == c + 1
    finally:
        st.close()


def test_from_facets_refusals(gpu_ctx):
    st = ob.FacetStore(gpu_ctx, 10)
    st.add_number_field("n", [1, 2], [1.0, 2.0])
    st.add_string_field("s", {"a": [1], "b": [2]})
    L, h = ob._lib.lib(), C.c_void_p()
    vv = np.asarray([1.0, np.nan])
    for args in [(None, 0, None), (st._h, 2, None), (st._h, 0, vv.ctypes.data), (st._h, 1, None), (st._h, 1, vv.ctypes.data)]:
        assert L.oc_sort_field_from_facets(*args, C.byref(h)) == -1 and not h.value, args
    assert L.oc_sort_field_from_facets(st._h, 0, None, None) == -1
    with pytest.raises(ob.InvalidSortField):
        ob.SortField.from_facets(st, "s")
    with pytest.raises(ob.SortFieldNotFound):
        ob.SortField.from_facets(st, "x")
    st.close()


# ---------------------------------------------------------------- 3. sorted searches: from_facets handle = created handle
def _same_arrays(a, b, tag):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape and x.tobytes() == y.tobytes(), (tag, i)


def test_sorted_searches_with_either_handle(gpu_ctx):
    n, vocab, B = 20000, 800, 8
    rng = np.random.default_rng(31)
    rows = synth.make_vectors(n, 384, seed=32)
    qv, _ = synth.make_vector_queries(rows, B, seed=33)
    data = synth.make_text_corpus(n, vocab, seed=34)
    texts = synth.make_text_queries(vocab, B, seed=35)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    st = _store(gpu_ctx, rng, n, n + 3)
    st.insert_numbers("price", rng.integers(0, n, 3000), rng.integers(-5, 5, 3000))
    st.delete(rng.integers(0, n, 500))
    st.commit(n + 3)
    gb = ob.GroupBy(st, ["cat"])
    tsc = ob.TokenScoreContext(gpu_ctx, emb, strs)
    handles = []
    for name in ("price", "when", "flag"):
        vv = [1.0 if k == "true" else 0.0 for k in st.fields[name]["keys"]] if name == "flag" else None
        handles.append((name, ob.SortField.from_facets(st, name), _created(gpu_ctx, st, name, vv)[0]))
    promote = [[PromoteItem(int(rng.integers(0, n)), int(rng.integers(0, 12)))] if q % 2 else [] for q in range(B)]
    try:
        for phase in ("before", "after"):
            for mode in (MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID):
                p = ob.TokenScoreParams(mode=mode, limit_hint=20, offset=3, similarity=0.0)
                t = texts if mode != MODE_VECTOR else None
                v = qv if mode != MODE_FULLTEXT else None
                for name, ff, cr in handles:
                    for order in ORDERS:
                        for pr in (None, promote):
                            tag = (phase, mode, name, order, pr is not None)
                            _same_arrays(ob.search_sorted_arrays(tsc, p, ff, order, promote=pr, texts=t, q_vecs=v),
                                         ob.search_sorted_arrays(tsc, p, cr, order, promote=pr, texts=t, q_vecs=v), tag)
                            _same_arrays(ob.search_groups_arrays(tsc, gb, p, 3, texts=t, q_vecs=v, promote=pr, sort_by=(ff, order)),
                                         ob.search_groups_arrays(tsc, gb, p, 3, texts=t, q_vecs=v, promote=pr, sort_by=(cr, order)),
                                         tag + ("groups",))
                    mix = lambda h: [None if q % 3 == 0 else (h, ORDERS[q % 2]) for q in range(B)]  # noqa: E731
                    _same_arrays(ob.engine.search_q_sorted_arrays(tsc, p, mix(ff), promote=promote, texts=t, q_vecs=v),
                                 ob.engine.search_q_sorted_arrays(tsc, p, mix(cr), promote=promote, texts=t, q_vecs=v),
                                 (phase, mode, name, "q_sorted"))
            strs.delete(np.arange(0, n, 3, dtype=np.uint64))   # rows shift: the rank -> row maps are rebuilt
            strs.commit()
    finally:
        for _, a, b in handles:
            a.close(); b.close()
        gb.close(); st.close(); emb.close(); strs.close()


# ---------------------------------------------------------------- 4. IndexLoader.sort_by over op streams
def check_loader_sorts(tag, ld, model, orc, stream, sorted_fields):
    fields = ld.sort_fields()
    for name in ("flag", "price", "when"):
        docs, vals = model.sort_values(name)
        assert_matches_spec(fields[name], docs, vals, model.nbits, (tag, name))
    ex = Expect(orc, model)
    try:
        batch = ld.resolve(stream.texts(6))
        qs = [batch.query(i) for i in range(batch.n_queries)]
        tq = ob.engine.TextQueryBatch(qs)
        tsc = ld.context()
        p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, offset=2)
        maps = [_as_dict(ex.ft(q)) for q in qs]
        for name, order in sorted_fields:
            f, o = ld.sort_by(ob.SortBy(name, order))
            assert f is fields[name]
            docs, vals = model.sort_values(name)
            rk = ranks(docs, vals + 0.0, o)
            sd, ss, sv, sn, sc, _, _ = ob.search_sorted_arrays(tsc, p, f, o, texts=tq)
            for i in range(len(qs)):
                check(sd[i, :sn[i]], ss[i, :sn[i]], sv[i, :sn[i]], expect_flat(maps[i], rk, 10, 2), True)
                assert int(sc[i]) == len(maps[i]), (tag, name, order, i)
    finally:
        ex.close()


def test_loader_sort_by_follows_refreshes(gpu_ctx, orc):
    stream = Stream(21, 16, 500)
    ld = IndexLoader(gpu_ctx, STRING_FIELDS, embedding_dim=16, **FILTERS)
    model = IndexModel(STRING_FIELDS, dim=16, **FILTERS)
    sorted_fields = [("price", "ASC"), ("price", "DESC"), ("when", "DESC"), ("flag", "ASC"), ("flag", "DESC")]
    try:
        for op in stream.round(500):
            ld.apply(op); model.apply(op)
        ld.commit(); model.commit()
        for r in range(4):
            check_loader_sorts(f"round {r} committed", ld, model, orc, stream, sorted_fields)
            old = ld.sort_fields()["price"]
            for op in stream.round(300):
                ld.apply(op); model.apply(op)
            # queued values do not move a sort before the refresh that publishes them
            assert ld.sort_fields()["price"] is old
            check_loader_sorts(f"round {r} queued", ld, model, orc, stream, sorted_fields)
            if r % 2:
                ld.refresh_facets(); model.refresh_facets()
            else:
                ld.commit(); model.commit()
            assert old._h is None                      # the previous version's handle is closed
            check_loader_sorts(f"round {r} published", ld, model, orc, stream, sorted_fields)
        for name, kind in (("cat", "StringFilter"), ("loc", "GeoPoint"), ("title", "String")):
            with pytest.raises(ob.InvalidSortField) as e:
                ld.sort_by(ob.SortBy(name))
            assert e.value.kind == kind
        with pytest.raises(ob.SortFieldNotFound):
            ld.sort_by(ob.SortBy("nope"))
    finally:
        ld.close()


# ---------------------------------------------------------------- 5. a build racing a commit of its store
def test_from_facets_during_a_commit(gpu_ctx):
    rng = np.random.default_rng(77)
    n = 3_000_000
    st = ob.FacetStore(gpu_ctx, n)
    st.add_number_field("price", np.arange(n), rng.integers(-1000, 1000, size=n).astype(np.float64))
    before = _created(gpu_ctx, st, "price")[0]
    m = 400_000
    st.insert_numbers("price", rng.integers(0, n, m), rng.normal(0, 100, m))
    st.clear("price", rng.integers(0, n, m // 4))
    st.delete(rng.integers(0, n, m // 8))
    stats = {}
    th = threading.Thread(target=lambda: stats.update(st.commit(n)))
    got = []
    th.start()
    while th.is_alive() and len(got) < 50:
        got.append(ob.SortField.from_facets(st, "price"))
    th.join()
    after = _created(gpu_ctx, st, "price")[0]
    got.append(ob.SortField.from_facets(st, "price"))
    try:
        assert stats["version"] == 1
        versions = [f.read()["facets_version"] for f in got]
        assert set(versions) <= {0, 1} and versions == sorted(versions) and versions[-1] == 1, versions
        for f, ver in zip(got, versions):
            assert_same_build(f, before if ver == 0 else after, ver)
    finally:
        for f in got + [before, after]:
            f.close()
        st.close()
