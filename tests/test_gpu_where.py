"""`where` clauses on the GPU (oc_filter_facet_variant / oc_filter_facet_range, FacetStore.leaf, where.evaluate_where,
IndexLoader.where_filter) against
  (1) the reference's own answers (src/tests/filter.rs, all ten tests), driven through IndexLoader op streams with the
      values the write side emits (FilterNumber2 / FilterBool2 / FilterString2 / FilterDate2);
  (2) the host restatement of tests/test_where_host.py, bit for bit, for every leaf kind and op and for random trees
      up to depth 4 with geopoint polygon leaves, over ~200 K documents with multi-valued fields, ids >= nbits and
      uncommitted deletes;
and checks that searches under a where-filter are byte-identical to the same bitmap passed as filter_bits, and that
every refused call creates nothing."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib
from oramacore_b200.hostindex import tokenize
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from oramacore_b200.where import evaluate_where, parse_where
from test_gpu_pins import N, _inputs, _tsc, corpus  # noqa: F401  (corpus: fixture)
from test_where_host import host_where

pytestmark = pytest.mark.gpu


def _ids(f):
    if f is None:
        return None
    try:
        bits = f.read()
        return set(np.flatnonzero(np.unpackbits(bits.view(np.uint8), bitorder="little")[:f.nbits]).tolist())
    finally:
        f.close()


# ---------------------------------------------------------------- the reference's answers (src/tests/filter.rs)
class Collection:
    """One index fed through IndexLoader with the ops the write side emits.  Every insert takes the next DocumentId.
    The loader publishes inserts at commit; the reference's searches see them at once, so `publish()` makes them
    searchable while deletes stay uncommitted."""

    def __init__(self, ctx, **fields):
        self.ctx, self.fields, self.ops, self.next = ctx, fields, [], 1
        self.ld = IndexLoader(ctx, ["text"], **fields)

    def insert(self, docs):
        for doc in docs:
            d, self.next = self.next, self.next + 1
            toks = tokenize(doc.get("text", ""))
            terms = {}
            for i, t in enumerate(toks):
                terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
            vals = [{"type": "ScoreString2", "field": "text", "field_length": len(toks), "terms": terms}]
            vals += [dict(v, field=k) for k, v in doc.get("filters", {}).items()]
            self.apply({"type": "Index", "doc_id": d, "indexed_values": vals})

    def apply(self, op):
        self.ops.append(op)
        self.ld.apply(op)

    def publish(self):
        self.ld.strs.commit()
        self.ld.refresh_facets()

    def commit(self):
        self.ld.commit()

    def reload(self):
        self.ld.close()
        self.ld = IndexLoader(self.ctx, ["text"], **self.fields)
        self.ld.apply_all(self.ops)
        self.ld.commit()

    def search(self, term, where):
        f = self.ld.where_filter(where)
        try:
            return self.ld.context().execute_batch(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, device_filter=f),
                                                   self.ld.resolve([term]))[0]
        finally:
            if f is not None:
                f.close()

    def count(self, term, where):
        return self.search(term, where).count

    def close(self):
        self.ld.close()


def num(x):
    return {"type": "FilterNumber2", "value": {"I64": {"Plain": x}} if isinstance(x, int) else {"F64": {"Plain": x}}}


def nums(xs):
    return {"type": "FilterNumber2", "value": {"I64": {"Array": xs}}}


def boo(b, array=False):
    return {"type": "FilterBool2", "value": {"Array": [b]} if array else {"Plain": b}}


def strf(s):
    return {"type": "FilterString2", "value": {"Plain": s}}


def date(ms):
    return {"type": "FilterDate2", "value": {"Plain": ms}}


@pytest.fixture
def make(gpu_ctx):
    made = []

    def mk(**fields):
        c = Collection(gpu_ctx, **fields)
        made.append(c)
        return c
    yield mk
    for c in made:
        c.close()


def test_search_on_unknown_field(make):   # :9-39
    c = make(number_fields=["number"])
    c.insert([{"text": "Doe", "filters": {"number": num(1)}}])
    c.publish()
    with pytest.raises(ob.FilterFieldNotFound):
        c.search("Doe", {"unknown_field": {"eq": 1}})


def test_filter_number(make):   # :41-183
    c = make(number_fields=["number"])
    c.insert([{"text": "text " * (i + 1), "filters": {"number": num(i)}} for i in range(100)])
    c.publish()
    h = c.search("text", {"number": {"eq": 50}})
    assert h.count == 1 and h.doc_ids.tolist() == [51]   # id "50" is the 51st insert
    for op, expect in [("gt", 97), ("gte", 98), ("lt", 2), ("lte", 3)]:
        assert c.count("text", {"number": {op: 2}}) == expect, op
    assert c.count("text", {"number": {"between": [2, 4]}}) == 3


def test_filter_number_float_boundary_exclusion(make):   # :185-301
    c = make(number_fields=["number"])
    c.insert([{"text": "text " * (i + 1), "filters": {"number": num(i)}} for i in range(11)])
    c.publish()
    for op, expect in [("gt", 5), ("lt", 5), ("gte", 6), ("lte", 6)]:
        assert c.count("text", {"number": {op: 5.0}}) == expect, op


def test_filter_bool(make):   # :303-385
    c = make(bool_fields=["bool"])
    c.insert([{"text": "text " * (i + 1), "filters": {"bool": boo(i % 2 == 0)}} for i in range(100)])
    c.publish()
    for b, parity in [(True, 0), (False, 1)]:
        h = c.search("text", {"bool": b})
        assert h.count == 50 and len(h.doc_ids) == 10
        assert all((int(d) - 1) % 2 == parity for d in h.doc_ids)


def test_filter_string(make):   # :387-424
    c = make(string_filter_fields=["text"])
    c.insert([{"text": f"text {str(i % 2 == 0).lower()}", "filters": {"text": strf(f"text {str(i % 2 == 0).lower()}")}}
              for i in range(100)])
    c.publish()
    assert c.count("text", {"text": "text true"}) == 50


def test_array_types(make):   # :426-495
    c = make(number_fields=["number"], bool_fields=["bool"])
    c.insert([{"text": "text " * (i + 1), "filters": {"number": nums([i]), "bool": boo(i % 2 == 0, array=True)}}
              for i in range(10)])
    c.publish()
    assert c.count("text", {}) == 10
    assert c.count("text", {"number": {"eq": 5}}) == 1
    assert c.count("text", {"bool": True}) == 5


def test_filter_and_or_not(make):   # :497-573
    c = make(number_fields=["number"], bool_fields=["bool"], string_filter_fields=["text"])
    c.insert([{"text": f"text {str(i % 3 == 0).lower()}",
               "filters": {"number": num(i), "bool": boo(i % 2 == 0), "text": strf(f"text {str(i % 3 == 0).lower()}")}}
              for i in range(100)])
    c.publish()
    assert c.count("text", {"and": [{"bool": True}, {"number": {"gte": 50}}]}) == 25
    assert c.count("text", {"or": [{"bool": True}, {"number": {"gte": 50}}]}) == 75
    assert c.count("text", {"not": {"bool": True}}) == 50


DAY0 = 1672531200000   # 2023-01-01T00:00:00Z


def test_date(make):   # :575-816
    c = make(date_fields=["date"])
    c.insert([{"text": "test", "filters": {"date": date(DAY0 + k * 86400000)}} for k in range(3)])

    def check():
        assert c.count("", {"date": {"gt": "2023-01-01T00:00:00Z"}}) == 2
        assert c.count("", {"date": {"lt": "2023-01-03T00:00:00Z"}}) == 2
        assert c.count("", {"date": {"gte": "2023-01-01T00:00:00Z"}}) == 3
        assert c.count("", {"date": {"lte": "2023-01-03T00:00:00Z"}}) == 3
        assert c.count("", {"date": {"between": ["2023-01-01T00:00:01Z", "2023-01-02T23:59:59Z"]}}) == 1
    c.publish()
    check()
    c.commit()
    check()
    c.reload()
    check()


def test_enum_strategy(make):   # :818-910: the Explicit strategy emits the parsed enum value
    c = make(string_filter_fields=["enum"])
    c.insert([{"text": "text " * (i + 1), "filters": {"enum": strf("even" if i % 2 == 0 else "odd")}} for i in range(100)])
    c.publish()
    assert c.count("text", {"enum": "even"}) == 50
    c.commit()
    c.reload()
    assert c.count("text", {"enum": "even"}) == 50


def test_long_strings_are_not_indexed_as_string_filter(make):   # :912-986: no FilterString2 for the long value
    c = make(string_filter_fields=["category"])
    c.insert([{"text": "hello world", "filters": {"category": strf("short")}}, {"text": "hello world"},
              {"text": "hello world", "filters": {"category": strf("short")}}])
    c.publish()
    assert c.count("hello", {"category": "short"}) == 2
    assert c.count("hello", {"category": "this string is way too long to be indexed"}) == 0


def test_loader_deletes_and_i64_refusal(make):
    c = make(number_fields=["n"], bool_fields=["b"])
    c.insert([{"text": "t", "filters": {"n": num(i), "b": boo(i % 2 == 0)}} for i in range(10)])
    c.commit()
    c.apply({"type": "DeleteDocuments", "doc_ids": [1, 2]})
    assert _ids(c.ld.where_filter({"n": {"lt": 4}})) == {3, 4}
    assert _ids(c.ld.where_filter({})) == set(range(c.ld.nbits)) - {1, 2}
    assert c.ld.where_filter({"or": []}) is not None   # is_empty, but the deletes still filter
    c.commit()
    assert c.ld.where_filter({}) is None
    assert _ids(c.ld.where_filter({"n": {"lt": 4}})) == {3, 4}
    with pytest.raises(ValueError):
        c.apply({"type": "Index", "doc_id": 50, "indexed_values": [{"type": "FilterNumber2", "field": "n",
                                                                      "value": {"I64": {"Plain": 2**53 + 1}}}]})


# ---------------------------------------------------------------- leaves and trees against the host restatement
ND, NBITS = 200_000, 190_000


@pytest.fixture(scope="module")
def store(gpu_ctx):
    rng = np.random.default_rng(5)
    docs = np.arange(ND)

    def multi(p_has, p_two):
        has = docs[rng.random(ND) < p_has]
        return np.concatenate([has, has[rng.random(has.shape[0]) < p_two]])
    fields = {}
    nd = multi(0.9, 0.3)
    nv = np.where(rng.random(nd.shape[0]) < 0.5, rng.integers(-50, 50, nd.shape[0]), rng.standard_normal(nd.shape[0]) * 30)
    nv[rng.random(nd.shape[0]) < 0.01] = -0.0
    fields["n"] = ("number", (nd, nv.astype(np.float64)))
    dd = multi(0.8, 0.2)
    fields["d"] = ("date", (dd, (rng.integers(-3 * 10**11, 2 * 10**12, dd.shape[0])).astype(np.float64)))
    bd = multi(0.9, 0.1)
    bv = rng.random(bd.shape[0]) < 0.5
    bm = {}
    for d_, b_ in zip(bd.tolist(), bv.tolist()):
        bm.setdefault(d_, set()).add(b_)
    fields["b"] = ("bool", bm)
    sd = multi(0.7, 0.4)
    keys = [f"k{i}" for i in range(12)]
    sm = {}
    for d_, k_ in zip(sd.tolist(), rng.integers(0, 12, sd.shape[0]).tolist()):
        sm.setdefault(d_, []).append(keys[k_])
    fields["s"] = ("string", sm)
    gd = multi(0.8, 0.2)
    glat, glon = rng.uniform(-60, 60, gd.shape[0]), rng.uniform(-120, 120, gd.shape[0])
    fields["g"] = ("geo", (gd, glat, glon))

    st = ob.FacetStore(gpu_ctx, NBITS)
    st.add_number_field("n", nd, nv)
    st.add_date_field("d", dd, fields["d"][1][1].astype(np.int64))
    st.add_bool_field("b", [d_ for d_, bs in bm.items() if True in bs], [d_ for d_, bs in bm.items() if False in bs])
    by_key = {}
    for d_, ks in sm.items():
        for k_ in ks:
            by_key.setdefault(k_, []).append(d_)
    st.add_string_field("s", by_key)
    geo = {"g": ob.GeoPointField(gpu_ctx, NBITS, gd, glat, glon)}
    deleted = rng.choice(ND, 3000, replace=False).tolist()
    yield st, geo, fields, deleted, rng, nv
    st.close()
    geo["g"].close()


def _num_bound(rng, nv):
    r = rng.random()
    if r < 0.3:
        return int(rng.integers(-60, 60))
    if r < 0.6:
        return float(nv[rng.integers(0, nv.shape[0])])   # a stored value (f32-rounded by the parser)
    return float(rng.choice([0.0, -0.0, 1e39, -1e39, 2.5, float(rng.standard_normal() * 40)]))


def _date_str(ms):
    import datetime
    t = datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc) + datetime.timedelta(milliseconds=int(ms))
    return t.strftime("%Y-%m-%dT%H:%M:%S.") + f"{t.microsecond // 1000:03d}Z"


def _leaf_json(rng, key, nv, fields):
    ops = ["eq", "gt", "gte", "lt", "lte", "between"]
    if key == "n":
        op = ops[rng.integers(0, 6)]
        v = [_num_bound(rng, nv), _num_bound(rng, nv)] if op == "between" else _num_bound(rng, nv)
        return {op: v}
    if key == "d":
        op = ops[rng.integers(0, 6)]
        vals = fields["d"][1][1]
        pick = lambda: _date_str(vals[rng.integers(0, vals.shape[0])] + rng.integers(-1, 2))  # noqa: E731
        return {op: [pick(), pick()] if op == "between" else pick()}
    if key == "b":
        return bool(rng.random() < 0.5)
    if key == "s":
        return f"k{rng.integers(0, 14)}"   # k12, k13: unknown keys
    if key == "g":
        c = rng.uniform(-40, 40, 2)
        a = np.linspace(0, 2 * np.pi, int(rng.integers(3, 9)), endpoint=False)
        rr = rng.uniform(5, 45)   # vertices stay within +-85 degrees of latitude
        return {"polygon": {"coordinates": [{"lat": float(c[0] + rr * np.sin(t)), "lon": float(c[1] + rr * np.cos(t))} for t in a],
                            "inside": bool(rng.random() < 0.7)}}
    return {"eq": 5}   # key "zz": not a field of the index


def _tree(rng, depth, nv, fields):
    w = {}
    for key in rng.choice(["n", "d", "b", "s", "g", "n", "zz"], int(rng.integers(0, 3)), replace=False):
        w[str(key)] = _leaf_json(rng, str(key), nv, fields)
    if depth < 4:
        if rng.random() < 0.4:
            w["and"] = [_tree(rng, depth + 1, nv, fields) for _ in range(int(rng.integers(0, 3)))]
        if rng.random() < 0.4:
            w["or"] = [_tree(rng, depth + 1, nv, fields) for _ in range(int(rng.integers(0, 3)))]
        if rng.random() < 0.3:
            w["not"] = _tree(rng, depth + 1, nv, fields)
    return w


def _check(store, where, deleted):
    st, geo, fields, _, _, _ = store
    w = parse_where(where)
    got = _ids(evaluate_where(w, st, geo, NBITS, deleted))
    assert got == host_where(w, fields, NBITS, deleted), where


@pytest.mark.parametrize("key", ["n", "d", "b", "s", "g"])
def test_every_leaf_kind_and_op(store, key):
    st, geo, fields, deleted, rng, nv = store
    for _ in range(40):
        _check(store, {key: _leaf_json(rng, key, nv, fields)}, ())
    for op in ("eq", "gt", "gte", "lt", "lte"):
        for b in ([0, -0.0, 0.0, 1e39, -1e39, 2**31, 5.5] if key == "n" else []):
            _check(store, {key: {op: b}}, ())
    _check(store, {key: {"between": [10, -10]} if key == "n" else True}, deleted[:10])
    # the wrong kind of filter for the field: empty
    for wrong in (True, "k1", {"gt": 0}, {"gt": "2000-01-01T00:00:00Z"}, {"radius": {"coordinates": {"lat": 0, "lon": 0}, "value": 1e7}}):
        if key != "g" or not isinstance(wrong, dict) or "radius" not in wrong:   # the host restatement has no radius (test_gpu_geo.py checks it)
            _check(store, {key: wrong}, ())


def test_random_trees(store):
    st, geo, fields, deleted, rng, nv = store
    for i in range(120):
        where = _tree(rng, 1, nv, fields)
        _check(store, where, deleted if i % 2 else ())


# ---------------------------------------------------------------- searches: where_filter == the same bitmap as filter_bits
@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
def test_searches_byte_identical_to_filter_bits(corpus, mode):
    c = corpus
    rng = np.random.default_rng(77)
    ctx = c["strs"].ctx
    st = ob.FacetStore(ctx, c["nbits"])
    try:
        st.add_number_field("price", c["ids"], rng.integers(0, 100, N).astype(np.float64))
        st.add_bool_field("ok", c["ids"][rng.random(N) < 0.6], c["ids"][rng.random(N) < 0.5])
        st.add_string_field("cat", {k: c["ids"][rng.random(N) < 0.3] for k in ("a", "b", "c")})
        tsc = _tsc(c, mode)
        texts, qv = _inputs(c, mode)
        for where in ({"price": {"between": [10, 60]}, "or": [{"ok": True}, {"cat": "b"}]},
                      {"not": {"cat": "a"}, "price": {"lt": 90.5}}):
            f = evaluate_where(parse_where(where), st, {}, c["nbits"], [5, 77, 4000])
            try:
                bits = f.read()
                assert 0 < f.count() < c["nbits"]
                for limit, offset in [(10, 0), (50, 7)]:
                    kw = dict(mode=mode, limit_hint=limit, offset=offset, similarity=0.0)
                    a = tsc.execute_batch_arrays(ob.TokenScoreParams(device_filter=f, **kw), texts, qv)
                    b = tsc.execute_batch_arrays(ob.TokenScoreParams(filtered_doc_ids=bits, filter_nbits=c["nbits"], **kw), texts, qv)
                    for x, y in zip(a, b):
                        assert x.tobytes() == y.tobytes(), (where, mode, limit)
            finally:
                f.close()
    finally:
        st.close()


# ---------------------------------------------------------------- refusals (through the C ABI)
def test_refusals_create_nothing(gpu_ctx):
    L = _lib.lib()
    st = ob.FacetStore(gpu_ctx, 100)
    try:
        st.add_bool_field("b", [1, 2], [3])
        st.add_number_field("n", [1, 2, 3], [1.0, 2.0, 3.0])
        fb, fn = st.fields["b"]["id"], st.fields["n"]["id"]
        calls = [
            lambda h: L.oc_filter_facet_variant(None, fb, 0, C.byref(h)),
            lambda h: L.oc_filter_facet_variant(st._h, fb, 0, None),
            lambda h: L.oc_filter_facet_variant(st._h, 7, 0, C.byref(h)),        # field out of range
            lambda h: L.oc_filter_facet_variant(st._h, fb, 2, C.byref(h)),       # variant out of range
            lambda h: L.oc_filter_facet_variant(st._h, fn, 0, C.byref(h)),       # number field
            lambda h: L.oc_filter_facet_range(None, fn, 0.0, 1.0, 0, C.byref(h)),
            lambda h: L.oc_filter_facet_range(st._h, fn, 0.0, 1.0, 0, None),
            lambda h: L.oc_filter_facet_range(st._h, 9, 0.0, 1.0, 0, C.byref(h)),
            lambda h: L.oc_filter_facet_range(st._h, fb, 0.0, 1.0, 0, C.byref(h)),  # bool field
            lambda h: L.oc_filter_facet_range(st._h, fn, float("nan"), 1.0, 0, C.byref(h)),
            lambda h: L.oc_filter_facet_range(st._h, fn, 0.0, float("nan"), 0, C.byref(h)),
            lambda h: L.oc_filter_facet_range(st._h, fn, 0.0, 1.0, 4, C.byref(h)),   # unknown flag bits
        ]
        for i, call in enumerate(calls):
            h = C.c_void_p(0xDEAD0)
            assert call(h) == -1, i
            assert h.value == 0xDEAD0, i   # *out untouched
        h = C.c_void_p()
        assert L.oc_filter_facet_range(st._h, fn, 1.0, 3.0, _lib.OC_RANGE_LO_OPEN | _lib.OC_RANGE_HI_OPEN, C.byref(h)) == 0
        assert _ids(ob.DeviceFilter(gpu_ctx, h, 100)) == {2}
        h = C.c_void_p()
        assert L.oc_filter_facet_range(st._h, fn, -np.inf, np.inf, 0, C.byref(h)) == 0
        assert _ids(ob.DeviceFilter(gpu_ctx, h, 100)) == {1, 2, 3}
    finally:
        st.close()
    st = ob.FacetStore(gpu_ctx, 10)
    try:
        st.add_date_field("d", [1], [0])
        with pytest.raises(ValueError):
            ob.GroupBy(st, ["d"])
    finally:
        st.close()
