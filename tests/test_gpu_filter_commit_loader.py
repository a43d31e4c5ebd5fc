"""IndexLoader driven through the device filter-field commit: after each of several commits, where_filter,
where_program, facet counts and groups equal, byte for byte, the same calls on stores the test builds from scratch from
its own record of the op stream (the per-document values IndexLoader.apply's rules give), with uncommitted deletes
before and after the commit.  Also: a store built by FacetStore.add_* with ties, mixed -0.0 / +0.0 and unsorted
documents takes commits like one built by commits."""
import copy

import numpy as np
import pytest

import filter_commit_spec as S
import oramacore_b200 as ob
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT
from oramacore_b200.where import evaluate_where, parse_where

pytestmark = pytest.mark.gpu

WORDS = ["alpha", "beta", "gamma", "delta"]


class Record:
    """The filter values IndexLoader.apply's rules give each live document (tests/filter_commit_spec.py)."""

    def __init__(self):
        self.b, self.n, self.s, self.d, self.g = {}, {}, {}, {}, {}

    def index(self, d, vals):
        for v in vals:
            t = v["type"]
            if t == "FilterBool":
                self.b[d] = {bool(v["value"])}
            elif t == "FilterBool2":
                self.b.setdefault(d, set()).update(bool(x) for x in v["value"]["Array"])
            elif t == "FilterNumber2":
                self.n.setdefault(d, []).extend(float(x) for x in v["value"]["F64"]["Array"])
            elif t == "FilterString2":
                self.s.setdefault(d, []).extend(v["value"]["Array"])
            elif t == "FilterDate2":
                self.d.setdefault(d, []).extend(int(x) for x in v["value"]["Array"])
            elif t == "FilterGeoPoint2":
                self.g.setdefault(d, []).extend((p["lat"], p["lon"]) for p in v["value"]["Array"])

    def delete(self, d):
        for m in (self.b, self.n, self.s, self.d, self.g):
            m.pop(d, None)

    def stores(self, ctx, nbits):
        """As IndexLoader built them before it committed on the device: string_filter keys sorted, only keys that hold
        documents."""
        st = ob.FacetStore(ctx, nbits)
        st.add_bool_field("b", [d for d, bs in self.b.items() if True in bs], [d for d, bs in self.b.items() if False in bs])
        st.add_number_field("n", [d for d, xs in self.n.items() for _ in xs], [x for xs in self.n.values() for x in xs])
        st.add_date_field("d", [d for d, xs in self.d.items() for _ in xs], [x for xs in self.d.values() for x in xs])
        by = {}
        for d, ks in self.s.items():
            for k in ks:
                by.setdefault(k, []).append(d)
        st.add_string_field("s", {k: by[k] for k in sorted(by)})
        g = ob.GeoPointField(ctx, nbits, [d for d, ps in self.g.items() for _ in ps], [p[0] for ps in self.g.values() for p in ps],
                             [p[1] for ps in self.g.values() for p in ps])
        return st, g


def _op(rng, d):
    toks = [WORDS[int(i)] for i in rng.integers(0, len(WORDS), int(rng.integers(1, 5)))]
    terms = {}
    for i, t in enumerate(toks):
        terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
    arr = lambda xs: {"Array": list(xs)}   # noqa: E731
    vals = [{"type": "ScoreString2", "field": "text", "field_length": len(toks), "terms": terms}]
    if rng.random() < 0.5:
        vals.append({"type": "FilterBool", "field": "b", "value": bool(rng.random() < 0.5)})
    if rng.random() < 0.5:
        vals.append({"type": "FilterBool2", "field": "b", "value": arr(bool(x) for x in rng.random(int(rng.integers(1, 3))) < 0.5)})
    vals.append({"type": "FilterNumber2", "field": "n",
                 "value": {"F64": arr(float(x) for x in rng.choice([-0.0, 0.0, 1.0, 2.0, 7.5], int(rng.integers(0, 3))))}})
    vals.append({"type": "FilterString2", "field": "s", "value": arr(f"k{int(x)}" for x in rng.integers(0, 6, int(rng.integers(0, 3))))})
    vals.append({"type": "FilterDate2", "field": "d", "value": arr(int(x) for x in rng.integers(0, 10**12, int(rng.integers(0, 2))))})
    vals.append({"type": "FilterGeoPoint2", "field": "g",
                 "value": arr({"lat": float(rng.uniform(-50, 50)), "lon": float(rng.uniform(-90, 90))} for _ in range(int(rng.integers(0, 2))))})
    return {"type": "Index", "doc_id": d, "indexed_values": vals}


CLAUSES = [{"b": True}, {"b": False}, {"n": {"between": [0, 2]}}, {"n": {"gt": 1}}, {"s": "k2"}, {"s": "k9"},
           {"d": {"lt": "2001-09-09T01:46:40Z"}},
           {"g": {"radius": {"coordinates": {"lat": 0, "lon": 0}, "value": 3000, "unit": "km", "inside": True}}},
           {"and": [{"b": True}, {"not": {"s": "k1"}}]}, {"or": [{"n": {"lte": 0}}, {"s": "k4"}]}, {}]


def _compare(ld, rec, tag):
    """rec: the record as of the last refresh_facets() / commit(); the deletes since the last commit are excluded."""
    st, g = rec.stores(ld.ctx, ld.nbits)
    deleted = sorted(ld._uncommitted_deleted)
    tsc = ld.context()
    texts = ld.resolve(["alpha beta"] * len(CLAUSES))
    kw = dict(mode=MODE_FULLTEXT, limit_hint=40)
    try:
        mine = [ld.where_filter(w) for w in CLAUSES]
        ref = [evaluate_where(parse_where(w), st, {"g": g}, ld.nbits, deleted, ctx=ld.ctx) for w in CLAUSES]
        try:
            for w, a, b in zip(CLAUSES, mine, ref):
                assert (a is None) == (b is None), (tag, w)
                if a is not None:
                    assert a.read().tobytes() == b.read().tobytes(), (tag, w)
            got = tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=[ld.where_program(w) for w in CLAUSES], **kw), texts)
            exp = tsc.execute_batch_arrays(ob.TokenScoreParams(device_filters=ref, **kw), texts)
            for x, y in zip(got, exp):
                assert x.tobytes() == y.tobytes(), tag
        finally:
            for h in mine + ref:
                if h is not None:
                    h.close()
        facets = {"b": {"true": True, "false": True}, "n": {"ranges": [{"from": 0, "to": 1}, {"from": -1, "to": 10}]}, "s": {}}
        p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10)
        f_ref = ob.search_facets(tsc, st, p, facets, texts=ld.resolve(["alpha"]))
        f_got = ob.search_facets(tsc, ld.facets, p, facets, texts=ld.resolve(["alpha"]))
        assert f_got == f_ref, tag
        g1, g2 = ob.GroupBy(ld.facets, ["b", "n"]), ob.GroupBy(st, ["b", "n"])
        try:
            assert g1.values == g2.values, tag
            a = ob.search_groups_arrays(tsc, g1, p, 3, texts=ld.resolve(["alpha"]))
            b = ob.search_groups_arrays(tsc, g2, p, 3, texts=ld.resolve(["alpha"]))
            for x, y in zip(a, b):
                assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), tag
        finally:
            g1.close(); g2.close()
    finally:
        st.close(); g.close()


def test_loader_commits_equal_stores_built_from_scratch(gpu_ctx):
    rng = np.random.default_rng(5)
    ld = IndexLoader(gpu_ctx, ["text"], bool_fields=["b"], number_fields=["n"], string_filter_fields=["s"], date_fields=["d"],
                     geopoint_fields=["g"])
    rec = Record()
    facets0, geo0 = ld.facets, ld.geo["g"]
    try:
        n_docs = 0
        for rnd in range(4):
            for _ in range(150):
                d = int(rng.integers(0, n_docs + 60))
                if rng.random() < 0.15 and n_docs:
                    ld.apply({"type": "DeleteDocuments", "doc_ids": [d]})
                    rec.delete(d)
                else:
                    op = _op(rng, d)
                    ld.apply(op)
                    rec.index(d, op["indexed_values"])
                    n_docs = max(n_docs, d + 1)
            ld.commit()
            assert ld.facets is facets0 and ld.geo["g"] is geo0   # the stores persist across commits
            _compare(ld, rec, ("committed", rnd))
            published = copy.deepcopy(rec)
            dels = [int(x) for x in rng.integers(0, n_docs, 5)]
            ld.apply({"type": "DeleteDocuments", "doc_ids": dels})   # uncommitted: excluded at once
            for x in dels:
                rec.delete(x)
            _compare(ld, published, ("uncommitted deletes", rnd))
            ld.refresh_facets()                                       # publish without a commit: deletes stay uncommitted
            _compare(ld, rec, ("published", rnd))
    finally:
        ld.close()


def test_commit_into_a_store_built_with_ties_and_signed_zeros(gpu_ctx):
    """add_number_field / add_field take documents in any order inside a run of equal values or a variant; commits
    merge into them as into a store built by commits."""
    st = ob.FacetStore(gpu_ctx, 20)
    try:
        st.add_number_field("n", [5, 3, 9, 2, 8], [1.0, 1.0, 0.0, -0.0, 0.0])
        st.add_string_field("s", {"a": [7, 2, 4], "b": [6, 1]})
        st.insert_numbers("n", [4, 1, 3], [1.0, -0.0, 1.0])
        st.insert_variants("s", [3, 5], ["a", "b"])
        st.delete([9])
        st.commit()
        prev_n = {"values": np.asarray([-0.0, 0.0, 0.0, 1.0, 1.0]), "docs": np.asarray([2, 8, 9, 3, 5], np.uint64)}
        ops_n = [("ins", 0, 4, 1.0, False), ("ins", 0, 1, -0.0, False), ("ins", 0, 3, 1.0, False), ("del", 9)]
        exp = S.commit("number", 0, prev_n, ops_n)
        got = st.read_field("n")
        assert S.same_up_to_ties("number", {"values": got["values"], "docs": got["doc_ids"]}, exp)
        assert got["values"].tolist() == sorted(got["values"].tolist())
        s = st.read_field("s")
        assert s["offsets"].tolist() == [0, 4, 7] and s["doc_ids"].tolist() == [2, 3, 4, 7, 1, 5, 6]
    finally:
        st.close()
