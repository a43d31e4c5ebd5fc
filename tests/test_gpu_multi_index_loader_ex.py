"""Facets and groupBy across the indexes of a collection through the loader (loader.search_collection_ex, one
oc_search_indexes_ex call): src/tests/facets.rs:461-576 (two indexes, one index empty), groupby.rs:9-175 and
groupby.rs:984-1062 (groups with a pin rule) with the documents split over two indexes, an index that lacks the group
property, and the error cases."""
import pytest

import oramacore_b200 as ob
from oramacore_b200.loader import IndexLoader, search_collection_ex
from oramacore_b200.types import MODE_FULLTEXT, FacetFieldNotFound
from test_gpu_loader import _index_op

pytestmark = pytest.mark.gpu


def _params(limit=10):
    return ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=limit)


def test_facets_on_multiple_index_collection(gpu_ctx):
    # facets.rs:461-519: two indexes of 10 documents each, category A / B alternating -> A: 10, B: 10
    a = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"])
    b = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"])
    try:
        a.apply_all([_index_op(i, f"title {i}", category="A" if i % 2 == 0 else "B") for i in range(10)])
        b.apply_all([_index_op(10 + i, f"title {i}", category="A" if i % 2 == 0 else "B") for i in range(10)])
        a.commit(); b.commit()
        r = search_collection_ex([a, b], [""], _params(), facets={"category": {}})[0]
        assert r["facets"]["category"]["values"] == {"A": 10, "B": 10}
        assert r["hits"].count == 20 and r["groups"] is None
    finally:
        a.close(); b.close()


def test_facets_with_different_shaped_index(gpu_ctx):
    # facets.rs:521-576: the first index is empty -> A: 5, B: 5
    a = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"])
    b = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"])
    try:
        b.apply_all([_index_op(i, f"title {i}", category="A" if i % 2 == 0 else "B") for i in range(10)])
        a.commit(); b.commit()
        r = search_collection_ex([a, b], [""], _params(), facets={"category": {}})[0]
        assert r["facets"]["category"]["values"] == {"A": 5, "B": 5}
    finally:
        a.close(); b.close()


def test_groupby_split_over_two_indexes(gpu_ctx):
    # groupby.rs:9-175: 100 documents "text " x (i+1), number i % 5, bool i % 2 == 0, split by parity of the id
    a = IndexLoader(gpu_ctx, ["text"], number_fields=["number"], bool_fields=["bool"])
    b = IndexLoader(gpu_ctx, ["text"], number_fields=["number"], bool_fields=["bool"])
    try:
        for i in range(100):
            (a if i % 2 == 0 else b).apply_all([_index_op(i, " ".join(["text"] * (i + 1)), number=float(i % 5), bool=i % 2 == 0)])
        a.commit(); b.commit()
        for props, expect in [(["number"], {(float(v),) for v in range(5)}),
                              (["number", "bool"], {(float(v), x) for v in range(5) for x in (True, False)})]:
            r = search_collection_ex([a, b], ["text"], _params(1), group_by={"properties": props, "max_results": 5})[0]
            assert r["hits"].count == 100
            got = {tuple(g["values"]) for g in r["groups"] if g["result"]}
            assert got == expect
            for g in r["groups"]:
                assert len(g["result"]) <= 5
                for d, _ in g["result"]:
                    assert float(d % 5) == g["values"][0]
                    if len(props) > 1:
                        assert (d % 2 == 0) == g["values"][1]
    finally:
        a.close(); b.close()


def test_group_by_with_pin_rules_score_based_split(gpu_ctx):
    # groupby.rs:984-1062: "apple" grouped by category, max_results 3, doc3 promoted at position 1 (the pin rule matched,
    # so the query is active) -> food = [doc1, doc3], tech = [doc2, doc5].  Split: doc1, doc2, doc5 on one index, doc3
    # (the promoted, non-matching member of food) and doc4 on the other.
    docs = {1: ("apple fruit", "food", 10.0), 2: ("apple phone", "tech", 100.0), 3: ("banana fruit", "food", 5.0),
            4: ("orange tech", "tech", 50.0), 5: ("apple laptop", "tech", 200.0)}
    a = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"], number_fields=["price"])
    b = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"], number_fields=["price"])
    try:
        for d, (t, c, pr) in docs.items():
            (a if d in (1, 2, 5) else b).apply_all([_index_op(d, t, category=c, price=pr)])
        a.commit(); b.commit()
        r = search_collection_ex([a, b], ["apple"], _params(), promote=[[(3, 1)]],
                                 group_by={"properties": ["category"], "max_results": 3})[0]
        groups = sorted(r["groups"], key=lambda g: g["values"][0])
        assert [g["values"] for g in groups] == [["food"], ["tech"]]
        assert [d for d, _ in groups[0]["result"]] == [1, 3]
        assert [d for d, _ in groups[1]["result"]] == [2, 5]
        assert groups[0]["result"][1][1] == 0.0   # doc3 is not a key of either index's score map
    finally:
        a.close(); b.close()


def test_groupby_index_without_property(gpu_ctx):
    # an index that lacks the property adds no groups (group.rs:104-168); the other index's groups are whole
    a = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"])
    b = IndexLoader(gpu_ctx, ["text"], number_fields=["price"])
    try:
        a.apply_all([_index_op(i, "item", category=["x", "y"][i % 2]) for i in range(6)])
        b.apply_all([_index_op(10 + i, "item", price=float(i)) for i in range(4)])
        a.commit(); b.commit()
        r = search_collection_ex([a, b], ["item"], _params(), group_by={"properties": ["category"], "max_results": 10})[0]
        assert r["hits"].count == 10
        assert {g["values"][0]: sorted(d for d, _ in g["result"]) for g in r["groups"]} == {"x": [0, 2, 4], "y": [1, 3, 5]}
    finally:
        a.close(); b.close()


def test_errors(gpu_ctx):
    a = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"], number_fields=["n"], date_fields=["d"])
    b = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["category"])
    try:
        a.apply_all([_index_op(0, "item", category="x", n=1.0)])
        b.apply_all([_index_op(1, "item", category="y")])
        a.commit(); b.commit()
        with pytest.raises(FacetFieldNotFound) as e:   # every missing field is listed (search.rs:452-464)
            search_collection_ex([a, b], ["item"], _params(), facets={"missing": {}, "category": {}, "gone": {}})
        assert e.value.names == ["missing", "gone"]
        with pytest.raises(ValueError):   # a range on a string_filter field
            search_collection_ex([a, b], ["item"], _params(), facets={"category": {"ranges": [{"from": 0, "to": 1}]}})
        with pytest.raises(ValueError):   # a number field without ranges
            search_collection_ex([a, b], ["item"], _params(), facets={"n": {}})
        with pytest.raises(ValueError):   # a date property
            search_collection_ex([a, b], ["item"], _params(), group_by={"properties": ["d"], "max_results": 1})
    finally:
        a.close(); b.close()
