"""The collection-level search over several IndexLoaders (loader.search_collection, one oc_search_indexes call): the
cases of src/tests/multi_index.rs — two indexes, one index empty, a filter on committed fields only, and sorting across
indexes.  Document ids are unique per collection, as the reference's DocumentId is."""
import pytest

import oramacore_b200 as ob
from oramacore_b200.loader import IndexLoader, search_collection
from oramacore_b200.types import MODE_FULLTEXT, SortBy
from oramacore_b200.where import FilterFieldNotFound
from test_gpu_loader import _index_op

pytestmark = pytest.mark.gpu


def _params(limit=10):
    return ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=limit)


def test_basic(gpu_ctx):
    a = IndexLoader(gpu_ctx, ["text"], number_fields=["number"])
    b = IndexLoader(gpu_ctx, ["text"], bool_fields=["bool"])
    try:
        a.apply_all([_index_op(i, " ".join(["text"] * (i + 1)), number=float(i)) for i in range(10)])
        b.apply_all([_index_op(10 + i, " ".join(["text"] * (i + 1)), bool=i % 2 == 0) for i in range(10)])
        a.commit(); b.commit()
        hits, _ = search_collection([a, b], ["text"], _params())
        assert hits[0].count == 20
        assert search_collection([a, b], ["text"], _params(), where={"bool": True})[0][0].count == 5      # only on b
        assert search_collection([a, b], ["text"], _params(), where={"number": {"gt": -1}})[0][0].count == 10   # only on a
        with pytest.raises(FilterFieldNotFound):
            search_collection([a, b], ["text"], _params(), where={"missing": True})
    finally:
        a.close(); b.close()


def test_one_index_empty(gpu_ctx):
    a = IndexLoader(gpu_ctx, ["text"], number_fields=["number"])
    b = IndexLoader(gpu_ctx, ["text"], number_fields=["number"])
    try:
        a.apply_all([_index_op(i, " ".join(["text"] * (i + 1)), number=float(i)) for i in range(10)])
        a.commit(); b.commit()
        assert search_collection([a, b], ["text"], _params())[0][0].count == 10
        assert search_collection([a, b], ["text"], _params(), where={"number": {"gt": -1}})[0][0].count == 10
        assert search_collection([a, b], ["text"], _params(), where={"number": {"eq": 3}})[0][0].count == 1
    finally:
        a.close(); b.close()


def test_committed_only_field_filter(gpu_ctx):
    a = IndexLoader(gpu_ctx, ["text"], string_filter_fields=["status"])
    try:
        a.apply_all([_index_op(1, "test", status="active"), _index_op(2, "test", status="inactive")])
        a.commit()
        assert search_collection([a], ["test"], _params(), where={"status": "active"})[0][0].count == 1
    finally:
        a.close()


def test_sorting_across_indexes(gpu_ctx):
    a = IndexLoader(gpu_ctx, ["text"], number_fields=["priority"])
    b = IndexLoader(gpu_ctx, ["text"], number_fields=["priority"])
    try:
        a.apply_all([_index_op(1, "item", priority=1.0), _index_op(2, "item", priority=3.0)])
        b.apply_all([_index_op(3, "item", priority=2.0), _index_op(4, "item", priority=4.0)])
        a.commit(); b.commit()
        hits, sv = search_collection([a, b], ["item"], _params(), sort_by=SortBy("priority", "ASC"))
        assert hits[0].count == 4 and hits[0].doc_ids.tolist() == [1, 3, 2, 4] and sv[0, :4].tolist() == [1, 2, 3, 4]
        hits, sv = search_collection([a, b], ["item"], _params(), sort_by=SortBy("priority", "DESC"))
        assert hits[0].count == 4 and hits[0].doc_ids.tolist() == [4, 2, 3, 1] and sv[0, :4].tolist() == [4, 3, 2, 1]
    finally:
        a.close(); b.close()
