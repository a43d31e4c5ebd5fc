"""The host helpers of groups and facets across indexes: the collection's group keys over the indexes' GroupBy values
(engine.collection_group_keys) and the collection's facet slots over the indexes' stores
(engine.collection_facet_requests).  No device."""
from types import SimpleNamespace

import numpy as np
import pytest

from oramacore_b200 import engine as E


def _gb(values):
    return SimpleNamespace(values=values, n_groups=len(values))


def test_group_keys_first_appearance_index_by_index():
    a = _gb([["x", True], ["y", True], ["x", False]])
    b = _gb([["y", True], ["z", False], ["x", True]])
    keys, maps = E.collection_group_keys([a, None, b])
    assert keys == [["x", True], ["y", True], ["x", False], ["z", False]]
    assert maps[0].tolist() == [0, 1, 2] and maps[1] is None and maps[2].tolist() == [1, 3, 0]
    assert maps[0].dtype == np.uint32


def test_group_keys_compare_values_with_eq():
    keys, maps = E.collection_group_keys([_gb([[-0.0], [1.5]]), _gb([[1.5], [0.0]])])
    assert len(keys) == 2 and maps[1].tolist() == [1, 0]
    # a bool is not the number 1.0, a string is not a number
    keys, maps = E.collection_group_keys([_gb([[True], [1.0], ["1"]]), _gb([[1.0], [True]])])
    assert len(keys) == 3 and maps[1].tolist() == [1, 0]


def test_group_keys_empty_handle():
    keys, maps = E.collection_group_keys([_gb([]), None])
    assert keys == [] and maps[0].shape == (1,) and maps[1] is None


def _store(fields):
    return SimpleNamespace(fields=fields)


def _strf(fid, keys):
    return {"id": fid, "kind": "string", "keys": keys, "variant": {k: j for j, k in enumerate(keys)}}


def test_facet_slots_union_and_order():
    s0 = _store({"cat": _strf(0, ["b", "a"]), "n": {"id": 1, "kind": "number"}})
    s1 = _store({"cat": _strf(3, ["a", "c"]),
                 "flag": {"id": 4, "kind": "bool", "keys": ["true", "false"], "variant": {"true": 0, "false": 1}}})
    facets = {"flag": {"true": True}, "cat": {}, "n": {"ranges": [{"from": 0, "to": 10}, {"from": 0.5, "to": 1}]}}
    labels, per = E.collection_facet_requests([s0, None, s1], facets)
    assert labels == [("flag", "true"), ("cat", "b"), ("cat", "a"), ("cat", "c"), ("n", "0-10"), ("n", "0.5-1")]
    (r0, sl0), (r1, sl1), (r2, sl2) = per
    assert r1 == [] and sl1 == []
    assert [labels[s] for s in sl0] == [("cat", "b"), ("cat", "a"), ("n", "0-10"), ("n", "0.5-1")]
    assert r0[0] == (0, 0, 0.0, 0.0) and r0[2] == (1, 0, 0.0, 10.0)
    assert [labels[s] for s in sl2] == [("flag", "true"), ("cat", "a"), ("cat", "c")]
    assert r2[0] == (4, 0, 0.0, 0.0) and r2[1] == (3, 0, 0.0, 0.0)


def test_facet_slots_errors():
    s0 = _store({"cat": _strf(0, ["a"]), "n": {"id": 1, "kind": "number"}, "d": {"id": 2, "kind": "date"}})
    with pytest.raises(KeyError):
        E.collection_facet_requests([s0, None], {"missing": {}})
    with pytest.raises(ValueError):
        E.collection_facet_requests([s0], {"cat": {"ranges": [{"from": 0, "to": 1}]}})
    with pytest.raises(ValueError):
        E.collection_facet_requests([s0], {"n": {}})
    with pytest.raises(ValueError):
        E.collection_facet_requests([s0], {"d": {}})
