"""sort_field_spec.py against a brute-force restatement of the host sort oc_sort_field_create ran before the build
moved to the device (std::sort with the same comparator, then each document at its first position), and the refusals
SortField.from_facets makes in Python before any device call."""
import functools
from types import SimpleNamespace

import numpy as np
import pytest

import oramacore_b200 as ob
from sort_field_spec import random_entries, rank_order, variant_entries


def host_create(doc_ids, values, nbits, order):
    e = [(float(v) + 0.0, int(d)) for d, v in zip(np.asarray(doc_ids).tolist(), np.asarray(values).tolist()) if int(d) < nbits]

    def cmp(a, b):
        if a[0] != b[0]:
            less = a[0] < b[0] if order == "ASC" else a[0] > b[0]
            return -1 if less else 1
        return (a[1] > b[1]) - (a[1] < b[1])
    e.sort(key=functools.cmp_to_key(cmp))
    seen, rd, rv = set(), [], []
    for v, d in e:
        if d not in seen:
            seen.add(d)
            rd.append(d)
            rv.append(v)
    return np.asarray(rd, np.uint64), np.asarray(rv, np.float64)


def _same(a, b):
    assert a[0].tolist() == b[0].tolist()
    assert a[1].view(np.uint64).tolist() == b[1].view(np.uint64).tolist()   # value bits: +0.0, never -0.0


@pytest.mark.parametrize("seed", range(12))
def test_spec_is_the_host_sort(seed):
    rng = np.random.default_rng(seed)
    for n, nbits in [(0, 1), (1, 1), (5, 3), (50, 10), (400, 97), (3000, 5000), (20000, 1500)]:
        d, v = random_entries(rng, n, nbits)
        for order in ("ASC", "DESC"):
            got = rank_order(d, v, nbits, order)
            _same(got, host_create(d, v, nbits, order))
            assert not np.signbit(got[1][got[1] == 0]).any()


def test_signed_zeros_ties_and_duplicates():
    d = np.asarray([4, 2, 2, 9, 1, 4, 3, 3], np.uint64)
    v = np.asarray([-0.0, 0.0, 7.0, 1.0, -0.0, 5.0, np.inf, -np.inf])
    # ASC: -inf (3), then 0.0 for 1, 2, 4 by id, then 1.0 (9); id 9 >= nbits 9 is dropped
    rd, rv = rank_order(d, v, 9, "ASC")
    assert rd.tolist() == [3, 1, 2, 4] and rv.view(np.uint64).tolist() == np.asarray([-np.inf, 0.0, 0.0, 0.0]).view(np.uint64).tolist()
    rd, rv = rank_order(d, v, 9, "DESC")
    assert rd.tolist() == [3, 2, 4, 1] and rv.tolist() == [np.inf, 7.0, 5.0, 0.0]
    _same(rank_order(np.repeat(d, 3), np.repeat(v, 3), 9, "ASC"), rank_order(d, v, 9, "ASC"))


def test_variant_entries():
    layout = {"offsets": np.asarray([1, 3, 3, 5], np.uint64), "doc_ids": np.asarray([8, 0, 4, 2, 4], np.uint64)}
    d, v = variant_entries(layout, [1.0, 9.0, 0.0])
    assert d.tolist() == [0, 4, 2, 4] and v.tolist() == [1.0, 1.0, 0.0, 0.0]
    # a bool field with both values on document 4: the max (true) for DESC, the min (false) for ASC
    assert rank_order(d, v, 10, "DESC")[0].tolist() == [0, 4, 2]
    assert rank_order(d, v, 10, "ASC")[0].tolist() == [2, 4, 0]


def test_from_facets_refusals_before_any_device_call():
    # a store stand-in without a device handle: a device call would fail on it, so each refusal happens first
    store = SimpleNamespace(ctx=None, _h=None, nbits=4, fields={"cat": {"id": 0, "kind": "string", "keys": ["a"], "variant": {"a": 0}}})
    with pytest.raises(ob.InvalidSortField) as e:
        ob.SortField.from_facets(store, "cat")
    assert e.value.args[1] == "StringFilter"
    with pytest.raises(ob.SortFieldNotFound):
        ob.SortField.from_facets(store, "nope")
