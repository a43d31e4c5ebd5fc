"""oc_merge_sorted (host): the multi-index union in field order against a restatement of MergeSortedIterator
(read/sort.rs:491-559) followed by apply_pin_rules_internal and skip/take; the sortBy property lookup
(IndexSortContext::execute, read/index/sort.rs:186-265) and SortField's create-time validation.  Runs without a GPU."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import PromoteItem
from test_pins_host import apply_pin_rules


def merge_sorted(lists, order, take):
    """MergeSortedIterator: lists[i] = [(doc, score, value)] in field order; strict comparison, so on equal values the
    index listed first wins."""
    head = [0] * len(lists)
    out = []
    while len(out) < take:
        best = -1
        for i, l in enumerate(lists):
            if head[i] >= len(l):
                continue
            if best < 0:
                best = i
                continue
            va, vb = l[head[i]][2], lists[best][head[best]][2]
            if (va < vb) if order == "ASC" else (va > vb):
                best = i
        if best < 0:
            break
        out.append(lists[best][head[best]])
        head[best] += 1
    return out


def expect(lists, order, limit, offset, items=()):
    """Per query: (docs, scores, sort values) of the page."""
    active = len(items) > 0
    top = merge_sorted(lists, order, (2 if active else 1) * (limit + offset))
    value = {d: v for d, _, v in top}
    score_map = {d: s for l in lists for d, s, _ in l}
    page = apply_pin_rules(list(items), score_map, [(d, s) for d, s, _ in top])[offset:offset + limit]
    promoted = {d for d, _ in items}
    return ([d for d, _ in page], [s for _, s in page],
            [float("nan") if (d in promoted and active) else value[d] for d, _ in page])


def _per_index(lists_per_q, stride, promote=None):
    """What oc_search_sorted returns per index (limit' = stride, apply = 0): hits, scores, values, n, count, and the
    per-item values when promote is given."""
    B = len(lists_per_q)
    docs, scores = np.zeros((B, stride), np.uint64), np.zeros((B, stride), np.float32)
    vals, n, cnt = np.zeros((B, stride), np.float64), np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    for q, l in enumerate(lists_per_q):
        t = l[:stride]
        n[q], cnt[q] = len(t), len(l) + 3   # the count also holds keys with no value in the field
        docs[q, :len(t)] = [d for d, _, _ in t]
        scores[q, :len(t)] = [s for _, s, _ in t]
        vals[q, :len(t)] = [v for _, _, v in t]
    if promote is None:
        return docs, scores, vals, n, cnt
    flat = [(q, d) for q in range(B) for d, _ in promote[q]]
    ps, pp = np.zeros(max(len(flat), 1), np.float32), np.zeros(max(len(flat), 1), np.uint8)
    for i, (q, d) in enumerate(flat):
        m = {dd: s for dd, s, _ in lists_per_q[q]}
        if d in m:
            ps[i], pp[i] = m[d], 1
    return docs, scores, vals, n, cnt, ps, pp


def _random_lists(rng, B, k, order):
    """Per index and query, a list of (doc, score, value) in field order: disjoint documents, many equal values across
    indexes, NaN scores, ties by ascending document id."""
    out = [[None] * B for _ in range(k)]
    for i in range(k):
        for q in range(B):
            ds = rng.choice(200, size=int(rng.integers(0, 40)), replace=False) * k + i
            vals = rng.choice([-1.5, 0.0, 2.0, 3.0, 7.25], size=ds.shape[0])
            scores = rng.choice([0.5, 1.0, np.nan], size=ds.shape[0]).astype(np.float32)
            l = [(int(d), float(s), float(v)) for d, s, v in zip(ds, scores, vals)]
            l.sort(key=lambda e: ((e[2] if order == "ASC" else -e[2]), e[0]))
            out[i][q] = l
    return out


def _check(res, vals, exp, q):
    hits = res[q]
    ed, es, ev = exp
    assert hits.doc_ids.tolist() == ed
    np.testing.assert_array_equal(hits.scores, np.asarray(es, np.float32))   # NaN kept, bit for bit
    np.testing.assert_array_equal(vals[q, :len(ed)], np.asarray(ev, np.float64))


@pytest.mark.parametrize("order", ["ASC", "DESC"])
@pytest.mark.parametrize("k", [1, 2, 3])
def test_merge_sorted_matches_restatement(order, k):
    rng = np.random.default_rng(7 + k)
    B, limit, offset = 9, 6, 3
    lists = _random_lists(rng, B, k, order)
    per = [_per_index(lists[i], limit + offset) for i in range(k)]
    res, vals = ob.merge_index_results_sorted(per, order, limit, offset)
    for q in range(B):
        _check(res, vals, expect([lists[i][q][:limit + offset] for i in range(k)], order, limit, offset), q)
        assert res[q].count == sum(len(lists[i][q]) + 3 for i in range(k))


def test_merge_sorted_equal_values_take_index_order():
    # index 1 holds the lower document ids, but on equal values index 0 (listed first) wins
    l0 = [[(10, 1.0, 5.0), (11, 1.0, 5.0), (12, 1.0, 6.0)]]
    l1 = [[(1, 2.0, 5.0), (2, 2.0, 6.0)]]
    for order, exp in [("ASC", [10, 11, 1, 12, 2]), ("DESC", [12, 2, 10, 11, 1])]:
        a, b = ([sorted(l[0], key=lambda e: (e[2] if order == "ASC" else -e[2], e[0]))] for l in (l0, l1))
        res, _ = ob.merge_index_results_sorted([_per_index(a, 5), _per_index(b, 5)], order, 5)
        assert res[0].doc_ids.tolist() == exp


def test_merge_sorted_reference_multi_index():
    # multi_index.rs:406-508: index 1 {doc1: 1, doc2: 3}, index 2 {doc3: 2, doc4: 4}
    i1 = {"ASC": [[(1, 0.5, 1.0), (2, 0.5, 3.0)]], "DESC": [[(2, 0.5, 3.0), (1, 0.5, 1.0)]]}
    i2 = {"ASC": [[(3, 0.5, 2.0), (4, 0.5, 4.0)]], "DESC": [[(4, 0.5, 4.0), (3, 0.5, 2.0)]]}
    for order, exp in [("ASC", [1, 3, 2, 4]), ("DESC", [4, 2, 3, 1])]:
        res, vals = ob.merge_index_results_sorted([_per_index(i1[order], 10), _per_index(i2[order], 10)], order, 10)
        assert res[0].doc_ids.tolist() == exp
        assert vals[0, :4].tolist() == sorted([1.0, 2.0, 3.0, 4.0], reverse=order == "DESC")


@pytest.mark.parametrize("order", ["ASC", "DESC"])
def test_merge_sorted_with_pins(order):
    rng = np.random.default_rng(41)
    B, k, limit, offset = 8, 2, 5, 2
    lists = _random_lists(rng, B, k, order)
    promote = []
    for q in range(B):
        pool = [d for i in range(k) for d, _, _ in lists[i][q]] + [9999]
        promote.append([(int(rng.choice(pool)), int(rng.choice([0, 1, 1, 4, 50]))) for _ in range(int(rng.integers(0, 4)))])
    stride = 2 * (limit + offset)
    per = [_per_index(lists[i], stride, promote) for i in range(k)]
    res, vals = ob.merge_index_results_sorted(per, order, limit, offset, promote=promote)
    for q in range(B):
        _check(res, vals, expect([lists[i][q][:stride] for i in range(k)], order, limit, offset, promote[q]), q)
    # apply = False: the plain merge of the same lists
    res0, vals0 = ob.merge_index_results_sorted(per, order, limit, offset, promote=promote, apply=False)
    for q in range(B):
        _check(res0, vals0, expect([lists[i][q][:stride] for i in range(k)], order, limit, offset), q)


def test_merge_sorted_refusals():
    l = [[(1, 1.0, 1.0), (2, 1.0, 2.0)]]
    per = [_per_index(l, 2)]
    with pytest.raises(ValueError):
        ob.merge_index_results_sorted(per, "SIDEWAYS", 2)
    keep = [np.ascontiguousarray(a) for a in per[0]]
    arr = [(C.c_void_p * 1)(a.ctypes.data) for a in keep]
    out = [np.zeros((1, 2), np.uint64), np.zeros((1, 2), np.float32), np.zeros((1, 2), np.float64), np.zeros(1, np.uint32),
           np.zeros(1, np.uint64)]
    for order in (2, -1):   # the C entry point refuses an order that is neither OC_SORT_ASC nor OC_SORT_DESC
        rc = ob.lib().oc_merge_sorted(1, 1, 2, 0, 2, order, *arr, None, None, None, *[o.ctypes.data for o in out])
        assert rc != 0 and not out[0].any()
    bad = list(_per_index(l, 2)); bad[3] = np.asarray([3], np.uint32)
    with pytest.raises(ob.OcError):   # n > in_stride
        ob.merge_index_results_sorted([tuple(bad)], "ASC", 2)
    with pytest.raises(ob.OcError):   # an active query needs in_stride >= 2 x (limit + offset)
        ob.merge_index_results_sorted([_per_index(l, 2, [[(1, 0)]])], "ASC", 2, promote=[[PromoteItem(1, 0)]])
    with pytest.raises(ob.OcError):   # limit 0
        ob.merge_index_results_sorted(per, "ASC", 0)


def test_resolve_sort_by_errors():
    # sort.rs:325-411: an unknown property, a geopoint property
    fields = {"position": "geopoint", "name": "string", "tag": "string_filter"}
    with pytest.raises(ob.SortFieldNotFound) as e:
        ob.resolve_sort_by(fields, ob.SortBy("unknown_field"))
    assert e.value.name == "unknown_field"
    for prop, kind in [("position", "GeoPoint"), ("name", "String"), ("tag", "StringFilter")]:
        with pytest.raises(ob.InvalidSortField) as e:
            ob.resolve_sort_by(fields, ob.SortBy(prop))
        assert (e.value.name, e.value.kind) == (prop, kind)
    with pytest.raises(ValueError):
        ob.resolve_sort_by(fields, ob.SortBy("position", "UP"))
    assert ob.SortBy("x").order == "ASC"   # the reference's default (types.rs:1350-1357)


def test_sort_field_create_time_validation():
    # refused on the host before the device is touched (ctx is not used)
    with pytest.raises(ValueError):
        ob.SortField(None, 10, [1, 2], [1.0, float("nan")], "number")
    with pytest.raises(ValueError):
        ob.SortField(None, 10, [1], [2 ** 53 + 1], "date")
    with pytest.raises(ValueError):
        ob.SortField(None, 10, [1, 2], [1.0], "number")
    with pytest.raises(ValueError):
        ob.SortField(None, 10, [1], [1.0], "geopoint")
