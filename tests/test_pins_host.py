"""oc_merge_pinned (host): the multi-index union with pin rules against a restatement of apply_pin_rules_internal
(read/sort.rs:285-391) over the union of the per-index score maps, and the reference's multi-index expectation
(src/tests/pin_rules.rs:109-239).  Runs without a GPU."""
import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import PromoteItem


def apply_pin_rules(items, score_map, top):
    """apply_pin_rules_internal: items = [(doc, position)] in consequence order; top = [(doc, score)] best first."""
    if not items:
        return list(top)
    promoted = {d for d, _ in items}
    top = [e for e in top if e[0] not in promoted]
    for d, pos in sorted(items, key=lambda it: it[1]):   # stable sort by position
        top.insert(min(pos, len(top)), (d, score_map.get(d, 0.0)))
    return top


def top_n(score_map, n):
    return sorted(((d, s) for d, s in score_map.items() if s == s), key=lambda e: (-np.float32(e[1]), e[0]))[:n]


def _per_index(maps, promote, stride):
    """What oc_search_pinned returns per index with limit' = stride, apply = 0: hits, counts, per-item values."""
    B = len(promote)
    flat = [d for q in promote for d, _ in q]
    per = []
    for m in maps:
        docs, scores = np.zeros((B, stride), np.uint64), np.zeros((B, stride), np.float32)
        n, cnt = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
        for q in range(B):
            t = top_n(m[q], stride)
            n[q], cnt[q] = len(t), len(m[q])
            docs[q, :len(t)] = [d for d, _ in t]
            scores[q, :len(t)] = [s for _, s in t]
        ps = np.zeros(max(len(flat), 1), np.float32)
        pp = np.zeros(max(len(flat), 1), np.uint8)
        i = 0
        for q in range(B):
            for d, _ in promote[q]:
                if d in m[q]:
                    ps[i], pp[i] = m[q][d], 1
                i += 1
        per.append((docs, scores, n, cnt, ps, pp))
    return per


def _random_case(rng, B, k, n_docs):
    maps = [[{} for _ in range(B)] for _ in range(k)]
    for q in range(B):
        for i in range(k):   # disjoint documents per index, many ties
            ds = rng.choice(n_docs, size=int(rng.integers(0, 60)), replace=False) * k + i
            for d in ds.tolist():
                maps[i][q][d] = float(np.float32(rng.choice([0.25, 0.5, 1.0, 1.5, 2.0])))
    return maps


def _check(maps, promote, limit, offset, apply=True):
    B = len(promote)
    stride = 2 * (limit + offset)
    per = _per_index(maps, promote, stride)
    hits = ob.merge_index_results_pinned(per, promote, limit, offset, apply=apply)
    for q in range(B):
        union = {}
        for m in maps:
            union.update(m[q])
        active = apply and len(promote[q]) > 0
        top = top_n(union, stride if active else limit + offset)
        if active:
            top = apply_pin_rules(promote[q], union, top)
        exp = top[offset:offset + limit]
        assert hits[q].doc_ids.tolist() == [d for d, _ in exp], (q, promote[q])
        assert hits[q].scores.tolist() == [np.float32(s) for _, s in exp]
        assert hits[q].count == len(union)
    return hits, per


def test_merge_pinned_against_the_restatement():
    rng = np.random.default_rng(7)
    B, k, n_docs = 24, 3, 200
    maps = _random_case(rng, B, k, n_docs)
    promote = []
    for q in range(B):
        kind = q % 8
        present = [d for m in maps for d in m[q]]
        pick = lambda: int(rng.choice(present)) if present and rng.random() < 0.7 else int(rng.integers(10 ** 6, 2 * 10 ** 6))  # noqa: E731
        if kind == 0:
            items = []                                               # inactive
        elif kind == 1:
            items = [(pick(), 2), (pick(), 2), (pick(), 2)]          # equal positions: the later one in front
        elif kind == 2:
            items = [(pick(), 0), (pick(), 10 ** 6)]                  # first slot, far beyond the length
        elif kind == 3:
            d = pick()
            items = [(d, 1), (d, 4)]                                 # one document promoted twice
        elif kind == 4:
            items = [(5 * 10 ** 6 + j, j) for j in range(4)]         # documents absent from every index
        else:
            items = [(pick(), int(rng.integers(0, 40))) for _ in range(int(rng.integers(1, 12)))]
        promote.append(items)
    for limit, offset in [(10, 0), (5, 3), (1, 0), (7, 20)]:
        _check(maps, promote, limit, offset)


def test_merge_pinned_equal_positions_and_overflow_order():
    m = [[{d: 1.0 for d in range(6)}]]
    hits, _ = _check(m, [[(10, 1), (11, 1), (12, 1)]], 10, 0)
    assert hits[0].doc_ids.tolist() == [0, 12, 11, 10, 1, 2, 3, 4, 5]
    hits, _ = _check(m, [[(10, 50), (11, 40)]], 10, 0)   # past the end: appended in position order
    assert hits[0].doc_ids.tolist() == [0, 1, 2, 3, 4, 5, 11, 10]
    hits, _ = _check(m, [[(3, 0), (3, 2)]], 10, 0)        # promoted twice: inserted twice
    assert hits[0].doc_ids.tolist() == [3, 0, 3, 1, 2, 4, 5]


def test_merge_pinned_inactive_is_merge_results():
    rng = np.random.default_rng(11)
    B, k = 16, 2
    maps = _random_case(rng, B, k, 100)
    promote = [[(int(rng.integers(0, 200)), int(rng.integers(0, 8)))] if q % 2 else [] for q in range(B)]
    for apply in (True, False):
        limit, offset = 6, 2
        hits, per = _check(maps, promote, limit, offset, apply=apply)
        plain = ob.merge_index_results([r[:4] for r in per], limit, offset)
        for q in range(B):
            if apply and promote[q]:
                continue
            assert hits[q].doc_ids.tolist() == plain[q].doc_ids.tolist()
            assert hits[q].scores.view(np.uint32).tolist() == plain[q].scores.view(np.uint32).tolist()
            assert hits[q].count == plain[q].count


def test_reference_multiple_indexes():
    # pin_rules.rs:109-239: docs 0-9 in one index, 10-19 in another, every document scores the same for "c";
    # rule 1 promotes 5 @ 1 and 7 @ 4, rule 2 promotes 11 @ 2 and 15 @ 3
    maps = [[{d: 0.75 for d in range(10)}], [{d: 0.75 for d in range(10, 20)}]]
    promote = [[PromoteItem(5, 1), PromoteItem(7, 4), PromoteItem(11, 2), PromoteItem(15, 3)]]
    per = _per_index(maps, [[(it.doc_id, it.position) for it in promote[0]]], 20)
    hits = ob.merge_index_results_pinned(per, promote, 10)
    assert hits[0].doc_ids.tolist() == [0, 5, 11, 15, 7, 1, 2, 3, 4, 6]
    assert hits[0].count == 20


def test_merge_pinned_rejections():
    maps = [[{1: 1.0}], [{2: 1.0}]]
    promote = [[(1, 0)]]
    per = _per_index(maps, promote, 4)
    with pytest.raises(ob.OcError) as e:   # the per-index lists must hold the top 2 x (limit + offset)
        ob.merge_index_results_pinned([tuple(a[:, :3] if a.ndim == 2 else a for a in r) for r in per], promote, 2)
    assert e.value.code == -1
    ob.merge_index_results_pinned(per, promote, 2)
    import ctypes as C
    from oramacore_b200 import _lib
    off = np.asarray([1, 0], np.uint32)   # not monotone
    doc, pos = np.zeros(1, np.uint64), np.zeros(1, np.uint32)
    pins = _lib.Pins(off.ctypes.data, doc.ctypes.data, pos.ctypes.data, 1)
    keep = [[np.ascontiguousarray(a) for a in r] for r in per]
    arr = lambda j: (C.c_void_p * 2)(*[r[j].ctypes.data for r in keep])  # noqa: E731
    out = [np.zeros(2, np.uint64), np.zeros(2, np.float32), np.zeros(1, np.uint32), np.zeros(1, np.uint64)]
    rc = _lib.lib().oc_merge_pinned(2, 1, 2, 0, 4, arr(0), arr(1), arr(2), arr(3), C.byref(pins), arr(4), arr(5),
                                    *[o.ctypes.data for o in out])
    assert rc == -1 and out[2][0] == 0 and out[3][0] == 0   # nothing written
