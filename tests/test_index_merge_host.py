"""The co-rank rules of index_merge_kernel (oc_search_indexes' device merge), restated in numpy and checked against the
host merges oc_merge_results / oc_merge_sorted / oc_merge_pinned on random lists.  Runs without a GPU."""
import numpy as np
import pytest

import oramacore_b200 as ob


def _before_score(s, d, ls, ld, le):
    """entries of one list (scores ls, docs ld, sorted by (score desc, doc asc)) before (s, d); le: ties count."""
    return int(np.sum((ls > s) | ((ls == s) & ((ld <= d) if le else (ld < d)))))


def _before_value(v, lv, desc, le):
    return int(np.sum((lv > v) | (le & (lv == v)))) if desc else int(np.sum((lv < v) | (le & (lv == v))))


def co_rank(lists, take, order=None):
    """lists: per index (docs, scores, values) of one query.  Places entry k of list i at k + the co-ranks in the other
    lists (index_merge.cuh) and returns the first `take` of the union as (docs, scores, values)."""
    M = min(take, sum(len(l[0]) for l in lists))
    out_d, out_s, out_v = np.zeros(M, np.uint64), np.zeros(M, np.float32), np.zeros(M, np.float64)
    seen = np.zeros(M, bool)
    for i, (d, s, v) in enumerate(lists):
        for k in range(len(d)):
            pos = k
            for j, (dj, sj, vj) in enumerate(lists):
                if j == i:
                    continue
                if order is None:
                    pos += _before_score(s[k], d[k], sj, dj, j < i)
                else:
                    pos += _before_value(v[k], vj, order == "DESC", j < i)
            if pos < M:
                assert not seen[pos]
                seen[pos] = True
                out_d[pos], out_s[pos], out_v[pos] = d[k], s[k], v[k]
    assert seen.all()
    return out_d, out_s, out_v


def _lists(rng, n_idx, B, stride, order=None, neg_zero=False, empty=()):
    per = []
    for i in range(n_idx):
        docs, scores = np.zeros((B, stride), np.uint64), np.zeros((B, stride), np.float32)
        vals = np.zeros((B, stride), np.float64)
        n = rng.integers(0, stride + 1, size=B).astype(np.uint32)
        if i in empty:
            n[:] = 0
        cnt = (n + rng.integers(0, 30, size=B)).astype(np.uint64)
        for q in range(B):
            k = int(n[q])
            s = rng.choice([0.0, 0.5, 1.0, 1.5], size=k).astype(np.float32)   # ties across indexes
            if neg_zero:
                s[rng.random(k) < 0.5] *= -1   # -0.0 among +0.0
            d = (rng.choice(500, size=k, replace=False) * n_idx + i).astype(np.uint64)
            v = rng.integers(0, 4, size=k).astype(np.float64)                 # equal values across indexes
            o = np.lexsort((d, -s)) if order is None else np.lexsort((d, v if order == "ASC" else -v))
            docs[q, :k], scores[q, :k], vals[q, :k] = d[o], s[o], v[o]
        per.append((docs, scores, vals, n, cnt))
    return per


@pytest.mark.parametrize("n_idx", [1, 2, 3, 5])
@pytest.mark.parametrize("neg_zero", [False, True])
def test_score_order_co_rank_equals_oc_merge_results(n_idx, neg_zero):
    rng = np.random.default_rng(n_idx * 2 + neg_zero)
    B, limit = 9, 6
    for offset in (0, 3, 40):   # 40: take beyond the union
        stride = limit + offset
        per = _lists(rng, n_idx, B, stride, neg_zero=neg_zero, empty=(1,) if n_idx > 2 else ())
        hits = ob.merge_index_results([(d, s, n, c) for d, s, _, n, c in per], limit, offset)
        for q in range(B):
            md, ms, _ = co_rank([(d[q, :n[q]], s[q, :n[q]], v[q, :n[q]]) for d, s, v, n, _ in per], limit + offset)
            assert np.array_equal(hits[q].doc_ids, md[offset:offset + limit])
            assert np.array_equal(hits[q].scores.view(np.uint32), ms[offset:offset + limit].view(np.uint32))
            assert hits[q].count == sum(int(c[q]) for *_, c in per)


@pytest.mark.parametrize("order", ["ASC", "DESC"])
@pytest.mark.parametrize("n_idx", [1, 2, 4])
def test_field_order_co_rank_equals_oc_merge_sorted(order, n_idx):
    rng = np.random.default_rng(7 + n_idx)
    B, limit = 8, 5
    for offset in (0, 4, 30):
        stride = limit + offset
        per = _lists(rng, n_idx, B, stride, order=order, empty=(0,) if n_idx > 1 else ())
        hits, ov = ob.merge_index_results_sorted(per, order, limit, offset)
        for q in range(B):
            md, ms, mv = co_rank([(d[q, :n[q]], s[q, :n[q]], v[q, :n[q]]) for d, s, v, n, _ in per], limit + offset, order)
            k = len(hits[q].doc_ids)
            assert np.array_equal(hits[q].doc_ids, md[offset:offset + limit])
            assert np.array_equal(hits[q].scores.view(np.uint32), ms[offset:offset + limit].view(np.uint32))
            assert np.array_equal(ov[q, :k], mv[offset:offset + k])


def _splice(top_d, top_s, items, item_scores):
    """apply_pin_rules_internal as pin_splice_block: drop promoted ids, insert items stably by position."""
    promoted = {d for d, _ in items}
    out = [(d, s) for d, s in zip(top_d.tolist(), top_s.tolist()) if d not in promoted]
    for j in sorted(range(len(items)), key=lambda j: items[j][1]):
        out.insert(min(items[j][1], len(out)), (items[j][0], item_scores[j]))
    return out


def test_pinned_co_rank_equals_oc_merge_pinned():
    rng = np.random.default_rng(11)
    B, n_idx, limit, offset = 6, 3, 4, 2
    stride = 2 * (limit + offset)
    per = _lists(rng, n_idx, B, stride)
    promote = [[] if q == 0 else [(int(d), int(p)) for d, p in zip(rng.integers(0, 1500, 3), rng.integers(0, 8, 3))]
               for q in range(B)]
    n_items = sum(len(p) for p in promote)
    pin_s = [rng.random(n_items).astype(np.float32) for _ in range(n_idx)]
    pin_p = [(rng.random(n_items) < 0.3).astype(np.uint8) for _ in range(n_idx)]
    hits = ob.merge_index_results_pinned([(d, s, n, c, pin_s[i], pin_p[i]) for i, (d, s, _, n, c) in enumerate(per)],
                                         promote, limit, offset)
    at = 0
    for q in range(B):
        items = promote[q]
        take = (limit + offset) * (2 if items else 1)
        md, ms, _ = co_rank([(d[q, :n[q]], s[q, :n[q]], v[q, :n[q]]) for d, s, v, n, _ in per], take)
        isc = []
        for j in range(len(items)):
            s = 0.0
            for i in range(n_idx):
                if pin_p[i][at + j]:
                    s = float(pin_s[i][at + j])
                    break
            isc.append(s)
        at += len(items)
        exp = _splice(md, ms, items, isc) if items else list(zip(md.tolist(), ms.tolist()))
        exp = exp[offset:offset + limit]
        assert hits[q].doc_ids.tolist() == [d for d, _ in exp]
        assert np.array_equal(hits[q].scores, np.asarray([s for _, s in exp], np.float32))
