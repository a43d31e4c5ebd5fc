"""oc_search_indexes_ex's facets across the indexes of a collection: each collection slot's count equals the sum of the
per-index oc_search_q_facets counts mapped to it (a query filtered on an index — a q_filters entry or a where program —
is counted there without its filter).  Bool, string_filter and number-range facets, a field only some indexes have, an
empty index, unfiltered and filtered queries in one batch, a commit between calls; hits and groups are byte-identical
to the call without facets."""
import dataclasses

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import engine as E
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID
from test_gpu_multi_index import N
from test_gpu_multi_index_groups import B, Collection, _part_b, where_programs
from test_gpu_multi_index_groups import cols, corpus  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu


def _facet_recipe(col, params, facets):
    """per query the per-index oc_search_q_facets counts, summed by label"""
    out = []
    for b, f in enumerate(facets):
        if not f:
            out.append({})
            continue
        tot = {}
        for part in col.parts:
            if part.store is None:
                continue
            present = {k: v for k, v in f.items() if k in part.store.fields}
            if not present:
                continue
            got = E.search_q_facets_arrays(_part_b(part, b).tsc, part.store, dataclasses.replace(params, **dict(_part_b(part, b).fields or {})),
                                           [present], texts=_part_b(part, b).texts, q_vecs=_part_b(part, b).q_vecs)
            fc, labels = got[12], got[14][0]
            for j, lab in enumerate(labels):
                tot[lab] = tot.get(lab, 0) + int(fc[j])
        out.append(tot)
    return out


FACETS = {"cat": {}, "flag": {"true": True, "false": True}, "num": {"ranges": [{"from": -3, "to": 0}, {"from": 0.5, "to": 10}]},
          "only1": {"true": True}}


@pytest.mark.parametrize("kind", ["q_filters", "where_programs"])
def test_facets_match_per_index_sums(gpu_ctx, cols, kind):
    col = cols(3, "mod", empty=True)
    base = list(col.parts)
    try:
        for i, part in enumerate(col.parts[:3]):   # queries 1, 3, ... filtered on index 0 only, query 2 on every index
            on = [(b % 2 == 1 and i == 0) or b == 2 for b in range(B)]
            if kind == "q_filters":
                docs = np.arange(N, dtype=np.uint64)[np.arange(N) % 3 == i]
                flt = ob.DeviceFilter.from_ids(gpu_ctx, docs[docs % 2 == 0], N)
                fields = {"device_filters": [flt if on[b] else None for b in range(B)]}
            else:
                fields = {"where_programs": where_programs(part, [{"flag": True} if on[b] else None for b in range(B)])}
            col.parts[i] = dataclasses.replace(part, fields=fields)
        facets = [None if b % 5 == 4 else FACETS if b % 2 == 0 else {"cat": {}} for b in range(B)]
        for mode in (MODE_FULLTEXT, MODE_HYBRID):
            p = ob.TokenScoreParams(mode=mode, limit_hint=10, similarity=0.0)
            groups = [(col.group_by(["cat"]), 3)] * B
            got = E.search_indexes_arrays(gpu_ctx, col.parts, p, groups=groups, facets=facets)
            alone = E.search_indexes_arrays(gpu_ctx, col.parts, p, groups=groups)
            for a, b2 in zip(got[:11], alone[:11]):   # hits and groups byte-identical to the call without facets
                assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b2).view(np.uint8))
            fc, foff, labels = got[13], got[14], got[15]
            exp = _facet_recipe(col, p, facets)
            for b in range(B):
                assert {lab: int(fc[foff[b] + j]) for j, lab in enumerate(labels[b])} == exp[b]
    finally:
        col.parts[:] = base


def test_facets_around_a_commit(gpu_ctx, corpus):
    col = Collection(gpu_ctx, corpus, 2, "range")
    try:
        p = ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10)
        facets = [FACETS] * B
        for step in range(2):
            got = E.search_indexes_arrays(gpu_ctx, col.parts, p, facets=facets)
            exp = _facet_recipe(col, p, facets)
            for b in range(B):
                assert {lab: int(got[13][got[14][b] + j]) for j, lab in enumerate(got[15][b])} == exp[b]
            for part in col.parts:
                docs = np.arange(N, dtype=np.uint64)[::11]
                part.store.delete(docs)
                part.store.commit(N)
                part.tsc.str.delete(docs)
                part.tsc.str.commit()
    finally:
        col.close()


