"""Per-query parameters in one batch (oc_search_params.q_params, TokenScoreParams.query_params): every query of a batch
has its own mode, limit, offset, similarity, threshold and vector_limit.

The rule: query b's outputs — ids, score bits, n, count, and in the q_sorted / q_groups / q_facets calls its sort values,
pin outputs, group rows and facet counts — equal, byte for byte, what it gets alone (B = 1 with its own scalars, filter,
sort, items, groups and facets).  The hit arrays of the batch have p->limit = the largest limit as row stride; a row's
entries past the query's own limit are 0.  Checked over mixed batches of fulltext / vector / hybrid queries with limits
1-200, offsets 0-100, several similarities, thresholds and vector_limits, on an fp32 store (fp16 sweep) and a bf16 store,
through the plain, threshold and multi-term fulltext scorers; entries equal to p's scalars against the plain call; the
sorted, grouped and faceted calls with q_filters, OMC and tombstones before and after a commit; the oracle's score maps;
and every refusal."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import _lib
from oramacore_b200.engine import _p
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from test_gpu_q_facets import _mix
from test_gpu_q_facets import faceting  # noqa: F401  (fixture)
from test_gpu_q_groups import _requests
from test_gpu_q_sorted import _promote, _sorts
from test_gpu_q_sorted import fields  # noqa: F401  (fixture)
from test_gpu_query_filters import N, OC_ERR_INVALID, OC_ERR_UNSUPPORTED, _assign, _inputs
from test_gpu_query_filters import corpus  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

_MODES = (MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID)


def _entries(B, seed, max_limit=200, thresholds=(None,), sims=(0.0, 0.5, 0.7), max_offset=100, vector_limits=True):
    """A third of each mode; limits 1..max_limit (the first queries take the largest), offsets 0..max_offset, some
    vector_limit."""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(B):
        lim = max_limit - b if b < 3 else int(rng.integers(1, max_limit + 1))
        vl = int(rng.integers(lim, lim + 40)) if rng.random() < 0.2 and vector_limits else 0
        thr = thresholds[int(rng.integers(0, len(thresholds)))]
        out.append(ob.QueryParams(mode=_MODES[b % 3], limit=lim, offset=int(rng.integers(0, max_offset + 1)),
                                  similarity=float(sims[int(rng.integers(0, len(sims)))]), threshold=thr, vector_limit=vl))
    return out


def _scalars(e):
    return dict(mode=e.mode, limit_hint=e.limit, offset=e.offset, similarity=e.similarity, threshold=e.threshold,
                vector_limit=e.vector_limit)


def _one_inputs(e, texts, qv, b):
    """A query alone: its text for a text part, its vector for a vector part."""
    return ([texts[b]] if e.mode != MODE_VECTOR else None), (qv[b:b + 1] if e.mode != MODE_FULLTEXT else None)


def _tsc(c, emb=None, strs=None):
    return ob.TokenScoreContext(c["ctx"], emb or c["emb"], strs or c["strs"])


def _row(x, b, L):
    """Query b's row of a batch output, cut to its own limit; the rest of the row must be 0."""
    assert not x[b, L:].any(), (b, L)
    return x[b, :L]


def _check_plain(tsc, entries, texts, qv, filters=None, **kw):
    got = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=MODE_HYBRID, query_params=entries, device_filters=filters, **kw),
                                   texts, qv)
    assert got[0].shape[1] == max(e.limit for e in entries)
    for b, e in enumerate(entries):
        t, q = _one_inputs(e, texts, qv, b)
        one = tsc.execute_batch_arrays(ob.TokenScoreParams(device_filter=None if filters is None else filters[b], **_scalars(e), **kw), t, q)
        for what, x, y in (("docs", _row(got[0], b, e.limit), one[0][0]), ("scores", _row(got[1], b, e.limit), one[1][0]),
                           ("n", got[2][b], one[2][0]), ("count", got[3][b], one[3][0])):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (b, what, e, kw)
    return got


@pytest.mark.parametrize("store", ["f32", "bf16"])
@pytest.mark.parametrize("variant", ["plain", "threshold", "multi_term", "deep", "filters_omc"])
def test_mixed_batch_equals_each_query_alone(corpus, store, variant):  # noqa: F811
    """plain: the register-folded scorer and the tensor-core sweep (depths <= 128); threshold: the threshold scorer;
    multi_term: the accumulator scorer; deep: depths up to 200 (the exact sweep); filters_omc: q_filters and OMC."""
    c = corpus
    B = 72
    tsc = _tsc(c, emb=c["embh"] if store == "bf16" else None)
    qv, texts = _inputs(B, 9100 + len(variant), c["rows"], multi=variant == "multi_term")
    max_limit = 200 if variant == "deep" else 120
    thresholds = (None, 0.0, 0.5, 1.0) if variant in ("threshold", "deep") else (None,)
    entries = _entries(B, 31 + len(variant), max_limit=max_limit, thresholds=thresholds)
    kw, filters = {}, None
    if variant == "filters_omc":
        filters = _assign(c["fs"], B, 5)
        rng = np.random.default_rng(19)
        od = np.sort(rng.choice(N, 3000, replace=False)).astype(np.uint64)
        kw.update(omc_doc_ids=od, omc_mult=rng.uniform(0.5, 3.0, od.shape[0]).astype(np.float32))
    _check_plain(tsc, entries, texts, qv, filters, **kw)


@pytest.mark.parametrize("mode", _MODES)
def test_entries_equal_to_the_scalars_give_the_plain_call(corpus, mode):  # noqa: F811
    c = corpus
    B = 40
    tsc = _tsc(c)
    qv, texts = _inputs(B, 9300, c["rows"])
    t, q = (texts if mode != MODE_VECTOR else None), (qv if mode != MODE_FULLTEXT else None)
    kw = dict(limit_hint=25, offset=7, similarity=0.5, threshold=0.5 if mode == MODE_HYBRID else None)
    plain = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=mode, **kw), t, q)
    entries = [ob.QueryParams(mode=mode, limit=25, offset=7, similarity=0.5, threshold=kw["threshold"])] * B
    got = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=mode, query_params=entries, **kw), t, q)
    for x, y in zip(got, plain):
        assert x.tobytes() == y.tobytes()


def test_q_sorted_mixed(corpus, fields):  # noqa: F811
    """Sorts and pins per query, with q_filters and OMC: each query equals oc_search_sorted / oc_search_pinned alone."""
    c = corpus
    B = 48
    tsc = _tsc(c)
    qv, texts = _inputs(B, 9500, c["rows"])
    entries = _entries(B, 41, max_limit=60, thresholds=(None, 0.5), max_offset=40)
    filters, sorts, promote = _assign(c["fs"], B, 7), _sorts(fields, B, 9), _promote(B, 11)
    rng = np.random.default_rng(23)
    od = np.sort(rng.choice(N, 2000, replace=False)).astype(np.uint64)
    kw = dict(omc_doc_ids=od, omc_mult=rng.uniform(0.5, 3.0, od.shape[0]).astype(np.float32))
    got = ob.search_q_sorted_arrays(tsc, ob.TokenScoreParams(mode=MODE_HYBRID, query_params=entries, device_filters=filters, **kw),
                                    sorts, promote, texts, qv)
    off = np.cumsum([0] + [len(x) for x in promote])
    for b, e in enumerate(entries):
        t, q = _one_inputs(e, texts, qv, b)
        one = ob.search_q_sorted_arrays(tsc, ob.TokenScoreParams(device_filter=filters[b], **_scalars(e), **kw), [sorts[b]],
                                        [promote[b]], t, q)
        for what, x, y in zip(("docs", "scores", "sort values"), got[:3], one[:3]):
            assert _row(x, b, e.limit).tobytes() == y[0].tobytes(), (b, what, e)
        for what, x, y in zip(("n", "count"), got[3:5], one[3:5]):
            assert x[b] == y[0], (b, what, e)
        for what, x, y in zip(("pin scores", "pin present"), got[5:7], one[5:7]):
            assert x[off[b]:off[b + 1]].tobytes() == y.tobytes(), (b, what, e)


def _check_grouped(tsc, st, entries, filters, groups, promote, facets, texts, qv, **kw):
    """oc_search_q_facets with per-query parameters: each query equals the same call with B = 1 and its own scalars."""
    B = len(entries)
    k = [len(x) for x in promote]
    S = max([1] + [(2 * int(g[1]) + k[b] if k[b] else int(g[1])) for b, g in enumerate(groups) if g is not None and g[0] is not None])
    got = ob.search_q_facets_arrays(tsc, st, ob.TokenScoreParams(mode=MODE_HYBRID, query_params=entries, device_filters=filters, **kw),
                                    facets, groups, promote, texts, qv, group_stride=S)
    off = np.cumsum([0] + k)
    rows, foff = got[11], got[13]
    for b, e in enumerate(entries):
        t, q = _one_inputs(e, texts, qv, b)
        one = ob.search_q_facets_arrays(tsc, st, ob.TokenScoreParams(device_filter=filters[b], **_scalars(e), **kw), [facets[b]],
                                        [groups[b]], [promote[b]], t, q, group_stride=S)
        L = e.limit
        for what, x, y in zip(("docs", "scores", "sort values"), got[:3], one[:3]):
            assert _row(x, b, L).tobytes() == y[0].tobytes(), (b, what, e)
        for what, x, y in zip(("n", "count"), got[3:5], one[3:5]):
            assert x[b] == y[0], (b, what, e)
        for what, x, y in zip(("pin scores", "pin present"), got[5:7], one[5:7]):
            assert x[off[b]:off[b + 1]].tobytes() == y.tobytes(), (b, what, e)
        for what, x, y in zip(("group docs", "group scores", "group sort values", "group n"), got[7:11], one[7:11]):
            assert x[rows[b]:rows[b + 1]].tobytes() == y.tobytes(), (b, what, e)
        assert got[12][foff[b]:foff[b + 1]].tolist() == one[12].tolist(), (b, "facets", e)


def test_q_groups_and_facets_mixed(corpus, fields, faceting):  # noqa: F811
    """Groups, sorts, pins and facets per query, with q_filters and OMC; then the same with tombstones in the string
    store, before and after a commit."""
    c = corpus
    B = 36
    qv, texts = _inputs(B, 9700, c["rows"])
    entries = _entries(B, 43, max_limit=40, thresholds=(None, 0.5), max_offset=30)
    filters = _assign(c["fs"], B, 13)
    groups = _requests(faceting["gbs"], fields, B, 17, with_1000=False)
    promote, facets = _promote(B, 19), _mix(B, 21)
    rng = np.random.default_rng(29)
    od = np.sort(rng.choice(N, 2000, replace=False)).astype(np.uint64)
    kw = dict(omc_doc_ids=od, omc_mult=rng.uniform(0.5, 3.0, od.shape[0]).astype(np.float32))
    _check_grouped(_tsc(c), faceting["st"], entries, filters, groups, promote, facets, texts, qv, **kw)
    strs = ob.StringFieldStorage(c["ctx"], c["data"])
    try:
        strs.delete(rng.choice(N, 600, replace=False).astype(np.uint64))
        tsc = _tsc(c, strs=strs)
        _check_grouped(tsc, faceting["st"], entries, filters, groups, promote, facets, texts, qv, **kw)
        strs.commit()
        _check_grouped(tsc, faceting["st"], entries, filters, groups, promote, facets, texts, qv, **kw)
    finally:
        strs.close()


def test_oracle(corpus, orc):  # noqa: F811
    c = corpus
    B = 30
    tsc = _tsc(c)
    qv, texts = _inputs(B, 9900, c["rows"])
    entries = _entries(B, 47, max_limit=50, thresholds=(None, 0.5), sims=(0.0,), max_offset=20, vector_limits=False)
    got = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=MODE_HYBRID, query_params=entries), texts, qv)
    sb = orc.SearchBatch(orc.StrIndex(c["data"]), orc.EmbStore(c["rows"]))
    for b, e in enumerate(entries):
        sb.add(e.mode, limit=e.limit, offset=e.offset, similarity=e.similarity, q_vec=qv[b], text=texts[b], threshold=e.threshold)
    od, os_, on, oc = sb.run(2)
    for b in range(B):
        assert int(got[3][b]) == int(oc[b]), b
        n = int(got[2][b])
        assert_topk_equal(got[0][b, :n], got[1][b, :n], od[b, :on[b]], os_[b, :on[b]])


def _raw(tsc, entries, texts, qv, limit=None, **kw):
    sp, keep, B = tsc._build_params(ob.TokenScoreParams(mode=MODE_HYBRID, query_params=entries, **kw), texts, qv)
    if limit is not None:
        sp.limit = limit
    L = max(int(sp.limit), 1)
    out = [np.full((B, L), 0xAB, np.uint64), np.full((B, L), 7.0, np.float32), np.full(B, 9, np.uint32), np.full(B, 9, np.uint64)]
    return sp, keep, out


def _untouched(out):
    assert (out[0] == 0xAB).all() and (out[1] == 7.0).all() and (out[2] == 9).all() and (out[3] == 9).all()


def test_refusals(corpus, fields, faceting):  # noqa: F811
    c = corpus
    B = 6
    lib = _lib.lib()
    qv, texts = _inputs(B, 9950, c["rows"])
    tsc = _tsc(c)
    base = _entries(B, 53, max_limit=20, max_offset=5)

    def search(t, entries, limit=None, no_emb=False, **kw):
        sp, keep, out = _raw(t, entries, texts, qv, limit, **kw)
        rc = lib.oc_search(t.ctx._h, None if no_emb else t.emb._h, t.str._h, C.byref(sp), *[_p(x) for x in out])
        _untouched(out)
        return rc

    def with_(b, **f):
        e = list(base)
        d = dict(_scalars(e[b]), **f)
        e[b] = ob.QueryParams(mode=d["mode"], limit=d["limit_hint"], offset=d["offset"], similarity=d["similarity"],
                              threshold=d["threshold"], vector_limit=d["vector_limit"])
        return e

    assert search(tsc, with_(2, mode=7)) == OC_ERR_INVALID
    assert search(tsc, with_(1, limit_hint=0)) == OC_ERR_INVALID
    assert search(tsc, base, limit=5) == OC_ERR_INVALID                      # an entry's limit above p->limit
    assert search(tsc, with_(0, limit_hint=1000, offset=100)) == OC_ERR_UNSUPPORTED
    assert search(tsc, with_(3, vector_limit=2000)) == OC_ERR_UNSUPPORTED
    assert search(tsc, base, no_emb=True) == OC_ERR_INVALID                  # a vector entry without a store
    assert search(tsc, base, sharded=True) == OC_ERR_UNSUPPORTED

    sp, keep, out = _raw(tsc, base, texts, qv)
    pins = (_lib.Pins)()
    offs = np.zeros(B + 1, np.uint32)
    pins.q_pin_offsets = _p(offs)
    sv = np.zeros(out[0].shape, np.float64)
    h = (tsc.ctx._h, tsc.emb._h, tsc.str._h)
    assert lib.oc_search_pinned(*h, C.byref(sp), C.byref(pins), _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]), None, None) == OC_ERR_UNSUPPORTED
    srt = _lib.Sort(fields["price"]._h, 0)
    assert lib.oc_search_sorted(*h, C.byref(sp), C.byref(srt), None, _p(out[0]), _p(out[1]), _p(sv), _p(out[2]), _p(out[3]),
                                None, None) == OC_ERR_UNSUPPORTED
    gb = faceting["gbs"][10]
    gd, gs, gn = np.zeros((gb.n_groups, 3), np.uint64), np.zeros((gb.n_groups, 3), np.float32), np.zeros(gb.n_groups, np.uint32)
    for fn in (lambda: lib.oc_search_groups(*h, gb._h, C.byref(sp), 3, _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]), _p(gd), _p(gs), _p(gn)),
               lambda: lib.oc_search_groups_pinned(*h, gb._h, C.byref(sp), 3, None, 3, _p(out[0]), _p(out[1]), _p(out[2]), _p(out[3]),
                                                   _p(gd), _p(gs), _p(gn)),
               lambda: lib.oc_search_groups_sorted(*h, gb._h, C.byref(sp), 3, C.byref(srt), None, 3, _p(out[0]), _p(out[1]), None,
                                                   _p(out[2]), _p(out[3]), _p(gd), _p(gs), None, _p(gn))):
        assert fn() == OC_ERR_UNSUPPORTED
        assert not gd.any() and not gn.any()
    reqs, _ = ob.facet_requests(faceting["st"], {"cat": {}})
    arr = (_lib.FacetReq * len(reqs))(*[_lib.FacetReq(*r) for r in reqs])
    fc = np.full(B * len(reqs), 5, np.uint64)
    assert lib.oc_search_facets(*h, faceting["st"]._h, C.byref(sp), arr, len(reqs), _p(fc)) == OC_ERR_UNSUPPORTED
    assert (fc == 5).all()
    _untouched(out)
    # an active pinned query with 2 x (limit + offset) > 1024 in oc_search_q_sorted
    e = with_(0, limit_hint=400, offset=200)
    sp, keep, out = _raw(tsc, e, texts, qv)
    offs = np.asarray([0, 1] + [1] * (B - 1), np.uint32)
    docs, pos = np.asarray([3], np.uint64), np.asarray([0], np.uint32)
    pins = _lib.Pins(_p(offs), _p(docs), _p(pos), 1)
    sorts = (_lib.Sort * B)()
    sv = np.zeros(out[0].shape, np.float64)
    assert lib.oc_search_q_sorted(*h, C.byref(sp), sorts, C.byref(pins), _p(out[0]), _p(out[1]), _p(sv), _p(out[2]), _p(out[3]),
                                  None, None) == OC_ERR_UNSUPPORTED
    _untouched(out)


@pytest.mark.parametrize("mixed", [True, False])
def test_batcher_mixed(corpus, mixed):  # noqa: F811
    """Threads through SearchBatcher(mixed=...) with random scalars, half of them with one index's OMC multipliers: each
    result equals the request alone.  mixed: requests merge across scalars and with OMC (no direct call); flag off: the
    old key, so every OMC request runs directly."""
    import threading
    c = corpus
    tsc = _tsc(c)
    T, PER = 24, 6
    B = T * PER
    qv, texts = _inputs(B, 9990, c["rows"])
    entries = _entries(B, 59, max_limit=40, thresholds=(None, 0.5), max_offset=20)
    rng = np.random.default_rng(61)
    od = np.sort(rng.choice(N, 2000, replace=False)).astype(np.uint64)
    om = rng.uniform(0.5, 3.0, od.shape[0]).astype(np.float32)
    with_omc = rng.random(B) < 0.5
    kws = [dict(omc_doc_ids=od, omc_mult=om) if with_omc[b] else {} for b in range(B)]
    got = [None] * B
    bat = ob.SearchBatcher(tsc, max_batch=64, max_wait_us=3000, mixed=mixed)
    errors = []

    def worker(t):
        try:
            for k in range(PER):
                b = t * PER + k
                e = entries[b]
                t_, q_ = _one_inputs(e, texts, qv, b)
                got[b] = bat.search(ob.TokenScoreParams(**_scalars(e), **kws[b]), None if t_ is None else t_[0],
                                    None if q_ is None else q_[0])
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)

    th = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
    st = bat.stats()
    with pytest.raises(ValueError):
        bat.search(ob.TokenScoreParams(mode=MODE_FULLTEXT, query_params=[entries[0]]), texts[0])
    bat.close()
    for b, e in enumerate(entries):
        t_, q_ = _one_inputs(e, texts, qv, b)
        one = tsc.execute_batch_arrays(ob.TokenScoreParams(**_scalars(e), **kws[b]), t_, q_)
        n = int(one[2][0])
        assert got[b].doc_ids.tobytes() == one[0][0, :n].tobytes(), (b, e)
        assert got[b].scores.tobytes() == one[1][0, :n].tobytes(), (b, e)
        assert got[b].count == int(one[3][0]), (b, e)
    assert st["queries"] + st["direct"] == B
    if mixed:
        assert st["direct"] == 0 and st["batches"] < st["queries"], st
    else:
        assert st["direct"] == int(with_omc.sum()), st
