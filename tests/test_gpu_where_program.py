"""Where clauses as programs evaluated inside the search call (oc_search_params.q_where, TokenScoreParams.where_programs,
IndexLoader.where_program, oc_filter_from_where, oc_where_check).

The bitmaps of programs (every leaf kind and op, random trees with geo leaves and deletes, FILTER-only programs, a
FILTER handle with a dirty tail) are checked against the host restatement of tests/test_where_host.py.  The rule for
searches: query b's outputs with q_where are byte for byte those it gets with q_filters[b] = the handle evaluate_where
builds from the same clause.  Both sides of that rule run the same planner and kernels, so it checks the in-call path
against the handle path only; tests/test_gpu_where_oracle.py checks the in-call programs against bitmaps computed on the
host.  Checked for oc_search / oc_search_q_sorted / oc_search_q_groups / oc_search_q_facets over fulltext, vector and
hybrid with mixed per-query parameters, for batches with duplicate programs, unfiltered queries, single leaves and
FILTER-only programs, for workspace reuse, for every refusal, for the launch count of the where stage and through the
batcher from many threads."""
import ctypes as C
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib
from oramacore_b200.engine import _p
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from oramacore_b200.where import WhereProgram, compile_where, evaluate_where, filter_from_program, pack_programs, parse_where
from test_gpu_q_groups import _facets, _requests
from test_gpu_q_sorted import _promote, _sorts, _tsc
from test_gpu_q_sorted import fields  # noqa: F401  (fixture)
from test_gpu_query_filters import MODES, N, OC_ERR_INVALID, OC_ERR_UNSUPPORTED, _inputs
from test_gpu_query_filters import corpus  # noqa: F401  (fixture)
from test_gpu_where import NBITS, _ids, _leaf_json, _tree
from test_gpu_where import store  # noqa: F401  (fixture)
from test_where_host import host_where

pytestmark = pytest.mark.gpu


def _bits(f):
    try:
        return f.read()
    finally:
        f.close()


def _live(ctx, deleted, nbits):
    d = ob.DeviceFilter.from_ids(ctx, deleted, nbits)
    try:
        return ~d
    finally:
        d.close()


# ---------------------------------------------------------------- bitmaps: oc_filter_from_where == the host restatement
def _check_bits(store, w, deleted, live):  # noqa: F811
    """The program of w (with the NOT(deletes) handle `live` as a FILTER node when there are deletes) is the set
    host_where computes."""
    st, geo, fields_, _, _, _ = store
    prog = compile_where(w, st, geo, NBITS, live if deleted else None)
    want = host_where(w, fields_, NBITS, deleted)
    assert (prog is None) == (want is None)
    if prog is not None:
        assert _ids(filter_from_program(st.ctx, prog)) == want


@pytest.mark.parametrize("key", ["n", "d", "b", "s", "g"])
def test_bits_every_leaf_kind(store, key):  # noqa: F811
    st, geo, fields_, deleted, rng, nv = store
    live = _live(st.ctx, deleted, NBITS)
    try:
        for i in range(30):
            where = {key: _leaf_json(rng, key, nv, fields_)}
            _check_bits(store, parse_where(where), deleted if i % 3 == 0 else [], live)
        for wrong in (True, "k1", {"gt": 0}):   # the wrong kind of filter for the field: empty
            _check_bits(store, parse_where({key: wrong}), [], live)
        # each op over two leaves, and the empty top level with deletes (a FILTER-only program)
        a, b = _leaf_json(rng, key, nv, fields_), _leaf_json(rng, key, nv, fields_)
        for where in ({"and": [{key: a}, {key: b}]}, {"or": [{key: a}, {key: b}]}, {"not": {key: a}}, {"or": []}, {}):
            _check_bits(store, parse_where(where), deleted, live)
    finally:
        live.close()


def test_bits_random_trees(store):  # noqa: F811
    st, geo, fields_, deleted, rng, nv = store
    live = _live(st.ctx, deleted, NBITS)
    try:
        for i in range(220):
            _check_bits(store, parse_where(_tree(rng, 1, nv, fields_)), deleted if i % 2 else [], live)
    finally:
        live.close()


def test_leaves_of_another_nbits_are_refused(store):  # noqa: F811
    """A store whose nbits differs from the nbits asked for is refused, for a tree of one leaf as for more."""
    st, geo, fields_, _, rng, nv = store
    for where in ({"b": True}, {"g": _leaf_json(rng, "g", nv, fields_)}, {"b": True, "s": "k1"}):
        with pytest.raises(_lib.OcError) as e:
            evaluate_where(parse_where(where), st, geo, NBITS + 1)
        assert e.value.code == OC_ERR_INVALID, where


# ---------------------------------------------------------------- searches: q_where == q_filters of the same handles
@pytest.fixture(scope="module")
def wcorpus(corpus):  # noqa: F811
    ctx = corpus["ctx"]
    st, gbs, _ = _facets(ctx, N, 5)
    rng = np.random.default_rng(31)
    ids = np.arange(N, dtype=np.uint64)
    geo = {"g": ob.GeoPointField(ctx, N, ids, rng.uniform(-60, 60, N), rng.uniform(-120, 120, N))}
    deleted = rng.choice(N, 500, replace=False).tolist()
    live = _live(ctx, deleted, N)
    yield dict(corpus, st=st, gbs=gbs, geo=geo, deleted=deleted, live=live)
    live.close()
    geo["g"].close()
    for gb in gbs.values():
        gb.close()
    st.close()


def _leaf(rng):
    k = ["cat", "flag", "num", "g", "num"][int(rng.integers(0, 5))]
    if k == "cat":
        return {k: f"c{int(rng.integers(0, 11))}"}   # c10: an unknown key
    if k == "flag":
        return {k: bool(rng.random() < 0.5)}
    if k == "num":
        lo = int(rng.integers(0, 1000))
        return {k: [{"gt": lo}, {"lte": lo}, {"between": [lo, lo + int(rng.integers(0, 400))]}, {"eq": lo}][int(rng.integers(0, 4))]}
    if rng.random() < 0.5:
        c = rng.uniform(-40, 40, 2)
        return {k: {"radius": {"coordinates": {"lat": float(c[0]), "lon": float(c[1])}, "value": float(rng.uniform(500, 3000)),
                               "unit": "km", "inside": bool(rng.random() < 0.7)}}}
    c, rr = rng.uniform(-40, 40, 2), rng.uniform(5, 40)
    a = np.linspace(0, 2 * np.pi, int(rng.integers(3, 8)), endpoint=False)
    return {k: {"polygon": {"coordinates": [{"lat": float(c[0] + rr * np.sin(t)), "lon": float(c[1] + rr * np.cos(t))} for t in a]}}}


def _clause(rng, depth=1):
    w = {}
    for _ in range(int(rng.integers(0, 3))):
        w.update(_leaf(rng))
    if depth < 3:
        if rng.random() < 0.4:
            w["and"] = [_clause(rng, depth + 1) for _ in range(int(rng.integers(1, 3)))]
        if rng.random() < 0.4:
            w["or"] = [_clause(rng, depth + 1) for _ in range(int(rng.integers(1, 3)))]
        if rng.random() < 0.2:
            w["not"] = _clause(rng, depth + 1)
    return w


def _batch(c, B, seed, deletes=True):
    """Per query a program and the handle evaluate_where builds for it: random trees, duplicates, unfiltered queries,
    single leaves and (with deletes) FILTER-only programs."""
    rng = np.random.default_rng(seed)
    live = c["live"] if deletes else None
    dele = c["deleted"] if deletes else []
    progs, handles, cache, srcs = [], [], {}, []
    for b in range(B):
        r = b % 6
        if r == 0:
            where = None
        elif r == 1:
            where = {}
        elif r == 2:
            where = _leaf(rng)
        elif r == 3 and b > 6:
            where = srcs[b - 6]   # a duplicate of an earlier clause
        else:
            where = _clause(rng)
        srcs.append(where)
        if where is None:
            progs.append(None); handles.append(None)
            continue
        w = parse_where(where)
        progs.append(compile_where(w, c["st"], c["geo"], N, live))
        key = repr(where)
        if key not in cache:
            cache[key] = evaluate_where(w, c["st"], c["geo"], N, dele, ctx=c["ctx"])
        handles.append(cache[key])
    return progs, handles, [h for h in cache.values() if h is not None]


def _qparams(B, seed):
    rng = np.random.default_rng(seed)
    return [ob.QueryParams(mode=[MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID][b % 3], limit=int(rng.integers(1, 30)),
                           offset=int(rng.integers(0, 5)), similarity=0.0) for b in range(B)]


def _same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (what, i)


@pytest.mark.parametrize("B", [1, 48])
@pytest.mark.parametrize("mode", list(MODES))
def test_search_identity(wcorpus, fields, mode, B):  # noqa: F811
    """In-call programs (q_where) give the outputs of q_filters set to the handles evaluate_where builds for the same
    clauses.  Both come from the same where_plan, so this shows the two paths agree, not that either is right:
    tests/test_gpu_where_oracle.py compares the in-call programs with independent host bitmaps and the oracle."""
    c = wcorpus
    m = MODES[mode]
    qv, texts = _inputs(B, 700 + B, c["rows"])
    progs, handles, owned = _batch(c, B, B + 1)
    if B == 1:
        progs, handles = progs[-1:], handles[-1:]
    t, q = (texts if m != MODE_VECTOR else None), (qv if m != MODE_FULLTEXT else None)
    tsc = _tsc(c, m)
    try:
        for kw in [dict(mode=m, limit_hint=20, similarity=0.0)] + ([dict(mode=m, query_params=_qparams(B, B))] if m == MODE_HYBRID else []):
            pw = ob.TokenScoreParams(where_programs=progs, **kw)
            pf = ob.TokenScoreParams(device_filters=handles, **kw)
            got = tsc.execute_batch_arrays(pw, t, q)
            _same(got, tsc.execute_batch_arrays(pf, t, q), "oc_search")
            for b in range(min(B, 4)):   # each query alone
                one = tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=[progs[b]], **{**kw, **(
                    {"query_params": [kw["query_params"][b]]} if "query_params" in kw else {})}),
                    None if t is None else [t[b]], None if q is None else q[b:b + 1])
                n = int(one[2][0])
                assert got[0][b, :n].tobytes() == one[0][0, :n].tobytes() and got[3][b] == one[3][0], b
            sorts, promote = _sorts(fields, B, B), _promote(B, B)
            _same(ob.search_q_sorted_arrays(tsc, pw, sorts, promote, t, q), ob.search_q_sorted_arrays(tsc, pf, sorts, promote, t, q),
                  "oc_search_q_sorted")
            groups = _requests(c["gbs"], fields, B, B + 3, with_1000=False)
            _same(ob.search_q_groups_arrays(tsc, pw, groups, promote, t, q), ob.search_q_groups_arrays(tsc, pf, groups, promote, t, q),
                  "oc_search_q_groups")
            facets = [{"cat": {}, "num": {"ranges": [{"from": 0, "to": 300}]}} if b % 2 else None for b in range(B)]
            a = ob.search_q_facets_arrays(tsc, c["st"], pw, facets, groups, promote, t, q)
            f = ob.search_q_facets_arrays(tsc, c["st"], pf, facets, groups, promote, t, q)
            _same(a[:13], f[:13], "oc_search_q_facets")
    finally:
        for h in owned:
            h.close()


def test_workspace_reuse(wcorpus):
    """A call with dense leaves, then one with sparse leaves in the same workspace: no stale bits."""
    c = wcorpus
    tsc = _tsc(c, MODE_FULLTEXT)
    _, texts = _inputs(16, 901, c["rows"])
    for where in ({"or": [{"num": {"gte": 0}}, {"flag": True}], "cat": "c1"}, {"and": [{"num": {"eq": 3}}, {"cat": "c3"}]},
                  {"num": {"eq": 3}, "not": {"flag": True}}):
        w = parse_where(where)
        prog = compile_where(w, c["st"], c["geo"], N, None)
        h = evaluate_where(w, c["st"], c["geo"], N, [], ctx=c["ctx"])
        try:
            kw = dict(mode=MODE_FULLTEXT, limit_hint=50)
            _same(tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=[prog] * 16, **kw), texts),
                  tsc.execute_batch_arrays(ob.TokenScoreParams(device_filters=[h] * 16, **kw), texts), where)
            assert _bits(filter_from_program(c["ctx"], prog)).tobytes() == h.read().tobytes()
        finally:
            h.close()


# ---------------------------------------------------------------- launch count of the where stage
def test_launch_count_is_bounded(wcorpus):
    c = wcorpus
    tsc = _tsc(c, MODE_FULLTEXT)
    deltas = []
    for B in (1, 256):
        _, texts = _inputs(B, 950 + B, c["rows"])
        for n_leaves in (1, 8):
            rng = np.random.default_rng(B + n_leaves)
            progs, handles = [], []
            for b in range(B):
                where = {"and": [_leaf(rng) for _ in range(n_leaves)]} if n_leaves > 1 else _leaf(rng)
                w = parse_where(where)
                progs.append(compile_where(w, c["st"], c["geo"], N, c["live"]))
                handles.append(evaluate_where(w, c["st"], c["geo"], N, c["deleted"], ctx=c["ctx"]))
            kw = dict(mode=MODE_FULLTEXT, limit_hint=10)
            try:
                x0 = c["ctx"].launch_count()
                tsc.execute_batch_arrays(ob.TokenScoreParams(device_filters=handles, **kw), texts)
                x1 = c["ctx"].launch_count()
                tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=progs, **kw), texts)
                x2 = c["ctx"].launch_count()
            finally:
                for h in handles:
                    h.close()
            deltas.append((x2 - x1) - (x1 - x0))
    assert all(0 <= d <= 3 for d in deltas), deltas
    assert deltas[1] == deltas[3], deltas   # 8 leaves per query: the same launches at B = 1 and B = 256


# ---------------------------------------------------------------- refusals
def test_refusals_write_nothing(wcorpus):
    c = wcorpus
    L = _lib.lib()
    ctx = c["ctx"]
    tsc = _tsc(c, MODE_FULLTEXT)
    _, texts = _inputs(2, 990, c["rows"])
    good = compile_where(parse_where({"num": {"gt": 5}, "g": {"polygon": {"coordinates": [{"lat": 0, "lon": 0}, {"lat": 1, "lon": 0},
                                                                                            {"lat": 0, "lon": 1}]}}}),
                         c["st"], c["geo"], N, c["live"])
    other = ob.Context(0)
    foreign = ob.DeviceFilter.from_ids(other, [1], N)
    small = ob.DeviceFilter.from_ids(ctx, [1], N - 1)
    try:
        st_h, g_h = c["st"]._h.value, c["geo"]["g"]._h.value
        num_id, cat_id = c["st"].fields["num"]["id"], c["st"].fields["cat"]["id"]
        V, R, GR, GP, FI = _lib.OC_WHERE_VARIANT, _lib.OC_WHERE_RANGE, _lib.OC_WHERE_GEO_RADIUS, _lib.OC_WHERE_GEO_POLYGON, _lib.OC_WHERE_FILTER
        A, O, NO = _lib.OC_WHERE_AND, _lib.OC_WHERE_OR, _lib.OC_WHERE_NOT
        nan = float("nan")
        bad = {   # name: nodes (op, field, arg, a, b, c, src, verts)
            "field": [(V, 99, 0, 0, 0, 0, st_h, None)],
            "kind": [(V, num_id, 0, 0, 0, 0, st_h, None)],
            "kind_range": [(R, cat_id, 0, 0, 1, 0, st_h, None)],
            "variant": [(V, cat_id, 99, 0, 0, 0, st_h, None)],
            "nan": [(R, num_id, 0, nan, 1, 0, st_h, None)],
            "flags": [(R, num_id, 4, 0, 1, 0, st_h, None)],
            "coords": [(GR, 0, 1, 91.0, 0, 10, g_h, None)],
            "radius": [(GR, 0, 1, 0, 0, -1.0, g_h, None)],
            "vertices": [(GP, 0, 1, 0, 0, 0, g_h, (np.zeros(2), np.zeros(2)))],
            "vertex": [(GP, 0, 1, 0, 0, 0, g_h, (np.array([0.0, 1.0, 95.0]), np.zeros(3)))],
            "foreign": [(FI, 0, 0, 0, 0, 0, foreign._h.value, None), (NO, 0, 0, 0, 0, 0, None, None)],
            "nbits": [(FI, 0, 0, 0, 0, 0, small._h.value, None), (NO, 0, 0, 0, 0, 0, None, None)],
            "underflow": [(R, num_id, 0, 0, 1, 0, st_h, None), (A, 0, 2, 0, 0, 0, None, None)],
            "two_left": [(R, num_id, 0, 0, 1, 0, st_h, None), (R, num_id, 0, 2, 3, 0, st_h, None)],
            "arity": [(R, num_id, 0, 0, 1, 0, st_h, None), (O, 0, 1, 0, 0, 0, None, None)],
            "op": [(77, 0, 0, 0, 0, 0, None, None)],
            "depth": [(R, num_id, 0, float(i), 1e9, 0, st_h, None) for i in range(_lib.OC_WHERE_MAX_DEPTH + 1)]
                     + [(A, 0, _lib.OC_WHERE_MAX_DEPTH + 1, 0, 0, 0, None, None)],
            "nodes": [(R, num_id, 0, 0, 1, 0, st_h, None)] + [(NO, 0, 0, 0, 0, 0, None, None)] * _lib.OC_WHERE_MAX_NODES,
        }
        cases = [(name, [good, WhereProgram(N, nodes)], OC_ERR_INVALID) for name, nodes in bad.items()]
        for name, progs, code in cases:
            w, keep = pack_programs(progs)
            assert L.oc_where_check(C.byref(w), 2) == code, name
            sp, keep2, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=5, where_programs=progs), texts)
            docs, sc = np.full((2, 5), 7, np.uint64), np.full((2, 5), 7, np.float32)
            n, cnt = np.full(2, 7, np.uint32), np.full(2, 7, np.uint64)
            rc = L.oc_search(ctx._h, None, tsc.str._h, C.byref(sp), _p(docs), _p(sc), _p(n), _p(cnt))
            assert rc == code, (name, rc)
            assert (docs == 7).all() and (sc == 7).all() and (n == 7).all() and (cnt == 7).all(), name
            h = C.c_void_p(0xDEAD0)
            assert L.oc_filter_from_where(ctx._h, C.byref(w), 1, C.byref(h)) == code and h.value == 0xDEAD0, name
        # q_where with filter / filter_bits / q_filters: invalid; sharded: unsupported; nothing written
        w, keep = pack_programs([good, good])
        fbits = np.full((N + 63) // 64, ~np.uint64(0), np.uint64)
        for what, code in (("filter", OC_ERR_INVALID), ("filter_bits", OC_ERR_INVALID), ("q_filters", OC_ERR_INVALID),
                           ("sharded", OC_ERR_UNSUPPORTED)):
            sp, keep2, _ = tsc._build_params(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=5, where_programs=[good, good]), texts)
            arr = (C.c_void_p * 2)(c["live"]._h.value, None)
            if what == "filter":
                sp.filter = c["live"]._h
            elif what == "filter_bits":
                sp.filter_bits, sp.filter_nbits = _p(fbits), N
            elif what == "q_filters":
                sp.q_filters = C.cast(arr, C.c_void_p)
            else:
                sp.sharded = 1
            docs, sc = np.full((2, 5), 7, np.uint64), np.full((2, 5), 7, np.float32)
            n, cnt = np.full(2, 7, np.uint32), np.full(2, 7, np.uint64)
            assert L.oc_search(ctx._h, None, tsc.str._h, C.byref(sp), _p(docs), _p(sc), _p(n), _p(cnt)) == code, what
            assert (docs == 7).all() and (n == 7).all() and (cnt == 7).all(), what
        assert L.oc_where_check(C.byref(w), 2) == 0
        # the entry points that refuse q_filters refuse q_where with the same code
        kw = dict(mode=MODE_FULLTEXT, limit_hint=5)
        for call in (lambda p: ob.search_pinned_arrays(tsc, p, [[], []], texts=texts),
                     lambda p: ob.search_groups_arrays(tsc, c["gbs"][10], p, 3, texts=texts)):
            codes = []
            for p in (ob.TokenScoreParams(where_programs=[good, good], **kw), ob.TokenScoreParams(device_filters=[c["live"], None], **kw)):
                with pytest.raises(_lib.OcError) as e:
                    call(p)
                codes.append(e.value.code)
            assert codes == [OC_ERR_UNSUPPORTED, OC_ERR_UNSUPPORTED], codes
    finally:
        foreign.close(); small.close(); other.close()


# ---------------------------------------------------------------- the batcher
def test_batcher_merges_where_requests(wcorpus):
    c = wcorpus
    tsc = _tsc(c, MODE_HYBRID)
    Q = 64
    qv, texts = _inputs(Q, 1234, c["rows"])
    progs, handles, owned = _batch(c, Q, 77)
    modes = [MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID]
    kws = [dict(mode=modes[i % 3], limit_hint=5 + i % 7, similarity=0.0) for i in range(Q)]
    try:
        expect = []
        for i in range(Q):
            one = tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=[progs[i]], **kws[i]),
                                           [texts[i]] if kws[i]["mode"] != MODE_VECTOR else None,
                                           qv[i:i + 1] if kws[i]["mode"] != MODE_FULLTEXT else None)
            expect.append(one)
        sb = ob.SearchBatcher(tsc, max_batch=64, max_wait_us=20000, mixed=True)
        got = [None] * Q
        bar = threading.Barrier(Q)

        def run(i):
            bar.wait()
            got[i] = sb.search(ob.TokenScoreParams(where_programs=[progs[i]], **kws[i]),
                               texts[i] if kws[i]["mode"] != MODE_VECTOR else None, qv[i] if kws[i]["mode"] != MODE_FULLTEXT else None)
        ts = [threading.Thread(target=run, args=(i,)) for i in range(Q)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        st = sb.stats()
        sb.close()
        for i in range(Q):
            d, s, n, cnt = expect[i]
            k = int(n[0])
            assert got[i].doc_ids.tobytes() == d[0, :k].tobytes() and got[i].scores.tobytes() == s[0, :k].tobytes(), i
            assert got[i].count == int(cnt[0]), i
        assert st["direct"] == 0 and st["batches"] < Q, st
    finally:
        for h in owned:
            h.close()


# ---------------------------------------------------------------- IndexLoader.where_program
def test_loader_where_program_equals_where_filter(gpu_ctx):
    from test_gpu_where import Collection, boo, num, strf
    c = Collection(gpu_ctx, number_fields=["n"], bool_fields=["b"], string_filter_fields=["s"])
    try:
        c.insert([{"text": "alpha " * (1 + i % 5), "filters": {"n": num(i), "b": boo(i % 3 == 0), "s": strf(f"k{i % 4}")}}
                  for i in range(300)])
        c.publish()
        c.apply({"type": "DeleteDocuments", "doc_ids": [3, 40, 41, 200]})
        clauses = [{}, {"n": {"gt": 100}}, {"b": True, "or": [{"s": "k1"}, {"n": {"lt": 20}}]}, {"not": {"s": "k2"}}]
        tsc, texts = c.ld.context(), c.ld.resolve(["alpha"] * len(clauses))
        progs = [c.ld.where_program(w) for w in clauses]
        assert progs[0] is not None and len(progs[0].nodes) == 1   # deletes only: one FILTER node
        assert progs[1].keep[0] is progs[0].keep[0]                 # one NOT(deletes) handle per set of deletes
        kw = dict(mode=MODE_FULLTEXT, limit_hint=50)
        got = tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=progs, **kw), texts)
        fs = [c.ld.where_filter(w) for w in clauses]
        try:
            _same(got, tsc.execute_batch_arrays(ob.TokenScoreParams(device_filters=fs, **kw), texts), "loader")
        finally:
            for f in fs:
                f.close()
        c.apply({"type": "DeleteDocuments", "doc_ids": [5]})
        assert c.ld.where_program({}).keep[0] is not progs[0].keep[0]   # new deletes: a new handle
    finally:
        c.close()


def test_loader_where_program_after_publish_without_commit(gpu_ctx):
    """Deletes stay uncommitted while refresh_facets() publishes documents with higher ids: the NOT(deletes) handle of
    where_program follows the new DocumentId space, as where_filter's does."""
    from test_gpu_where import Collection, num
    c = Collection(gpu_ctx, number_fields=["n"])
    try:
        c.insert([{"text": "alpha", "filters": {"n": num(i)}} for i in range(50)])
        c.publish()
        c.apply({"type": "DeleteDocuments", "doc_ids": [4, 9]})
        assert c.ld.where_program({}) is not None
        c.insert([{"text": "alpha", "filters": {"n": num(100 + i)}} for i in range(80)])   # ids beyond the old nbits
        c.publish()
        clauses = [{}, {"n": {"gte": 10}}]
        progs = [c.ld.where_program(w) for w in clauses]
        assert all(p.nbits == c.ld.nbits for p in progs) and progs[0].keep[0].nbits == c.ld.nbits
        tsc, texts = c.ld.context(), c.ld.resolve(["alpha"] * len(clauses))
        kw = dict(mode=MODE_FULLTEXT, limit_hint=200)
        got = tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=progs, **kw), texts)
        fs = [c.ld.where_filter(w) for w in clauses]
        try:
            _same(got, tsc.execute_batch_arrays(ob.TokenScoreParams(device_filters=fs, **kw), texts), "published")
        finally:
            for f in fs:
                f.close()
        assert int(got[3][0]) == 130 - 2   # every published document but the two deleted ones
    finally:
        c.close()


def test_filter_node_with_a_dirty_tail(store):  # noqa: F811
    """A FILTER handle whose padding bits are set (oc_filter_from_bits): And / Or / Not in a program clear them in the
    result."""
    st, geo, _, _, rng, _ = store
    assert NBITS % 64
    ctx = st.ctx
    words = (NBITS + 63) // 64
    tail = np.full(words, ~np.uint64(0), np.uint64)
    tail[-1] = np.uint64((1 << (NBITS % 64)) - 1)
    d = rng.integers(0, np.iinfo(np.uint64).max, words, dtype=np.uint64, endpoint=True)
    d[-1] |= ~tail[-1]
    dirty = ob.DeviceFilter.from_bits(ctx, d, NBITS)
    fid = st.fields["b"]["id"]
    leaf = st.leaf("b", True)
    try:
        assert (dirty.read() == d).all()
        lb = leaf.read()
        F, V = (_lib.OC_WHERE_FILTER, 0, 0, 0.0, 0.0, 0.0, dirty._h.value, None), (_lib.OC_WHERE_VARIANT, fid, 0, 0.0, 0.0, 0.0, st._h.value, None)
        for nodes, want in (([F, V, (_lib.OC_WHERE_OR, 0, 2, 0.0, 0.0, 0.0, None, None)], (d | lb) & tail),
                            ([F, V, (_lib.OC_WHERE_AND, 0, 2, 0.0, 0.0, 0.0, None, None)], d & lb & tail),
                            ([F, (_lib.OC_WHERE_NOT, 0, 0, 0.0, 0.0, 0.0, None, None)], ~d & tail)):
            prog = WhereProgram(NBITS, nodes, [dirty])
            assert _bits(filter_from_program(ctx, prog)).tobytes() == want.tobytes(), nodes[-1][0]
    finally:
        dirty.close(); leaf.close()


def test_batcher_refuses_a_foreign_program_alone(wcorpus):
    """A request whose program names a store of another ctx gets OC_ERR_INVALID; the requests around it are served."""
    c = wcorpus
    tsc = _tsc(c, MODE_FULLTEXT)
    Q = 16
    _, texts = _inputs(Q, 4321, c["rows"])
    other = ob.Context(0)
    st2 = ob.FacetStore(other, N)
    st2.add_number_field("num", np.arange(N, dtype=np.uint64), np.arange(N, dtype=np.float64))
    try:
        good = [compile_where(parse_where(_leaf(np.random.default_rng(i))), c["st"], c["geo"], N, c["live"]) for i in range(Q)]
        bad = compile_where(parse_where({"num": {"gt": 5}}), st2, {}, N, None)
        progs = [bad if i == 5 else good[i] for i in range(Q)]
        kw = dict(mode=MODE_FULLTEXT, limit_hint=10)
        expect = [tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=[progs[i]], **kw), [texts[i]]) if i != 5 else None
                  for i in range(Q)]
        sb = ob.SearchBatcher(tsc, max_batch=Q, max_wait_us=20000)
        got, err = [None] * Q, [None] * Q
        bar = threading.Barrier(Q)

        def run(i):
            bar.wait()
            try:
                got[i] = sb.search(ob.TokenScoreParams(where_programs=[progs[i]], **kw), texts[i])
            except _lib.OcError as e:
                err[i] = e.code
        ts = [threading.Thread(target=run, args=(i,)) for i in range(Q)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        st = sb.stats()
        sb.close()
        assert err[5] == OC_ERR_INVALID and got[5] is None
        for i in range(Q):
            if i == 5:
                continue
            assert err[i] is None, (i, err[i])
            d, s, n, cnt = expect[i]
            k = int(n[0])
            assert got[i].doc_ids.tobytes() == d[0, :k].tobytes() and got[i].count == int(cnt[0]), i
        assert st["queries"] == Q - 1 and st["batches"] < Q - 1, st
    finally:
        st2.close(); other.close()
