"""Where programs on the GPU against an independent host evaluation (tests/where_spec.py), never against the device
evaluator itself: oc_filter_from_where bitmaps, programs at the evaluator's limits, in-call programs (q_where) of every
search entry point, the oracle, IndexLoader and the batcher.

Two corpora of filter fields, built from seeds here: bool, string_filter (with a key no document holds), number (-0.0
and +0.0, runs of equal values at the query bounds, the i32 extremes, integers that round to f32, +-inf, entries with a
document id >= nbits), date, and geopoint with several points per document (the poles, lon +-180, the vertices and
horizontal edges of the polygons queried, exact duplicates at a radius-0 centre).
  * small: NS = 69 989 documents (nbits = 37 mod 64), with a text and embedding corpus over the same documents;
  * large: NL = 3 000 001 documents (nbits = 1 mod 64): several grid-stride passes of where_scatter_kernel and
    where_geo_kernel, and 46 876 words per bitmap.
Legs and sizes:
  0. small programs of every shape (small corpus) — first, so a wrong combinator fails before any program large enough
     to need it right;
  1. random trees with every leaf kind, radius included, with and without NOT(deletes): both corpora;
  2. programs at the limits (depth OC_WHERE_MAX_DEPTH, OC_WHERE_MAX_NODES nodes, And / Or of several hundred
     arguments, a long Not chain, one leaf pushed many times, a 2048-vertex concave self-intersecting polygon, radius 0,
     tiny, >= pi R and at a pole): large corpus;
  3. in-call programs of a 512-query batch against q_filters = DeviceFilter.from_bits(the host bitmap), byte for byte,
     for oc_search / oc_search_q_sorted / oc_search_q_groups / oc_search_q_facets in fulltext, vector and hybrid mode:
     small corpus;
  4. the plain search of leg 3 against the oracle with the host bitmaps as filter_bits: small corpus;
  5. IndexLoader.where_program over uncommitted deletes and after a commit against the host evaluation of the model's
     fields (tests/index_model.py), and programs sent through SearchBatcher from many threads: own small corpora.
Radius leaves are compared outside a 1e-9 relative band of the boundary; in legs 3 and 4 a clause whose radius has a
point in the band is redrawn, so every comparison there is exact."""
import threading

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import _lib, synth
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from oramacore_b200.where import _NARY, WhereFilter, WhereProgram, compile_where, filter_from_program, parse_where
from index_model import IndexModel
from test_gpu_q_groups import _facets
from test_gpu_q_sorted import _promote
from where_spec import from_host_fields, unpack, where_masks, where_spec

pytestmark = pytest.mark.gpu

NS = 64 * 1093 + 37        # 69 989
NL = 64 * 46875 + 1        # 3 000 001
DIM, VOCAB = 64, 2000
MODES = {"fulltext": MODE_FULLTEXT, "vector": MODE_VECTOR, "hybrid": MODE_HYBRID}


def f32(x):
    return float(np.float32(x))


DUP = (f32(12.345678), f32(-98.7654321))   # a radius-0 centre several points sit on exactly
# polygons with horizontal edges, concave and self-intersecting; (lat, lon), f32 values
SQUARE = [(10.0, 20.0), (10.0, 30.0), (20.0, 30.0), (20.0, 20.0)]
NOTCH = [(-30.0, -60.0), (-30.0, -40.0), (-25.0, -40.0), (-25.0, -50.0), (-15.0, -50.0), (-15.0, -40.0), (-10.0, -40.0),
         (-10.0, -60.0)]
BOWTIE = [(40.0, 100.0), (50.0, 120.0), (50.0, 100.0), (40.0, 120.0)]
EDGE = [(-5.0, 170.0), (-5.0, 180.0), (5.0, 180.0), (5.0, 170.0)]   # on the antimeridian


def big_polygon(n=_lib.OC_GEO_MAX_VERTICES):
    """n vertices around (-45, 150) visited five times round (self-intersecting, even-odd matters) at alternating radii
    (concave)."""
    k = np.arange(n)
    a = 2 * np.pi * ((k * 5) % n) / n
    r = np.where(k % 2 == 0, 2.0, 1.2)
    return [(f32(-45.0 + r_ * np.sin(t)), f32(150.0 + r_ * np.cos(t))) for r_, t in zip(r, a)]


BIG = big_polygon()
FIXED = [SQUARE, NOTCH, BOWTIE, EDGE, BIG]


def _poly_json(p, inside=True):
    return {"polygon": {"coordinates": [{"lat": a, "lon": b} for a, b in p], "inside": inside}}


def _special_points(rng):
    """Points every geo leaf has to get right: the poles, lon +-180, the fixed polygons' vertices, edge midpoints and
    points on the horizontal lines through their vertices, and the radius-0 centre six times over."""
    lat = [np.array([90.0, 90.0, 90.0, -90.0, -90.0]), rng.uniform(-80, 80, 300), np.full(6, DUP[0])]
    lon = [np.array([0.0, 77.0, -180.0, 180.0, 12.0]), np.where(rng.random(300) < 0.5, -180.0, 180.0), np.full(6, DUP[1])]
    for p in FIXED:
        vl, vo = np.array([x[0] for x in p]), np.array([x[1] for x in p])
        nx = np.roll(np.arange(len(p)), -1)
        lat += [vl, (vl + vl[nx]) / 2, vl, vl]
        lon += [vo, (vo + vo[nx]) / 2, rng.uniform(vo.min() - 1, vo.max() + 1, len(p)).clip(-180, 180),
                np.nextafter(vo, 200).clip(-180, 180)]
    return np.concatenate(lat).clip(-90, 90), np.concatenate(lon)


def _make_fields(ctx, nbits, seed):
    """Spec fields (where_spec's layout) and the device FacetStore / GeoPointField over [0, nbits)."""
    rng = np.random.default_rng(seed)
    n = nbits
    docs = np.arange(n, dtype=np.int64)
    beyond = nbits + np.arange(40, dtype=np.int64)   # store entries no leaf may pass

    def multi(p_has, p_two):
        has = docs[rng.random(n) < p_has]
        return np.concatenate([has, has[rng.random(has.shape[0]) < p_two], beyond])

    F = {}
    bd = multi(0.85, 0.15)
    bv = rng.random(bd.shape[0]) < 0.5
    F["b"] = ("bool", bd, bv)
    sd = multi(0.7, 0.3)
    sv = np.array([f"k{i}" for i in range(12)])[rng.integers(0, 12, sd.shape[0])]
    F["s"] = ("string", sd, sv)
    nd = multi(0.9, 0.2)
    special = np.array([-0.0, 0.0, np.inf, -np.inf, 2147483647.0, -2147483648.0, 2147483648.0, 2147483649.0, 3e9, 3e9 + 1,
                        16777216.0, 16777217.0, 16777218.0, 0.5, 2.5, -2.5, 1e30])
    r = rng.random(nd.shape[0])
    nv = np.where(r < 0.5, rng.integers(-50, 51, nd.shape[0]).astype(np.float64),
                  np.where(r < 0.8, rng.standard_normal(nd.shape[0]) * 30, special[rng.integers(0, special.shape[0], nd.shape[0])]))
    F["n"] = ("number", nd, nv)
    dd = multi(0.8, 0.2)
    dv = (1_600_000_000_000 + rng.integers(-400, 400, dd.shape[0]) * 86_400_000 + rng.integers(-1, 2, dd.shape[0])).astype(np.float64)
    F["d"] = ("date", dd, dv)
    gd = multi(0.8, 0.2)[:-40]
    glat, glon = np.degrees(np.arcsin(rng.uniform(-1, 1, gd.shape[0]))), rng.uniform(-180, 180, gd.shape[0])
    slat, slon = _special_points(rng)
    sdoc = rng.integers(0, n, slat.shape[0])
    gd, glat, glon = np.concatenate([gd, sdoc]), np.concatenate([glat, slat]), np.concatenate([glon, slon])
    F["g"] = ("geo", gd, (glat, glon))

    st = ob.FacetStore(ctx, nbits)
    st.add_bool_field("b", bd[bv], bd[~bv])
    by_key = {k: sd[sv == k] for k in np.unique(sv).tolist()}
    by_key["ghost"] = []                                   # a key no document holds
    st.add_string_field("s", by_key)
    st.add_number_field("n", nd, nv)
    st.add_date_field("d", dd, dv.astype(np.int64))
    perm = rng.permutation(gd.shape[0])
    geo = {"g": ob.GeoPointField(ctx, nbits, gd[perm], glat[perm], glon[perm])}
    return dict(F=F, st=st, geo=geo, nbits=nbits, ctx=ctx, deleted=rng.choice(n, max(n // 200, 10), replace=False))


def _close_fields(c):
    c["st"].close()
    c["geo"]["g"].close()


@pytest.fixture(scope="module")
def small(gpu_ctx):
    c = _make_fields(gpu_ctx, NS, 11)
    rows = synth.make_vectors(NS, DIM, seed=12)
    data = synth.make_text_corpus(NS, VOCAB, seed=13)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall", dim=DIM)
    emb.insert_batch(np.arange(NS, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    live = _live(gpu_ctx, c["deleted"], NS)
    c.update(rows=rows, data=data, emb=emb, strs=strs, live=live)
    yield c
    live.close(); emb.close(); strs.close()
    _close_fields(c)


@pytest.fixture(scope="module")
def large(gpu_ctx):
    c = _make_fields(gpu_ctx, NL, 21)
    c["live"] = _live(gpu_ctx, c["deleted"], NL)
    yield c
    c["live"].close()
    _close_fields(c)


def _live(ctx, deleted, nbits):
    d = ob.DeviceFilter.from_ids(ctx, np.asarray(deleted, np.uint64), nbits)
    try:
        return ~d
    finally:
        d.close()


def _raw(f):
    try:
        return f.read()
    finally:
        f.close()


# ---------------------------------------------------------------- random clauses
def _num_bound(rng):
    return [0, -0.0, 0.0, 5, -5, 2.5, -2.5, 0.5, 2**31 - 1, -2**31, 2**31, 2**31 + 1, 3000000001, 16777217, 16777216,
            1e39, -1e39, 1e30, int(rng.integers(-50, 51)), int(rng.integers(-50, 51))][int(rng.integers(0, 20))]


def _date_str(ms):
    import datetime
    t = datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc) + datetime.timedelta(milliseconds=int(ms))
    return t.strftime("%Y-%m-%dT%H:%M:%S.") + f"{t.microsecond // 1000:03d}Z"


def _radius(rng):
    r = rng.random()
    inside = bool(rng.random() < 0.7)
    if r < 0.15:
        c, v, u = DUP, 0.0, "m"
    elif r < 0.3:
        c, v, u = (float(rng.choice([90.0, -90.0])), float(rng.uniform(-180, 180))), float(rng.uniform(100, 3000)), "km"
    elif r < 0.4:
        c, v, u = (float(rng.uniform(-60, 60)), float(rng.uniform(-180, 180))), 21000.0, "km"
    else:
        c, v, u = (float(rng.uniform(-70, 70)), float(rng.uniform(-180, 180))), float(rng.uniform(50, 3000)), "km"
    return {"radius": {"coordinates": {"lat": c[0], "lon": c[1]}, "value": v, "unit": u, "inside": inside}}


def _leaf(rng, key=None):
    key = key or ["n", "d", "b", "s", "g", "g", "n", "zz"][int(rng.integers(0, 8))]
    ops = ["eq", "gt", "gte", "lt", "lte", "between"]
    if key == "n":
        op = ops[int(rng.integers(0, 6))]
        return {key: {op: [_num_bound(rng), _num_bound(rng)] if op == "between" else _num_bound(rng)}}
    if key == "d":
        op = ops[int(rng.integers(0, 6))]
        pick = lambda: _date_str(1_600_000_000_000 + int(rng.integers(-400, 400)) * 86_400_000 + int(rng.integers(-1, 2)))  # noqa: E731
        return {key: {op: [pick(), pick()] if op == "between" else pick()}}
    if key == "b":
        return {key: bool(rng.random() < 0.5)}
    if key == "s":
        return {key: ["k1", "k5", "k11", "ghost", "nobody", f"k{int(rng.integers(0, 12))}"][int(rng.integers(0, 6))]}
    if key == "g":
        r = rng.random()
        if r < 0.4:
            return {key: _radius(rng)}
        if r < 0.7:
            return {key: _poly_json(FIXED[int(rng.integers(0, 4))], bool(rng.random() < 0.7))}
        c, rr = rng.uniform(-60, 60, 2), rng.uniform(2, 20)
        a = np.sort(rng.uniform(0, 2 * np.pi, int(rng.integers(3, 9))))
        return {key: _poly_json([(float(c[0] + rr * np.sin(t)), float(c[1] + rr * np.cos(t))) for t in a], bool(rng.random() < 0.7))}
    return {"zz": True}   # not a filter field: the node is empty


def _tree(rng, depth=1, max_depth=4):
    w = {}
    for _ in range(int(rng.integers(0, 3))):
        w.update(_leaf(rng))
    if depth < max_depth:
        if rng.random() < 0.4:
            w["and"] = [_tree(rng, depth + 1, max_depth) for _ in range(int(rng.integers(0, 4)))]
        if rng.random() < 0.4:
            w["or"] = [_tree(rng, depth + 1, max_depth) for _ in range(int(rng.integers(0, 4)))]
        if rng.random() < 0.3:
            w["not"] = _tree(rng, depth + 1, max_depth)
    return w


# ---------------------------------------------------------------- comparing a device bitmap with the host evaluation
def _device_bits(c, w, deletes):
    prog = compile_where(w, c["st"], c["geo"], c["nbits"], c["live"] if deletes else None)
    return None if prog is None else _raw(filter_from_program(c["ctx"], prog))


def _check(c, w, deletes, got=None, cache=None, what=""):
    """The device bitmap of w equals where_spec on every decided document, and its padding bits are clear."""
    nbits = c["nbits"]
    if got is None:
        got = _device_bits(c, w, deletes)
    m = where_masks(w, c["F"], nbits, c["deleted"] if deletes else (), cache)
    assert (got is None) == (m is None), what
    if got is None:
        return 0
    t, f = m
    assert got.shape == ((nbits + 63) // 64,), what
    assert nbits % 64 == 0 or int(got[-1]) >> (nbits % 64) == 0, ("dirty tail", what)
    g = unpack(got, nbits)
    known = t | f
    bad = np.flatnonzero(known & (g != t))
    assert bad.size == 0, (what, bad[:10].tolist(), int(bad.size))
    return int((~known).sum())


# ---------------------------------------------------------------- leg 0: small programs of every shape
def test_small_programs(small):
    """Two- and three-leaf And / Or, Not, leaves shared within a program, and FILTER nodes: each at most a few nodes."""
    c = small
    rng = np.random.default_rng(3)
    lv = [_leaf(rng, k) for k in ("b", "s", "n", "d", "n")]
    b, s, n, d, n2 = lv
    for where in ({"and": [b, s]}, {"or": [b, s]}, {"and": [s, n, d]}, {"or": [n, d, b]}, {"not": b}, {"not": {"or": [s, n]}},
                  {"and": [n, n2]}, {"or": [b, {"not": b}]}, {"and": [n, {"not": n}]}, {**b, "or": [s, n]}):
        for deletes in (False, True):
            _check(c, parse_where(where), deletes, what=(where, deletes))
    # the combinators must matter here: every pair of parts differs
    for where in ({"and": [b, s]}, {"or": [b, s]}, {"and": [s, n, d]}):
        w = parse_where(where)
        full = where_masks(w, c["F"], NS)[0]
        first = where_masks(WhereFilter(and_=[(w.and_ or w.or_)[0]]), c["F"], NS)[0]
        assert (full != first).any(), where


# ---------------------------------------------------------------- leg 1: random trees at scale
@pytest.mark.parametrize("size, n_trees", [("small", 120), ("large", 24)])
def test_bitmaps_random_trees(request, size, n_trees):
    c = request.getfixturevalue(size)
    rng = np.random.default_rng(100 + n_trees)
    cache, undecided, nonempty = {}, 0, 0
    for i in range(n_trees):
        where = _tree(rng)
        w = parse_where(where)
        for deletes in (False, True):
            got = _device_bits(c, w, deletes)
            undecided += _check(c, w, deletes, got=got, cache=cache, what=(i, deletes, where))
            nonempty += got is not None and bool(got.any())
    assert nonempty >= n_trees // 2
    assert undecided <= 64 * n_trees, undecided   # the band is thin: nearly every document is compared


@pytest.mark.parametrize("size", ["small", "large"])
def test_every_leaf_kind_at_scale(request, size):
    """Each leaf kind alone and under Not, with and without deletes; the number bounds at -0.0, the i32 extremes,
    integers that round to f32 and +-inf with every op."""
    c = request.getfixturevalue(size)
    rng = np.random.default_rng(7)
    cache = {}
    clauses = [_leaf(rng, k) for k in ("b", "s", "d", "g", "g", "g", "g") for _ in range(3)]
    clauses += [{"n": {op: b}} for op in ("eq", "gt", "gte", "lt", "lte")
                for b in (0, -0.0, 2**31 - 1, -2**31, 2**31, 2**31 + 1, 3000000001, 16777217, 1e39, -1e39, 2.5, 5)]
    clauses += [{"n": {"between": [5, -5]}}, {"n": {"between": [-0.0, 0]}}, {"n": {"between": [-1e39, 1e39]}},
                {"s": "ghost"}, {"s": "nobody"}, {"b": "k1"}, {"s": {"gt": 1}}, {"g": True}, {"n": _poly_json(SQUARE)}]
    for i, where in enumerate(clauses):
        w = parse_where(where)
        _check(c, w, i % 2 == 1, cache=cache, what=where)
        _check(c, parse_where({"not": where}), i % 2 == 0, cache=cache, what=("not", where))


# ---------------------------------------------------------------- leg 2: programs at the limits
def _leaf_node(c, where):
    """The one node compile_where makes of a single leaf, and the leaf as a parsed tree."""
    w = parse_where(where)
    nodes = compile_where(w, c["st"], c["geo"], c["nbits"]).nodes
    assert len(nodes) == 1, where
    return nodes[0], w


def _postfix(c, tokens, leaves):
    """A program from postfix tokens ("leaf", i) / ("and", k) / ("or", k) / ("not",) over `leaves` (_leaf_node pairs),
    and the same program as a where tree for the host evaluation."""
    nodes, stack = [], []
    for t in tokens:
        if t[0] == "leaf":
            nodes.append(leaves[t[1]][0])
            stack.append(leaves[t[1]][1])
        elif t[0] == "not":
            nodes.append((_lib.OC_WHERE_NOT, 0, 0, 0.0, 0.0, 0.0, None, None))
            stack.append(WhereFilter(not_=stack.pop()))
        else:
            k = t[1]
            args = stack[-k:]
            del stack[-k:]
            op = _lib.OC_WHERE_AND if t[0] == "and" else _lib.OC_WHERE_OR
            nodes.append((op, 0, k, 0.0, 0.0, 0.0, None, None))
            stack.append(WhereFilter(and_=args) if t[0] == "and" else WhereFilter(or_=[x for x in args]))
    assert len(stack) == 1
    return WhereProgram(c["nbits"], nodes), stack[0]


def _depth(tokens):
    sp = top = 0
    for t in tokens:
        sp += 1 if t[0] == "leaf" else 0 if t[0] == "not" else 1 - t[1]
        top = max(top, sp)
    return top


def _run_postfix(c, tokens, leaves, cache, what):
    prog, tree = _postfix(c, tokens, leaves)
    _check(c, tree, False, got=_raw(filter_from_program(c["ctx"], prog)), cache=cache, what=what)


@pytest.fixture(scope="module")
def limit_leaves(large):
    rng = np.random.default_rng(41)
    keys = ["b", "s", "n", "d", "n", "s", "d", "n"]
    ls = [_leaf_node(large, _leaf(rng, keys[i % len(keys)])) for i in range(40)]
    ls += [_leaf_node(large, {"g": _poly_json(p, inside)}) for p in (SQUARE, NOTCH, BOWTIE) for inside in (True, False)]
    return ls


# leaves each of which holds a few per cent of the documents or less: an Or of them and an And of their Nots are neither
# empty nor everything, and every operand of such a node changes its result
NARROW = ([{"s": f"k{i}"} for i in range(12)] + [{"n": {"eq": v}} for v in range(-50, 51)]
          + [{"d": {"eq": _date_str(1_600_000_000_000 + k * 86_400_000)}} for k in range(-20, 20, 2)])


@pytest.fixture(scope="module")
def narrow_leaves(large):
    return [_leaf_node(large, w) for w in NARROW]


def _spec_of(c, tokens, leaves, cache):
    """The host result (certainly in) of a postfix program; every document is decided for these leaves."""
    t, f = where_masks(_postfix(c, tokens, leaves)[1], c["F"], c["nbits"], cache=cache)
    assert (t | f).all()
    return t


def test_program_of_max_depth(large, limit_leaves, narrow_leaves):
    D = _lib.OC_WHERE_MAX_DEPTH
    cache, L, N = {}, limit_leaves, narrow_leaves
    # D leaves and one D-ary node, the stack full once: an Or of narrow leaves and an And of their Nots, each neither
    # empty nor what its first D - 1 operands give
    for op in ("and", "or"):
        leaf_toks = [[("leaf", i)] + ([("not",)] if op == "and" else []) for i in range(D)]
        toks = [t for lt in leaf_toks for t in lt] + [(op, D)]
        assert _depth(toks) == D
        _run_postfix(large, toks, N, cache, (op, D))
        full = _spec_of(large, toks, N, cache)
        assert 0 < full.sum() < NL and (full != _spec_of(large, [t for lt in leaf_toks[:-1] for t in lt] + [(op, D - 1)], N, cache)).any()
    # D leaves, then D - 1 binary nodes alternating And / Or and a Not between them
    toks = [("leaf", i) for i in range(D)]
    for k in range(D - 1):
        toks += [("and" if k % 2 else "or", 2)] + ([("not",)] if k % 3 == 0 else [])
    assert _depth(toks) == D
    _run_postfix(large, toks, L, cache, "binary")


def _max_nodes_program(rng, n_leaves):
    """Postfix tokens of exactly OC_WHERE_MAX_NODES nodes over narrow leaves, and the token count at each level's end.
    From a running value X, levels alternate X And (Or of k leaves) and X Or (And of k Nots of leaves), so X neither
    empties nor fills and every level changes it."""
    toks, ends = [("leaf", 0)], []

    def level(kind, k):
        pick = [("leaf", int(i)) for i in rng.integers(0, n_leaves, k)]
        if kind == "and":
            toks.extend(pick + [("or", k), ("and", 2)])
        else:
            toks.extend([t for p in pick for t in (p, ("not",))] + [("and", k), ("or", 2)])
        ends.append(len(toks))

    M = _lib.OC_WHERE_MAX_NODES
    i = 0
    while M - len(toks) > 64:
        level("and" if i % 2 == 0 else "or", 15)
        i += 1
    rem = M - len(toks)             # 33 .. 64: an Or level of k1 Nots and a last And level of k2 leaves fill it
    k1 = min(15, (rem - 8) // 2)
    level("or", k1)
    level("and", M - len(toks) - 2)
    assert len(toks) == M and 2 <= toks[-2][1] <= 31
    return toks, ends


def test_program_of_max_nodes(large, narrow_leaves):
    """OC_WHERE_MAX_NODES nodes, each level changing the running value: the result is neither the program's first leaf
    nor what it is halfway or before its last level, so a program cut short or a level combined wrongly fails."""
    cache, N = {}, narrow_leaves
    toks, ends = _max_nodes_program(np.random.default_rng(5), len(N))
    assert _depth(toks) <= _lib.OC_WHERE_MAX_DEPTH
    _run_postfix(large, toks, N, cache, "max nodes")
    full = _spec_of(large, toks, N, cache)
    half = min(ends, key=lambda e: abs(e - len(toks) // 2))
    assert 0 < full.sum() < NL
    for cut in (1, half, ends[-2]):
        assert (full != _spec_of(large, toks[:cut], N, cache)).any(), cut


def test_not_chain_and_repeated_leaf(large, limit_leaves):
    cache, L = {}, limit_leaves
    for n_not in (255, 256):
        _run_postfix(large, [("leaf", 3)] + [("not",)] * n_not, L, cache, ("not chain", n_not))
    # one leaf pushed many times, with other leaves between
    toks = [("leaf", 2)]
    for i in range(300):
        toks += [("leaf", 2 if i % 3 else 7), ("or" if i % 2 else "and", 2)]
    _run_postfix(large, toks, L, cache, "repeated leaf")
    toks = [("leaf", 4)] * 32 + [("or", 32), ("leaf", 4), ("and", 2)]
    _run_postfix(large, toks, L, cache, "one leaf 33 times")


def test_wide_and_or(large):
    """An And / Or of several hundred arguments, as a where clause: compile_where folds it into nodes the planner
    accepts, and the bitmap is the host's.  The Or is over narrow leaves and the And over their Nots, the last part a
    broad one: neither is empty or everything, and neither is what its first _NARY parts give."""
    rng = np.random.default_rng(9)
    cache = {}
    for op, n in (("or", 300), ("and", 300), ("or", 33), ("and", 17)):
        parts = [NARROW[int(i)] for i in rng.integers(0, len(NARROW), n - 1)] + [{"b": True}]
        if op == "and":
            parts = [{"not": p} for p in parts]
        w = parse_where({op: parts})
        t = where_masks(w, large["F"], NL, cache=cache)[0]
        head = where_masks(parse_where({op: parts[:_NARY]}), large["F"], NL, cache=cache)[0]
        assert 0 < t.sum() < NL and (t != head).any(), (op, n)
        _check(large, w, True, cache=cache, what=(op, n))
        nested = parse_where({"or": [{"and": [{op: parts[:40]}, parts[0]]}, {op: parts[40:]}]})
        _check(large, nested, False, cache=cache, what=("nested", op, n))


def test_polygon_of_max_vertices(large):
    assert len(BIG) == _lib.OC_GEO_MAX_VERTICES
    cache = {}
    for inside in (True, False):
        w = parse_where({"g": _poly_json(BIG, inside)})
        m = where_masks(w, large["F"], NL, cache=cache)[0]
        assert 100 < m.sum() < NL - 100
        _check(large, w, False, cache=cache, what=("big polygon", inside))
        _check(large, parse_where({"g": _poly_json(BIG, inside), "b": True}), True, cache=cache, what=("big polygon and", inside))


def test_radius_edges(large):
    clauses = [
        {"g": {"radius": {"coordinates": {"lat": DUP[0], "lon": DUP[1]}, "value": 0}}},                # radius 0
        {"g": {"radius": {"coordinates": {"lat": DUP[0], "lon": DUP[1]}, "value": 0, "inside": False}}},
        {"g": {"radius": {"coordinates": {"lat": DUP[0], "lon": DUP[1]}, "value": 1, "unit": "cm"}}},  # tiny
        {"g": {"radius": {"coordinates": {"lat": 0, "lon": 0}, "value": 20016, "unit": "km"}}},        # >= pi R
        {"g": {"radius": {"coordinates": {"lat": 0, "lon": 0}, "value": 20016, "unit": "km", "inside": False}}},
        {"g": {"radius": {"coordinates": {"lat": 90, "lon": 0}, "value": 1, "unit": "m"}}},           # at a pole
        {"g": {"radius": {"coordinates": {"lat": -90, "lon": 45}, "value": 2000, "unit": "km"}}},
        {"g": {"radius": {"coordinates": {"lat": 0, "lon": 180}, "value": 500, "unit": "km"}}},
    ]
    for where in clauses:
        w = parse_where(where)
        _check(large, w, False, what=where)
        _check(large, parse_where({"not": where, "b": True}), True, what=("not", where))
    t, _ = where_masks(parse_where(clauses[0]), large["F"], NL)
    assert 1 <= t.sum() <= 6   # the duplicates at the centre, and only they


# ---------------------------------------------------------------- leg 3: in-call programs == q_filters of the host bitmaps
def _decided_clause(c, rng, gen):
    """A clause (from gen(rng)) whose host evaluation decides every document: radius leaves with a point in the band
    are redrawn."""
    for _ in range(50):
        where = gen(rng)
        m = where_masks(parse_where(where), c["F"], c["nbits"])
        if m is None or (m[0] | m[1]).all():
            return where
    raise AssertionError("no decided clause in 50 draws")


def _batch(c, B, seed):
    """Per query (program or None, host bitmap or None): random trees, duplicates, unfiltered queries, single leaves,
    FILTER-only programs, and a few hundred distinct leaves; queries of even index carry the deletes."""
    rng = np.random.default_rng(seed)
    progs, bits, srcs = [], [], []
    for b in range(B):
        r = b % 8
        deletes = b % 2 == 0
        if r == 1:
            where = None
        elif r == 2:
            where = {}   # with deletes: a FILTER-only program, else unfiltered
        elif r in (3, 5):
            where = _decided_clause(c, rng, _leaf)
        elif r == 4 and b > 16:
            where, deletes = srcs[b - 16]   # a duplicate of an earlier query
        else:
            where = _decided_clause(c, rng, lambda g: _tree(g, max_depth=3))
        srcs.append((where, deletes))
        if where is None:
            progs.append(None); bits.append(None)
            continue
        w = parse_where(where)
        progs.append(compile_where(w, c["st"], c["geo"], c["nbits"], c["live"] if deletes else None))
        bits.append(where_spec(w, c["F"], c["nbits"], c["deleted"] if deletes else ()))
    return progs, bits


@pytest.fixture(scope="module")
def search_setup(small):
    c = small
    ctx = c["ctx"]
    B = 512
    progs, bits = _batch(c, B, 17)
    handles, by_key = [], {}
    for x in bits:
        if x is None:
            handles.append(None)
            continue
        k = x.tobytes()
        if k not in by_key:
            by_key[k] = ob.DeviceFilter.from_bits(ctx, x, NS)   # a plain upload: no where program involved
        handles.append(by_key[k])
    n_leaves = len({(n[0], n[1], n[2], n[3], n[4], n[5], n[6]) for p in progs if p is not None for n in p.nodes
                    if n[0] not in (_lib.OC_WHERE_AND, _lib.OC_WHERE_OR, _lib.OC_WHERE_NOT) and n[7] is None})
    assert n_leaves >= 200, n_leaves
    fst, gbs, _ = _facets(ctx, NS, 5)
    rng = np.random.default_rng(23)
    ids = np.arange(NS, dtype=np.uint64)
    sfs = [ob.SortField(ctx, NS, ids, rng.uniform(0, 1000, NS).round(2), "number"),
           ob.SortField(ctx, NS, ids, rng.integers(0, 30, NS).astype(np.float64), "number")]
    qv, _ = synth.make_vector_queries(c["rows"], B, seed=29)
    texts = synth.make_text_queries(VOCAB, B, seed=30)
    yield dict(B=B, progs=progs, bits=bits, handles=handles, fst=fst, gbs=gbs, sfs=sfs, qv=qv, texts=texts)
    for h in by_key.values():
        h.close()
    for x in list(gbs.values()) + sfs:
        x.close()
    fst.close()


def _same(a, b, what):
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), (what, i)


def _qparams(B, seed):
    rng = np.random.default_rng(seed)
    return [ob.QueryParams(mode=[MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID][b % 3], limit=int(rng.integers(1, 40)),
                           offset=int(rng.integers(0, 6)), similarity=0.0) for b in range(B)]


def _tsc(c, m):
    return ob.TokenScoreContext(c["ctx"], c["emb"] if m != MODE_FULLTEXT else None, c["strs"] if m != MODE_VECTOR else None)


@pytest.mark.parametrize("mode", list(MODES))
def test_in_call_programs_equal_host_bitmaps(small, search_setup, mode):
    c, s = small, search_setup
    m, B = MODES[mode], s["B"]
    t, q = (s["texts"] if m != MODE_VECTOR else None), (s["qv"] if m != MODE_FULLTEXT else None)
    tsc = _tsc(c, m)
    kws = [dict(mode=m, limit_hint=20, similarity=0.0)] + ([dict(mode=m, query_params=_qparams(B, 3))] if m == MODE_HYBRID else [])
    rng = np.random.default_rng(31)
    sorts_mix = [None, (s["sfs"][0], "ASC"), (s["sfs"][0], "DESC"), (s["sfs"][1], "ASC"), (s["sfs"][1], "DESC")]
    sorts = [sorts_mix[int(rng.integers(0, 5))] for _ in range(B)]
    promote = _promote(B, 37, n=NS)
    kinds = [10, 20, None, 1, 1000, 10]
    groups = [None if kinds[b % 6] is None else (s["gbs"][kinds[b % 6]], [1, 3, 10, 0][b % 4], sorts[b]) for b in range(B)]
    facets = [{"cat": {}, "num": {"ranges": [{"from": 0, "to": 300}]}} if b % 2 else None for b in range(B)]
    for kw in kws:
        pw = ob.TokenScoreParams(where_programs=s["progs"], **kw)
        pf = ob.TokenScoreParams(device_filters=s["handles"], **kw)
        got = tsc.execute_batch_arrays(pw, t, q)
        _same(got, tsc.execute_batch_arrays(pf, t, q), "oc_search")
        assert int((got[3] > 0).sum()) > B // 4   # the filters leave hits to compare
        _same(ob.search_q_sorted_arrays(tsc, pw, sorts, promote, t, q), ob.search_q_sorted_arrays(tsc, pf, sorts, promote, t, q),
              "oc_search_q_sorted")
        _same(ob.search_q_groups_arrays(tsc, pw, groups, promote, t, q), ob.search_q_groups_arrays(tsc, pf, groups, promote, t, q),
              "oc_search_q_groups")
        a = ob.search_q_facets_arrays(tsc, s["fst"], pw, facets, groups, promote, t, q)
        f = ob.search_q_facets_arrays(tsc, s["fst"], pf, facets, groups, promote, t, q)
        _same(a[:13], f[:13], "oc_search_q_facets")


# ---------------------------------------------------------------- leg 4: the plain search against the oracle
def test_in_call_programs_against_the_oracle(small, search_setup, orc):
    c, s = small, search_setup
    B = 192
    entries = _qparams(B, 43)
    tsc = _tsc(c, MODE_HYBRID)
    texts = synth.make_text_queries(VOCAB, B, seed=30)
    got = tsc.execute_batch_arrays(ob.TokenScoreParams(mode=MODE_HYBRID, query_params=entries, where_programs=s["progs"][:B]),
                                   texts, s["qv"][:B])
    sb = orc.SearchBatch(orc.StrIndex(c["data"]), orc.EmbStore(c["rows"]))
    for b, e in enumerate(entries):
        fb = s["bits"][b]
        kw = {} if fb is None else dict(filter_bits=fb, filter_nbits=NS)
        sb.add(e.mode, limit=e.limit, offset=e.offset, similarity=e.similarity, q_vec=s["qv"][b], text=texts[b], **kw)
    od, os_, on, oc = sb.run(4)
    for b in range(B):
        assert int(got[3][b]) == int(oc[b]), b
        n = int(got[2][b])
        assert_topk_equal(got[0][b, :n], got[1][b, :n], od[b, :on[b]], os_[b, :on[b]])


# ---------------------------------------------------------------- leg 5: IndexLoader and the batcher
def _loader_ops(rng, d0, n):
    ops = []
    for d in range(d0, d0 + n):
        toks = [f"w{int(t)}" for t in rng.integers(0, 50, int(rng.integers(2, 6)))]
        terms = {}
        for i, t in enumerate(toks):
            terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
        x = [int(rng.integers(-50, 51)) for _ in range(int(rng.integers(1, 3)))]
        vals = [{"type": "ScoreString2", "field": "text", "field_length": len(toks), "terms": terms},
                {"type": "FilterBool2", "field": "b", "value": {"Array": [bool(v) for v in rng.random(int(rng.integers(1, 3))) < 0.5]}},
                {"type": "FilterNumber2", "field": "n", "value": {"I64": {"Array": x}}},
                {"type": "FilterString2", "field": "s", "value": {"Plain": f"k{int(rng.integers(0, 12))}"}},
                {"type": "FilterDate2", "field": "d",
                 "value": {"Plain": 1_600_000_000_000 + int(rng.integers(-400, 400)) * 86_400_000}},
                {"type": "FilterGeoPoint2", "field": "g", "value": {"Array": [
                    {"lat": float(rng.uniform(-60, 60)), "lon": float(rng.uniform(-180, 180))} for _ in range(int(rng.integers(1, 3)))]}}]
        if d % 7 == 0:
            vals[2] = {"type": "FilterNumber2", "field": "n", "value": {"F64": {"Plain": float(rng.choice([-0.0, 0.0, 2.5, -2.5]))}}}
        ops.append({"type": "Index", "doc_id": d, "indexed_values": vals})
    return ops


def test_loader_where_program(gpu_ctx):
    rng = np.random.default_rng(61)
    kw = dict(bool_fields=["b"], number_fields=["n"], string_filter_fields=["s"], date_fields=["d"], geopoint_fields=["g"])
    ld, model = IndexLoader(gpu_ctx, ["text"], **kw), IndexModel(["text"], **kw)
    try:
        def feed(ops):
            for op in ops:
                ld.apply(op)
                model.apply(op)

        def check(tag):
            fields = from_host_fields(model.filter_values())
            assert ld.nbits == model.nbits
            for i in range(40):
                where = _tree(rng, max_depth=3) if i else {}
                while "'zz'" in repr(where):   # the loader refuses a key that is not a filter field
                    where = _tree(rng, max_depth=3)
                prog = ld.where_program(where)
                w = parse_where(where)
                m = where_masks(w, fields, model.nbits, sorted(model.uncommitted_deleted))
                assert (prog is None) == (m is None), (tag, where)
                if prog is not None:
                    c = dict(nbits=model.nbits, F=fields, deleted=sorted(model.uncommitted_deleted))
                    _check(c, w, bool(model.uncommitted_deleted), got=_raw(filter_from_program(gpu_ctx, prog)), what=(tag, i, where))
        feed(_loader_ops(rng, 0, 3000))
        ld.commit(); model.commit()
        check("committed")
        dele = {"type": "DeleteDocuments", "doc_ids": rng.choice(3000, 120, replace=False).tolist()}
        feed([dele] + _loader_ops(rng, 3000, 500))
        ld.refresh_facets(); model.refresh_facets()
        check("uncommitted deletes")
        ld.commit(); model.commit()
        check("after commit")
    finally:
        ld.close()


def test_batcher_equals_one_at_a_time(small, search_setup):
    c, s = small, search_setup
    tsc = _tsc(c, MODE_HYBRID)
    Q = 64
    modes = [MODE_FULLTEXT, MODE_VECTOR, MODE_HYBRID]
    kws = [dict(mode=modes[i % 3], limit_hint=5 + i % 9, similarity=0.0) for i in range(Q)]
    args = [(s["texts"][i] if kws[i]["mode"] != MODE_VECTOR else None, s["qv"][i] if kws[i]["mode"] != MODE_FULLTEXT else None)
            for i in range(Q)]
    expect = []
    for i in range(Q):
        t, q = args[i]
        one = tsc.execute_batch_arrays(ob.TokenScoreParams(where_programs=[s["progs"][i]], **kws[i]),
                                       None if t is None else [t], None if q is None else q[None])
        expect.append(one)
    sb = ob.SearchBatcher(tsc, max_batch=64, max_wait_us=20000, mixed=True)
    got = [None] * Q
    bar = threading.Barrier(Q)

    def run(i):
        bar.wait()
        got[i] = sb.search(ob.TokenScoreParams(where_programs=[s["progs"][i]], **kws[i]), *args[i])
    ts = [threading.Thread(target=run, args=(i,)) for i in range(Q)]
    for x in ts:
        x.start()
    for x in ts:
        x.join()
    st = sb.stats()
    sb.close()
    for i in range(Q):
        d, sc, n, cnt = expect[i]
        k = int(n[0])
        assert got[i].doc_ids.tobytes() == d[0, :k].tobytes() and got[i].scores.tobytes() == sc[0, :k].tobytes(), i
        assert got[i].count == int(cnt[0]), i
    assert st["direct"] == 0 and st["batches"] < Q, st
