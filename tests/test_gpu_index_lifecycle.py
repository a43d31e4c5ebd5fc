"""Long random write streams through IndexLoader (strings, embeddings and every filter kind changing together, with
commits in between), every search compared with the oracle run over tests/index_model.py's plain model of the index.

Each round applies one stretch of the stream and checks three states: (a) before any commit (pending strings
invisible, deletes and N live), (b) after refresh_facets() alone, (c) after commit() (string commit, embedding
compaction, filter commit).  At each: fulltext queries resolved by the loader (exact, prefix, tolerance 1 / 2,
properties, boosts, thresholds) bit for bit at several pages; vector and hybrid queries at the K2 and K1 depths; random
where trees through where_filter and where_program; and, in fulltext mode bit for bit and in hybrid mode within ATOL,
facets, groups, sortBy and pins against their restatements over the oracle's score map."""
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import oramacore_b200 as ob
from index_model import IndexModel
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from oramacore_b200.where import parse_where
from helpers import assert_topk_equal
from test_gpu_facets import _oracle_counts
from test_gpu_groups import _check_groups, _oracle_groups
from test_gpu_parity import ATOL
from test_gpu_pins import _compare, _expect_flat
from test_gpu_sort import check as check_sorted
from test_gpu_sort import expect_flat, ranks
from test_gpu_topn_paths import _eq, _sorted, page
from test_where_host import host_where

pytestmark = pytest.mark.gpu

STRING_FIELDS = ["title", "body"]
FILTERS = dict(bool_fields=["flag"], number_fields=["price"], string_filter_fields=["cat"], date_fields=["when"],
               geopoint_fields=["loc"])
KEYS = [f"k{i}" for i in range(7)]
FT_PAGES = [(1, 0), (10, 0), (10, 23), (300, 0)]
VEC_LIMITS = [10, 128, 129, 300]          # K2 (<= 128) and K1 depths
SIMS = [0.0, 0.3]
TILE = 8192                               # BM25 tile rows
RANGES = [(-50, 0), (0, 20.5), (20.5, 1e9)]


def _words(n, seed):
    rng = np.random.default_rng(seed)
    out, seen = [], set()
    while len(out) < n:
        w = "".join(chr(97 + int(c)) for c in rng.integers(0, 26, int(rng.integers(4, 9))))
        if w not in seen:
            seen.add(w)
            out.append(w)
    return out


class Stream:
    """The op-stream generator: Index ops over two string fields with a Zipf vocabulary (hot terms take the dense
    form), documents without strings, IndexEmbedding ops of 0-3 chunks (some a round late, some exact duplicates of
    another document's), gaps in the doc ids, updates (delete + new id), plain deletes (unknown and repeated ids
    included) and filter values of every kind (bool, number with +-0.0, string_filter, date, geopoint)."""

    def __init__(self, seed, dim, vocab):
        self.rng = np.random.default_rng(seed)
        self.dim = dim
        self.words = _words(vocab, seed + 1)
        p = 1.0 / np.arange(1, vocab + 1) ** 1.05
        self.p = p / p.sum()
        self.perm = [self.rng.permutation(vocab), self.rng.permutation(vocab)]
        self.next_id = 0
        self.live, self.dead, self.gaps = [], [], []
        self.late = []                          # (doc, chunks) carried to the next round
        self.vectors = []                       # every chunk inserted so far (duplicates are drawn from it)

    def _field(self, fi, lo, hi):
        rng = self.rng
        n = int(rng.integers(lo, hi + 1))
        toks = [self.words[int(self.perm[fi][k])] for k in rng.choice(len(self.words), n, p=self.p)]
        terms = {}
        for i, t in enumerate(toks):
            e = terms.setdefault(t, {"exact_positions": [], "positions": []})
            (e["positions"] if rng.random() < 0.1 else e["exact_positions"]).append(i)
        return {"type": "ScoreString2", "field": STRING_FIELDS[fi], "field_length": n, "terms": terms}

    def _filters(self):
        rng, vals = self.rng, []
        r = rng.random
        if r() < 0.85:
            vals.append({"type": "FilterBool", "field": "flag", "value": bool(r() < 0.4)} if r() < 0.7 else
                        {"type": "FilterBool2", "field": "flag", "value": {"Array": [True, False]} if r() < 0.3 else {"Plain": bool(r() < 0.5)}})
        if r() < 0.85:
            x = float(rng.choice([0.0, -0.0, float(rng.integers(-30, 60)), round(float(rng.normal(20, 30)), 2)]))
            vals.append({"type": "FilterNumber", "field": "price", "value": x} if r() < 0.7 else
                        {"type": "FilterNumber2", "field": "price", "value": {"F64": {"Array": [x, -x]}} if r() < 0.5 else
                         {"I64": {"Plain": int(rng.integers(-40, 80))}}})
        if r() < 0.8:
            vals.append({"type": "FilterString", "field": "cat", "value": KEYS[int(rng.integers(0, 6))]} if r() < 0.7 else
                        {"type": "FilterString2", "field": "cat", "value": {"Array": [KEYS[int(k)] for k in rng.integers(0, 7, 2)]}})
        if r() < 0.8:
            ms = int(rng.integers(-10**11, 2 * 10**12))
            vals.append({"type": "FilterDate", "field": "when", "value": ms} if r() < 0.7 else
                        {"type": "FilterDate2", "field": "when", "value": {"Array": [ms, ms + int(rng.integers(0, 10**9))]}})
        if r() < 0.8:
            pt = lambda: {"lat": float(rng.uniform(-60, 60)), "lon": float(rng.uniform(-120, 120))}  # noqa: E731
            vals.append({"type": "FilterGeoPoint2", "field": "loc", "value": {"Plain": pt()} if r() < 0.7 else {"Array": [pt(), pt()]}})
        return vals

    def _chunks(self):
        rng = self.rng
        n = int(rng.choice(4, p=[0.1, 0.35, 0.3, 0.25]))
        out = []
        for _ in range(n):
            if self.vectors and rng.random() < 0.04:
                v = self.vectors[int(rng.integers(0, len(self.vectors)))]        # an exact duplicate: a tie
            else:
                v = rng.standard_normal(self.dim).astype(np.float32)
            self.vectors.append(v)
            out.append(v)
        return out

    def _new_doc(self, emb):
        rng = self.rng
        if rng.random() < 0.05:                                                  # a gap in the doc ids
            g = int(rng.integers(1, 4))
            self.gaps += range(self.next_id, self.next_id + g)
            self.next_id += g
        d = self.next_id
        self.next_id += 1
        vals = []
        if rng.random() < 0.92:
            if rng.random() < 0.85:
                vals.append(self._field(0, 1, 6))
            if rng.random() < 0.8:
                vals.append(self._field(1, 4, 40))
            if rng.random() < 0.02:
                vals.append({"type": "ScoreString2", "field": "body", "field_length": 0, "terms": {}})
        vals += self._filters()
        self.live.append(d)
        if rng.random() < 0.95:
            (self.late if rng.random() < 0.1 else emb).append((d, self._chunks()))
        return {"type": "Index", "doc_id": d, "indexed_values": vals}

    def _take_live(self):
        i = int(self.rng.integers(0, len(self.live)))
        self.live[i], self.live[-1] = self.live[-1], self.live[i]
        d = self.live.pop()
        self.dead.append(d)
        return d

    def round(self, n_new):
        rng = self.rng
        ops, emb = [], list(self.late)
        self.late = []

        def flush():
            nonlocal emb
            dead = set(self.dead)
            data = [(d, c) for d, c in emb if d not in dead]
            if data:
                ops.append({"type": "IndexEmbedding", "data": data})
            emb = []
        made = 0
        while made < n_new:
            r = rng.random()
            if r < 0.06 and len(self.live) > 10:                                 # update: delete + a new id
                ops.append({"type": "DeleteDocuments", "doc_ids": [self._take_live()]})
                ops.append(self._new_doc(emb))
                made += 1
            elif r < 0.1 and len(self.live) > 10:                                # plain delete
                ids = [self._take_live() for _ in range(int(rng.integers(1, 3)))]
                if rng.random() < 0.3 and self.gaps:
                    ids.append(int(rng.choice(self.gaps)))                         # never indexed
                if rng.random() < 0.3:
                    ids.append(int(rng.choice(self.dead)))                         # deleted already, or twice in one op
                ops.append({"type": "DeleteDocuments", "doc_ids": ids})
            elif r < 0.13:
                flush()
            else:
                ops.append(self._new_doc(emb))
                made += 1
        flush()
        return ops

    def texts(self, n):
        """Query strings of 1-3 words: vocabulary words, prefixes, one-letter typos, an unknown word."""
        rng, out = self.rng, []
        for _ in range(n):
            ws = []
            for _ in range(int(rng.integers(1, 4))):
                w = self.words[int(rng.choice(len(self.words), p=self.p))]
                r = rng.random()
                if r < 0.2 and len(w) > 4:
                    w = w[:len(w) - 2]
                elif r < 0.4:
                    i = int(rng.integers(0, len(w)))
                    w = w[:i] + chr(97 + int(rng.integers(0, 26))) + w[i + 1:]
                elif r < 0.45:
                    w = "zzzzq"
                ws.append(w)
            out.append(" ".join(ws))
        return out

    def qvecs(self, n):
        """Half near an inserted chunk, half random."""
        rng = self.rng
        q = rng.standard_normal((n, self.dim)).astype(np.float32)
        for i in range(0, n, 2):
            if self.vectors:
                q[i] = self.vectors[int(rng.integers(0, len(self.vectors)))] + 0.3 * q[i]
        return q


# ---------------------------------------------------------------- the oracle over the model
class Expect:
    """One checkpoint's oracle inputs: the model's committed strings with the live N, the filter its tombstones
    apply, and its live embedding rows."""

    def __init__(self, orc, model):
        self.orc, self.m = orc, model
        self.ix = orc.StrIndex(model.string_index())
        live = model.live_rows()
        self.nbits_rows = int(model.rows()[-1]) + 1 if model.rows().size else 1
        self.alive = None if live is None else orc.make_filter_bits(live.tolist(), self.nbits_rows)
        self.st = model.emb_store(orc)
        self.pool = ThreadPoolExecutor(8)

    def ft(self, q, threshold=None, where=None):
        if where is not None:
            return self.orc.fulltext(self.ix, q, threshold=threshold, filter_bits=where[0], filter_nbits=where[1])
        if self.alive is not None:
            return self.orc.fulltext(self.ix, q, threshold=threshold, filter_bits=self.alive, filter_nbits=self.nbits_rows)
        return self.orc.fulltext(self.ix, q, threshold=threshold)

    def vec(self, qv, limit, sim, where=None):
        if where is not None:
            return self.orc.vector(self.st, qv, limit, sim, where[0], where[1])
        return self.orc.vector(self.st, qv, limit, sim)

    def hybrid(self, q, qv, limit, sim, where=None):
        return self.orc.hybrid_combine(self.vec(qv, limit, sim, where), self.ft(q, where=where))

    def map(self, fn, items):
        return list(self.pool.map(lambda a: fn(*a), items))

    def close(self):
        self.pool.shutdown()


def _as_dict(m):
    return dict(zip(m[0].tolist(), m[1].tolist()))


def _resolve(ld, rng, texts):
    """Each query with its own exact, tolerance, properties and boost."""
    B = len(texts)
    exact = [bool(rng.random() < 0.2) for _ in range(B)]
    tol = [None if e else [None, None, 1, 2][int(rng.integers(0, 4))] for e in exact]
    props = [[0, 1] if rng.random() < 0.6 else [int(rng.integers(0, 2))] for _ in range(B)]
    boost = [[1.0, 1.0] if rng.random() < 0.5 else [float(rng.choice([0.5, 2.0, 3.0])), float(rng.choice([1.0, 0.25]))]
             for _ in range(B)]
    return ld.resolve(texts, exact=exact, tolerance=tol, properties=props, boost=boost)


# ---------------------------------------------------------------- checks of one state
def check_fulltext(tag, ld, ex, batch, thresholds):
    tsc = ld.context()
    B = batch.n_queries
    qs = [batch.query(i) for i in range(B)]
    refs = ex.map(lambda q, t: _sorted(*ex.ft(q, threshold=t)), list(zip(qs, thresholds)))
    for limit, offset in FT_PAGES:
        qp = [ob.QueryParams(MODE_FULLTEXT, limit, offset, 0.0, thresholds[i]) for i in range(B)]
        hits = tsc.execute_batch(ob.TokenScoreParams(mode=MODE_FULLTEXT, query_params=qp), batch)
        for i, h in enumerate(hits):
            _eq(h, page(refs[i], limit, offset), (tag, "fulltext", i, qs[i].term_id[:8], thresholds[i], limit, offset))
    small = ob.engine.TextQueryBatch(qs[:3])                                     # B < 8
    for i, h in enumerate(tsc.execute_batch(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10), small)):
        _eq(h, page(_sorted(*ex.ft(qs[i])), 10, 0), (tag, "fulltext B=3", i))
    return qs


def check_vector_hybrid(tag, ld, ex, qs, qv):
    tsc = ld.context()
    B = qv.shape[0]
    tq = ob.engine.TextQueryBatch(qs[:B])
    for limit in VEC_LIMITS:
        for sim in SIMS:
            vmaps = ex.map(lambda i: ex.vec(qv[i], limit, sim), [(i,) for i in range(B)])
            hmaps = ex.map(lambda i: ex.orc.hybrid_combine(vmaps[i], ex.ft(qs[i])), [(i,) for i in range(B)])
            for mode, maps in ((MODE_VECTOR, vmaps), (MODE_HYBRID, hmaps)):
                hits = tsc.execute_batch(ob.TokenScoreParams(mode=mode, limit_hint=limit, similarity=sim),
                                         None if mode == MODE_VECTOR else tq, qv)
                for i, h in enumerate(hits):
                    d, s, count = page(_sorted(*maps[i]), limit, 0)
                    ctx = (tag, "vector" if mode == MODE_VECTOR else "hybrid", i, limit, sim)
                    assert h.count == count, (ctx, h.count, count)
                    assert_topk_equal(h.doc_ids, h.scores, d, s, atol=ATOL)


def _leaf(rng, key):
    ops = ["eq", "gt", "gte", "lt", "lte", "between"]
    op = ops[int(rng.integers(0, 6))]
    if key == "flag":
        return bool(rng.random() < 0.5)
    if key == "cat":
        return KEYS[int(rng.integers(0, len(KEYS)))] if rng.random() < 0.9 else "k99"
    if key == "price":
        b = lambda: float(rng.choice([0.0, -0.0, float(rng.integers(-30, 60)), 20.5]))  # noqa: E731
        return {op: [b(), b()] if op == "between" else b()}
    if key == "when":
        import datetime
        ms = lambda: int(rng.integers(-10**11, 2 * 10**12))  # noqa: E731
        s = lambda x: (datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc) +  # noqa: E731
                       datetime.timedelta(milliseconds=x)).strftime("%Y-%m-%dT%H:%M:%S.%f")[:-3] + "Z"
        return {op: [s(ms()), s(ms())] if op == "between" else s(ms())}
    c = rng.uniform(-40, 40, 2)
    a = np.linspace(0, 2 * np.pi, int(rng.integers(3, 8)), endpoint=False)
    rr = rng.uniform(10, 45)
    return {"polygon": {"coordinates": [{"lat": float(c[0] + rr * np.sin(t)), "lon": float(c[1] + rr * np.cos(t))} for t in a],
                        "inside": bool(rng.random() < 0.7)}}


def _tree(rng, depth=1):
    w = {}
    for key in rng.choice(["flag", "price", "cat", "when", "loc"], int(rng.integers(1, 3)), replace=False):
        w[str(key)] = _leaf(rng, str(key))
    if depth < 3 and rng.random() < 0.4:
        w["not"] = _tree(rng, depth + 1)
    if depth < 3 and rng.random() < 0.3:
        w["or"] = [_tree(rng, depth + 1) for _ in range(2)]
    return w


def check_where(tag, ld, ex, model, rng, qs, qv):
    tsc = ld.context()
    B = qv.shape[0]
    tq = ob.engine.TextQueryBatch(qs[:B])
    for k in range(4):
        where = _tree(rng)
        allowed = host_where(parse_where(where), model.filter_values(), model.nbits, model.uncommitted_deleted)
        wb = None if allowed is None else (ex.orc.make_filter_bits(sorted(allowed), model.nbits), model.nbits)
        f, prog = ld.where_filter(where), ld.where_program(where)
        try:
            for mode in (MODE_FULLTEXT, MODE_HYBRID):
                maps = ex.map(lambda i: ex.ft(qs[i], where=wb) if mode == MODE_FULLTEXT else ex.hybrid(qs[i], qv[i], 10, 0.0, wb),
                              [(i,) for i in range(B)])
                p = dict(mode=mode, limit_hint=10, similarity=0.0)
                a = tsc.execute_batch(ob.TokenScoreParams(device_filter=f, **p), tq, qv)
                b = tsc.execute_batch(ob.TokenScoreParams(where_programs=[prog] * B, **p), tq, qv)
                for i in range(B):
                    ctx = (tag, "where", k, where, "fulltext" if mode == MODE_FULLTEXT else "hybrid", i)
                    assert a[i].count == b[i].count and np.array_equal(a[i].doc_ids, b[i].doc_ids) \
                        and np.array_equal(a[i].scores, b[i].scores), ctx
                    d, s, count = page(_sorted(*maps[i]), 10, 0)
                    if mode == MODE_FULLTEXT:
                        _eq(a[i], (d, s, count), ctx)
                    else:
                        assert a[i].count == count, ctx
                        assert_topk_equal(a[i].doc_ids, a[i].scores, d, s, atol=ATOL)
        finally:
            if f is not None:
                f.close()


def _facet_variants(model):
    """Each facet value's documents, once per matching entry: bools are a set per document (FilterBool2 inserts are
    unique), while a string_filter key or a number listed twice for a document is listed twice and counts twice
    (filter_commit_spec.py's append rule, as test_gpu_facets._oracle_counts counts)."""
    fv = model.filter_values()
    flag, cat = fv["flag"][1], fv["cat"][1]
    pd, pv = fv["price"][1]
    return {
        "flag": {"true": [d for d, bs in flag.items() if True in bs], "false": [d for d, bs in flag.items() if False in bs]},
        "cat": {k: [d for d, ks in cat.items() for x in ks if x == k] for k in KEYS},
        "price": {f"{ob.engine._number_label(a)}-{ob.engine._number_label(b)}": pd[(pv >= a) & (pv <= b)].tolist()
                  for a, b in RANGES},
    }


def _members(model, gb):
    fv = model.filter_values()
    flag, cat = fv["flag"][1], fv["cat"][1]
    out = []
    for fl, k in gb.values:
        out.append(((fl, k), {d for d, bs in flag.items() if fl in bs} & {d for d, ks in cat.items() if k in ks}))
    return out


def _promote(rng, sm, model, stream, B):
    pending = [d for op in model.pending if op[0] == "insert" for d in [op[2]]]
    pools = [list(sm)[:20], stream.dead[-50:], pending[-50:], stream.gaps[-5:] + [10**9 + 7]]
    out = []
    for _ in range(B):
        items = []
        for pool in pools:
            if pool:
                d = int(pool[int(rng.integers(0, len(pool)))])
                if d not in [x for x, _ in items]:
                    items.append((d, int(rng.choice([0, 1, 3, 9, 40]))))
        out.append(items)
    return out


def check_derived(tag, ld, ex, model, stream, rng, qs, qv, mode):
    """Facets, groups, sortBy and pins over the score map: exact in fulltext mode; in hybrid mode doc sets exact and
    scores within ATOL, on the queries whose fp64 cosine gap at the vector depth (10) exceeds 1e-4.  Returns the
    number of hybrid queries that passed that guard."""
    tsc = ld.context()
    B = qv.shape[0]
    tq = ob.engine.TextQueryBatch(qs[:B])
    exact = mode == MODE_FULLTEXT
    if exact:
        keep = list(range(B))
        maps = ex.map(lambda i: ex.ft(qs[i]), [(i,) for i in range(B)])
    else:
        keep = []
        for i in range(B):
            d, c = ex.orc.vector_f64(ex.st, qv[i], 11)
            if c.shape[0] < 11 or c[9] - c[10] > 1e-4:
                keep.append(i)
        maps = ex.map(lambda i: ex.hybrid(qs[i], qv[i], 10, 0.0), [(i,) for i in range(B)])
    sms = [_as_dict(m) for m in maps]
    p = ob.TokenScoreParams(mode=mode, limit_hint=10, similarity=0.0)
    vin = None if mode == MODE_FULLTEXT else qv
    # facets
    variants = _facet_variants(model)
    req = {"flag": {"true": True, "false": True}, "cat": {}, "price": {"ranges": [{"from": a, "to": b} for a, b in RANGES]}}
    got = ob.search_facets(tsc, ld.facets, p, req, texts=tq, q_vecs=vin)
    for i in keep:
        for name in req:
            exp = _oracle_counts(sms[i].keys(), variants[name])
            g = got[i][name]["values"]
            for label in set(exp) | set(g):
                assert g.get(label, 0) == exp.get(label, 0), (tag, "facets", mode, i, name, label, g, exp)
    # groups: flag x cat, 3 per group
    gb = ob.GroupBy(ld.facets, ["flag", "cat"])
    try:
        res = ob.search_groups(tsc, gb, p, max_results=3, texts=tq, q_vecs=vin)
        members = _members(model, gb)
        for i in keep:
            exp = _oracle_groups(maps[i], members, 3)
            try:
                _check_groups(res[i][1], exp, exact)
            except AssertionError as e:
                raise AssertionError((tag, "groups", mode, i)) from e
    finally:
        gb.close()
    # sortBy: number ASC / DESC, date
    for field, kind, order in (("price", "number", "ASC"), ("price", "number", "DESC"), ("when", "date", "ASC")):
        docs, vals = model.sort_values(field)
        sf = ob.SortField(ld.ctx, model.nbits, docs, vals, kind)
        try:
            sd, ss, sv, sn, sc, _, _ = ob.engine.search_sorted_arrays(tsc, p, sf, order, texts=tq, q_vecs=vin)
            rk = ranks(docs, vals, order)
            for i in keep:
                try:
                    check_sorted(sd[i, :sn[i]], ss[i, :sn[i]], sv[i, :sn[i]], expect_flat(sms[i], rk, 10, 0), exact)
                except AssertionError as e:
                    raise AssertionError((tag, "sortBy", field, order, mode, i)) from e
                assert int(sc[i]) == len(sms[i]), (tag, "sortBy count", mode, i)
        finally:
            sf.close()
    # pins: a ranked document, a deleted one, a pending one and an unknown id
    promote = _promote(rng, sms[0], model, stream, B)
    hits = ob.search_pinned(tsc, p, promote, texts=tq, q_vecs=vin)
    for i in keep:
        try:
            _compare(hits[i].doc_ids, hits[i].scores, _expect_flat(sms[i], promote[i], 10, 0), promote[i], exact)
        except AssertionError as e:
            raise AssertionError((tag, "pins", mode, i, promote[i])) from e
    return len(keep)


def check_state(tag, ld, model, stream, orc, rng):
    ex = Expect(orc, model)
    try:
        texts = stream.texts(12)
        batch = _resolve(ld, rng, texts)
        thresholds = [None if rng.random() < 0.6 else float(rng.choice([0.5, 1.0])) for _ in range(12)]
        qs = check_fulltext(tag, ld, ex, batch, thresholds)
        assert ld.document_count == model.document_count, (tag, ld.document_count, model.document_count)
        qv = stream.qvecs(8)
        check_vector_hybrid(tag, ld, ex, qs, qv)
        check_where(tag, ld, ex, model, rng, qs, qv)
        check_derived(tag, ld, ex, model, stream, rng, qs, qv, MODE_FULLTEXT)
        return check_derived(tag, ld, ex, model, stream, rng, qs, qv, MODE_HYBRID)
    finally:
        ex.close()


# first: the stretch committed before the first checkpoint, so that round 0's state (a) already scores committed rows
SIZES = {"small": dict(seed=3, dim=100, vocab=600, first=600, rounds=[400] * 6),
         "large": dict(seed=4, dim=384, vocab=4000, first=40000, rounds=[9000, 7000, 6000])}


@pytest.mark.parametrize("size", list(SIZES))
def test_op_streams_against_the_model(gpu_ctx, orc, size):
    cfg = SIZES[size]
    stream = Stream(cfg["seed"], cfg["dim"], cfg["vocab"])
    ld = IndexLoader(gpu_ctx, STRING_FIELDS, embedding_dim=cfg["dim"], **FILTERS)
    model = IndexModel(STRING_FIELDS, dim=cfg["dim"], **FILTERS)
    rng = np.random.default_rng(cfg["seed"] + 100)
    guarded = total = 0
    try:
        for op in stream.round(cfg["first"]):
            ld.apply(op)
            model.apply(op)
        ld.commit()
        model.commit()
        for r, n_new in enumerate(cfg["rounds"]):
            for op in stream.round(n_new):
                ld.apply(op)
                model.apply(op)
            guarded += check_state(f"{size} round {r} (a) before commit", ld, model, stream, orc, rng)
            ld.refresh_facets()
            model.refresh_facets()
            guarded += check_state(f"{size} round {r} (b) after refresh_facets", ld, model, stream, orc, rng)
            ld.commit()
            model.commit()
            guarded += check_state(f"{size} round {r} (c) after commit", ld, model, stream, orc, rng)
            total += 3 * 8
            # the dictionary hands out term ids in first-seen order, as the model assumes
            for fi in range(2):
                assert ld.dict.size(fi) == len(model.term_ids[fi])
            if size == "large":
                assert model.rows().shape[0] > TILE and ld.emb.info()["num_rows"] > TILE
        assert guarded >= 0.75 * total, (guarded, total)
    finally:
        ld.close()


def test_document_count_set_during_a_commit_is_kept(gpu_ctx, orc):
    """Index / DeleteDocuments ops applied while the string store's commit runs push their N (oc_str_set_global); the
    snapshot the commit publishes must carry the latest one, not the one it started from."""
    stream = Stream(9, 16, 3000)
    ld = IndexLoader(gpu_ctx, STRING_FIELDS)
    strip = lambda op: {**op, "indexed_values": [v for v in op["indexed_values"] if v["type"] == "ScoreString2"]} \
        if op["type"] == "Index" else op  # noqa: E731
    ops = [strip(op) for op in stream.round(60000) if op["type"] != "IndexEmbedding"]
    for op in ops:
        ld.apply(op)
    late = [strip(op) for op in stream.round(300) if op["type"] != "IndexEmbedding"]
    th = threading.Thread(target=ld.strs.commit)
    th.start()
    for op in late:
        ld.apply(op)
    overlapped = th.is_alive()
    th.join()
    assert ld.strs.read_rows()["document_count"] == ld.document_count, overlapped
    # and searches score with it: the oracle over the committed snapshot read back, with the live N
    rows = ld.strs.read_rows()
    fields = [ob.FieldPostings(float(f["avg_field_len"]), f["term_offsets"], f["post_row"], f["post_tf"], f["post_len"])
              for f in (ld.strs.read_field(i) for i in range(2))]
    ix = orc.StrIndex(ob.StringIndexData(fields, rows["row_doc_ids"].shape[0], ld.document_count, rows["row_doc_ids"]))
    dead = np.isin(rows["row_doc_ids"], np.asarray([int(d) for op in late if op["type"] == "DeleteDocuments" for d in op["doc_ids"]], np.uint64))
    alive = orc.make_filter_bits(rows["row_doc_ids"][~dead].tolist(), int(rows["row_doc_ids"][-1]) + 1)
    batch = ld.resolve(stream.texts(8))
    hits = ld.context().execute_batch(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10), batch)
    for i, h in enumerate(hits):
        ref = _sorted(*orc.fulltext(ix, batch.query(i), filter_bits=alive, filter_nbits=int(rows["row_doc_ids"][-1]) + 1))
        _eq(h, page(ref, 10, 0), ("during commit", i))
    ld.close()
