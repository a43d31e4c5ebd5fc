"""oc_dict_resolve_q without a ctx: every query of a batch with its own exact / tolerance / boost / properties, byte
for byte against the same query alone through oc_dict_resolve and against hostindex.resolve.  Host only."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib
from oramacore_b200.hostindex import HostStringIndex

FIELDS = ("title", "body")


def _index(docs):
    h = HostStringIndex(FIELDS)
    for d, doc in docs:
        h.insert(d, doc)
    h.commit()
    d = ob.TermDictionary(len(FIELDS))
    for fi in range(len(FIELDS)):
        d.add_terms(fi, h.terms[fi])
    return h, d


def _same(a, b):
    for x, y in ((a.token_term_offsets, b.token_term_offsets), (a.term_field, b.term_field), (a.term_id, b.term_id)):
        assert np.array_equal(x, y), (x, y)
    assert a.term_weight.view(np.uint32).tolist() == b.term_weight.view(np.uint32).tolist()


def _random_case(seed, n_words=2500, n_docs=300):
    rng = np.random.default_rng(seed)
    words = sorted({"".join(rng.choice(list("abcdef"), size=int(rng.integers(1, 8)))) for _ in range(n_words)})
    docs = [(i, {"title": " ".join(rng.choice(words, size=3)), "body": " ".join(rng.choice(words, size=8))}) for i in range(n_docs)]
    h, d = _index(docs)
    texts = [" ".join(rng.choice(words, size=int(rng.integers(1, 4)))) for _ in range(48)] + ["", "a", "zz", "abcdefabcdef", "  "]
    return rng, h, d, texts


def _options(rng, B):
    """per query: (exact, tolerance, boost per field or None, properties or None)"""
    out = []
    for _ in range(B):
        exact = bool(rng.random() < 0.2)
        tol = [None, 0, 1, 2, 8][int(rng.integers(0, 5))]
        boost = None if rng.random() < 0.5 else [float(rng.choice([0.5, 1.0, 2.5])), float(rng.choice([1.0, 3.0]))]
        props = [None, [0], [1], [0, 1]][int(rng.integers(0, 4))]
        out.append((exact, tol, boost, props))
    return out


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_mixed_batch_matches_each_query_alone_and_hostindex(seed):
    rng, h, d, texts = _random_case(seed)
    opts = _options(rng, len(texts))
    batch = d.resolve_batch(texts, exact=[o[0] for o in opts], tolerance=[o[1] for o in opts],
                            boost=[o[2] for o in opts], properties=[o[3] for o in opts])
    assert batch.n_queries == len(texts)
    for i, (t, (exact, tol, boost, props)) in enumerate(zip(texts, opts)):
        alone = d.resolve_batch([t], exact=exact, tolerance=tol, boost=boost, properties=props).query(0)
        _same(batch.query(i), alone)
        hb = None if boost is None else dict(zip(FIELDS, boost))
        hp = None if props is None else [FIELDS[f] for f in props]
        _same(batch.query(i), h.resolve(t, exact=exact, tolerance=tol, boost=hb, properties=hp))
    d.close()


def test_exact_match_boost_and_stemmer_per_query():
    rng, h, d, texts = _random_case(7, n_words=600, n_docs=80)
    d.set_stemmer(lambda t: t[:-1] if len(t) > 2 else None)
    opts = _options(rng, len(texts))
    kw = dict(exact=[o[0] for o in opts], tolerance=[o[1] for o in opts], boost=[o[2] for o in opts],
              properties=[o[3] for o in opts], exact_match_boost=3.5)
    batch = d.resolve_batch(texts, **kw)
    for i, (t, (exact, tol, boost, props)) in enumerate(zip(texts, opts)):
        _same(batch.query(i), d.resolve_batch([t], exact=exact, tolerance=tol, boost=boost, properties=props,
                                                exact_match_boost=3.5).query(0))
    d.close()


@pytest.mark.parametrize("kw", [dict(), dict(exact=True), dict(tolerance=0), dict(tolerance=1), dict(tolerance=2),
                                dict(boost=[2.0, 0.5], properties=[1])])
def test_without_per_query_options_equals_oc_dict_resolve(kw):
    _, _, d, texts = _random_case(11)
    rp = _lib.ResolveParams()
    arr = (C.c_char_p * len(texts))(*[t.encode() for t in texts])
    rp.texts, rp.n_queries = arr, len(texts)
    rp.exact, rp.tolerance = int(kw.get("exact", False)), kw.get("tolerance", -1)
    fb = np.asarray(kw.get("boost", [1.0, 1.0]), np.float32)
    fm = np.zeros(2, np.uint8)
    fm[kw.get("properties", [0, 1])] = 1
    rp.field_boost, rp.field_mask = fb.ctypes.data, fm.ctypes.data
    L = _lib.lib()

    def arrays(fn):
        res = C.c_void_p()
        _lib.check(fn(C.byref(res)))
        ptrs = [C.c_void_p() for _ in range(5)]
        nt, ne = C.c_uint32(), C.c_uint32()
        L.oc_resolved_arrays(res, *[C.byref(x) for x in ptrs], C.byref(nt), C.byref(ne))
        sizes = [len(texts) + 1, nt.value + 1, ne.value, ne.value, ne.value]
        out = [C.string_at(p, 4 * n) for p, n in zip(ptrs, sizes)]
        L.oc_resolved_free(res)
        return out
    plain = arrays(lambda out: L.oc_dict_resolve(d._h, C.byref(rp), out))
    assert plain == arrays(lambda out: L.oc_dict_resolve_q(d._h, None, C.byref(rp), None, out))
    d.close()


def test_refusals_write_nothing():
    _, _, d, texts = _random_case(5, n_words=100, n_docs=10)
    L = _lib.lib()
    arr = (C.c_char_p * 2)(b"abc", b"de")
    rp = _lib.ResolveParams()
    rp.texts, rp.n_queries, rp.tolerance = arr, 2, -1
    q = (_lib.ResolveQuery * 2)()
    q[0].tolerance, q[1].tolerance = 1, 9
    sentinel = C.c_void_p(0x1234)
    out = C.c_void_p(sentinel.value)
    assert L.oc_dict_resolve_q(d._h, None, C.byref(rp), q, C.byref(out)) == -4 and out.value == sentinel.value
    rp.tolerance = 9                                                      # p's tolerance is checked when q is NULL
    assert L.oc_dict_resolve_q(d._h, None, C.byref(rp), None, C.byref(out)) == -4 and out.value == sentinel.value
    q[1].tolerance = 8                                                    # ... and ignored when q is given
    assert L.oc_dict_resolve_q(d._h, None, C.byref(rp), q, C.byref(out)) == 0 and out.value != sentinel.value
    L.oc_resolved_free(out)
    out = C.c_void_p(sentinel.value)
    assert L.oc_dict_resolve_q(None, None, C.byref(rp), q, C.byref(out)) == -1 and out.value == sentinel.value
    assert L.oc_dict_resolve_q(d._h, None, None, q, C.byref(out)) == -1 and out.value == sentinel.value
    assert L.oc_dict_resolve_q(d._h, None, C.byref(rp), q, None) == -1
    arr[1] = None
    assert L.oc_dict_resolve_q(d._h, None, C.byref(rp), q, C.byref(out)) == -1 and out.value == sentinel.value
    with pytest.raises(ValueError):
        d.resolve_batch(["a", "b"], tolerance=[1])                        # one value per query
    d.close()


def test_bytes_above_0x7f_and_long_tokens_through_the_stemmer():
    d = ob.TermDictionary(1)
    terms = ["café", "cafe", "caffè", "naïve", "naive", "a" * 70, "a" * 69 + "b", "a" * 65]
    d.add_terms(0, terms)
    d.set_stemmer(lambda t: {"cafx": "café", "naivx": "naïv"}.get(t, "a" * 70 if t == "aaaa" else None))
    texts = ["cafx", "naivx", "aaaa", "cafe"]
    batch = d.resolve_batch(texts, tolerance=[1, 2, 2, 1])
    for i, (t, tol) in enumerate(zip(texts, [1, 2, 2, 1])):
        _same(batch.query(i), d.resolve_batch([t], tolerance=tol).query(0))
    q = batch.query(0)                              # "cafx" and its stem "caf\xc3\xa9" (5 bytes)
    assert q.n_tokens == 2
    d.close()
