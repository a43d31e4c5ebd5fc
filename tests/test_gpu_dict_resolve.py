"""oc_dict_resolve_q with a ctx: the typo-tolerant expansions run on the device (csrc/dict_dev.cuh) and must equal the
host walk (ctx = NULL) byte for byte — token ranges, fields, term ids, order inside a token and weight bits."""
import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_HYBRID

pytestmark = pytest.mark.gpu


def _words(n, seed, shared_prefixes=False, alphabet=26, lo=3, hi=11):
    rng = np.random.default_rng(seed)
    m = int(n * (2 if shared_prefixes else 1.3 if alphabet == 26 else 3))   # small alphabets repeat short words
    lens = rng.integers(lo, hi, size=m)
    buf = rng.integers(97, 97 + alphabet, size=int(lens.sum()), dtype=np.uint8).tobytes().decode()
    offs = np.concatenate([[0], np.cumsum(lens)])
    words = [buf[offs[i]:offs[i + 1]] for i in range(m)]
    if shared_prefixes:   # a few thousand stems, each with many short suffixes over a small alphabet
        stems, si = words[:20000], rng.integers(0, 20000, size=m)
        suf = rng.integers(97, 102, size=(m, 4), dtype=np.uint8)
        k = rng.integers(0, 5, size=m)
        words = [stems[si[i]] + suf[i, :k[i]].tobytes().decode() for i in range(m)]
    words = list(dict.fromkeys(words))[:n]
    assert len(words) == n
    return words


def _typo(rng, w):
    """w with one random edit (or none)"""
    i = int(rng.integers(0, len(w) + 1))
    c = chr(int(rng.integers(97, 123)))
    return [w, w[:i] + c + w[i:], w[:i] + w[i + 1:], w[:i] + c + w[i + 1:]][int(rng.integers(0, 4))] or w


def _texts(rng, words, B, per=3):
    return [" ".join(_typo(rng, words[int(i)]) for i in rng.integers(0, len(words), size=per)) for _ in range(B)]


def _dict(words_per_field):
    d = ob.TermDictionary(len(words_per_field))
    for f, ws in enumerate(words_per_field):
        d.add_terms(f, ws)
    return d


def _same(a, b):
    assert a.n_queries == b.n_queries
    for name in ("q_token_offsets", "token_term_offsets", "term_field", "term_id"):
        x, y = getattr(a, name), getattr(b, name)
        assert np.array_equal(x, y), name
    assert np.array_equal(a.term_weight.view(np.uint32), b.term_weight.view(np.uint32))


def _check(d, ctx, texts, **kw):
    dev = d.resolve_batch(texts, ctx=ctx, **kw)
    _same(dev, d.resolve_batch(texts, **kw))
    return dev


@pytest.fixture(scope="module")
def vocabs():
    return {("200K", False): _words(200_000, 1), ("200K", True): _words(200_000, 2, shared_prefixes=True),
            ("1M", False): _words(1_000_000, 3), ("1M", True): _words(1_000_000, 4, shared_prefixes=True)}


@pytest.mark.parametrize("size", ["200K", "1M"])
@pytest.mark.parametrize("shared", [False, True])
def test_device_equals_host_on_large_vocabularies(gpu_ctx, vocabs, size, shared):
    words = vocabs[(size, shared)]
    d = _dict([words])
    rng = np.random.default_rng(10)
    for tol, B in ((1, 64), (2, 32), (3, 16), (8, 4)):
        dev = _check(d, gpu_ctx, _texts(rng, words, B), tolerance=tol)
        assert dev.term_id.size >= B
    # the mirror holds the term bytes, 8 B of offset and 4 B of permutation per term
    nbytes = sum(len(w) for w in words)
    assert d.device_bytes(gpu_ctx) == nbytes + (len(words) + 1) * 8 + len(words) * 4
    d.close()


def test_mixed_options_per_query_and_two_fields(gpu_ctx):
    rng = np.random.default_rng(3)
    a, b = _words(30_000, 5, alphabet=6), _words(20_000, 6, alphabet=8, lo=1, hi=7)
    d = _dict([a, b])
    B = 96
    texts = _texts(rng, a, B // 2) + _texts(rng, b, B // 2 - 3) + ["", "   ", "a"]
    tol = [[None, 0, 1, 2, 3, 8][int(i)] for i in rng.integers(0, 6, size=B)]
    exact = (rng.random(B) < 0.15).tolist()
    boost = [None if rng.random() < 0.5 else [float(rng.choice([0.5, 2.0])), 1.5] for _ in range(B)]
    props = [[None, [0], [1]][int(i)] for i in rng.integers(0, 3, size=B)]
    _check(d, gpu_ctx, texts, exact=exact, tolerance=tol, boost=boost, properties=props, exact_match_boost=3.0)
    d.close()


def test_token_lengths_1_to_64_and_beyond(gpu_ctx):
    rng = np.random.default_rng(4)
    base = _words(20_000, 7, alphabet=4, lo=1, hi=11)
    long_ = ["".join(rng.choice(list("abcd"), size=n)) for n in range(9, 80) for _ in range(40)]
    # terms one edit away from the long ones, so long tokens have neighbours at every distance
    words = list(dict.fromkeys(base + long_ + [_typo(rng, w) for w in long_]))
    d = _dict([words])
    texts = [w for w in long_[::7]] + [_typo(rng, w) for w in long_[3::11]] + ["a", "ab", "b" * 64, "c" * 65]
    for tol in (1, 2, 3, 8):
        _check(d, gpu_ctx, texts, tolerance=tol)
    d.close()


def test_terms_with_bytes_above_0x7f(gpu_ctx):
    rng = np.random.default_rng(6)
    ascii_ = _words(5000, 8, alphabet=5, lo=2, hi=8)
    accented = [w.replace("a", "á").replace("c", "ç") for w in ascii_[:2000]] + [w + "ü" for w in ascii_[2000:3000]]
    d = _dict([ascii_ + accented])
    d.set_stemmer(lambda t: t.replace("b", "ß") if "b" in t else None)   # stems with multi-byte characters
    texts = _texts(rng, ascii_, 60)
    for tol in (1, 2, 3):
        _check(d, gpu_ctx, texts, tolerance=tol)
    d.close()


def test_dictionary_growing_between_calls(gpu_ctx):
    rng = np.random.default_rng(8)
    words = _words(60_000, 9, alphabet=8, lo=2, hi=8)
    d = ob.TermDictionary(1)
    d.add_terms(0, words[::3])
    texts = _texts(rng, words, 48)
    _check(d, gpu_ctx, texts, tolerance=2)
    before = d.device_bytes(gpu_ctx)
    d.add_terms(0, words[1::3])                       # new ids whose terms sort into the middle of the old ones
    _check(d, gpu_ctx, texts, tolerance=2)
    assert d.device_bytes(gpu_ctx) > before
    d.add_terms(0, words[2::3] + words[:10])          # known terms keep their ids
    _check(d, gpu_ctx, texts, tolerance=1)
    _check(d, gpu_ctx, texts, tolerance=1)            # nothing changed: the mirror is reused as it is
    d.close()


def test_two_dicts_on_one_ctx_and_one_dict_on_two_ctxs(gpu_ctx):
    rng = np.random.default_rng(9)
    wa, wb = _words(20_000, 10, alphabet=6), _words(25_000, 11, alphabet=6)
    da, db = _dict([wa]), _dict([wb])
    ta, tb = _texts(rng, wa, 32), _texts(rng, wb, 32)
    ctx2 = ob.Context(0)
    try:
        for _ in range(2):
            _check(da, gpu_ctx, ta, tolerance=1)
            _check(db, gpu_ctx, tb, tolerance=2)
            _check(da, ctx2, ta, tolerance=2)
        assert da.device_bytes(gpu_ctx) == da.device_bytes(ctx2) > 0
        assert db.device_bytes(ctx2) == 0 and db.device_bytes(gpu_ctx) > 0
    finally:
        ctx2.close()
    da.close(); db.close()


def test_dict_destroyed_before_shutdown_and_the_reverse():
    rng = np.random.default_rng(12)
    words = _words(20_000, 13, alphabet=6)
    texts = _texts(rng, words, 16)
    # the dictionary goes first: the ctx frees its mirror on its next device resolve and at shutdown
    ctx = ob.Context(0)
    d1 = _dict([words])
    _check(d1, ctx, texts, tolerance=1)
    d1.close()
    d2 = _dict([words])
    _check(d2, ctx, texts, tolerance=2)
    ctx.close()
    # the ctx goes first: the dictionary keeps working on the host and on another ctx, and is destroyed afterwards
    ctx = ob.Context(0)
    _check(d2, ctx, texts, tolerance=1)
    ctx.close()
    ref = d2.resolve_batch(texts, tolerance=1)
    ctx = ob.Context(0)
    _same(d2.resolve_batch(texts, tolerance=1, ctx=ctx), ref)
    d2.close()
    ctx.close()


def _index_op(doc_id, text):
    toks = text.lower().split()
    terms = {}
    for i, t in enumerate(toks):
        terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
    return {"type": "Index", "doc_id": doc_id,
            "indexed_values": [{"type": "ScoreString2", "field": "text", "field_length": len(toks), "terms": terms}]}


def test_index_loader_resolves_typos_on_the_device(gpu_ctx):
    ld = IndexLoader(gpu_ctx, ["text"], embedding_dim=32)
    # the reference pin (fulltext_search.rs:956-1018): "Mxin" with tolerance 1 reaches "main" only
    ld.apply_all([_index_op(1, "Main Street"), _index_op(2, "Maple Avenue"), _index_op(3, "Another Street")])
    ld.commit()
    q = ld.resolve(["Mxin"], tolerance=1).query(0)
    assert q.term_id.tolist() == [ld.dict.lookup(0, "main")]
    assert ld.dict.device_bytes(gpu_ctx) > 0
    # a hybrid search over device-resolved typos equals the same search over host-resolved ones
    rng = np.random.default_rng(14)
    words = _words(3000, 15, alphabet=7, lo=3, hi=8)
    ld.apply_all([_index_op(10 + i, " ".join(rng.choice(words, size=6))) for i in range(2000)])
    vecs = rng.standard_normal((2010, 32)).astype(np.float32)
    ld.apply({"type": "IndexEmbedding", "data": [(i, [vecs[i]]) for i in range(2010)]})
    ld.commit()
    texts = _texts(rng, words, 16, per=2)
    dev, host = ld.resolve(texts, tolerance=2), ld.dict.resolve_batch(texts, tolerance=2)
    _same(dev, host)
    tsc, p = ld.context(), ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, limit_hint=20)
    a, b = tsc.execute_batch(p, dev, vecs[:16]), tsc.execute_batch(p, host, vecs[:16])
    for x, y in zip(a, b):
        assert x.count == y.count and x.doc_ids.tolist() == y.doc_ids.tolist()
        assert np.array_equal(x.scores.view(np.uint32), y.scores.view(np.uint32))
    ld.close()
