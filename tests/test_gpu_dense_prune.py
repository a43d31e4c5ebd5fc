"""The dense-scan skip of the register-folded BM25 scorers (K3c bm25_tile3_kernel, K3d bm25_warp_kernel): when the
tile maxima of an item's hot-term (dense) tokens, folded in token order, stay below the query's running threshold, no
row scored by those tokens alone can become a candidate, and the scan of their arrays is replaced by a count over their
presence bitmaps.  Every case here must return the same bytes as K3b (OC_BM25_TILE3=0), which scores every row, and
agree with the oracle; last_timing()'s bm25_dense_items / bm25_dense_skipped show whether the skip ran.  The
environment switches are read per launch."""
import os

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import synth
from oramacore_b200.types import TextQuery
from test_gpu_parity import _check, _oracle_batch

pytestmark = pytest.mark.gpu


class _env:
    def __init__(self, **kw):
        self.kw, self.old = kw, {}

    def __enter__(self):
        for k, v in self.kw.items():
            self.old[k] = os.environ.get(k)
            os.environ[k] = v

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.count == y.count
        assert np.array_equal(x.doc_ids, y.doc_ids)
        assert np.array_equal(x.scores, y.scores)


def _queries(vocab, rng, n, ntok, hot_only=False, weight=1.0):
    """Hot (dense-form), mid and rare terms per query; hot_only: only the 8 hottest terms (a cold threshold)."""
    out = []
    for _ in range(n):
        ids = []
        while len(ids) < ntok:
            r = 0.0 if hot_only else rng.random()
            t = int(rng.integers(0, 8)) if r < 0.4 else (int(rng.integers(8, 200)) if r < 0.75 else int(rng.integers(200, vocab)))
            if t not in ids:
                ids.append(t)
        out.append(TextQuery.single_terms(ids, weight=weight))
    return out


def _run(ctx, strs, texts, route, emb=None, qv=None, **kw):
    """One search through `route` ("K3d", "K3c" or "K3b"); returns the hits and the call's dense-pass counters."""
    env = {"K3d": {"OC_BM25_TILE3": "1", "OC_BM25_WARP": "1"}, "K3c": {"OC_BM25_TILE3": "1", "OC_BM25_WARP": "0"},
           "K3b": {"OC_BM25_TILE3": "0"}}[route]
    with _env(**env):
        if emb is None:
            h = ob.search(ctx, None, strs, "fulltext", texts=texts, **kw)
        else:
            h = ob.search(ctx, emb, strs, "hybrid", texts=texts, q_vecs=qv, similarity=0.0, **kw)
    t = ctx.last_timing()
    assert t["bm25_dense_skipped"] <= t["bm25_dense_items"], t
    return h, (t["bm25_dense_items"], t["bm25_dense_skipped"])


@pytest.mark.parametrize("n_docs,vocab,ntok,limit,offset", [(70000, 3000, 3, 10, 0), (70000, 3000, 4, 7, 5),
                                                            (30000, 500, 2, 40, 10), (9000, 300, 3, 10, 0),
                                                            (400000, 5000, 3, 10, 0), (400000, 5000, 3, 40, 10)])
def test_mixed_queries_match_tile2_and_oracle(gpu_ctx, orc, n_docs, vocab, ntok, limit, offset):
    """Queries mixing dense and list tokens: rows of the list tokens are excluded from the count pass (`touched`).
    The 400K-document corpora have 49 tiles, so many items of one query run while other CTAs raise its threshold; at
    limit + offset > 32 both routes run K3c (a CTA per item)."""
    data = synth.make_text_corpus(n_docs, vocab, seed=n_docs + ntok)
    texts = _queries(vocab, np.random.default_rng(n_docs + 1), 48, ntok)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=limit, offset=offset)
    h2, c2 = _run(gpu_ctx, strs, texts, "K3b", limit=limit, offset=offset)
    assert c2 == (0, 0)                                   # (K3b scans every row and counts nothing)
    _check(h2, ref, exact_scores=True)
    for route in ("K3d", "K3c"):
        h, (items, skipped) = _run(gpu_ctx, strs, texts, route, limit=limit, offset=offset)
        _same(h, h2)
        if n_docs >= 70000 and ntok == 3 and limit == 10 and route == "K3d":
            # hot terms score low next to a rare list term: most dense items cannot reach the threshold
            assert items > 0 and skipped > 0, (items, skipped)
    strs.close()


def test_all_dense_queries(gpu_ctx, orc):
    """Only hot terms: the threshold starts cold (the seed falls back to the first rows of the store)."""
    n_docs, vocab = 70000, 3000
    data = synth.make_text_corpus(n_docs, vocab, seed=31)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    for ntok in (1, 2, 3):
        texts = _queries(vocab, np.random.default_rng(ntok), 24, ntok, hot_only=True)
        ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10)
        h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10)
        _check(h2, ref, exact_scores=True)
        for route in ("K3d", "K3c"):
            h, (items, _) = _run(gpu_ctx, strs, texts, route, limit=10)
            assert items > 0
            _same(h, h2)
    strs.close()


def test_cache_hit_repeats_the_bytes(gpu_ctx, orc):
    """A second identical call reads the kept arrays and their summaries (the dense-array cache) as they are."""
    n_docs, vocab = 70000, 3000
    data = synth.make_text_corpus(n_docs, vocab, seed=41)
    texts = _queries(vocab, np.random.default_rng(42), 48, 3)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10)
    first, c1 = _run(gpu_ctx, strs, texts, "K3d", limit=10)
    second, c2 = _run(gpu_ctx, strs, texts, "K3d", limit=10)
    _same(first, h2)
    _same(second, h2)
    assert c1[0] == c2[0] and c2[1] > 0, (c1, c2)
    with _env(OC_BM25_DENSE_CACHE_MB="0"):               # every array (and summary) built into the call's buffer
        fresh, c0 = _run(gpu_ctx, strs, texts, "K3d", limit=10)
    _same(fresh, h2)
    assert c0[1] > 0, c0
    _check(second, _oracle_batch(orc, data, None, 0, texts=texts, limit=10), exact_scores=True)
    strs.close()


def test_filter_and_tombstones(gpu_ctx, orc):
    """A filter and uncommitted deletes leave the skip out: they make the call count corpus df on the device, so no
    dense array is built and every route runs K3b.  Pins that routing (no dense pass is counted) and the results."""
    n_docs, vocab = 50000, 2000
    data = synth.make_text_corpus(n_docs, vocab, seed=51)
    rng = np.random.default_rng(52)
    texts = _queries(vocab, rng, 32, 3)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    fb = orc.make_filter_bits(np.flatnonzero(rng.random(n_docs) < 0.4).tolist(), n_docs)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10, filter_bits=fb, filter_nbits=n_docs)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10, filtered_doc_ids=fb, filter_nbits=n_docs)
    _check(h2, ref, exact_scores=True)
    for route in ("K3d", "K3c"):
        h, c = _run(gpu_ctx, strs, texts, route, limit=10, filtered_doc_ids=fb, filter_nbits=n_docs)
        _same(h, h2)
        assert c == (0, 0), (route, c)
    gone = sorted({int(h.doc_ids[0]) for h in h2 if len(h.doc_ids)})
    for d in gone:
        strs.delete(d)
    keep = orc.make_filter_bits(sorted(set(range(n_docs)) - set(gone)), n_docs)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10, filter_bits=keep, filter_nbits=n_docs)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10)
    _check(h2, ref, exact_scores=True)
    for route in ("K3d", "K3c"):
        h, c = _run(gpu_ctx, strs, texts, route, limit=10)
        _same(h, h2)
        assert c == (0, 0), (route, c)
    strs.close()


def test_hybrid(gpu_ctx, orc):
    """Hybrid: the fusion normalises by each query's fulltext maximum, which skipped rows never hold."""
    n, dim, vocab = 70000, 384, 3000
    rows = synth.make_vectors(n, dim, seed=61)
    qv, _ = synth.make_vector_queries(rows, 32, seed=62)
    data = synth.make_text_corpus(n, vocab, seed=63)
    texts = _queries(vocab, np.random.default_rng(64), 32, 3)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, rows, 2, texts=texts, qv=qv, limit=10, similarity=0.0)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", emb, qv, limit=10)
    _check(h2, ref)
    for route in ("K3d", "K3c"):
        h, (items, skipped) = _run(gpu_ctx, strs, texts, route, emb, qv, limit=10)
        _same(h, h2)
        assert skipped > 0, (route, items, skipped)
    emb.close()
    strs.close()


def test_negative_boost_never_skips(gpu_ctx, orc):
    """A negative weight makes contributions negative: the bound argument does not hold, and no item is skipped."""
    n_docs, vocab = 70000, 3000
    data = synth.make_text_corpus(n_docs, vocab, seed=71)
    texts = _queries(vocab, np.random.default_rng(72), 32, 3, weight=-0.5)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10)
    _check(h2, ref, exact_scores=True)
    for route in ("K3d", "K3c"):
        h, (items, skipped) = _run(gpu_ctx, strs, texts, route, limit=10)
        _same(h, h2)
        assert items > 0 and skipped == 0, (route, items, skipped)
    strs.close()
