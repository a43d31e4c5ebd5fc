"""The per-item paths of the warp BM25 scorer (K3d, bm25_warp_kernel) that its bookkeeping shortcuts touch, each
compared byte for byte with K3b (bm25_tile2_kernel, OC_BM25_TILE3=0), which scores every row, and with the oracle:
  * count-only items (dense tokens skipped, no list token): every lane's extrema stay 0 and their reduction is skipped;
  * items with 2-4 list tokens (per-token ownership bitmaps in use) whose bitmaps are cleared after each item;
  * a cold threshold (no seed) that overflows the candidate buffer and redoes the item;
and the hybrid point lookups, which start once the side stream has put up their inputs and run under the tile scorer:
their results must equal the single-stream order (OC_SIDE_STREAM=0).  The environment switches are read per call."""
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


def _queries(rng, n, n_hot, n_list, vocab):
    """n_hot of the 8 hottest terms (dense form) and n_list mid / rare terms (posting lists) per query."""
    out = []
    for _ in range(n):
        hot = rng.choice(8, size=n_hot, replace=False).tolist()
        lst = rng.choice(np.arange(20, vocab), size=n_list, replace=False).tolist()
        ids = hot + lst
        rng.shuffle(ids)
        out.append(TextQuery.single_terms([int(t) for t in ids]))
    return out


def _run(ctx, strs, texts, route, emb=None, qv=None, env=None, **kw):
    e = {"K3d": {"OC_BM25_TILE3": "1", "OC_BM25_WARP": "1"}, "K3b": {"OC_BM25_TILE3": "0"}}[route]
    e.update(env or {})
    with _env(**e):
        if emb is None:
            h = ob.search(ctx, None, strs, "fulltext", texts=texts, **kw)
        else:
            h = ob.search(ctx, emb, strs, "hybrid", texts=texts, q_vecs=qv, similarity=0.0, **kw)
    t = ctx.last_timing()
    return h, (t["bm25_dense_items"], t["bm25_dense_skipped"])


@pytest.fixture(scope="module")
def corpus():
    n_docs, vocab = 200000, 3000   # 25 tiles: items of one query run while other warps raise its threshold
    return n_docs, vocab, synth.make_text_corpus(n_docs, vocab, seed=81)


@pytest.mark.parametrize("n_hot,n_list", [(0, 2), (0, 4), (1, 2), (1, 3), (2, 2)])
def test_list_token_items(gpu_ctx, orc, corpus, n_hot, n_list):
    """2-4 list tokens per item: rows held by several lists, ownership by the first, bitmaps cleared per item."""
    n_docs, vocab, data = corpus
    texts = _queries(np.random.default_rng(n_hot * 10 + n_list), 48, n_hot, n_list, vocab)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10)
    _check(h2, ref, exact_scores=True)
    for seed in ("1", "0"):
        h, _ = _run(gpu_ctx, strs, texts, "K3d", env={"OC_BM25_SEED": seed}, limit=10)
        _same(h, h2)
    strs.close()


def test_count_only_items(gpu_ctx, orc, corpus):
    """Two hot terms and a rare one: the rare term warms the threshold (the seed) and is absent from most tiles, so
    most items are a count of the dense tokens' presence bits and nothing else."""
    n_docs, vocab, data = corpus
    texts = _queries(np.random.default_rng(3), 48, 2, 1, vocab)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10)
    _check(h2, ref, exact_scores=True)
    h, (items, skipped) = _run(gpu_ctx, strs, texts, "K3d", limit=10)
    _same(h, h2)
    assert skipped > 0, (items, skipped)
    strs.close()


def test_cold_threshold_redo(gpu_ctx, orc, corpus):
    """No seed and hot terms only: the first tiles of each query pass a cold threshold, overflow the 256-key buffer
    and are redone with a tighter one (scanned items, extrema reduced)."""
    n_docs, vocab, data = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)
    for n_hot, n_list in ((1, 0), (2, 1), (3, 1)):
        texts = _queries(np.random.default_rng(7 + n_hot), 32, n_hot, n_list, vocab)
        ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10)
        h2, _ = _run(gpu_ctx, strs, texts, "K3b", limit=10)
        _check(h2, ref, exact_scores=True)
        h, (items, _) = _run(gpu_ctx, strs, texts, "K3d", env={"OC_BM25_SEED": "0"}, limit=10)
        assert items > 0
        _same(h, h2)
    strs.close()


@pytest.mark.parametrize("limit", [1, 10, 32])
def test_hybrid_lookups_under_the_scorer(gpu_ctx, orc, limit):
    """Hybrid on the side stream (the point lookups wait for the uploaded descriptors, the fusion for the tiles) against
    one stream for everything and against K3b."""
    n, dim, vocab = 120000, 384, 3000
    rows = synth.make_vectors(n, dim, seed=91)
    qv, _ = synth.make_vector_queries(rows, 64, seed=92)
    data = synth.make_text_corpus(n, vocab, seed=93)
    texts = _queries(np.random.default_rng(94), 64, 1, 2, vocab)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, rows, 2, texts=texts, qv=qv, limit=limit, similarity=0.0)
    one, _ = _run(gpu_ctx, strs, texts, "K3d", emb, qv, env={"OC_SIDE_STREAM": "0"}, limit=limit)
    _check(one, ref)
    h2, _ = _run(gpu_ctx, strs, texts, "K3b", emb, qv, limit=limit)
    _same(h2, one)
    for _ in range(2):   # the second call reads the kept dense arrays
        h, _ = _run(gpu_ctx, strs, texts, "K3d", emb, qv, limit=limit)
        _same(h, one)
    emb.close()
    strs.close()
