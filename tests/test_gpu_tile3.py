"""K3c / K3d (bm25_tile3_kernel, bm25_warp_kernel: register-folded scorers, no accumulator arrays; a CTA resp. a warp per
item) against the oracle and against K3b
(bm25_tile2_kernel) on the same inputs — bit-identical scores, same ids, same counts — over the shapes that steer
its code paths: items with only list tokens, only dense tokens, both (ownership bitmap + binary search in the other
lists), rows present in several list tokens, filters / tombstones (batches with device-counted df are routed to K3b by
default: the comparison then pins that routing), cold thresholds overflowing the candidate buffer (the redo with a tighter threshold), the warm-start seed,
n_keep > 32 (bitonic keep) and 4-token queries.  The environment switches are read per launch."""
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


def _queries(vocab, rng, n, ntok):
    """Mix of hot (dense-form), mid and rare terms per query."""
    out = []
    for _ in range(n):
        ids = []
        while len(ids) < ntok:
            r = rng.random()
            t = int(rng.integers(0, 8)) if r < 0.35 else (int(rng.integers(8, 200)) if r < 0.7 else int(rng.integers(200, vocab)))
            if t not in ids:
                ids.append(t)
        out.append(TextQuery.single_terms(ids))
    return out


@pytest.mark.parametrize("n_docs,vocab,ntok,limit,offset", [(70000, 3000, 3, 10, 0), (70000, 3000, 4, 7, 5), (30000, 500, 2, 40, 10),
                                                            (9000, 300, 3, 10, 0)])
def test_tile3_matches_tile2_and_oracle(gpu_ctx, orc, n_docs, vocab, ntok, limit, offset):
    data = synth.make_text_corpus(n_docs, vocab, seed=n_docs + ntok)
    rng = np.random.default_rng(n_docs)
    texts = _queries(vocab, rng, 32, ntok)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=limit, offset=offset)
    with _env(OC_BM25_TILE3="1", OC_BM25_SEED="1"):
        h3 = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=limit, offset=offset)
    with _env(OC_BM25_TILE3="1", OC_BM25_SEED="0"):
        h3n = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=limit, offset=offset)
    with _env(OC_BM25_TILE3="1", OC_BM25_WARP="0"):          # the CTA-per-item form of the same scorer
        h3b = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=limit, offset=offset)
    with _env(OC_BM25_TILE3="1", OC_BM25_WARP="0", OC_BM25_SEED="0"):
        h3bn = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=limit, offset=offset)
    with _env(OC_BM25_TILE3="0"):
        h2 = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=limit, offset=offset)
    _check(h3, ref, exact_scores=True)
    _same(h3, h2)
    _same(h3n, h2)
    _same(h3b, h2)
    _same(h3bn, h2)
    strs.close()


def test_tile3_filter_and_tombstones(gpu_ctx, orc):
    n_docs, vocab = 50000, 2000
    data = synth.make_text_corpus(n_docs, vocab, seed=11)
    rng = np.random.default_rng(5)
    texts = _queries(vocab, rng, 24, 3)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    allowed = np.flatnonzero(rng.random(n_docs) < 0.4)
    fb = orc.make_filter_bits(allowed.tolist(), n_docs)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10, filter_bits=fb, filter_nbits=n_docs)
    with _env(OC_BM25_TILE3="1"):
        h3 = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=10, filtered_doc_ids=fb, filter_nbits=n_docs)
    with _env(OC_BM25_TILE3="1", OC_BM25_WARP="0"):
        h3b = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=10, filtered_doc_ids=fb, filter_nbits=n_docs)
    with _env(OC_BM25_TILE3="0"):
        h2 = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=10, filtered_doc_ids=fb, filter_nbits=n_docs)
    _check(h3, ref, exact_scores=True)
    _same(h3, h2)
    _same(h3b, h2)
    # uncommitted deletes == filtered out (string_field.rs:180-182)
    gone = sorted({int(h.doc_ids[0]) for h in h3 if len(h.doc_ids)})
    for d in gone:
        strs.delete(d)
    keep = orc.make_filter_bits([d for d in range(n_docs) if d not in set(gone)], n_docs)
    ref = _oracle_batch(orc, data, None, 0, texts=texts, limit=10, filter_bits=keep, filter_nbits=n_docs)
    with _env(OC_BM25_TILE3="1"):
        h3 = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=10)
    with _env(OC_BM25_TILE3="0"):
        h2 = ob.search(gpu_ctx, None, strs, "fulltext", texts=texts, limit=10)
    _check(h3, ref, exact_scores=True)
    _same(h3, h2)
    strs.close()


def test_tile3_hybrid(gpu_ctx, orc):
    n, dim, vocab = 30000, 384, 1500
    rows = synth.make_vectors(n, dim, seed=21)
    qv, _ = synth.make_vector_queries(rows, 16, seed=22)
    data = synth.make_text_corpus(n, vocab, seed=23)
    texts = _queries(vocab, np.random.default_rng(3), 16, 3)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    ref = _oracle_batch(orc, data, rows, 2, texts=texts, qv=qv, limit=10, similarity=0.0)
    with _env(OC_BM25_TILE3="1"):
        h3 = ob.search(gpu_ctx, emb, strs, "hybrid", texts=texts, q_vecs=qv, limit=10, similarity=0.0)
    with _env(OC_BM25_TILE3="0"):
        h2 = ob.search(gpu_ctx, emb, strs, "hybrid", texts=texts, q_vecs=qv, limit=10, similarity=0.0)
    _check(h3, ref)
    _same(h3, h2)
    emb.close()
    strs.close()
