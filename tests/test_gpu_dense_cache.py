"""The ctx's cache of hot-term dense contribution arrays (OC_BM25_DENSE_CACHE_MB): a search that reads kept arrays
returns the same bytes as one that builds every array from scratch (budget 0), across rotating batches that share hot
terms, a commit that changes a hot term's postings, other bm25 k and b, a budget small enough to evict, filters and
tombstones (the cache is bypassed) and a bf16 embedding store; and it matches the CPU oracle."""
import os

import numpy as np
import pytest

import oramacore_b200 as ob
import oramacore_b200.engine as engine
from helpers import assert_topk_equal
from oramacore_b200 import synth
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, TextQuery

pytestmark = pytest.mark.gpu

N, VOCAB, DIM, B = 200_000, 5000, 128, 64
ENV = "OC_BM25_DENSE_CACHE_MB"


@pytest.fixture(scope="module")
def corpus():
    data = synth.make_text_corpus(N, VOCAB, seed=71)
    rows = synth.make_vectors(N, DIM, seed=72)
    texts = [synth.make_text_queries(VOCAB, B, seed=73 + i) for i in range(4)]
    qv = [synth.make_vector_queries(rows, B, seed=83 + i)[0] for i in range(4)]
    return data, rows, texts, qv


@pytest.fixture
def budget():
    old = os.environ.get(ENV)

    def set_budget(mb):
        os.environ[ENV] = str(mb)
    yield set_budget
    if old is None:
        os.environ.pop(ENV, None)
    else:
        os.environ[ENV] = old


def hot_terms(data):
    offs = data.fields[0].term_offsets
    lens = (offs[1:] - offs[:-1]).astype(np.int64)
    return np.flatnonzero(lens >= max(512, N // 16))


def run(ctx, emb, strs, mode, texts, qv=None, **kw):
    p = ob.TokenScoreParams(mode=mode, limit_hint=10, similarity=0.0, **kw)
    docs, scores, n, cnt = ob.TokenScoreContext(ctx, emb, strs).execute_batch_arrays(p, texts, qv)
    return docs.tobytes() + scores.tobytes() + n.tobytes() + cnt.tobytes(), (docs, scores, n, cnt)


def both(ctx, emb, strs, budget, mode, texts, qv=None, mb=2048, **kw):
    """The same call with the cache (budget mb) and with budget 0: returns both results."""
    budget(mb)
    a = run(ctx, emb, strs, mode, texts, qv, **kw)
    budget(0)
    z = run(ctx, emb, strs, mode, texts, qv, **kw)
    return a, z


def test_hot_terms_present(corpus):
    data, _, texts, _ = corpus
    hot = set(hot_terms(data).tolist())
    assert len(hot) >= 20
    for batch in texts:   # the batches share hot terms, so later calls hit what earlier ones built
        assert len(hot & {t for q in batch for t in q.term_id.tolist()}) >= 10


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID])
def test_rotating_batches_identical(gpu_ctx, corpus, budget, mode):
    data, rows, texts, qv = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)
    emb = None
    if mode == MODE_HYBRID:
        emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
        emb.insert_batch(np.arange(N, dtype=np.uint64), rows)
    for _ in range(3):
        for i in range(len(texts)):
            a, z = both(gpu_ctx, emb, strs, budget, mode, texts[i], qv[i] if emb else None)
            assert a[0] == z[0]


def test_steady_state_skips_the_build(gpu_ctx, corpus, budget):
    """Every hot term of the batch kept: the call launches no precompute kernel (one launch fewer than budget 0)."""
    data, _, texts, _ = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)

    def launches(mb):
        budget(mb)
        l0 = gpu_ctx.launch_count()
        out = run(gpu_ctx, None, strs, MODE_FULLTEXT, texts[0])[0]
        return gpu_ctx.launch_count() - l0, out
    run(gpu_ctx, None, strs, MODE_FULLTEXT, texts[0])   # b derived, arrays built
    l_kept, o_kept = launches(2048)
    l_kept2, o_kept2 = launches(2048)
    l_zero, o_zero = launches(0)
    assert o_kept == o_kept2 == o_zero
    assert l_kept == l_kept2 == l_zero - 1, (l_kept, l_kept2, l_zero)


def test_commit_invalidates(gpu_ctx, corpus, budget):
    """Re-inserting a document that holds a hot term with another tf leaves the term's df, N, weight and idf as they
    were: only the snapshot's identity tells the kept array is stale."""
    data, _, _, _ = corpus
    hot = hot_terms(data)
    t = int(hot[0])
    f = data.fields[0]
    rows_t = f.post_row[int(f.term_offsets[t]):int(f.term_offsets[t + 1])]
    d = int(rows_t[0])
    texts = [TextQuery.single_terms([t])] + [TextQuery.single_terms([t, int(hot[1 + i % 5]), 100 + i]) for i in range(B - 1)]
    strs = ob.StringFieldStorage(gpu_ctx, data)
    a0, z0 = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts)
    assert a0[0] == z0[0]
    budget(2048)
    run(gpu_ctx, None, strs, MODE_FULLTEXT, texts)   # kept arrays read
    strs.insert(d, 0, 3, {t: 40})
    strs.commit()
    a1, z1 = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts)
    assert a1[0] == z1[0]
    assert int(a1[1][0][0, 0]) == d                  # tf 40 in a 3-token field: d tops the query on t alone
    assert a1[0] != a0[0]


def test_bm25_k_and_b_miss(gpu_ctx, corpus, budget, monkeypatch):
    data, _, texts, _ = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)
    a0, z0 = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0])
    assert a0[0] == z0[0]
    monkeypatch.setattr(engine, "BM25_K", 1.7)
    a1, z1 = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0])
    assert a1[0] == z1[0] and a1[0] != a0[0]
    monkeypatch.setattr(engine, "BM25_B", 0.3)
    a2, z2 = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0])
    assert a2[0] == z2[0] and a2[0] != a1[0]
    monkeypatch.undo()
    a3, z3 = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0])
    assert a3[0] == z3[0] == a0[0]


def test_small_budget_evicts(gpu_ctx, corpus, budget):
    """4 MB holds 5 of the batch's 0.8 MB arrays: every call evicts and builds the rest in its own buffer."""
    data, rows, texts, qv = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM)
    emb.insert_batch(np.arange(N, dtype=np.uint64), rows)
    for _ in range(2):
        for i in range(len(texts)):
            a, z = both(gpu_ctx, emb, strs, budget, MODE_HYBRID, texts[i], qv[i], mb=4)
            assert a[0] == z[0]
            a, z = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[(i + 1) % len(texts)], mb=1)
            assert a[0] == z[0]


def test_filters_and_tombstones(gpu_ctx, corpus, budget):
    data, _, texts, _ = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)
    budget(2048)
    run(gpu_ctx, None, strs, MODE_FULLTEXT, texts[0])   # kept arrays of the unfiltered batch
    flt = ob.DeviceFilter.from_ids(gpu_ctx, np.arange(0, N, 3, dtype=np.uint64), N)
    a, z = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0], device_filter=flt)
    assert a[0] == z[0]
    strs.delete(np.arange(0, N, 7, dtype=np.uint64))
    a, z = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0])
    assert a[0] == z[0]
    strs.commit()   # tombstones dropped: the cache is used again, on the new snapshot
    a, z = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0])
    assert a[0] == z[0]
    a2, _ = both(gpu_ctx, None, strs, budget, MODE_FULLTEXT, texts[0])
    assert a2[0] == a[0]


def test_bf16_store(gpu_ctx, corpus, budget):
    data, rows, texts, qv = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=DIM, dtype="bf16")
    emb.insert_batch(np.arange(N, dtype=np.uint64), rows)
    for _ in range(2):
        for i in range(len(texts)):
            a, z = both(gpu_ctx, emb, strs, budget, MODE_HYBRID, texts[i], qv[i])
            assert a[0] == z[0]


def test_kept_arrays_match_oracle(gpu_ctx, corpus, budget, orc):
    data, _, texts, _ = corpus
    strs = ob.StringFieldStorage(gpu_ctx, data)
    budget(2048)
    for i in range(len(texts)):
        run(gpu_ctx, None, strs, MODE_FULLTEXT, texts[i])
    ix = orc.StrIndex(data)
    for i in range(len(texts)):   # every hot term of these calls is kept by now
        _, (docs, scores, n, cnt) = run(gpu_ctx, None, strs, MODE_FULLTEXT, texts[i])
        sb = orc.SearchBatch(ix, None)
        for q in texts[i]:
            sb.add(MODE_FULLTEXT, limit=10, text=q)
        od, os_, on, oc = sb.run(1)
        for q in range(B):
            assert int(cnt[q]) == int(oc[q])
            assert int(n[q]) == int(on[q])
            assert_topk_equal(docs[q, :n[q]], scores[q, :n[q]], od[q, :on[q]], os_[q, :on[q]])
