"""K2 (wgmma batched scan: gather every row within 2*eps of the limit-th best approximate score, exact
re-score of those) against K1 (exact sweep) and the oracle.  The tensor-core path must return bit-identical
hits to the exact path: the low-precision sweep only selects candidates; every returned score is
re-computed with K1's fp32 arithmetic.  Includes the adversarial inputs for a selection scheme:
near-duplicate clusters, exact duplicates, large limits."""
import os

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import synth

pytestmark = pytest.mark.gpu


def _both_paths(ctx, emb, qv, limit, sim, fb=None, nb=0):
    os.environ.pop("OC_DISABLE_GEMM", None)
    d1, s1, c1 = emb.search_batch(qv, limit, sim, fb, nb)
    t1 = ctx.last_timing()
    return (d1, s1, c1), t1


@pytest.mark.parametrize("n,dim,model,B", [(20000, 768, "BGEBase", 32), (70001, 384, "BGESmall", 130),
                                            (40000, 384, "BGESmall", 600),   # 5 query groups: odd super-group tail

                                            (9000, 1024, "BGELarge", 8), (50000, 768, "MultilingualE5Base", 256)])
def test_gemm_path_matches_oracle(gpu_ctx, orc, n, dim, model, B):
    rows = synth.make_vectors(n, dim, seed=n)
    qv, planted = synth.make_vector_queries(rows, B, seed=n + 1)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, model)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    st = orc.EmbStore(rows, is_e5=model.startswith("MultilingualE5"))
    for limit, sim in ((10, -1.0), (25, 0.0)):
        (docs, scores, counts), t = _both_paths(gpu_ctx, emb, qv, limit, sim)
        assert t["scan_tensor_core"] == 1, t
        assert t["scan_launches"] >= 1
        for i in list(range(0, B, max(1, B // 16))):
            ed, es = orc.vector(st, qv[i], limit, sim)
            order = np.argsort(-es, kind="stable")
            assert counts[i] == len(ed), (i, counts[i], len(ed))
            assert_topk_equal(docs[i, :counts[i]], scores[i, :counts[i]], ed[order], es[order], atol=1e-5)
        if limit == 10 and sim < 0:
            assert np.all(docs[:, 0] == planted)
    emb.close()


def test_gemm_path_with_filter_delete_and_zero_query(gpu_ctx, orc):
    n, dim, B = 30000, 768, 16
    rows = synth.make_vectors(n, dim, seed=3)
    qv, _ = synth.make_vector_queries(rows, B, seed=4)
    qv[5] = 0.0                                   # zero query: fails the proof -> exact re-run
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGEBase")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    deleted = np.zeros(n, np.uint8)
    for d in (7, 8, 9):
        emb.delete(d)
        deleted[d] = 1
    rng = np.random.default_rng(0)
    allowed = np.flatnonzero(rng.random(n) < 0.4)
    fb = orc.make_filter_bits(allowed.tolist(), n)
    (docs, scores, counts), t = _both_paths(gpu_ctx, emb, qv, 10, -1.0, fb, n)
    assert t["scan_tensor_core"] == 1 and t["scan_unproven"] >= 1
    st = orc.EmbStore(rows, deleted=deleted)
    for i in range(B):
        ed, es = orc.vector(st, qv[i], 10, -1.0, fb, n)
        order = np.argsort(-es, kind="stable")
        assert_topk_equal(docs[i, :counts[i]], scores[i, :counts[i]], ed[order], es[order], atol=1e-5)
    emb.close()


# `pair` (here and in test_bf16_store_parity) names the cases after the CTA-pair switch of the Blackwell kernels;
# the H100 build has a single sweep kernel, so the value selects nothing and the cases keep their ids.
@pytest.mark.parametrize("n,B,pair", [(120000, 64, "1"), (150001, 300, "1"), (150001, 300, "0"), (4100, 256, "1")])
def test_gemm_equals_exact_sweep_bitwise(gpu_ctx, n, B, pair):
    """B <= 128: one query group; B > 128: several query groups, each swept by its own CTAs (300: a partial
    last group) — all must equal the exact sweep bit for bit."""
    dim = 768
    rows = synth.make_vectors(n, dim, seed=13)
    qv, _ = synth.make_vector_queries(rows, B, seed=14)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGEBase")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    d1, s1, c1 = emb.search_batch(qv, 10, 0.0)
    assert gpu_ctx.last_timing()["scan_tensor_core"] == 1
    os.environ["OC_DISABLE_GEMM"] = "1"
    try:
        d2, s2, c2 = emb.search_batch(qv, 10, 0.0)
        assert gpu_ctx.last_timing()["scan_tensor_core"] == 0
    finally:
        os.environ.pop("OC_DISABLE_GEMM", None)
    assert np.array_equal(d1, d2) and np.array_equal(s1, s2) and np.array_equal(c1, c2)
    emb.close()


@pytest.mark.parametrize("n,dim,model,B,pair", [(30000, 1024, "BGELarge", 5, None), (30000, 1024, "BGELarge", 200, None),
                                                 (50000, 768, "BGEBase", 64, None), (20000, 384, "BGESmall", 130, None),
                                                 (30000, 1024, "BGELarge", 200, "1")])
def test_bf16_store_parity(gpu_ctx, orc, n, dim, model, B, pair):
    """OC_DTYPE_BF16 store (BASELINE configs[4] shape, reduced): rows are bf16 values; every score is
    exact fp32 arithmetic on those values, so the oracle runs on the bf16-rounded rows."""
    rows = ob.from_bf16(ob.to_bf16(synth.make_vectors(n, dim, seed=n + dim)))
    qv, planted = synth.make_vector_queries(rows, B, seed=n + 1)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, model, dtype="bf16")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    assert emb.info()["device_bytes"] < n * dim * 2 * 1.7
    st = orc.EmbStore(rows)
    docs, scores, counts = emb.search_batch(qv, 10, -1.0)
    t = gpu_ctx.last_timing()
    assert t["scan_tensor_core"] == (1 if B >= 8 else 0)
    assert np.all(docs[:, 0] == planted)
    for i in list(range(0, B, max(1, B // 12))):
        ed, es = orc.vector(st, qv[i], 10, -1.0)
        order = np.argsort(-es, kind="stable")
        assert_topk_equal(docs[i, :counts[i]], scores[i, :counts[i]], ed[order], es[order], atol=1e-5)
    if B >= 8:   # tensor-core path == exact sweep, bit for bit
        os.environ["OC_DISABLE_GEMM"] = "1"
        try:
            d2, s2, c2 = emb.search_batch(qv, 10, -1.0)
        finally:
            os.environ.pop("OC_DISABLE_GEMM", None)
        assert np.array_equal(docs, d2) and np.array_equal(scores, s2)
    emb.close()


@pytest.mark.parametrize("n,B,cents,sigma", [(60000, 64, 100, 0.1), (150000, 300, 300, 0.1), (150000, 256, 50, 0.02)])
def test_gemm_on_near_duplicate_clusters(gpu_ctx, orc, n, B, cents, sigma):
    """Hundreds of rows within ~1e-3 (sigma 0.02: ~1e-4) of every query's best hit: the 10th and the 64th best
    are closer than the sweep's rounding error, so a fixed candidate depth cannot certify the answer.  The
    scan must stay on the tensor cores (no exact re-run) and equal the exact sweep bit for bit."""
    dim = 768
    rows = synth.make_clustered_vectors(n, dim, n_centroids=cents, sigma=sigma, seed=n)
    qv, _ = synth.make_vector_queries(rows, B, seed=n + 1)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGEBase")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    d1, s1, c1 = emb.search_batch(qv, 10, 0.0)
    t = gpu_ctx.last_timing()
    assert t["scan_tensor_core"] == 1
    per_cluster = n // cents
    assert t["scan_unproven"] == 0 or per_cluster > 2000, t     # the whole cluster fits the re-score budget
    assert t["scan_rescored"] >= min(per_cluster, 2000) // 4, t   # ... and it is the cluster that gets re-scored
    os.environ["OC_DISABLE_GEMM"] = "1"
    try:
        d2, s2, c2 = emb.search_batch(qv, 10, 0.0)
    finally:
        os.environ.pop("OC_DISABLE_GEMM", None)
    assert np.array_equal(d1, d2) and np.array_equal(s1, s2) and np.array_equal(c1, c2)
    st = orc.EmbStore(rows)
    for i in range(0, B, max(1, B // 8)):
        ed, es = orc.vector(st, qv[i], 10, 0.0)
        order = np.argsort(-es, kind="stable")
        assert_topk_equal(d1[i, :c1[i]], s1[i, :c1[i]], ed[order], es[order], atol=1e-5)
    emb.close()


def test_gemm_exact_duplicates_overflow_to_the_exact_sweep(gpu_ctx, orc):
    """5000 copies of one vector tie exactly: more rows within 2*eps of the 10th best than the re-score budget
    -> those queries are flagged and served by the exact sweep (ties resolve to the lowest doc ids)."""
    n, dim, B = 40000, 384, 16
    rows = synth.make_vectors(n, dim, seed=77)
    rows[10000:15000] = rows[123]
    qv, _ = synth.make_vector_queries(rows, B, seed=78)
    qv[3] = rows[123] * 1.5
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    docs, scores, counts = emb.search_batch(qv, 10, -1.0)
    t = gpu_ctx.last_timing()
    assert t["scan_tensor_core"] == 1 and t["scan_unproven"] >= 1
    assert docs[3, :10].tolist() == [123] + list(range(10000, 10009))
    assert np.all(np.abs(scores[3, :10] - 1.0) < 1e-5)
    st = orc.EmbStore(rows)
    for i in range(B):
        ed, es = orc.vector(st, qv[i], 10, -1.0)
        order = np.argsort(-es, kind="stable")
        assert_topk_equal(docs[i, :counts[i]], scores[i, :counts[i]], ed[order], es[order], atol=1e-5)
    emb.close()


@pytest.mark.parametrize("limit", [33, 100, 128])
def test_gemm_serves_large_limits(gpu_ctx, limit):
    """limit in (32, 128] used to fall off the tensor-core path (64 exact sweeps per 256-query batch)."""
    n, dim, B = 90000, 384, 48
    rows = synth.make_vectors(n, dim, seed=5)
    qv, _ = synth.make_vector_queries(rows, B, seed=6)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGESmall")
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    d1, s1, c1 = emb.search_batch(qv, limit, -1.0)
    t = gpu_ctx.last_timing()
    assert t["scan_tensor_core"] == 1 and t["scan_unproven"] == 0, t
    os.environ["OC_DISABLE_GEMM"] = "1"
    try:
        d2, s2, c2 = emb.search_batch(qv, limit, -1.0)
    finally:
        os.environ.pop("OC_DISABLE_GEMM", None)
    assert np.array_equal(d1, d2) and np.array_equal(s1, s2) and np.array_equal(c1, c2)
    emb.close()
