"""The fp16 sweep of fp32 stores (OC_SCAN_TC_F16): an fp32 store keeps a power-of-two scaled fp16 copy of its rows and
the tensor-core sweep selects candidates from it; every returned score is still K1's exact fp32 arithmetic on the fp32
rows.  So the results must be byte-identical to the exact sweep (OC_DISABLE_GEMM=1) and to the tf32 sweep of the same
store (OC_EMB_F16=0 at search time), at every dimension, batch size (one query group, CTA pairs, an odd number of
groups), limit, filter, tombstone, degenerate query and row, and on clustered data.  OC_EMB_F16=0 at creation gives a
store without the copy, served through tf32."""
import os

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import _lib, synth

pytestmark = pytest.mark.gpu

F16, TF32, EXACT = _lib.OC_SCAN_TC_F16, _lib.OC_SCAN_TC_TF32, _lib.OC_SCAN_EXACT


def _with_env(key, value, fn):
    old = os.environ.get(key)
    os.environ[key] = value
    try:
        return fn()
    finally:
        if old is None:
            os.environ.pop(key, None)
        else:
            os.environ[key] = old


def _three_ways(ctx, search):
    """search() through the fp16 sweep, the tf32 sweep and the exact sweep -> (results, timings) each; asserts the
    variants and that the three results are byte-identical."""
    os.environ.pop("OC_DISABLE_GEMM", None)
    os.environ.pop("OC_EMB_F16", None)
    r16 = search()
    t16 = ctx.last_timing()
    r32 = _with_env("OC_EMB_F16", "0", search)
    t32 = ctx.last_timing()
    rex = _with_env("OC_DISABLE_GEMM", "1", search)
    tex = ctx.last_timing()
    assert t16["scan_tensor_core"] == 1 and t16["scan_variant"] == F16, t16
    assert t32["scan_tensor_core"] == 1 and t32["scan_variant"] == TF32, t32
    assert tex["scan_tensor_core"] == 0 and tex["scan_variant"] == EXACT, tex
    for a, b, c in zip(r16, r32, rex):
        assert a.tobytes() == b.tobytes(), "fp16 sweep != tf32 sweep"
        assert a.tobytes() == c.tobytes(), "fp16 sweep != exact sweep"
    return r16, t16, t32


def _store(ctx, rows, model="BGEBase", chunks=1):
    emb = ob.EmbeddingFieldStorage(ctx, model, dim=rows.shape[1])
    n = rows.shape[0]
    cuts = np.linspace(0, n, chunks + 1).astype(np.int64)
    for a, b in zip(cuts[:-1], cuts[1:]):
        emb.insert_batch(np.arange(a, b, dtype=np.uint64), rows[a:b])
    return emb


@pytest.mark.parametrize("dim,B,limit", [(300, 8, 10), (384, 64, 33), (768, 130, 10), (768, 256, 10), (1024, 300, 128),
                                         (768, 1024, 10), (384, 256, 128), (1024, 64, 33), (300, 130, 128)])
def test_f16_sweep_equals_tf32_and_exact(gpu_ctx, dim, B, limit):
    """B = 8 / 64: one query group; 130 / 256 / 1024: an even number of groups (CTA pairs); 300: three groups (unpaired)."""
    n = 40000
    rows = synth.make_vectors(n, dim, seed=dim + B)
    qv, planted = synth.make_vector_queries(rows, B, seed=dim + B + 1)
    emb = _store(gpu_ctx, rows)
    (docs, _, _), t16, t32 = _three_ways(gpu_ctx, lambda: emb.search_batch(qv, limit, -1.0))
    assert np.all(docs[:, 0] == planted)
    assert t16["scan_unproven"] == 0 and t32["scan_unproven"] == 0, (t16, t32)
    assert 0 < t16["scan_rescored"] <= t32["scan_rescored"], (t16["scan_rescored"], t32["scan_rescored"])
    assert t16["scan_bytes"] == n * (emb_stride(dim) * 2 + 8)
    emb.close()


def emb_stride(dim):
    s = (dim + 127) // 128
    return 128 * (s + 1 if s in (5, 7) else s)


def test_f16_with_filter_tombstones_zero_query_and_degenerate_rows(gpu_ctx, orc):
    n, dim, B = 30000, 768, 16
    rng = np.random.default_rng(3)
    rows = synth.make_vectors(n, dim, seed=3)
    qv, _ = synth.make_vector_queries(rows, B, seed=4)
    # extreme norms (the cosine does not change) and degenerate rows
    rows *= (10.0 ** rng.uniform(-15, 15, (n, 1))).astype(np.float32)
    rows[100] *= np.float32(1e-25)        # |x|^2 underflows in fp32: inverse norm 0
    rows[101] *= np.float32(1e25)         # |x|^2 overflows: inverse norm 0
    rows[102, 5] = np.inf
    rows[103, 9] = np.nan
    rows[104] = 0.0
    qv[5] = 0.0                           # zero query: fails the proof -> exact re-run
    qv[6] *= np.float32(1e-15)
    qv[7] *= np.float32(1e15)
    emb = _store(gpu_ctx, rows)
    emb.delete([7, 8, 9])
    allowed = np.flatnonzero(rng.random(n) < 0.4)
    fb = orc.make_filter_bits(allowed.tolist(), n)
    for f, nb in ((None, 0), (fb, n)):
        (docs, scores, counts), t16, _ = _three_ways(gpu_ctx, lambda: emb.search_batch(qv, 10, -1.0, f, nb))
        assert t16["scan_unproven"] >= 1          # the zero query
        assert not np.any(np.isin(docs[counts > 0], [7, 8, 9, 102, 103]))
    emb.close()


def test_f16_with_per_query_filters(gpu_ctx):
    n, dim, B = 40000, 384, 64
    rng = np.random.default_rng(11)
    rows = synth.make_vectors(n, dim, seed=11)
    qv, _ = synth.make_vector_queries(rows, B, seed=12)
    emb = _store(gpu_ctx, rows, "BGESmall")
    emb.delete(list(range(50, 60)))
    ids = np.arange(n, dtype=np.uint64)
    fs = [ob.DeviceFilter.from_ids(gpu_ctx, ids[rng.random(n) < p], n) for p in (0.3, 0.7, 0.001)]
    filters = [None if i % 4 == 3 else fs[i % 3] for i in range(B)]
    tsc = ob.TokenScoreContext(gpu_ctx, emb, None)
    p = ob.TokenScoreParams(mode=ob.MODE_VECTOR, limit_hint=10, similarity=-1.0, device_filters=filters)
    _three_ways(gpu_ctx, lambda: tsc.execute_batch_arrays(p, None, qv))
    for f in fs:
        f.close()
    emb.close()


def test_f16_store_grown_over_several_inserts(gpu_ctx, orc):
    n, dim, B = 50001, 768, 256
    rows = synth.make_vectors(n, dim, seed=21)
    qv, planted = synth.make_vector_queries(rows, B, seed=22)
    emb = _store(gpu_ctx, rows, chunks=7)     # each insert past the capacity grows the fp32 rows and the fp16 copy
    info = emb.info()
    (docs, scores, counts), _, _ = _three_ways(gpu_ctx, lambda: emb.search_batch(qv, 10, 0.0))
    assert np.all(docs[:, 0] == planted)
    st = orc.EmbStore(rows)
    for i in range(0, B, 32):
        ed, es = orc.vector(st, qv[i], 10, 0.0)
        order = np.argsort(-es, kind="stable")
        assert_topk_equal(docs[i, :counts[i]], scores[i, :counts[i]], ed[order], es[order], atol=1e-5)
    emb.close()
    # the same store created with OC_EMB_F16=0: no copy (2 B per element and a scale per row less), the tf32 sweep
    plain = _with_env("OC_EMB_F16", "0", lambda: _store(gpu_ctx, rows, chunks=7))
    stride = emb_stride(dim)
    cap = info["device_bytes"] // (stride * 4 + 12 + stride * 2 + 4)
    assert info["device_bytes"] == cap * (stride * 4 + 12 + stride * 2 + 4)
    assert plain.info()["device_bytes"] == cap * (stride * 4 + 12)
    d2, s2, c2 = plain.search_batch(qv, 10, 0.0)
    t = gpu_ctx.last_timing()
    assert t["scan_variant"] == TF32 and t["scan_bytes"] == n * (stride * 4 + 4), t
    assert d2.tobytes() == docs.tobytes() and s2.tobytes() == scores.tobytes() and c2.tobytes() == counts.tobytes()
    plain.close()


@pytest.mark.parametrize("n,B,cents,sigma", [(60000, 64, 100, 0.1), (150000, 300, 300, 0.1), (150000, 256, 50, 0.02)])
def test_f16_on_near_duplicate_clusters(gpu_ctx, orc, n, B, cents, sigma):
    dim = 768
    rows = synth.make_clustered_vectors(n, dim, n_centroids=cents, sigma=sigma, seed=n)
    qv, _ = synth.make_vector_queries(rows, B, seed=n + 1)
    emb = _store(gpu_ctx, rows)
    (d1, s1, c1), t16, t32 = _three_ways(gpu_ctx, lambda: emb.search_batch(qv, 10, 0.0))
    per_cluster = n // cents
    assert t16["scan_unproven"] == 0 or per_cluster > 2000, t16
    assert t16["scan_rescored"] >= min(per_cluster, 2000) // 4, t16
    assert t16["scan_rescored"] <= t32["scan_rescored"], (t16["scan_rescored"], t32["scan_rescored"])
    print(f"\n[f16 clusters] n={n} B={B} sigma={sigma}: rows re-scored per query fp16 {t16['scan_rescored']} "
          f"tf32 {t32['scan_rescored']}; unproven fp16 {t16['scan_unproven']} tf32 {t32['scan_unproven']}")
    st = orc.EmbStore(rows)
    for i in range(0, B, max(1, B // 8)):
        ed, es = orc.vector(st, qv[i], 10, 0.0)
        order = np.argsort(-es, kind="stable")
        assert_topk_equal(d1[i, :c1[i]], s1[i, :c1[i]], ed[order], es[order], atol=1e-5)
    emb.close()


def test_f16_exact_duplicates_overflow_to_the_exact_sweep(gpu_ctx):
    n, dim, B = 40000, 384, 16
    rows = synth.make_vectors(n, dim, seed=77)
    rows[10000:15000] = rows[123]
    qv, _ = synth.make_vector_queries(rows, B, seed=78)
    qv[3] = rows[123] * 1.5
    emb = _store(gpu_ctx, rows, "BGESmall")
    (docs, scores, _), t16, _ = _three_ways(gpu_ctx, lambda: emb.search_batch(qv, 10, -1.0))
    assert t16["scan_unproven"] >= 1
    assert docs[3, :10].tolist() == [123] + list(range(10000, 10009))
    emb.close()


def test_f16_hybrid_matches_the_oracle(gpu_ctx, orc):
    n, dim, vocab, B = 30000, 768, 5000, 64
    rows = synth.make_vectors(n, dim, seed=31)
    qv, _ = synth.make_vector_queries(rows, B, seed=32)
    data = synth.make_text_corpus(n, vocab, seed=33)
    texts = synth.make_text_queries(vocab, B, seed=34)
    emb = _store(gpu_ctx, rows)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    tsc = ob.TokenScoreContext(gpu_ctx, emb, strs)
    p = ob.TokenScoreParams(mode=ob.MODE_HYBRID, limit_hint=10, similarity=0.0)
    (docs, scores, nhit, cnt), t16, _ = _three_ways(gpu_ctx, lambda: tsc.execute_batch_arrays(p, texts, qv))
    ix, st = orc.StrIndex(data), orc.EmbStore(rows)
    sb = orc.SearchBatch(ix, st)
    for i in range(B):
        sb.add(2, limit=10, similarity=0.0, q_vec=qv[i], text=texts[i])
    od, os_, on, oc = sb.run(1)
    for i in range(B):
        assert int(cnt[i]) == int(oc[i]) and int(nhit[i]) == int(on[i]), i
        assert np.allclose(scores[i, :nhit[i]], os_[i, :on[i]], rtol=0, atol=1e-5)
        assert set(docs[i, :nhit[i]].tolist()) == set(od[i, :on[i]].tolist())
    strs.close()
    emb.close()
