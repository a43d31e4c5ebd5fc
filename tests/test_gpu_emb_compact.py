"""oc_emb_compact on the GPU (EmbeddingFieldStorage compact(), index/mod.rs:583-590): the tombstoned rows leave the
store in place and in order, and no search can tell — ids, score bits, counts and tie order are those of the store
with its tombstones, and those of a store that never held the dead rows."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import _lib, synth
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_HYBRID, MODE_VECTOR

pytestmark = pytest.mark.gpu

N_DOCS = 4600        # documents; the string store holds all of them
N_ROWS = 9001        # embedding rows: 35 whole 256-row tiles and a partial one
LIMIT = 10
CONFIGS = {"f32": ("f32", False), "f32_nocopy": ("f32", True), "bf16": ("bf16", False)}


@pytest.fixture(scope="module")
def text(gpu_ctx):
    data = synth.make_text_corpus(N_DOCS, 800, seed=41)
    strs = ob.StringFieldStorage(gpu_ctx, data)
    yield strs, synth.make_text_queries(800, 64, seed=42)
    strs.close()


def _row_docs(n_rows, n_docs, seed):
    """Several chunks per document, documents out of id order: row -> DocumentId."""
    rng = np.random.default_rng(seed)
    docs = np.concatenate([rng.permutation(n_docs), rng.integers(0, n_docs, n_rows - n_docs)]).astype(np.uint64)
    return docs[rng.permutation(n_rows)] if n_rows >= n_docs else docs[:n_rows]


def _make_store(ctx, monkeypatch, cfg, dim, row_docs, rows):
    dtype, no_copy = CONFIGS[cfg]
    if no_copy:
        monkeypatch.setenv("OC_EMB_F16", "0")   # read at creation and by every search of the test
    emb = ob.EmbeddingFieldStorage(ctx, dim=dim, dtype=dtype)
    emb.insert_batch(row_docs, rows)
    return emb


def _dead_docs(pattern, row_docs):
    """The documents to delete, chosen so that their rows are the named rows."""
    n = row_docs.shape[0]
    rng = np.random.default_rng(7)
    if pattern == "scattered":
        return np.unique(row_docs[rng.random(n) < 0.2])
    if pattern == "all_but_one":
        keep = row_docs[n // 2]
        return np.unique(row_docs[row_docs != keep])
    raise AssertionError(pattern)


def _canon(docs, scores, counts):
    return [(int(c), docs[i, :c].tobytes(), scores[i, :c].tobytes()) for i, c in enumerate(counts)]


def _hits(hs):
    return [(h.count, np.asarray(h.doc_ids, np.uint64).tobytes(), np.asarray(h.scores, np.float32).tobytes()) for h in hs]


def _snapshot(ctx, emb, qv, text=None, filters=None):
    """Everything a caller can see of the store through the search entry points."""
    out = {}
    for B in (1, 4, 64):      # the exact sweep at 1 and 4 queries, the tensor-core sweep at 64
        out["emb", B] = _canon(*emb.search_batch(qv[:B], LIMIT, -1.0))
    out["vector"] = _hits(ob.search(ctx, emb, None, "vector", q_vecs=qv, limit=LIMIT, similarity=0.0))
    if text is not None:
        strs, texts = text
        omc_docs = np.arange(0, N_DOCS, 3, dtype=np.uint64)
        omc_mult = np.linspace(0.5, 2.0, omc_docs.shape[0]).astype(np.float32)
        out["hybrid"] = _hits(ob.search(ctx, emb, strs, "hybrid", texts=texts, q_vecs=qv, limit=LIMIT, similarity=0.0))
        out["hybrid_omc_qf"] = _hits(ob.search(ctx, emb, strs, "hybrid", texts=texts, q_vecs=qv, limit=LIMIT, similarity=0.0,
                                               omc_doc_ids=omc_docs, omc_mult=omc_mult, device_filters=filters))
        out["vector_qf"] = _hits(ob.search(ctx, emb, None, "vector", q_vecs=qv, limit=LIMIT, similarity=0.0, device_filters=filters))
        out["hybrid_200"] = _hits(ob.search(ctx, emb, strs, "hybrid", texts=texts[:8], q_vecs=qv[:8], limit=200, similarity=0.0))
    return out


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k] == b[k], k


@pytest.fixture(scope="module")
def q_filters(gpu_ctx):
    rng = np.random.default_rng(5)
    fs = [ob.DeviceFilter.from_ids(gpu_ctx, np.flatnonzero(rng.random(N_DOCS) < p), N_DOCS + 1) for p in (0.5, 0.1)]
    yield [None if b % 3 == 0 else fs[b % 2] for b in range(64)]
    for f in fs:
        f.close()


# ---- 1, 2, 6: invisible to searches, equal to a store that never held the dead rows


@pytest.mark.parametrize("dim,window", [(384, 64 << 10), (768, 1 << 20), (1000, 256 << 10)])
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_compaction_is_invisible_to_searches(gpu_ctx, monkeypatch, text, q_filters, cfg, dim, window):
    monkeypatch.setenv("OC_EMB_COMPACT_WINDOW", str(window))   # the stores span many staging windows
    rows = synth.make_vectors(N_ROWS, dim, seed=dim)
    rows[17] = 0.0                                  # a live row whose inverse norm says nothing about deadness
    qv, _ = synth.make_vector_queries(rows, 64, seed=dim + 1)
    row_docs = _row_docs(N_ROWS, N_DOCS, seed=dim)
    for pattern in ("scattered", "run", "first", "last", "all_but_one"):
        cur_docs = row_docs
        if pattern in ("scattered", "all_but_one"):
            dead_docs = _dead_docs(pattern, row_docs)
        else:
            # the rows of a range die together when the range has documents of its own (two chunks each)
            lo, hi = {"run": (3000, 5500), "first": (0, 2100), "last": (N_ROWS - 1900, N_ROWS)}[pattern]
            cur_docs = row_docs.copy()
            cur_docs[lo:hi] = N_DOCS + np.arange(hi - lo, dtype=np.uint64) // 2
            dead_docs = np.unique(cur_docs[lo:hi])
        emb = _make_store(gpu_ctx, monkeypatch, cfg, dim, cur_docs, rows)
        emb.delete(dead_docs)
        alive = ~np.isin(cur_docs, dead_docs)
        n_live = int(alive.sum())
        assert emb.info()["num_embeddings"] == n_live and emb.info()["num_rows"] == N_ROWS
        before = _snapshot(gpu_ctx, emb, qv, text, q_filters)
        bytes_before = emb.info()["device_bytes"]
        st = emb.compact()
        first_dead = int(np.flatnonzero(~alive)[0])
        assert st["rows_before"] == N_ROWS and st["rows_after"] == n_live and st["rows_moved"] == n_live - first_dead
        assert 0 < st["workspace_bytes"] <= 256 << 20 and st["device_ms"] > 0
        assert st["device_bytes_after"] == st["device_bytes_before"] == bytes_before       # capacity kept
        info = emb.info()
        assert info["num_rows"] == info["num_embeddings"] == n_live and info["device_bytes"] == bytes_before
        _assert_same(before, _snapshot(gpu_ctx, emb, qv, text, q_filters))
        # a store filled with the surviving rows only, in the same order
        twin = _make_store(gpu_ctx, monkeypatch, cfg, dim, cur_docs[alive], rows[alive])
        _assert_same(before, _snapshot(gpu_ctx, twin, qv, text, q_filters))
        st2 = emb.compact(shrink=True)
        assert st2["rows_moved"] == 0 and st2["device_bytes_after"] < st2["device_bytes_before"]
        ti, ei = twin.info(), emb.info()
        assert (ei["num_rows"], ei["num_embeddings"], ei["device_bytes"]) == (ti["num_rows"], ti["num_embeddings"], ti["device_bytes"])
        _assert_same(before, _snapshot(gpu_ctx, emb, qv, text, q_filters))
        twin.close()
        emb.close()


# ---- 3: ties


def test_tie_order_survives_compaction(gpu_ctx):
    dim = 128
    rng = np.random.default_rng(1)
    v = rng.standard_normal(dim).astype(np.float32)
    filler = synth.make_vectors(600, dim, seed=2)
    rows = filler.copy()
    dup_rows = np.arange(5, 600, 7)                  # the same vector under many documents...
    rows[dup_rows] = v
    row_docs = rng.permutation(600).astype(np.uint64) + 100     # ...inserted out of doc-id order
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=dim)
    emb.insert_batch(row_docs, rows)
    emb.delete(row_docs[dup_rows[::3]])              # some of the equal rows
    emb.delete(row_docs[np.arange(0, 600, 11)])      # and some others, shifting the rest
    q = np.stack([v, filler[0]])
    d0, s0, c0 = emb.search_batch(q, 40, -1.0)
    assert c0[0] == 40 and np.all(s0[0, :20] == s0[0, 0])       # a run of exactly equal scores
    st = emb.compact()
    assert st["rows_moved"] > 0
    d1, s1, c1 = emb.search_batch(q, 40, -1.0)
    assert _canon(d0, s0, c0) == _canon(d1, s1, c1)
    emb.close()


# ---- 4: life after compaction


def test_life_after_compaction(gpu_ctx, monkeypatch):
    monkeypatch.setenv("OC_EMB_COMPACT_WINDOW", str(128 << 10))
    dim, n = 256, 3000
    rows = synth.make_vectors(n + 500, dim, seed=3)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=dim)
    # an empty store
    st = emb.compact()
    assert (st["rows_before"], st["rows_after"], st["rows_moved"], st["device_ms"]) == (0, 0, 0, 0.0)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows[:n])
    # an already compact store launches nothing
    launches = gpu_ctx.launch_count()
    st = emb.compact()
    assert st["rows_moved"] == 0 and st["workspace_bytes"] == 0 and gpu_ctx.launch_count() == launches
    emb.delete(np.arange(0, n, 4, dtype=np.uint64))
    emb.compact()
    assert gpu_ctx.launch_count() > launches
    alive = np.ones(n, bool); alive[::4] = False
    # insert, delete (of moved rows: doc_rows follows the move), re-insert of a deleted document, compact again
    emb.insert_batch(np.arange(n, n + 500, dtype=np.uint64), rows[n:])
    emb.delete(np.asarray([1, 2, 2999, n + 3], np.uint64))
    emb.insert(0, [rows[0], rows[4]])
    emb.insert(2, [rows[2]])
    docs = np.concatenate([np.flatnonzero(alive), np.arange(n, n + 500), [0, 0, 2]]).astype(np.uint64)
    vecs = np.concatenate([rows[:n][alive], rows[n:], rows[[0, 4, 2]]])
    keep = ~np.isin(np.arange(docs.shape[0]), np.flatnonzero(np.isin(docs[:-3], [1, 2, 2999, n + 3])))
    qv, _ = synth.make_vector_queries(rows, 16, seed=4)
    before = _snapshot(gpu_ctx, emb, np.tile(qv, (4, 1)))
    st = emb.compact()
    assert st["rows_before"] == docs.shape[0] and st["rows_after"] == int(keep.sum()) and st["rows_moved"] > 0
    _assert_same(before, _snapshot(gpu_ctx, emb, np.tile(qv, (4, 1))))
    twin = ob.EmbeddingFieldStorage(gpu_ctx, dim=dim)
    twin.insert_batch(docs[keep], vecs[keep])
    _assert_same(before, _snapshot(gpu_ctx, twin, np.tile(qv, (4, 1))))
    twin.close()
    # every row dead
    emb.delete(np.unique(docs[keep]))
    assert emb.info()["num_embeddings"] == 0
    st = emb.compact()
    assert st["rows_after"] == 0 and st["rows_moved"] == 0 and emb.info()["num_rows"] == 0
    assert emb.search_batch(qv, LIMIT, -1.0)[2].tolist() == [0] * 16
    emb.insert_batch(np.arange(5, dtype=np.uint64), rows[:5])
    d, s, c = emb.search_batch(rows[3:4], LIMIT, -1.0)
    assert c[0] == 5 and d[0, 0] == 3
    st = emb.compact(shrink=True)       # nothing dead: only the capacity goes
    assert st["rows_moved"] == 0 and st["device_bytes_after"] < st["device_bytes_before"]
    assert emb.search_batch(rows[3:4], LIMIT, -1.0)[0][0, 0] == 3
    emb.close()


# ---- 5: oracle


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_compacted_store_matches_the_oracle(gpu_ctx, orc, dtype):
    n, dim = 9000, 768
    rows = synth.make_vectors(n, dim, seed=8)
    if dtype == "bf16":
        rows = ob.from_bf16(ob.to_bf16(rows))
    ids = np.arange(n, dtype=np.uint64) * 3 + 1
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGEBase", dtype=dtype)
    emb.insert_batch(ids, rows)
    rng = np.random.default_rng(9)
    dead = rng.random(n) < 0.4
    emb.delete(ids[dead])
    emb.compact()
    qv, _ = synth.make_vector_queries(rows, 12, seed=10)
    st = orc.EmbStore(rows[~dead], ids[~dead])
    for B in (4, 12):
        docs, scores, counts = emb.search_batch(qv[:B], LIMIT, 0.0)
        for i in range(B):
            ed, es = orc.vector(st, qv[i], LIMIT, 0.0)
            order = np.argsort(-es, kind="stable")
            assert counts[i] == len(ed)
            assert_topk_equal(docs[i, :counts[i]], scores[i, :counts[i]], ed[order], es[order], atol=1e-5)
    emb.close()


# ---- 6: memory


def test_shrink_and_kept_capacity(gpu_ctx):
    dim, n = 384, 8192
    rows = synth.make_vectors(n, dim, seed=12)
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=dim)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    full = emb.info()["device_bytes"]
    emb.delete(np.arange(0, n, 2, dtype=np.uint64))
    st = emb.compact()
    assert st["workspace_bytes"] <= 256 << 20 and st["device_bytes_after"] == full
    # the capacity was kept: as many rows as left fit again without a new allocation
    emb.insert_batch(np.arange(n, n + n // 2, dtype=np.uint64), rows[:n // 2])
    assert emb.info()["device_bytes"] == full and emb.info()["num_rows"] == n
    emb.delete(np.arange(n, n + n // 2, dtype=np.uint64))
    st = emb.compact(shrink=True)
    assert st["rows_after"] == n // 2 and st["device_bytes_after"] < st["device_bytes_before"] == full
    assert emb.info()["device_bytes"] == st["device_bytes_after"] == full // 2
    d, s, c = emb.search_batch(rows[1:2], LIMIT, -1.0)
    assert d[0, 0] == 1
    emb.close()


# ---- 7: loader


def _index_op(doc_id, text):
    toks = text.split()
    terms = {}
    for i, t in enumerate(toks):
        terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
    return {"type": "Index", "doc_id": doc_id,
            "indexed_values": [{"type": "ScoreString2", "field": "text", "field_length": len(toks), "terms": terms}]}


def test_loader_commit_compacts_the_embedding_store(gpu_ctx):
    dim, n = 64, 300
    rng = np.random.default_rng(0)
    vecs = rng.standard_normal((2 * n, dim)).astype(np.float32)
    words = ["alpha", "beta", "gamma", "delta"]

    def feed(ld):
        ld.apply_all([_index_op(i, " ".join(words[(i + j) % 4] for j in range(1 + i % 5))) for i in range(n)])
        ld.apply({"type": "IndexEmbedding", "data": [(i, [vecs[i], vecs[n + i]] if i % 3 == 0 else [vecs[i]]) for i in range(n)]})
        ld.commit()
        # an update is a delete and an insert: every fifth document is re-indexed with a new vector
        upd = list(range(0, n, 5))
        ld.apply({"type": "DeleteDocuments", "doc_ids": upd + [7, 8]})
        ld.apply_all([_index_op(i, "alpha beta") for i in upd])
        ld.apply({"type": "IndexEmbedding", "data": [(i, [vecs[n + i]]) for i in upd]})

    ld = IndexLoader(gpu_ctx, ["text"], embedding_dim=dim)
    feed(ld)
    info = ld.emb.info()
    assert info["num_rows"] > info["num_embeddings"]
    tsc = ld.context()
    qv = vecs[[0, 7, 33, n + 5]]
    p = ob.TokenScoreParams(mode=MODE_VECTOR, similarity=0.0, limit_hint=20)
    before = _hits(tsc.execute_batch(p, None, qv))
    ld.commit()
    info = ld.emb.info()
    assert info["num_rows"] == info["num_embeddings"]
    assert _hits(tsc.execute_batch(p, None, qv)) == before
    # hybrid: the same ops through a loader whose embedding store is compacted by hand give the same results
    other = IndexLoader(gpu_ctx, ["text"], embedding_dim=dim)
    feed(other)
    other.strs.commit()
    other.strs.set_global(max(other.document_count, 0))
    ph = ob.TokenScoreParams(mode=MODE_HYBRID, similarity=0.0, limit_hint=20)
    q = ld.resolve(["alpha", "beta gamma", "delta", "alpha"])
    uncompacted = _hits(other.context().execute_batch(ph, other.resolve(["alpha", "beta gamma", "delta", "alpha"]), qv))
    assert _hits(tsc.execute_batch(ph, q, qv)) == uncompacted
    other.emb.compact()
    assert _hits(other.context().execute_batch(ph, other.resolve(["alpha", "beta gamma", "delta", "alpha"]), qv)) == uncompacted
    other.close()
    ld.close()


# ---- 8: refusals


def test_refusals(gpu_ctx):
    emb = ob.EmbeddingFieldStorage(gpu_ctx, dim=64)
    L = ob.lib()
    st = _lib.EmbCompact()
    assert L.oc_emb_compact(None, 0, C.byref(st)) == -1
    assert L.oc_emb_compact(emb._h, 2, C.byref(st)) == -1 and "flags" in L.oc_last_error().decode()
    assert L.oc_emb_compact(emb._h, 0xffffffff, None) == -1
    assert L.oc_emb_compact(emb._h, 0, None) == 0          # the statistics are optional
    emb.close()
