"""Sharded string stores that follow writes: oc_str_sync_global rebuilds the corpus-wide df tables and average field
lengths on the devices after a commit, and IndexLoader(shard=(lo, hi)) feeds one rank of a document-sharded index from
the whole op stream.  W contexts on device 0 joined by Context.comm_init_local, one thread per rank (the pool /
Sharded helpers of test_gpu_sharded_local).

  1. A static corpus loaded without tables and synced equals the shards loaded with the replicated tables: the same
     tables, the same averages, byte-identical batches of every kind, the same scorer route.
  2. A live stream: W sharded loaders and one unsharded loader take the same ops; every search is byte-identical on
     every rank and to the unsharded loader (vector and hybrid: within ATOL at the depth cut, where exact duplicate
     rows tie), before and after each commit.
  3. Refusals: different n_fields on the ranks, a ctx without a comm; oc_str_set_global(N, NULL) keeps the tables."""
import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal
from oramacore_b200 import synth
from oramacore_b200.engine import TokenScoreContext, TokenScoreParams
from oramacore_b200.loader import IndexLoader
from oramacore_b200.sharding import shard_range, shard_string_index
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, FieldPostings, StringIndexData
from test_gpu_index_lifecycle import FILTERS, STRING_FIELDS, Stream, _resolve
from test_gpu_parity import ATOL
from test_gpu_sharded_local import Sharded, _join, pool, zipf  # noqa: F401  (module fixtures)
from test_gpu_topn_paths import KINDS, N_ZIPF, _kind

gpu = pytest.mark.gpu
OC_ERR_INVALID, OC_ERR_COMM = -1, -5   # include/oramacore_b200.h


def _row_len_mean(f: FieldPostings) -> np.float32:
    """The average oc_str_commit computes: the mean of the non-zero row lengths, one per row, as f32 of a double."""
    rows, first = np.unique(f.post_row, return_index=True)
    ln = f.post_len[first].astype(np.int64)
    ln = ln[ln > 0]
    return np.float32(float(int(ln.sum())) / float(ln.size))


def _synced_shards(sh, data, bounds):
    """The shards of `sh`, loaded again without df tables and with a wrong average, then synced on every rank."""
    stores = []
    for r, ctx in enumerate(sh.ctxs):
        sd, _ = shard_string_index(data, *bounds[r])
        sd = StringIndexData([FieldPostings(1.0, f.term_offsets, f.post_row, f.post_tf, f.post_len) for f in sd.fields],
                             sd.n_rows, sd.document_count, sd.row_doc_ids)
        stores.append(ob.StringFieldStorage(ctx, sd))
    stats, errs = sh.on_ranks(lambda r: stores[r].sync_global())
    assert errs == [None] * sh.W, errs
    return stores, stats


# ------------------------------------------------------------------ 1. static corpus
@gpu
@pytest.mark.parametrize("layout", ["W2", "W3", "W4", "W8", "W16", "empty"])
def test_static_sync_equals_load_time_tables(pool, gpu_ctx, orc, zipf, layout):  # noqa: F811
    W = 3 if layout == "empty" else int(layout[1:])
    bounds = [shard_range(N_ZIPF, r, W) for r in range(W)]
    if layout == "empty":   # rank 1 holds no row
        bounds[1] = (bounds[1][0], bounds[1][0])
        bounds[2] = (bounds[1][0], bounds[2][1])
    sh = Sharded(_join(pool, W), gpu_ctx, orc, data=zipf, bounds=bounds)
    replicated = sh.strs
    synced, stats = _synced_shards(sh, zipf, bounds)
    try:
        for r in range(W):
            assert stats[r]["rows_global"] == N_ZIPF, stats[r]
        for i, f in enumerate(zipf.fields):
            want = _row_len_mean(f)
            assert np.float32(f.avg_field_len) == want   # the premise of the byte comparisons below
            gdf = np.diff(f.term_offsets.astype(np.int64)).astype(np.uint32)
            for r in range(W):
                assert np.array_equal(synced[r].read_global_df(i), gdf), (layout, r, i)
                assert synced[r].read_field(i)["avg_field_len"] == want, (layout, r, i)
        for kind in KINDS:
            texts, skw, _, _ = _kind(kind)
            for limit, offset in ((10, 0), (100, 0), (7, 500)):
                kw = dict(limit_hint=limit, offset=offset, **skw)
                sh.strs = replicated
                res_rep, tim_rep = sh.sharded("fulltext", texts, **kw)
                sh.strs = synced
                tim_syn = sh.check("fulltext", texts, oracle=None, ctx=(layout, kind, limit, offset), **kw)
                res_syn, _ = sh.sharded("fulltext", texts, **kw)
                for r in range(W):
                    for a, b in zip(res_rep[r], res_syn[r]):
                        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), (layout, kind, r)
                    # the same route: hot terms take the dense form on both (the item count itself also counts the
                    # re-runs after a candidate-buffer overflow, which depend on the running thresholds)
                    d_rep, d_syn = tim_rep[r]["bm25_dense_items"], tim_syn[r]["bm25_dense_items"]
                    assert (d_rep > 0) == (d_syn > 0), (layout, kind, r, d_rep, d_syn)
    finally:
        sh.strs = replicated
        for s in synced:
            s.close()
        sh.close()


# ------------------------------------------------------------------ 2. live stream
def _on_ranks(n, fn):
    import threading
    out, errs = [None] * n, [None] * n

    def go(r):
        try:
            out[r] = fn(r)
        except ob.OcError as e:
            errs[r] = e
    th = [threading.Thread(target=go, args=(r,)) for r in range(n)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert errs == [None] * n, errs
    return out


def _same_bytes(a, b, ctx):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), ctx


class Live:
    def __init__(self, ctxs, single, cuts, dim):
        W = len(ctxs)
        kw = dict(embedding_dim=dim, **FILTERS)
        self.one = IndexLoader(single, STRING_FIELDS, **kw)
        self.lds = [IndexLoader(c, STRING_FIELDS, shard=(cuts[r], cuts[r + 1] if r + 1 < W else None), **kw)
                    for r, c in enumerate(ctxs)]

    def apply(self, ops):
        for ld in [self.one] + self.lds:
            ld.apply_all(ops)

    def commit(self):
        self.one.commit()
        _on_ranks(len(self.lds), lambda r: self.lds[r].commit())

    def close(self):
        for ld in [self.one] + self.lds:
            ld.close()

    def search(self, mode, batch, qv=None, where=None, **kw):
        """(every rank's arrays, the unsharded loader's arrays)"""
        def params(ld, sharded):
            f = ld.where_filter(where) if where is not None else None
            p = TokenScoreParams(mode=mode, omc_store=ld.omc() if mode == MODE_FULLTEXT else None, device_filter=f, sharded=sharded,
                                 shard_tombstones=sharded and ld.shard_tombstones, **kw)
            return p, f

        def run(ld, sharded):
            p, f = params(ld, sharded)
            try:
                tsc = TokenScoreContext(ld.ctx, ld.emb if mode != MODE_FULLTEXT else None, ld.strs if mode != MODE_VECTOR else None)
                return tsc.execute_batch_arrays(p, batch if mode != MODE_VECTOR else None, qv)
            finally:
                if f is not None:
                    f.close()
        return _on_ranks(len(self.lds), lambda r: run(self.lds[r], True)), run(self.one, False)


def _check_state(tag, lv, stream, rng, committed):
    W = len(lv.lds)
    for fi in range(len(STRING_FIELDS)):
        sizes = {ld.dict.size(fi) for ld in lv.lds + [lv.one]}
        assert len(sizes) == 1, (tag, fi, sizes)
    texts = stream.texts(12)
    batch = _resolve(lv.lds[0], rng, texts)
    where = {"flag": True} if rng.random() < 0.5 else {"price": {"gte": 0.0}}
    for limit, offset, thr, wh in ((10, 0, None, None), (100, 0, None, None), (10, 23, 0.5, None), (10, 0, None, where),
                                   (50, 0, 1.0, where)):
        kw = dict(limit_hint=limit, offset=offset, threshold=thr)
        ranks, one = lv.search(MODE_FULLTEXT, batch, where=wh, **kw)
        ctx = (tag, limit, offset, thr, wh)
        for r in range(W):
            _same_bytes(ranks[r], ranks[0], ctx + ("rank", r))
        _same_bytes(ranks[0], one, ctx + ("unsharded",))
        if committed:
            counted, _ = lv.search(MODE_FULLTEXT, batch, where=wh, shard_count_df=True, **kw)
            for r in range(W):
                _same_bytes(counted[r], ranks[0], ctx + ("count_df", r))
    qv = stream.qvecs(8)
    small = ob.engine.TextQueryBatch([batch.query(i) for i in range(8)])
    for mode in (MODE_VECTOR, MODE_HYBRID):
        for limit in (10, 129):
            ranks, one = lv.search(mode, small, qv, limit_hint=limit, similarity=0.0)
            for r in range(W):
                _same_bytes(ranks[r], ranks[0], (tag, mode, limit, "rank", r))
            d0, s0, n0, c0 = ranks[0]
            d1, s1, n1, c1 = one
            assert np.array_equal(c0, c1) and np.array_equal(n0, n1), (tag, mode, limit, c0, c1)
            for i in range(d0.shape[0]):
                assert_topk_equal(d0[i, :n0[i]], s0[i, :n0[i]], d1[i, :n1[i]], s1[i, :n1[i]], atol=ATOL)


@gpu
@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("layout", ["first_round", "spread"])
def test_live_stream(pool, gpu_ctx, W, layout):  # noqa: F811
    dim, rounds, per_round = 32, 3, 700
    stream = Stream(100 + W, dim, 1500)
    ops, ends = [], []
    omc_rng = np.random.default_rng(7)
    for _ in range(rounds):
        ops.append(stream.round(per_round))
        ends.append(stream.next_id)
        for op in ops[-1]:   # Index2 with a multiplier for some documents: every rank's OMC store takes all of them
            if op["type"] == "Index" and omc_rng.random() < 0.2:
                op["type"], op["omc"] = "Index2", float(omc_rng.choice([0.0, 0.5, 2.0, 3.0]))
    top = ends[0] if layout == "first_round" else ends[-1]
    cuts = [(top * r) // W for r in range(W)]
    lv = Live(_join(pool, W), gpu_ctx, cuts, dim)
    rng = np.random.default_rng(W)
    try:
        for k, round_ops in enumerate(ops):
            lv.apply(round_ops)
            _check_state((layout, W, k, "before commit"), lv, stream, rng, committed=False)
            lv.commit()
            _check_state((layout, W, k, "after commit"), lv, stream, rng, committed=True)
    finally:
        lv.close()


# ------------------------------------------------------------------ 3. refusals and set_global
def _tiny(n_fields, lo, hi):
    data = synth.make_text_corpus(hi - lo, 50, seed=lo + 1)
    return StringIndexData([data.fields[0]] * n_fields, data.n_rows, 3000, np.arange(lo, hi, dtype=np.uint64))


@gpu
def test_sync_refusals_and_set_global(pool, gpu_ctx):  # noqa: F811
    ctxs = _join(pool, 3)
    stores = [ob.StringFieldStorage(c, _tiny(2 if r == 1 else 1, 1000 * r, 1000 * r + 900)) for r, c in enumerate(ctxs)]
    try:
        out = [None] * 3

        def go(r):
            try:
                stores[r].sync_global()
            except ob.OcError as e:
                out[r] = e.code
        import threading
        th = [threading.Thread(target=go, args=(r,)) for r in range(3)]
        [t.start() for t in th]
        [t.join() for t in th]
        assert out == [OC_ERR_INVALID] * 3, out
        stores[1].close()
        stores[1] = ob.StringFieldStorage(ctxs[1], _tiny(1, 1000, 1900))
        _on_ranks(3, lambda r: stores[r].sync_global())   # the group is still usable
        texts = synth.make_text_queries(50, 4, seed=3)
        res = _on_ranks(3, lambda r: TokenScoreContext(ctxs[r], None, stores[r]).execute_batch_arrays(
            TokenScoreParams(mode=MODE_FULLTEXT, sharded=True), texts))
        for r in range(3):
            _same_bytes(res[r], res[0], ("rank", r))
        df, avg = stores[0].read_global_df(0), stores[0].read_field(0)["avg_field_len"]
        stores[0].set_global(5000)
        assert np.array_equal(stores[0].read_global_df(0), df)
        assert stores[0].read_field(0)["avg_field_len"] == avg
    finally:
        for s in stores:
            s.close()
    lone = ob.Context(0)
    s = ob.StringFieldStorage(lone, _tiny(1, 0, 100))
    try:
        with pytest.raises(ob.OcError) as e:
            s.sync_global()
        assert e.value.code == OC_ERR_COMM
        assert s.read_global_df(0) is None
    finally:
        s.close()
        lone.close()


# ------------------------------------------------------------------ 4. two GPUs over NCCL
@gpu
def test_sync_two_gpus_nccl():
    """One rank per GPU (torchrun): commit and sync over NCCL, then the checks of test 1 on that path."""
    import os
    import subprocess
    import sys

    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29613",
                        os.path.join(root, "tests", "sharded_sync_worker.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "SYNC_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
