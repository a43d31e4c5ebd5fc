"""OMC through IndexLoader with the ops the reference's write side emits (Index2, write/index/mod.rs:451-472): the cases
of src/tests/omc_test.rs, and random Index / Index2 / IndexEmbedding / DeleteDocuments streams against IndexModel
extended with the index's OMC rule (omc_spec.IndexOmc), searched before a commit (IndexLoader.omc(): the log over the
committed map) and after commit()."""
import numpy as np
import pytest

import oramacore_b200 as ob
import omc_spec as spec
from helpers import assert_topk_equal
from index_model import IndexModel
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from test_gpu_index_lifecycle import FILTERS, STRING_FIELDS, Expect, Stream
from test_gpu_loader import _index_op
from test_gpu_parity import ATOL
from test_gpu_topn_paths import _eq, _sorted, page

pytestmark = pytest.mark.gpu


def _index2(doc_id, text, omc=None):
    op = _index_op(doc_id, text)
    op["type"] = "Index2"
    op["omc"] = omc
    return op


def _scores(ld, term, omc=True):
    kw = dict(omc_store=ld.omc()) if omc else {}
    h = ld.context().execute_batch(ob.TokenScoreParams(mode=MODE_FULLTEXT, **kw), ld.resolve([term]))[0]
    return dict(zip(h.doc_ids.tolist(), h.scores.tolist())), h.count


def test_multiplies_and_persists(gpu_ctx):
    # omc_test.rs:8-139: two identical documents, one with _omc 2.0 (3.0): its score is 2x (3x), before and after commit
    for m in (2.0, 3.0):
        ld = IndexLoader(gpu_ctx, ["text"])
        ld.apply_all([_index2(1, "machine learning", m), _index2(2, "machine learning")])
        ld.commit()
        s, cnt = _scores(ld, "machine learning")
        assert cnt == 2 and s[1] == np.float32(np.float32(s[2]) * np.float32(m))
        ld.commit()   # a commit with nothing queued keeps the map
        assert _scores(ld, "machine learning")[0] == s
        ld.close()


def test_removed_on_delete_and_updated(gpu_ctx):
    # omc_test.rs:205-371: a deleted document's multiplier is gone; an update (delete + Index2 with a new id) carries the
    # new multiplier
    ld = IndexLoader(gpu_ctx, ["text"])
    ld.apply_all([_index2(1, "machine learning", 2.0), _index2(2, "machine learning"), _index2(3, "machine learning", 5.0)])
    ld.commit()
    ld.apply({"type": "DeleteDocuments", "doc_ids": [1]})
    ld.apply(_index2(4, "machine learning", 0.5))       # the update of document 1
    ld.apply({"type": "DeleteDocuments", "doc_ids": [3]})
    ld.commit()
    s, cnt = _scores(ld, "machine learning")
    assert cnt == 2 and set(s) == {2, 4}
    assert s[4] == np.float32(np.float32(s[2]) * np.float32(0.5))   # 2 and 4 hold the same text
    d, m, _ = ld.omc_store.read()
    assert d.tolist() == [4] and m.tolist() == [0.5]    # 1 and 3 left the map at the commit
    ld.close()


def test_various_and_fractional_and_none(gpu_ctx):
    # omc_test.rs:422-560: several multipliers and fractional ones; omc None leaves the score
    mults = [None, 1.5, 0.25, 10.0, 0.75, 4.0]
    ld = IndexLoader(gpu_ctx, ["text"])
    ld.apply_all([_index2(i, "search engine", m) for i, m in enumerate(mults)])
    ld.commit()
    s, _ = _scores(ld, "search engine")
    plain, _ = _scores(ld, "search engine", omc=False)
    for i, m in enumerate(mults):
        assert s[i] == (plain[i] if m is None else np.float32(np.float32(plain[i]) * np.float32(m))), (i, m)
    assert sorted(s, key=lambda d: (-s[d], d))[:2] == [3, 5]
    ld.close()


def test_visible_before_commit(gpu_ctx):
    # get_all_omc (mod.rs:1720-1739): a new multiplier counts at once; embeddings are searchable at once too
    dim = 16
    rng = np.random.default_rng(3)
    v = rng.standard_normal((3, dim)).astype(np.float32)
    ld = IndexLoader(gpu_ctx, ["text"], embedding_dim=dim)
    ld.apply_all([_index2(i, "alpha") for i in range(3)])
    ld.apply({"type": "IndexEmbedding", "data": [(i, [v[i].tolist()]) for i in range(3)]})
    tsc = ld.context()
    p = lambda **kw: ob.TokenScoreParams(mode=MODE_VECTOR, limit_hint=3, similarity=-1.0, **kw)  # noqa: E731
    before = tsc.execute_batch(p(omc_store=ld.omc()), None, v[:1])[0]
    ld.apply(_index2(7, None, 6.0))                      # a document with a multiplier only ...
    ld.apply({"type": "Index2", "doc_id": 1, "indexed_values": [], "omc": 3.0})   # ... and document 1 again
    after = tsc.execute_batch(p(omc_store=ld.omc()), None, v[:1])[0]
    sb, sa = dict(zip(before.doc_ids.tolist(), before.scores.tolist())), dict(zip(after.doc_ids.tolist(), after.scores.tolist()))
    assert sa[1] == np.float32(np.float32(sb[1]) * np.float32(3.0)) and sa[0] == sb[0]
    ld.close()


# ---------------------------------------------------------------- random streams against the model
class OmcModel(IndexModel):
    """IndexModel with the index's OMC state: Index2 is Index plus the OMC log; commit merges it."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.omc = spec.IndexOmc()

    def apply(self, op):
        if op["type"] == "Index2":
            self.omc.index2(op["doc_id"], op["omc"])
            op = {**op, "type": "Index"}
        elif op["type"] == "DeleteDocuments":
            self.omc.delete(op["doc_ids"])
        super().apply(op)

    def commit(self):
        super().commit()
        self.omc.commit()


def _with_omc(ops, rng):
    out = []
    for op in ops:
        if op["type"] == "Index" and rng.random() < 0.8:
            op = {**op, "type": "Index2", "omc": None if rng.random() < 0.3 else float(rng.choice([0.5, 2.0, 3.0, 1.25, 0.1]))}
        out.append(op)
    return out


def _check(tag, ld, model, orc, stream, rng):
    ex = Expect(orc, model)
    try:
        d, m = spec.as_arrays(model.omc.all_omc())
        store = ld.omc()
        rd, rm, _ = store.read()
        assert np.array_equal(rd, d) and rm.tobytes() == m.tobytes(), tag
        tsc = ld.context()
        texts = stream.texts(10)
        batch = ld.resolve(texts)
        qs = [batch.query(i) for i in range(batch.n_queries)]
        qv = stream.qvecs(len(qs))
        omc = lambda mp: orc.apply_omc(mp, d, m) if d.shape[0] else mp  # noqa: E731
        for limit, offset in [(10, 0), (7, 20)]:
            hits = tsc.execute_batch(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=limit, offset=offset, omc_store=store), batch)
            for i, h in enumerate(hits):
                _eq(h, page(_sorted(*omc(ex.ft(qs[i]))), limit, offset), (tag, "fulltext", i, limit, offset))
        for mode in (MODE_VECTOR, MODE_HYBRID):
            hits = tsc.execute_batch(ob.TokenScoreParams(mode=mode, limit_hint=20, similarity=0.0, omc_store=store),
                                     None if mode == MODE_VECTOR else batch, qv)
            for i, h in enumerate(hits):
                mp = ex.vec(qv[i], 20, 0.0) if mode == MODE_VECTOR else ex.hybrid(qs[i], qv[i], 20, 0.0)
                ed, es, cnt = page(_sorted(*omc(mp)), 20, 0)
                assert h.count == cnt, (tag, mode, i, h.count, cnt)
                assert_topk_equal(h.doc_ids, h.scores, ed, es, atol=ATOL)
    finally:
        ex.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_streams_against_the_model(gpu_ctx, orc, seed):
    dim = 32
    stream = Stream(seed, dim, 600)
    rng = np.random.default_rng(seed + 50)
    ld = IndexLoader(gpu_ctx, STRING_FIELDS, embedding_dim=dim, **FILTERS)
    model = OmcModel(STRING_FIELDS, dim=dim, **FILTERS)
    try:
        for rnd in range(3):
            for op in _with_omc(stream.round(400), rng):
                ld.apply(op)
                model.apply(op)
            _check((seed, rnd, "before commit"), ld, model, orc, stream, rng)
            ld.commit()
            model.commit()
            _check((seed, rnd, "after commit"), ld, model, orc, stream, rng)
    finally:
        ld.close()
