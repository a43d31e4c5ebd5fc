"""omc_spec.py against a dict replay of the same ops, IndexLoader's OMC handling (Index2, omc(), commit()) against the
reference's rule over random op streams, and the refusals of the OMC store and the loader that need no device.

The loader runs here on stand-ins for its device stores: only its own bookkeeping (which sets and deletes reach the
OMC store, and when) is under test, and the stand-in store applies omc_spec.commit, the rule the device commit is
checked against in test_gpu_omc.py."""
import ctypes as C

import numpy as np
import pytest

import omc_spec as spec
import oramacore_b200 as ob
from oramacore_b200 import _lib
from oramacore_b200.loader import IndexLoader


@pytest.mark.parametrize("seed", range(6))
def test_spec_matches_replay(seed):
    rng = np.random.default_rng(seed)
    doc, mult = spec.as_arrays({})
    state = {}
    for _ in range(8):
        ops = spec.random_ops(rng, int(rng.integers(0, 300)), int(rng.choice([5, 50, 2000])))
        doc, mult = spec.commit(doc, mult, ops)
        state = spec.replay(ops, state)
        d2, m2 = spec.as_arrays(state)
        assert np.array_equal(doc, d2)
        assert mult.tobytes() == m2.tobytes()
        assert np.all(np.diff(doc.astype(np.int64)) > 0)


def test_spec_call_order():
    # the last op for a document wins, whatever the order of the documents
    ops = [("set", 5, 2.0), ("set", 3, 1.5), ("delete", 5), ("set", 5, 4.0), ("set", 3, 0.5), ("delete", 9), ("set", 1, 3.0),
           ("delete", 1)]
    d, m = spec.commit(np.asarray([1, 2, 9], np.uint64), np.asarray([7.0, 8.0, 9.0], np.float32), ops)
    assert d.tolist() == [2, 3, 5] and m.tolist() == [8.0, 0.5, 4.0]
    d, m = spec.commit(d, m, [])
    assert d.tolist() == [2, 3, 5]


class _Stub:
    def __getattr__(self, name):
        return lambda *a, **k: None


class _SpecStore:
    """The OMC store's interface over omc_spec.commit."""

    def __init__(self):
        self.doc, self.mult, self.version, self.ops = np.zeros(0, np.uint64), np.zeros(0, np.float32), 0, []

    def set(self, doc_ids, mults):
        m = np.asarray(mults, np.float32)
        assert np.all(np.isfinite(m))
        self.ops += [("set", int(d), float(x)) for d, x in zip(doc_ids, m)]

    def delete(self, doc_ids):
        self.ops += [("delete", int(d)) for d in doc_ids]

    def commit(self):
        self.doc, self.mult = spec.commit(self.doc, self.mult, self.ops)
        self.ops, self.version = [], self.version + 1
        return {"version": self.version}

    def read(self):
        return self.doc, self.mult, self.version


def _loader():
    ld = IndexLoader.__new__(IndexLoader)
    ld.string_fields, ld.strs, ld.emb, ld.facets, ld.geo = [], _Stub(), None, None, {}
    ld.document_count, ld.max_doc_id, ld.nbits = 0, -1, 1
    ld._uncommitted_deleted, ld._live, ld._retired, ld._sorts = set(), None, [], {}
    ld.omc_store, ld._omc_log = _SpecStore(), []
    return ld


def _stream(rng, n_ops):
    """Index / Index2 / DeleteDocuments / commit ops as the write side emits them: an update deletes the old id and
    indexes a new one, and now and then a deleted id is indexed again before the commit (the loader's re-insert)."""
    nxt, live, out = 0, [], []
    vals = [None, None, 2.0, 0.5, 3.0, 1.25, 0.1]
    for _ in range(n_ops):
        r = rng.random()
        if r < 0.45 or not live:
            kind = "Index2" if rng.random() < 0.8 else "Index"
            op = {"type": kind, "doc_id": nxt, "indexed_values": []}
            if kind == "Index2":
                op["omc"] = vals[rng.integers(0, len(vals))]
            out.append(op)
            live.append(nxt)
            nxt += 1
        elif r < 0.65:   # update
            old = live.pop(int(rng.integers(0, len(live))))
            out.append({"type": "DeleteDocuments", "doc_ids": [old]})
            out.append({"type": "Index2", "doc_id": nxt, "indexed_values": [], "omc": vals[rng.integers(2, len(vals))]})
            live.append(nxt)
            nxt += 1
        elif r < 0.78:
            k = int(rng.integers(1, 4))
            gone = [live.pop(int(rng.integers(0, len(live)))) for _ in range(min(k, len(live)))]
            out.append({"type": "DeleteDocuments", "doc_ids": gone})
            if gone and rng.random() < 0.3:   # indexed again before the commit
                out.append({"type": "Index2", "doc_id": gone[0], "indexed_values": [], "omc": 9.5})
                live.append(gone[0])
        elif r < 0.9:
            out.append({"type": "commit"})
        else:
            out.append({"type": "search"})
    return out


@pytest.mark.parametrize("seed", range(8))
def test_loader_omc_rule(seed):
    rng = np.random.default_rng(100 + seed)
    ld, ref = _loader(), spec.IndexOmc()
    for op in _stream(rng, 250):
        t = op["type"]
        if t == "commit":
            ld.commit()
            ref.commit()
            doc, mult, _ = ld.omc_store.read()
            want = spec.as_arrays(ref.committed)
        elif t == "search":
            doc, mult, _ = ld.omc().read()
            want = spec.as_arrays(ref.all_omc())
        else:
            ld.apply(op)
            if t == "DeleteDocuments":
                ref.delete(op["doc_ids"])
            else:
                if int(op["doc_id"]) in ref.deleted:   # the loader's re-insert: the document is live again
                    ref.deleted.discard(int(op["doc_id"]))
                ref.index2(op["doc_id"], op.get("omc"))
            continue
        assert np.array_equal(doc, want[0]) and mult.tobytes() == want[1].tobytes(), (seed, op)


def test_loader_omc_before_commit_and_refusal():
    ld = _loader()
    ld.apply({"type": "Index2", "doc_id": 3, "indexed_values": [], "omc": 2.0})
    ld.apply({"type": "Index", "doc_id": 4, "indexed_values": []})
    ld.apply({"type": "Index2", "doc_id": 5, "indexed_values": [], "omc": None})
    assert ld.document_count == 3
    assert ld.omc_store.read()[0].tolist() == []          # nothing published yet
    assert ld.omc().read()[0].tolist() == [3]             # omc() publishes the log
    ld.apply({"type": "DeleteDocuments", "doc_ids": [3]})
    assert ld.omc().read()[0].tolist() == [3]             # a delete leaves the map at commit
    ld.commit()
    assert ld.omc_store.read()[0].tolist() == []
    for bad in (float("nan"), float("inf"), 1e39):        # 1e39 overflows f32
        with pytest.raises(ValueError):
            with np.errstate(over="ignore"):
                ld.apply({"type": "Index2", "doc_id": 9, "indexed_values": [], "omc": bad})
    assert ld.document_count == 2 and ld._omc_log == []


def test_c_refusals_without_device():
    L = ob.lib()
    d = np.asarray([1, 2], np.uint64)
    m = np.asarray([1.0, 2.0], np.float32)
    h = C.c_void_p()
    assert L.oc_omc_create(None, C.byref(h)) == -1
    assert not h.value
    assert L.oc_omc_set(None, d.ctypes.data, m.ctypes.data, 2) == -1
    assert L.oc_omc_delete(None, d.ctypes.data, 2) == -1
    assert L.oc_omc_commit_ex(None, None) == -1
    n = C.c_uint64(0)
    assert L.oc_omc_read(None, C.byref(n), None, None, None) == -1
    sizes = (C.c_size_t * 4)()
    L.oc_abi_sizes(sizes)
    assert sizes[0] == C.sizeof(_lib.SearchParams)
