"""Host checks of tests/index_model.py, the plain model of one index the lifecycle tests compare the loader with: its
string side against str_commit_spec.commit on random op streams, the document-count rule of the reference
(read/index/mod.rs:1417-1423, 1460) on small hand-written streams, and its where-sets (host_where over the values it
publishes) for uncommitted deletes and for values queued but not yet published."""
import numpy as np
import pytest

import str_commit_spec as spec
from index_model import IndexModel
from oramacore_b200.where import parse_where
from test_gpu_index_lifecycle import FILTERS, STRING_FIELDS, Stream, _tree
from test_where_host import host_where


def _index(d, **values):
    vals = []
    for f, text in values.items():
        if f in STRING_FIELDS:
            toks = text.split()
            terms = {}
            for i, t in enumerate(toks):
                terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
            vals.append({"type": "ScoreString2", "field": f, "field_length": len(toks), "terms": terms})
        elif isinstance(text, bool):
            vals.append({"type": "FilterBool", "field": f, "value": text})
        elif isinstance(text, str):
            vals.append({"type": "FilterString", "field": f, "value": text})
        else:
            vals.append({"type": "FilterNumber", "field": f, "value": text})
    return {"type": "Index", "doc_id": d, "indexed_values": vals}


def _delete(*ids):
    return {"type": "DeleteDocuments", "doc_ids": list(ids)}


def _spec_ops(ops, term_ids):
    """The string side of an op stream as str_commit_spec ops, with term ids given out in first-seen order."""
    out = []
    for op in ops:
        if op["type"] == "DeleteDocuments":
            out += [spec.delete(d) for d in op["doc_ids"]]
        elif op["type"] == "Index":
            for v in op["indexed_values"]:
                if v["type"] == "ScoreString2":
                    fi = STRING_FIELDS.index(v["field"])
                    pairs = [(term_ids[fi].setdefault(t, len(term_ids[fi])),
                              max(1, len(p["exact_positions"]) + len(p["positions"]))) for t, p in v["terms"].items()]
                    out.append(spec.insert(fi, op["doc_id"], v["field_length"], pairs))
    return out


def _same(a, b):
    assert a.n_rows == b.n_rows and np.array_equal(spec.row_docs(a), spec.row_docs(b))
    for fa, fb in zip(a.fields, b.fields):
        assert fa.avg_field_len == fb.avg_field_len
        for x in ("term_offsets", "post_row", "post_tf", "post_len"):
            assert np.array_equal(getattr(fa, x), getattr(fb, x)), x


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_string_side_matches_the_commit_spec(seed):
    stream = Stream(seed, 4, 300)
    model = IndexModel(STRING_FIELDS, dim=4, **FILTERS)
    snap, term_ids = spec.empty(2), [{}, {}]
    for n_new in (200, 150, 150, 100):
        ops = stream.round(n_new)
        for op in ops:
            model.apply(op)
        model.commit()
        snap = spec.commit(snap, _spec_ops(ops, term_ids))
        got = model.string_index()
        _same(got, snap)
        # document_count is where the two part: the spec counts rows, the model follows Index::document_count
        assert snap.document_count == snap.n_rows
        n_index = sum(op["type"] == "Index" for op in ops)
        assert got.document_count == model.document_count and n_index > 0
    assert model.term_ids == term_ids


def test_document_count_rule():
    m = IndexModel(STRING_FIELDS)
    m.apply(_index(0, title="a b"))
    m.apply(_index(1))                                   # no string value: still a document
    assert m.document_count == 2                         # pending Index ops count at once
    assert m.string_index().document_count == 2 and m.string_index().n_rows == 0
    m.commit()
    m.apply(_index(2, body="c"))                         # counted, but not searchable before the commit
    assert m.string_index().document_count == 3 and m.string_index().n_rows == 1
    m.apply(_delete(77))                                 # an id never indexed subtracts one
    assert m.document_count == 2
    m.apply(_delete(0))
    m.apply(_delete(0))                                  # and so does a second delete of the same id
    assert m.document_count == 0
    m.apply(_delete(1, 2, 3))                            # never below 0
    assert m.document_count == 0
    m.apply(_index(4, title="d"))
    assert m.document_count == 1
    m.commit()
    assert m.string_index().document_count == 1 and m.rows().tolist() == [4]


def test_uncommitted_deletes_and_tombstones():
    m = IndexModel(STRING_FIELDS, dim=2)
    m.apply(_index(0, title="a"))
    m.apply(_index(1, title="a b"))
    m.apply({"type": "IndexEmbedding", "data": [(0, [[1, 0]]), (1, [[0, 1], [1, 1]])]})
    m.commit()
    m.apply(_delete(1))
    assert m.rows().tolist() == [0, 1]                   # the row stays until the commit ...
    assert m.live_rows().tolist() == [0]                 # ... tombstoned
    assert list(m.emb_rows) == [0]                       # embedding rows go at once
    m.apply(_index(2, title="b"))
    m.apply(_delete(2))                                  # cancels its own pending insert
    m.commit()
    assert m.rows().tolist() == [0] and m.live_rows() is None


def test_last_insert_wins_and_avg_field_len():
    m = IndexModel(["title"])
    m.apply(_index(5, title="a a b"))
    m.apply(_index(6, title=""))                         # a row without postings: no length
    m.commit()
    s = m.string_index()
    assert s.fields[0].avg_field_len == 3.0 and s.n_rows == 2
    m.apply(_index(9, title="c d"))
    m.commit()
    assert m.string_index().fields[0].avg_field_len == 2.5
    assert m.string_index().fields[0].post_tf.tolist() == [2, 1, 1, 1]


def test_where_sets_follow_publish_and_deletes():
    m = IndexModel(STRING_FIELDS, **FILTERS)
    for d in range(6):
        m.apply(_index(d, flag=d % 2 == 0, cat="k1" if d < 3 else "k2", price=float(d)))
    w = parse_where({"flag": True})
    assert host_where(w, m.filter_values(), m.nbits, m.uncommitted_deleted) == set()   # queued, not published
    m.refresh_facets()
    assert m.nbits == 7
    assert host_where(w, m.filter_values(), m.nbits, m.uncommitted_deleted) == {0, 2, 4}
    m.apply(_delete(2))                                  # visible at once
    assert host_where(w, m.filter_values(), m.nbits, m.uncommitted_deleted) == {0, 4}
    m.apply(_index(8, flag=True))                        # queued: beyond the published DocumentId space as well
    nw = parse_where({"not": {"cat": "k1"}})
    assert host_where(nw, m.filter_values(), m.nbits, m.uncommitted_deleted) == {3, 4, 5, 6}
    m.commit()
    assert m.nbits == 10 and not m.uncommitted_deleted
    assert host_where(w, m.filter_values(), m.nbits, m.uncommitted_deleted) == {0, 4, 8}
    # the deleted document's values are gone with the commit; a `not` covers the whole DocumentId space
    assert host_where(nw, m.filter_values(), m.nbits, m.uncommitted_deleted) == {2, 3, 4, 5, 6, 7, 8, 9}


def test_generated_where_clauses_on_the_model():
    """The generated trees over the model's published values: a document deleted since the last publish is in no
    where-set, and a document whose values are only queued is in a set only through a `not`."""
    stream = Stream(5, 4, 200)
    m = IndexModel(STRING_FIELDS, dim=4, **FILTERS)
    rng = np.random.default_rng(0)
    for op in stream.round(300):
        m.apply(op)
    m.refresh_facets()
    published = set().union(*[set(v) for v in m.published.values()])
    for op in stream.round(100):
        m.apply(op)
    queued = set().union(*[set(v) for v in m.values.values()]) - published
    assert m.uncommitted_deleted and queued
    for _ in range(200):
        where = _tree(rng)
        s = host_where(parse_where(where), m.filter_values(), m.nbits, m.uncommitted_deleted)
        assert not s & m.uncommitted_deleted
        assert not s & queued or "not" in str(where)
