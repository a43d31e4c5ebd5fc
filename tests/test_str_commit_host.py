"""The numpy restatement of the string store's commit (str_commit_spec.py) on hand-worked cases; the GPU tests
(test_gpu_str_commit.py) hold the device commit to it byte for byte."""
import numpy as np
import pytest

import str_commit_spec as spec
from oramacore_b200.types import FieldPostings, StringIndexData


def csr(n_terms, posts, avg=0.0):
    """posts: (term, row, tf, len), any order."""
    posts = sorted(posts)
    offs = np.searchsorted(np.asarray([p[0] for p in posts], np.int64), np.arange(n_terms + 1)).astype(np.uint64)
    return FieldPostings(avg, offs, np.asarray([p[1] for p in posts], np.uint32), np.asarray([p[2] for p in posts], np.uint16),
                         np.asarray([p[3] for p in posts], np.uint16))


def posts_of(f):
    term = np.repeat(np.arange(f.n_terms), np.diff(f.term_offsets.astype(np.int64)))
    return list(zip(term.tolist(), f.post_row.tolist(), f.post_tf.tolist(), f.post_len.tolist()))


def test_ops_apply_in_order():
    s = spec.commit(spec.empty(1), [
        spec.insert(0, 1, 4, [(0, 1), (1, 3)]), spec.insert(0, 2, 2, [(1, 2)]),
        spec.insert(0, 1, 3, [(1, 1), (2, 2)]),              # the last insert of doc 1 wins
        spec.insert(0, 7, 5, [(1, 5)]), spec.delete(7),     # inserted then deleted: never a row
        spec.delete(9), spec.insert(0, 9, 1, [(2, 1)])])    # deleted then inserted: a new document
    assert s.row_doc_ids.tolist() == [1, 2, 9] and s.n_rows == 3 and s.document_count == 3
    f = s.fields[0]
    assert f.term_offsets.tolist() == [0, 0, 2, 4]
    assert posts_of(f) == [(1, 0, 1, 3), (1, 1, 2, 2), (2, 0, 2, 3), (2, 2, 1, 1)]
    assert f.avg_field_len == 2.0
    s2 = spec.commit(s, [spec.delete(2)])
    assert s2.row_doc_ids.tolist() == [1, 9] and s2.document_count == 2
    assert s2.fields[0].term_offsets.tolist() == [0, 0, 1, 3]
    assert posts_of(s2.fields[0]) == [(1, 0, 1, 3), (2, 0, 2, 3), (2, 1, 1, 1)]


def three_fields():
    return StringIndexData([csr(2, [(0, 0, 1, 5), (1, 1, 2, 7)], 6.0), csr(1, [(0, 0, 1, 3)], 3.0), csr(3, [(2, 1, 1, 4)], 4.0)],
                           2, 2, np.asarray([10, 20], np.uint64))


def test_reinsert_in_one_of_three_fields_keeps_the_others():
    s = spec.commit(three_fields(), [spec.insert(1, 10, 9, [(5, 2)])])   # term 5 is past the field's n_terms
    assert s.row_doc_ids.tolist() == [10, 20]
    assert posts_of(s.fields[0]) == [(0, 0, 1, 5), (1, 1, 2, 7)] and s.fields[0].avg_field_len == 6.0
    assert s.fields[1].n_terms == 6 and posts_of(s.fields[1]) == [(5, 0, 2, 9)] and s.fields[1].avg_field_len == 9.0
    assert posts_of(s.fields[2]) == [(2, 1, 1, 4)]


def test_insert_without_terms():
    s = spec.commit(three_fields(), [spec.insert(0, 30, 6, []), spec.insert(2, 20, 2, [])])
    assert s.row_doc_ids.tolist() == [10, 20, 30] and s.document_count == 3
    assert posts_of(s.fields[0]) == [(0, 0, 1, 5), (1, 1, 2, 7)]   # doc 30: a row, no postings, no length
    assert posts_of(s.fields[2]) == [] and s.fields[2].n_terms == 3   # doc 20's field 2 emptied
    assert s.fields[2].avg_field_len == 4.0                           # no length left: the old average stays


def test_identity_and_sparse_ids():
    base = StringIndexData([csr(1, [(0, r, 1, 2) for r in range(4)], 2.0)], 4, 4, None)
    s = spec.commit(base, [spec.insert(0, 4, 2, [(0, 1)])])
    assert s.row_doc_ids.tolist() == [0, 1, 2, 3, 4]
    s = spec.commit(base, [spec.delete(0), spec.insert(0, 1000, 2, [(0, 1)])])
    assert s.row_doc_ids.tolist() == [1, 2, 3, 1000]
    assert posts_of(s.fields[0]) == [(0, r, 1, 2) for r in range(4)]


def test_row_length_is_the_len_of_its_largest_term():
    # a loaded field may carry several len values per row: the posting of the largest term id decides
    base = StringIndexData([csr(4, [(0, 0, 1, 5), (3, 0, 1, 8), (1, 1, 1, 0), (2, 1, 1, 6), (3, 1, 1, 0)], 1.0)], 2, 2, None)
    s = spec.commit(base, [spec.insert(0, 2, 3, [(1, 1)])])
    assert s.fields[0].avg_field_len == float(np.float32((8 + 3) / 2))   # row 1's largest term has len 0: not counted


def test_empty_commit_keeps_everything():
    b = three_fields()
    s = spec.commit(b, [])
    assert s.row_doc_ids.tolist() == b.row_doc_ids.tolist() and s.document_count == 2
    for a, c in zip(b.fields, s.fields):
        assert posts_of(a) == posts_of(c) and a.term_offsets.tolist() == c.term_offsets.tolist()
        assert c.avg_field_len == a.avg_field_len


def test_duplicate_term_fails():
    with pytest.raises(spec.DuplicateTerm) as e:
        spec.commit(spec.empty(2), [spec.insert(1, 3, 2, [(4, 1), (4, 2)])])
    assert e.value.field == 1 and e.value.term == 4


def test_caller_owned_values_stay():
    s = spec.commit(three_fields(), [spec.insert(0, 40, 100, [(0, 1)])], global_count=True, global_avg=True)
    assert s.document_count == 2 and s.n_rows == 3
    assert [f.avg_field_len for f in s.fields] == [6.0, 3.0, 4.0]
