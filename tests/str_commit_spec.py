"""The commit contract of the string store (oc_str_commit), restated in numpy.

From the published snapshot and the ops since the last commit, in call order, `commit` gives the next snapshot: its
row -> document map, every field's CSR, avg_field_len and document_count.  The rules:

  - a delete tombstones the committed rows of its document and cancels the inserts of that document made before it;
    an insert after the delete is a new document;
  - per (field, document) the last insert that no later delete cancelled wins, and it replaces every posting the
    document had in that field, whether it lists terms or not; the document's other fields keep their postings;
  - the rows of the next snapshot are the alive committed documents and the documents with a winning insert in any
    field, ascending;
  - postings are term-major, rows ascending inside a term; n_terms = max(old n_terms, largest inserted term + 1);
  - a term listed twice in one insert of a document fails the commit (DuplicateTerm);
  - a row's length in a field is the `len` of its posting with the largest term id; avg_field_len is the mean of the
    non-zero lengths (sum in integers, then float(sum / count) in double) and keeps its old value when no row has one;
  - document_count is the number of rows.
  `global_count` / `global_avg` (oc_str_set_global): the caller owns document_count / avg_field_len, which stay."""
from typing import List, Sequence, Tuple

import numpy as np

from oramacore_b200.types import FieldPostings, StringIndexData

U64_32 = np.uint64(32)


class DuplicateTerm(ValueError):
    def __init__(self, field: int, term: int):
        super().__init__(f"field {field}: term {term} listed twice in one insert of a document")
        self.field, self.term = field, term


def empty(n_fields: int) -> StringIndexData:
    e = FieldPostings(0.0, np.zeros(1, np.uint64), np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(0, np.uint16))
    return StringIndexData([FieldPostings(e.avg_field_len, e.term_offsets.copy(), e.post_row, e.post_tf, e.post_len)
                            for _ in range(n_fields)], 0, 0, np.zeros(0, np.uint64))


def row_docs(s: StringIndexData) -> np.ndarray:
    return np.arange(s.n_rows, dtype=np.uint64) if s.row_doc_ids is None else np.asarray(s.row_doc_ids, np.uint64)


def insert(field: int, doc: int, field_len: int, pairs: Sequence[Tuple[int, int]]):
    """An insert op: pairs are (term id, tf), in the order the caller lists them."""
    return ("insert", int(field), int(doc), int(field_len), [(int(t), int(f)) for t, f in pairs])


def delete(doc: int):
    return ("delete", int(doc))


def commit(base: StringIndexData, ops: List[tuple], global_count: bool = False, global_avg: bool = False) -> StringIndexData:
    nf = len(base.fields)
    old_docs = row_docs(base)
    alive = np.ones(base.n_rows, bool)
    deleted_at, last = {}, [dict() for _ in range(nf)]
    for seq, op in enumerate(ops, 1):
        if op[0] == "delete":
            deleted_at[op[1]] = seq
            r = int(np.searchsorted(old_docs, np.uint64(op[1])))
            if r < base.n_rows and int(old_docs[r]) == op[1]:
                alive[r] = False
        else:
            _, f, doc, flen, pairs = op
            last[f][doc] = (seq, flen, pairs)
    wins = [{d: v for d, v in lf.items() if v[0] > deleted_at.get(d, 0)} for lf in last]
    pdocs = np.asarray(sorted(set().union(*[w.keys() for w in wins])), np.uint64)
    docs = np.union1d(old_docs[alive], pdocs).astype(np.uint64)
    new_of_old = np.searchsorted(docs, old_docs).astype(np.int64)
    fields = []
    for fi, of in enumerate(base.fields):
        off = of.term_offsets.astype(np.int64)
        term_of = np.repeat(np.arange(of.n_terms, dtype=np.uint64), np.diff(off))
        replaced = np.zeros(docs.shape[0] + 1, bool)
        replaced[np.searchsorted(docs, np.asarray(list(wins[fi].keys()), np.uint64))] = True
        nr = new_of_old[of.post_row]
        keep = alive[of.post_row] & ~replaced[nr]
        old_key = (term_of[keep] << U64_32) | nr[keep].astype(np.uint64)
        pt, pr, ptf, plen = [], [], [], []
        for doc, (_, flen, pairs) in wins[fi].items():
            row = int(np.searchsorted(docs, np.uint64(doc)))
            for t, tf in pairs:
                pt.append(t); pr.append(row); ptf.append(tf); plen.append(flen)
        pend_key = (np.asarray(pt, np.uint64) << U64_32) | np.asarray(pr, np.uint64)
        order = np.argsort(pend_key, kind="stable")
        pend_key = pend_key[order]
        dup = np.nonzero(pend_key[1:] == pend_key[:-1])[0]
        if dup.size:
            raise DuplicateTerm(fi, int(pend_key[dup[0] + 1] >> U64_32))
        # the survivors are already in (term, row) order: the pending postings merge in at their sorted places
        n = old_key.shape[0] + pend_key.shape[0]
        at_pend = np.searchsorted(old_key, pend_key) + np.arange(pend_key.shape[0])
        is_old = np.ones(n, bool)
        is_old[at_pend] = False
        key = np.empty(n, np.uint64)
        key[is_old], key[at_pend] = old_key, pend_key
        tf = np.empty(n, np.uint16)
        tf[is_old], tf[at_pend] = of.post_tf[keep], np.asarray(ptf, np.uint16)[order]
        ln = np.empty(n, np.uint16)
        ln[is_old], ln[at_pend] = of.post_len[keep], np.asarray(plen, np.uint16)[order]
        terms = key >> U64_32
        rows = (key & np.uint64(0xffffffff)).astype(np.uint32)
        n_terms = max(of.n_terms, int(max(pt)) + 1 if pt else 0)
        offs = np.searchsorted(terms, np.arange(n_terms + 1, dtype=np.uint64)).astype(np.uint64)
        avg = of.avg_field_len
        if not global_avg:
            last_post = np.full(docs.shape[0], -1, np.int64)   # per row: its posting of the largest term id
            np.maximum.at(last_post, rows.astype(np.int64), np.arange(n, dtype=np.int64))
            lens = ln[last_post[last_post >= 0]].astype(np.int64)
            lens = lens[lens > 0]
            if lens.size:
                avg = float(np.float32(float(int(lens.sum())) / float(lens.size)))
        fields.append(FieldPostings(avg, offs, rows, tf, ln))
    dc = base.document_count if global_count else int(docs.shape[0])
    return StringIndexData(fields, int(docs.shape[0]), dc, docs)
