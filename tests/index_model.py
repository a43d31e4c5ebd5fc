"""A plain-Python model of one index, fed the same operation dicts as IndexLoader.apply (the JSON shape of the
reference's IndexWriteOperation), with no device code.  The end-to-end tests compare every search of the loader with
the oracle run over what this model says the index holds.

Rules taken from the reference's read side:
  * document_count: +1 per Index op (read/index/mod.rs:1460), -len(doc_ids) per DeleteDocuments op whether or not an id
    was live, stopping at 0 (mod.rs:1417-1423).  It is the index's live count, and every search reads it as N of the
    idf (token_score.rs:221, read/index/mod.rs:411, read/search.rs:305-318): committed or not.
  * A delete takes effect at once in every store: string rows and embedding rows are tombstoned
    (string_field.rs:180-182, embedding_field.rs:240-242), and execute_filter excludes the uncommitted deletes from
    every where-set (filter.rs:344-392).
  * The chunks of one document sum their scores (embedding_field.rs:268-276) and the vector stage's depth is the
    query's limit (search.rs:330-336): both are the oracle's to apply, over the rows `emb_store` returns.
  * An update is DeleteDocuments(old id) then Index(new id) (write/index/mod.rs:375-410), so a document id is never
    reused; the model assumes that and the streams it is fed respect it.

Rules this project chose where the reference's storage crates are not vendored (loader.py's docstring,
str_commit_spec.py, DESIGN.md §0 rows f1 and f15):
  * String inserts become searchable at commit().  Per (field, document) the last insert wins and replaces the
    document's postings in that field; a delete cancels the inserts of its document made before it.
  * A row's length in a field is the insert's field_length, and avg_field_len is the mean of the non-zero lengths of
    the rows that hold a posting in that field (str_commit_spec.py); it keeps its old value when there is none.
  * A term's id is its position in the order the field's terms were first seen (the native dictionary hands out the
    next id to a new term); tf is the number of positions (exact + stemmed), at least 1, and tf and field_length are
    clamped to u16.
  * Embedding inserts are searchable at once.
  * Filter values become visible at refresh_facets() / commit(); filter deletes at once.  The DocumentId space of the
    filters is [0, max document id seen + 2), grown at each refresh (IndexLoader.refresh_facets)."""
from __future__ import annotations

import copy
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from oramacore_b200.types import FieldPostings, StringIndexData

U16_MAX = 65535


def _plain_or_array(v) -> list:
    return [v["Plain"]] if "Plain" in v else list(v["Array"])


class IndexModel:
    def __init__(self, string_fields: Sequence[str], dim: Optional[int] = None, bool_fields: Sequence[str] = (),
                 number_fields: Sequence[str] = (), string_filter_fields: Sequence[str] = (),
                 date_fields: Sequence[str] = (), geopoint_fields: Sequence[str] = ()):
        self.string_fields = list(string_fields)
        self.dim = dim
        nf = max(len(self.string_fields), 1)
        self.document_count = 0
        self.max_doc_id = -1
        self.nbits = 1
        self.uncommitted_deleted: set = set()
        # strings: per field {term: id}; committed {doc: (field_length, {term id: tf})}; ops since the last commit
        self.term_ids: List[Dict[str, int]] = [dict() for _ in range(nf)]
        self.committed: List[Dict[int, Tuple[int, Dict[int, int]]]] = [dict() for _ in range(nf)]
        self.avg = [0.0] * nf
        self.n_terms = [0] * nf
        self.pending: List[tuple] = []
        self._fields: Optional[list] = None                     # string_index's postings, built once per commit
        # embeddings: the live rows of each document with their insert sequence numbers
        self.emb_rows: Dict[int, List[Tuple[int, np.ndarray]]] = {}
        self._emb_seq = 0
        # filters: what apply() has seen (deletes applied) and what the last refresh published
        self.kinds = {**{f: "bool" for f in bool_fields}, **{f: "number" for f in number_fields},
                      **{f: "string" for f in string_filter_fields}, **{f: "date" for f in date_fields},
                      **{f: "geo" for f in geopoint_fields}}
        self.values: Dict[str, Dict[int, list]] = {f: {} for f in self.kinds}
        self.published: Dict[str, Dict[int, list]] = {f: {} for f in self.kinds}

    # ---------------------------------------------------------------- the op stream
    def apply(self, op: Dict) -> None:
        kind = op["type"]
        if kind == "Index":
            d = int(op["doc_id"])
            self.document_count += 1
            self.max_doc_id = max(self.max_doc_id, d)
            for v in op["indexed_values"]:
                self._value(d, v)
        elif kind == "IndexEmbedding":
            for d, vectors in op["data"]:
                self.max_doc_id = max(self.max_doc_id, int(d))
                for x in np.asarray(vectors, np.float32).reshape(-1, self.dim):
                    self.emb_rows.setdefault(int(d), []).append((self._emb_seq, x.copy()))
                    self._emb_seq += 1
        elif kind == "DeleteDocuments":
            ids = [int(x) for x in op["doc_ids"]]
            self.document_count = max(self.document_count - len(ids), 0)
            gone = set(ids)
            self.uncommitted_deleted |= gone
            self.pending += [("delete", d) for d in ids]
            for d in gone:
                self.emb_rows.pop(d, None)
                for vals in self.values.values():
                    vals.pop(d, None)
        else:
            raise ValueError(kind)

    def _value(self, d: int, v: Dict) -> None:
        t = v["type"]
        if t == "ScoreString2":
            fi = self.string_fields.index(v["field"])
            ids = self.term_ids[fi]
            tf = {}
            for name, pos in v["terms"].items():
                tid = ids.setdefault(name, len(ids))
                tf[tid] = min(max(1, len(pos.get("exact_positions", ())) + len(pos.get("positions", ()))), U16_MAX)
            self.pending.append(("insert", fi, d, min(int(v["field_length"]), U16_MAX), tf))
            return
        f = v["field"]
        cur = self.values[f]
        if t == "FilterBool":                            # replaces the document's value
            cur[d] = [bool(v["value"])]
        elif t == "FilterBool2":                         # adds to the document's set of bools
            cur.setdefault(d, []).extend(bool(b) for b in _plain_or_array(v["value"]))
        elif t == "FilterNumber":
            cur.setdefault(d, []).append(float(v["value"]))
        elif t == "FilterNumber2":
            (store, val), = v["value"].items()
            cur.setdefault(d, []).extend(float(int(x)) if store == "I64" else float(x) for x in _plain_or_array(val))
        elif t == "FilterString":
            cur.setdefault(d, []).append(str(v["value"]))
        elif t == "FilterString2":
            cur.setdefault(d, []).extend(str(x) for x in _plain_or_array(v["value"]))
        elif t in ("FilterDate", "FilterDate2"):
            xs = [v["value"]] if t == "FilterDate" else _plain_or_array(v["value"])
            cur.setdefault(d, []).extend(float(int(x)) for x in xs)
        elif t == "FilterGeoPoint2":
            cur.setdefault(d, []).extend((float(p["lat"]), float(p["lon"])) for p in _plain_or_array(v["value"]))
        else:
            raise ValueError(t)

    def refresh_facets(self) -> None:
        self.nbits = max(self.nbits, self.max_doc_id + 2)
        self.published = copy.deepcopy(self.values)

    def commit(self) -> None:
        nf = len(self.committed)
        work = [dict(c) for c in self.committed]
        fresh = [set() for _ in range(nf)]               # documents whose postings this commit wrote
        for op in self.pending:
            if op[0] == "delete":
                for fi in range(nf):
                    work[fi].pop(op[1], None)
                    fresh[fi].discard(op[1])
            else:
                _, fi, d, flen, tf = op
                work[fi][d] = (flen, tf)
                fresh[fi].add(d)
        for fi in range(nf):
            tids = [t for d in fresh[fi] for t in work[fi][d][1]]
            self.n_terms[fi] = max([self.n_terms[fi]] + [t + 1 for t in tids])
            lens = [flen for flen, tf in work[fi].values() if tf and flen > 0]
            if lens:
                self.avg[fi] = float(np.float32(float(sum(lens)) / float(len(lens))))
        self.committed, self.pending = work, []
        self._fields = None
        self.uncommitted_deleted = set()
        self.refresh_facets()

    # ---------------------------------------------------------------- what a search sees
    def rows(self) -> np.ndarray:
        """The committed string rows' document ids, ascending."""
        return np.asarray(sorted(set().union(*[c.keys() for c in self.committed])), np.uint64)

    def string_index(self) -> StringIndexData:
        """The committed string documents, with N = the live document_count."""
        docs = self.rows()
        if self._fields is None:
            row_of = {int(d): r for r, d in enumerate(docs.tolist())}
            self._fields = []
            for fi, c in enumerate(self.committed):
                # term-major, rows ascending inside a term
                post = sorted((t, row_of[d], tf, flen) for d, (flen, tfs) in c.items() for t, tf in tfs.items())
                terms = np.asarray([p[0] for p in post], np.int64)
                offs = np.searchsorted(terms, np.arange(self.n_terms[fi] + 1)).astype(np.uint64)
                col = lambda i, t: np.asarray([p[i] for p in post], t)  # noqa: E731
                self._fields.append(FieldPostings(self.avg[fi], offs, col(1, np.uint32), col(2, np.uint16), col(3, np.uint16)))
        return StringIndexData(self._fields, int(docs.shape[0]), self.document_count, docs)

    def live_rows(self) -> Optional[np.ndarray]:
        """The committed string rows not deleted since, or None when none was: the filter a fulltext search of the
        committed snapshot applies through its tombstones."""
        docs = self.rows()
        dead = np.isin(docs, np.asarray(sorted(self.uncommitted_deleted), np.uint64))
        return docs[~dead] if dead.any() else None

    def emb_store(self, orc):
        """An oracle.EmbStore of the live embedding rows, in insert order, with their document ids."""
        e = sorted((seq, d, x) for d, xs in self.emb_rows.items() for seq, x in xs)
        rows = np.asarray([x for _, _, x in e], np.float32).reshape(-1, self.dim)
        return orc.EmbStore(rows, row_doc_ids=np.asarray([d for _, d, _ in e], np.uint64))

    def filter_values(self) -> Dict[str, tuple]:
        """The published filter values as test_where_host.host_where takes them: bool {doc: {bools}}, string
        {doc: [keys]}, number / date (docs, f64 values), geo (docs, lat, lon)."""
        out = {}
        for f, kind in self.kinds.items():
            vals = self.published[f]
            if kind == "bool":
                out[f] = ("bool", {d: set(bs) for d, bs in vals.items()})
            elif kind == "string":
                out[f] = ("string", {d: list(ks) for d, ks in vals.items()})
            elif kind == "geo":
                e = [(d, la, lo) for d, ps in sorted(vals.items()) for la, lo in ps]
                out[f] = ("geo", tuple(np.asarray([x[i] for x in e], np.float64 if i else np.int64) for i in range(3)))
            else:
                docs, xs = self.sort_values(f)
                out[f] = (kind, (docs.astype(np.int64), xs))
        return out

    def sort_values(self, field: str) -> Tuple[np.ndarray, np.ndarray]:
        """(docs, f64 values) of a published number, date or bool field, a document once per value."""
        e = [(d, float(x)) for d, xs in sorted(self.published[field].items()) for x in xs]
        return np.asarray([d for d, _ in e], np.uint64), np.asarray([x for _, x in e], np.float64)
