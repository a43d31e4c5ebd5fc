"""Loader / refresher of the device-resident stores from the reference's own write-operation stream.

The reference's read side is fed by `Index::update_data(IndexWriteOperation)` (read/index/mod.rs:1436-1705):
  * `Index { doc_id, indexed_values }` — `document_count += 1`, then per value
      ScoreString2(field, IndexedValue{field_length: u16, terms: {term -> TermData{exact_positions, positions}}})
                                              -> StringFieldStorage::insert   (string_field.rs:155-177, mod.rs:1509-1515)
      FilterBool / FilterNumber / FilterString -> the filter fields the facets and filters read (mod.rs:1461-1497)
      FilterGeoPoint2(field, Plain(point) | Array([points]))  -> the geopoint fields of the where-filter (mod.rs:1556-1565, 1678-1687)
      FilterBool2 / FilterString2 / FilterDate / FilterDate2 / FilterNumber2 -> the same filter fields as the write side
                                              emits them today (write/index/fields.rs:312-325, 345-353, 401-423, 467-504)
  * `IndexEmbedding { data: field -> [(doc_id, vectors)] }` -> EmbeddingFieldStorage::insert (mod.rs:1688-1698)
  * `DeleteDocuments { doc_ids }` — uncommitted deletes, excluded from every search at once (mod.rs:1346-1427)
and `commit` / `compact` lay the pending data out (`CURRENT` + `versions/<n>`, embedding_field.rs:91-95).

`IndexLoader.apply(op)` takes the same operations as plain dicts (the JSON shape of the reference's enum), resolves
terms to stable term ids through the native dictionary (oc_dict_*), and drives the C ABI: oc_str_insert /
oc_str_delete / oc_str_commit (snapshot swap: searches keep running on the previous version while a commit builds
the next), oc_emb_insert / oc_emb_delete (live) and oc_emb_compact at commit.  `refresh_facets()` lays the accumulated filter fields out for
oc_search_facets and rebuilds the geopoint field handles (`geo`, oc_geo_field_*); `where_filter(where)` evaluates a
where-clause over them (where.py).  tf of a term = number of positions (exact + stemmed), as StringStorage counts them."""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np

from .engine import (Context, DeviceFilter, EmbeddingFieldStorage, FacetStore, GeoPointField, StringFieldStorage,
                     TermDictionary, TokenScoreContext)
from .where import WhereFilter, WhereProgram, check_where_keys, compile_where, evaluate_where, parse_where

_F64_INT_MAX = 1 << 53   # I64 values beyond +-2^53 would not survive the trip through a double


def _plain_or_array(v) -> list:
    """oramacore_fields' IndexedValue: {"Plain": x} or {"Array": [x, ...]}."""
    return [v["Plain"]] if "Plain" in v else list(v["Array"])


def _exact_i64(x, what: str) -> float:
    if abs(int(x)) > _F64_INT_MAX:
        raise ValueError(f"{what} {x}: beyond +-2^53, not exact as a double")
    return float(int(x))


class IndexLoader:
    def __init__(self, ctx: Context, string_fields: Sequence[str], embedding_model: Optional[str] = None,
                 embedding_dim: Optional[int] = None, bool_fields: Sequence[str] = (), number_fields: Sequence[str] = (),
                 string_filter_fields: Sequence[str] = (), geopoint_fields: Sequence[str] = (), date_fields: Sequence[str] = ()):
        self.ctx = ctx
        self.string_fields = list(string_fields)
        self.dict = TermDictionary(max(len(self.string_fields), 1))
        self.strs = StringFieldStorage.empty(ctx, max(len(self.string_fields), 1))
        self.emb = EmbeddingFieldStorage(ctx, embedding_model or "BGESmall", dim=embedding_dim) if (embedding_model or embedding_dim) else None
        self._bool = {f: ({}) for f in bool_fields}            # field -> {doc: bool} (FilterBool) or {doc: {bools}}
        self._num = {f: ({}) for f in number_fields}           # field -> {doc: [numbers]}
        self._strf = {f: ({}) for f in string_filter_fields}   # field -> {doc: [keys]}
        self._geo = {f: ({}) for f in geopoint_fields}         # field -> {doc: [(lat, lon)]}
        self._date = {f: ({}) for f in date_fields}            # field -> {doc: [ms]}
        self.document_count = 0
        self.max_doc_id = -1
        self._deleted: set = set()
        self._uncommitted_deleted: set = set()                 # deletes since the last commit (filter.rs:344-392)
        self.facets: Optional[FacetStore] = None
        self.geo: Dict[str, GeoPointField] = {}
        self.nbits = 1                                         # DocumentId space of `facets` and `geo`
        self._live: Optional[DeviceFilter] = None              # NOT(uncommitted deletes) of where_program, built once
        self._retired: List[DeviceFilter] = []                 # earlier ones, which programs may still point at

    # ---- Index::update_data
    def apply(self, op: Dict) -> None:
        kind = op["type"]
        if kind == "Index":
            d = int(op["doc_id"])
            self.document_count += 1
            self.max_doc_id = max(self.max_doc_id, d)
            self._deleted.discard(d)
            if d in self._uncommitted_deleted:
                self._uncommitted_deleted.discard(d)
                self._retire_live()
            for v in op["indexed_values"]:
                t = v["type"]
                if t == "ScoreString2":
                    fi = self.string_fields.index(v["field"])
                    terms = v["terms"]                                  # {term: {"exact_positions": [...], "positions": [...]}}
                    names = list(terms)
                    ids = self.dict.add_terms(fi, names) if names else np.zeros(0, np.uint32)
                    tf = {int(i): max(1, len(terms[n].get("exact_positions", ())) + len(terms[n].get("positions", ()))) for i, n in zip(ids, names)}
                    self.strs.insert(d, fi, int(v["field_length"]), tf)
                elif t == "FilterBool":
                    self._bool[v["field"]][d] = bool(v["value"])
                elif t == "FilterNumber":
                    self._num[v["field"]].setdefault(d, []).append(float(v["value"]))
                elif t == "FilterString":
                    self._strf[v["field"]].setdefault(d, []).append(str(v["value"]))
                elif t == "FilterGeoPoint2":
                    # GeoPointIndexedValue: {"Plain": {"lat", "lon"}} or {"Array": [{"lat", "lon"}, ...]}
                    val = v["value"]
                    pts = [val["Plain"]] if "Plain" in val else list(val["Array"])
                    self._geo[v["field"]].setdefault(d, []).extend((float(p["lat"]), float(p["lon"])) for p in pts)
                elif t == "FilterBool2":
                    bs = self._bool[v["field"]].get(d)
                    bs = self._bool[v["field"]][d] = {bs} if isinstance(bs, bool) else (bs or set())
                    bs.update(bool(b) for b in _plain_or_array(v["value"]))
                elif t == "FilterNumber2":
                    # NumberFieldIndexedValue: {"I64": {"Plain": x} | {"Array": [...]}} or {"F64": ...}
                    (store, val), = v["value"].items()
                    xs = _plain_or_array(val)
                    xs = [_exact_i64(x, "I64 value") for x in xs] if store == "I64" else [float(x) for x in xs]
                    self._num[v["field"]].setdefault(d, []).extend(xs)
                elif t == "FilterString2":
                    self._strf[v["field"]].setdefault(d, []).extend(str(x) for x in _plain_or_array(v["value"]))
                elif t in ("FilterDate", "FilterDate2"):
                    xs = [v["value"]] if t == "FilterDate" else _plain_or_array(v["value"])
                    self._date[v["field"]].setdefault(d, []).extend(int(x) for x in xs)
                else:
                    raise ValueError(f"unsupported indexed value {t!r} (outside the search hot path)")
        elif kind == "IndexEmbedding":
            for d, vectors in op["data"]:
                self.max_doc_id = max(self.max_doc_id, int(d))
                self.emb.insert(int(d), vectors)
        elif kind == "DeleteDocuments":
            ids = [int(x) for x in op["doc_ids"]]
            self.strs.delete(ids)
            if self.emb is not None:
                self.emb.delete(ids)
            for d in ids:
                if d not in self._deleted:
                    self._deleted.add(d)
                    self.document_count -= 1
                self._uncommitted_deleted.add(d)
                for m in list(self._bool.values()) + list(self._num.values()) + list(self._strf.values()) + list(self._geo.values()) + list(self._date.values()):
                    m.pop(d, None)
            self._retire_live()
        else:
            raise ValueError(f"unsupported operation {kind!r}")

    def apply_all(self, ops: Iterable[Dict]) -> None:
        for op in ops:
            self.apply(op)

    def commit(self) -> None:
        """ReadSide::commit -> field compact(): publish the next snapshot of the string store (searches on the
        previous one keep running meanwhile), drop the deleted rows of the embedding store (index/mod.rs:583-590) and
        refresh the facet layout and the geopoint fields."""
        self.strs.commit()
        if self.emb is not None:
            self.emb.compact()
        # N of the idf is Index::document_count (mod.rs:1460: +1 per Index op, also for documents without string fields)
        self.strs.set_global(max(self.document_count, 0))
        self._uncommitted_deleted.clear()
        self.refresh_facets()

    def refresh_facets(self) -> None:
        """Lay the filter fields out again: the facet store and one GeoPointField per geopoint field, both over
        DocumentId [0, max_doc_id + 2).  Handles built earlier are closed."""
        for g in self.geo.values():
            g.close()
        self.geo = {}
        self._retire_live()       # nbits changes: the deletes handle is rebuilt over the new DocumentId space
        for f in self._retired:   # programs built before now point at the closed facet store and fields as well
            f.close()
        self._retired = []
        self.nbits = self.max_doc_id + 2
        for f, m in self._geo.items():
            docs = [d for d, ps in m.items() for _ in ps]
            self.geo[f] = GeoPointField(self.ctx, self.max_doc_id + 2, docs, [p[0] for ps in m.values() for p in ps],
                                        [p[1] for ps in m.values() for p in ps])
        if not (self._bool or self._num or self._strf or self._date):
            return
        if self.facets is not None:
            self.facets.close()
        st = FacetStore(self.ctx, self.max_doc_id + 2)
        for f, m in self._bool.items():
            has = {d: ({b} if isinstance(b, bool) else b) for d, b in m.items()}
            st.add_bool_field(f, [d for d, bs in has.items() if True in bs], [d for d, bs in has.items() if False in bs])
        for f, m in self._num.items():
            docs = [d for d, vs in m.items() for _ in vs]
            vals = [x for vs in m.values() for x in vs]
            st.add_number_field(f, docs, vals)
        for f, m in self._strf.items():
            keys: Dict[str, List[int]] = {}
            for d, ks in m.items():
                for k in ks:
                    keys.setdefault(k, []).append(d)
            st.add_string_field(f, {k: keys[k] for k in sorted(keys)})
        for f, m in self._date.items():
            st.add_date_field(f, [d for d, ms in m.items() for _ in ms], [x for ms in m.values() for x in ms])
        self.facets = st

    def filter_fields(self) -> List[str]:
        return list(self._bool) + list(self._num) + list(self._strf) + list(self._date) + list(self._geo)

    def where_filter(self, where) -> Optional[DeviceFilter]:
        """The where-clause `where` (a JSON object or a parsed WhereFilter) over this index as execute_filter
        (filter.rs:344-392) computes it: None when nothing is filtered, else a DeviceFilter to pass as
        TokenScoreParams.device_filter.  Raises FilterFieldNotFound for a key that is not a filter field
        (search.rs:435-449) before any device work, and ValueError for a clause serde would refuse.  The fields are
        the ones laid out by the last refresh_facets() / commit(); the deletes since the last commit are excluded."""
        w = where if isinstance(where, WhereFilter) else parse_where(where)
        check_where_keys(w, [self.filter_fields()])
        return evaluate_where(w, self.facets, self.geo, self.nbits, sorted(self._uncommitted_deleted), ctx=self.ctx)

    def where_program(self, where) -> Optional[WhereProgram]:
        """The counterpart of where_filter: the same clause as a program for TokenScoreParams.where_programs, which the
        search call evaluates itself.  Nothing runs on the device here except, once per set of uncommitted deletes, the
        NOT(deletes) handle the program carries.  A program is valid until the next refresh_facets() / commit()."""
        w = where if isinstance(where, WhereFilter) else parse_where(where)
        check_where_keys(w, [self.filter_fields()])
        if self._uncommitted_deleted and self._live is None:
            dele = DeviceFilter.from_ids(self.ctx, sorted(self._uncommitted_deleted), self.nbits)
            try:
                self._live = ~dele
            finally:
                dele.close()
        return compile_where(w, self.facets, self.geo, self.nbits, self._live)

    def _retire_live(self) -> None:
        if self._live is not None:
            self._retired.append(self._live)
            self._live = None

    def context(self) -> TokenScoreContext:
        return TokenScoreContext(self.ctx, self.emb, self.strs)

    def resolve(self, texts: Sequence[str], **kw):
        """token_score.rs:196-209 + the FST expansion: the packed query arrays oc_search takes.  Typo-tolerant
        expansions run on this index's device."""
        return self.dict.resolve_batch(list(texts), ctx=self.ctx, **kw)

    def close(self):
        for x in [self.facets, self.emb, self.strs, self.dict, self._live] + list(self.geo.values()) + self._retired:
            if x is not None:
                x.close()
