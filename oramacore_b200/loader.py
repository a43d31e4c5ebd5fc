"""Loader / refresher of the device-resident stores from the reference's own write-operation stream.

The reference's read side is fed by `Index::update_data(IndexWriteOperation)` (read/index/mod.rs:1436-1705):
  * `Index { doc_id, indexed_values }` — `document_count += 1`, then per value
      ScoreString2(field, IndexedValue{field_length: u16, terms: {term -> TermData{exact_positions, positions}}})
                                              -> StringFieldStorage::insert   (string_field.rs:155-177, mod.rs:1509-1515)
      FilterBool / FilterNumber / FilterString -> the filter fields the facets and filters read (mod.rs:1461-1497)
      FilterGeoPoint2(field, Plain(point) | Array([points]))  -> the geopoint fields of the where-filter (mod.rs:1556-1565, 1678-1687)
      FilterBool2 / FilterString2 / FilterDate / FilterDate2 / FilterNumber2 -> the same filter fields as the write side
                                              emits them today (write/index/fields.rs:312-325, 345-353, 401-423, 467-504)
  * `Index2 { doc_id, indexed_values, omc }` — what the write side emits today (write/index/mod.rs:451-472): `Index`,
      and `omc` (when not None) appended to the index's OMC log (mod.rs:1566-1580)
  * `IndexEmbedding { data: field -> [(doc_id, vectors)] }` -> EmbeddingFieldStorage::insert (mod.rs:1688-1698)
  * `DeleteDocuments { doc_ids }` — `document_count -= len(doc_ids)` (saturating), uncommitted deletes, excluded
      from every search at once (mod.rs:1346-1427)
and `commit` / `compact` lay the pending data out (`CURRENT` + `versions/<n>`, embedding_field.rs:91-95).

`IndexLoader.apply(op)` takes the same operations as plain dicts (the JSON shape of the reference's enum), resolves
terms to stable term ids through the native dictionary (oc_dict_*), and drives the C ABI: oc_str_insert /
oc_str_delete / oc_str_commit (snapshot swap: searches keep running on the previous version while a commit builds
the next), oc_emb_insert / oc_emb_delete (live) and oc_emb_compact at commit.  Filter values and deletes are queued on
the facet store and the geopoint fields as apply() sees them (tests/filter_commit_spec.py states the per-kind rules as
ops); `refresh_facets()` merges them into the next version of every field on the device (oc_facets_commit_ex,
oc_geo_field_commit_ex), `where_filter(where)` evaluates a where-clause over them (where.py), and `sort_by(SortBy)`
sorts by a number, date or bool field of the published version (oc_sort_field_from_facets).  No host copy of the
filter values is kept.  OMC multipliers go to a device-resident OmcStore: `omc()` publishes the ones applied so far
(get_all_omc, mod.rs:1720-1739: visible before a commit), and `commit()` also removes the uncommitted deletes' entries
(mod.rs:604-627).  tf of a term = number of positions (exact + stemmed), as StringStorage counts them.

`IndexLoader(..., shard=(lo, hi))` is one rank of a document-sharded index (sharding.py): every rank applies the whole
stream but stores only the documents in its doc-id range [lo, hi) (hi None: open-ended; ranges ascend with rank).  The
dictionary, N, the OMC map, the DocumentId space and the deletes follow every op, so every rank resolves queries to the
same term ids; `commit()` ends with the collective that rebuilds the corpus-wide df tables and averages
(StringFieldStorage.sync_global), so it must run on every rank concurrently (one thread or process per rank)."""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

from .engine import (Context, DeviceFilter, EmbeddingFieldStorage, FacetStore, GeoPointField, GroupBy, IndexPart, OmcStore, SortField,
                     StringFieldStorage, TermDictionary, TokenScoreContext, TokenScoreParams, _facet_result, resolve_sort_by,
                     search_indexes_arrays)
from .types import FacetFieldNotFound, SearchHits
from .types import SortBy
from .where import WhereFilter, WhereProgram, check_where_keys, compile_where, filter_from_program, parse_where

_F64_INT_MAX = 1 << 53   # I64 values beyond +-2^53 would not survive the trip through a double


def _plain_or_array(v) -> list:
    """oramacore_fields' IndexedValue: {"Plain": x} or {"Array": [x, ...]}."""
    return [v["Plain"]] if "Plain" in v else list(v["Array"])


def _exact_i64(x, what: str) -> float:
    if abs(int(x)) > _F64_INT_MAX:
        raise ValueError(f"{what} {x}: beyond +-2^53, not exact as a double")
    return float(int(x))


class IndexLoader:
    shard: Optional[Tuple[int, Optional[int]]] = None    # this rank's doc-id range [lo, hi); None: the whole index
    _deletes_since_commit = False                         # sharded: some rank's store may hold tombstones

    def __init__(self, ctx: Context, string_fields: Sequence[str], embedding_model: Optional[str] = None,
                 embedding_dim: Optional[int] = None, bool_fields: Sequence[str] = (), number_fields: Sequence[str] = (),
                 string_filter_fields: Sequence[str] = (), geopoint_fields: Sequence[str] = (), date_fields: Sequence[str] = (),
                 shard: Optional[Tuple[int, Optional[int]]] = None):
        if shard is not None and (shard[0] < 0 or (shard[1] is not None and shard[1] < shard[0])):
            raise ValueError(f"shard {shard!r}: want (lo, hi) with 0 <= lo <= hi, or (lo, None)")
        self.ctx = ctx
        self.shard = shard
        self.string_fields = list(string_fields)
        self.dict = TermDictionary(max(len(self.string_fields), 1))
        self.strs = StringFieldStorage.empty(ctx, max(len(self.string_fields), 1))
        self.emb = EmbeddingFieldStorage(ctx, embedding_model or "BGESmall", dim=embedding_dim) if (embedding_model or embedding_dim) else None
        self._bool, self._num = list(bool_fields), list(number_fields)
        self._strf, self._date, self._geo = list(string_filter_fields), list(date_fields), list(geopoint_fields)
        self.document_count = 0                                # N of the idf, live between commits (see _push_count)
        self.max_doc_id = -1
        self._uncommitted_deleted: set = set()                 # deletes since the last commit (filter.rs:344-392)
        self.nbits = 1                                         # DocumentId space of `facets` and `geo`
        # one store and one geopoint field per field for the life of the loader; values queue until refresh_facets()
        self.facets: Optional[FacetStore] = None
        if self._bool or self._num or self._strf or self._date:
            self.facets = FacetStore(ctx, self.nbits)
            for f in self._bool:
                self.facets.add_bool_field(f, [], [])
            for f in self._num:
                self.facets.add_number_field(f, [], [])
            for f in self._date:
                self.facets.add_date_field(f, [], [])
            # a string_filter field joins the store with its first key (a field needs one variant)
        self.geo: Dict[str, GeoPointField] = {f: GeoPointField(ctx, self.nbits, [], [], []) for f in self._geo}
        self._live: Optional[DeviceFilter] = None              # NOT(uncommitted deletes) of where_program, built once
        self._retired: List[object] = []                       # earlier ones, which programs may still point at, and
                                                               # this version's group handles
        self._sorts: Dict[str, SortField] = {}                 # sort fields of the published version, built when asked
        self._groups: Dict[Tuple[str, ...], GroupBy] = {}      # group handles of the published version, built when asked
        self.omc_store = OmcStore(ctx)                         # the OMC map; sets queue in _omc_log until omc() / commit()
        self._omc_log: List[tuple] = []

    # ---- Index::update_data
    def apply(self, op: Dict) -> None:
        kind = op["type"]
        if kind in ("Index", "Index2"):
            d = int(op["doc_id"])
            omc = op.get("omc") if kind == "Index2" else None
            if omc is not None:
                omc = np.float32(omc)
                if not np.isfinite(omc):
                    raise ValueError(f"document {d}: omc {op['omc']!r} is not a finite f32")
            self.document_count += 1                            # mod.rs:1460
            if omc is not None:                                 # the uncommitted OMC log (mod.rs:1573-1579)
                self._omc_log.append((d, omc))
            self.max_doc_id = max(self.max_doc_id, d)
            if d in self._uncommitted_deleted:
                self._uncommitted_deleted.discard(d)
                self._retire_live()
            own = self.owns(d)
            for v in op["indexed_values"]:
                t = v["type"]
                if t == "ScoreString2":
                    fi = self.string_fields.index(v["field"])
                    terms = v["terms"]                                  # {term: {"exact_positions": [...], "positions": [...]}}
                    names = list(terms)
                    # registered on every rank, stored or not: the ranks' dictionaries hand out the same ids
                    ids = self.dict.add_terms(fi, names) if names else np.zeros(0, np.uint32)
                    if own:
                        tf = {int(i): max(1, len(terms[n].get("exact_positions", ())) + len(terms[n].get("positions", ()))) for i, n in zip(ids, names)}
                        self.strs.insert(d, fi, int(v["field_length"]), tf)
                elif not own:
                    continue
                elif t == "FilterBool":                         # replaces the document's value
                    f = self._field(self._bool, v["field"])
                    self.facets.clear(f, [d])
                    self.facets.insert_variants(f, [d], [bool(v["value"])])
                elif t == "FilterNumber":
                    self.facets.insert_numbers(self._field(self._num, v["field"]), [d], [float(v["value"])])
                elif t == "FilterString":
                    self._insert_keys(v["field"], d, [str(v["value"])])
                elif t == "FilterGeoPoint2":
                    # GeoPointIndexedValue: {"Plain": {"lat", "lon"}} or {"Array": [{"lat", "lon"}, ...]}
                    val = v["value"]
                    pts = [val["Plain"]] if "Plain" in val else list(val["Array"])
                    self.geo[self._field(self._geo, v["field"])].insert([d] * len(pts), [float(p["lat"]) for p in pts],
                                                                        [float(p["lon"]) for p in pts])
                elif t == "FilterBool2":                        # adds to the document's set of bools
                    bs = [bool(b) for b in _plain_or_array(v["value"])]
                    self.facets.insert_variants(self._field(self._bool, v["field"]), [d] * len(bs), bs)
                elif t == "FilterNumber2":
                    # NumberFieldIndexedValue: {"I64": {"Plain": x} | {"Array": [...]}} or {"F64": ...}
                    f = self._field(self._num, v["field"])
                    (store, val), = v["value"].items()
                    xs = _plain_or_array(val)
                    xs = [_exact_i64(x, "I64 value") for x in xs] if store == "I64" else [float(x) for x in xs]
                    self.facets.insert_numbers(f, [d] * len(xs), xs)
                elif t == "FilterString2":
                    self._insert_keys(v["field"], d, [str(x) for x in _plain_or_array(v["value"])])
                elif t in ("FilterDate", "FilterDate2"):
                    xs = [int(x) for x in ([v["value"]] if t == "FilterDate" else _plain_or_array(v["value"]))]
                    self.facets.insert_numbers(self._field(self._date, v["field"]), [d] * len(xs), xs)
                else:
                    raise ValueError(f"unsupported indexed value {t!r} (outside the search hot path)")
            self._push_count()
        elif kind == "IndexEmbedding":
            for d, vectors in op["data"]:
                self.max_doc_id = max(self.max_doc_id, int(d))
                if self.owns(int(d)):
                    self.emb.insert(int(d), vectors)
        elif kind == "DeleteDocuments":
            ids = [int(x) for x in op["doc_ids"]]
            self.strs.delete(ids)
            if self.emb is not None:
                self.emb.delete(ids)
            # mod.rs:1417-1423: the count drops by the number of ids in the op, whether or not each was a live
            # document, and stops at 0
            self.document_count = max(self.document_count - len(ids), 0)
            self._push_count()
            self._uncommitted_deleted.update(ids)
            self._deletes_since_commit = True
            if self.facets is not None:
                self.facets.delete(ids)
            for g in self.geo.values():
                g.delete(ids)
            self._retire_live()
        else:
            raise ValueError(f"unsupported operation {kind!r}")

    def owns(self, doc_id: int) -> bool:
        """Whether this loader stores the document (always, unless it is one shard)."""
        if self.shard is None:
            return True
        lo, hi = self.shard
        return doc_id >= lo and (hi is None or doc_id < hi)

    @property
    def shard_tombstones(self) -> bool:
        """The OC_SHARD_TOMBSTONES flag (TokenScoreParams.shard_tombstones) of a sharded search on this loader: a
        delete since the last commit, which may have tombstoned rows on any rank.  The same on every rank."""
        return self._deletes_since_commit

    def _push_count(self) -> None:
        """N of the idf is Index::document_count (mod.rs:1460: +1 per Index op, also for documents without string
        fields), read by every search whether or not it was committed (token_score.rs:221, search.rs:305-318).  So the
        string store gets it after every op that changes it, and again after its commit."""
        self.strs.set_global(self.document_count)

    @staticmethod
    def _field(names: List[str], name: str) -> str:
        if name not in names:
            raise KeyError(name)
        return name

    def _insert_keys(self, name: str, d: int, keys: List[str]) -> None:
        """FilterString / FilterString2 append (a key listed twice is listed twice); a new key gets the next variant."""
        self._field(self._strf, name)
        if not keys:
            return
        if name not in self.facets.fields:
            self.facets.add_string_field(name, {keys[0]: []})
        self.facets.insert_variants(name, [d] * len(keys), keys)

    def apply_all(self, ops: Iterable[Dict]) -> None:
        for op in ops:
            self.apply(op)

    def commit(self) -> None:
        """ReadSide::commit -> field compact(): publish the next snapshot of the string store (searches on the
        previous one keep running meanwhile), drop the deleted rows of the embedding store (index/mod.rs:583-590) and
        refresh the facet layout and the geopoint fields.  A shard then rebuilds the corpus-wide df tables and
        averages with the other ranks (a collective: every rank's commit() runs concurrently)."""
        self.strs.commit()
        if self.emb is not None:
            self.emb.compact()
        self._push_count()
        # mod.rs:604-627: the log merges into the committed map, then the uncommitted deletes leave it
        self._publish_omc(sorted(self._uncommitted_deleted))
        self._uncommitted_deleted.clear()
        self._deletes_since_commit = False
        self.refresh_facets()
        if self.shard is not None:
            self.strs.sync_global()

    def omc(self) -> OmcStore:
        """The OMC store with every multiplier applied so far published (get_all_omc, mod.rs:1720-1739: the log over
        the committed map, last writer wins), for TokenScoreParams.omc_store.  Deletes leave the map at commit()."""
        self._publish_omc([])
        return self.omc_store

    def _publish_omc(self, deleted: List[int]) -> None:
        if not self._omc_log and not deleted:
            return
        if self._omc_log:
            self.omc_store.set([d for d, _ in self._omc_log], [m for _, m in self._omc_log])
        if deleted:
            self.omc_store.delete(deleted)
        self.omc_store.commit()
        self._omc_log = []

    def refresh_facets(self) -> dict:
        """Publish every filter value applied so far over DocumentId [0, max_doc_id + 2): the queued values and deletes
        merge into the next version of the facet store and of every geopoint field on the device; the objects stay
        the same.  The uncommitted deletes stay uncommitted.  NOT(deletes) handles built earlier are closed (nbits may
        change).  Returns the commits' statistics by field kind ("facets", and the geopoint field names)."""
        self._retire_live()       # nbits changes: the deletes handle is rebuilt over the new DocumentId space
        for f in self._retired:   # programs built before now carry the earlier nbits
            f.close()
        self._retired = []
        self._groups = {}         # (their handles were retired with them)
        for f in self._sorts.values():   # the sorts of the previous version
            f.close()
        self._sorts = {}
        self.nbits = max(self.nbits, self.max_doc_id + 2)
        stats = {}
        if self.facets is not None:
            stats["facets"] = self.facets.commit(self.nbits)
        for name, g in self.geo.items():
            stats[name] = g.commit(self.nbits)
        return stats

    def filter_fields(self) -> List[str]:
        return self._bool + self._num + self._strf + self._date + self._geo

    def where_filter(self, where) -> Optional[DeviceFilter]:
        """The where-clause `where` (a JSON object or a parsed WhereFilter) over this index as execute_filter
        (filter.rs:344-392) computes it: None when nothing is filtered, else a DeviceFilter to pass as
        TokenScoreParams.device_filter.  Raises FilterFieldNotFound for a key that is not a filter field
        (search.rs:435-449) before any device work, and ValueError for a clause serde would refuse.  The fields are
        the ones laid out by the last refresh_facets() / commit(); the deletes since the last commit are excluded."""
        prog = self.where_program(where)
        return None if prog is None else filter_from_program(self.ctx, prog)

    def where_program(self, where) -> Optional[WhereProgram]:
        """The counterpart of where_filter: the same clause as a program for TokenScoreParams.where_programs, which the
        search call evaluates itself.  Nothing runs on the device here except, once per set of uncommitted deletes, the
        NOT(deletes) handle the program carries.  A program is valid until the next refresh_facets() / commit()."""
        w = where if isinstance(where, WhereFilter) else parse_where(where)
        check_where_keys(w, [self.filter_fields()])
        return self._compile_where(w)

    def _compile_where(self, w: WhereFilter) -> Optional[WhereProgram]:
        """where_program without the key check: a key that is not a filter field of this index filters out everything."""
        if self._uncommitted_deleted and self._live is None:
            dele = DeviceFilter.from_ids(self.ctx, sorted(self._uncommitted_deleted), self.nbits)
            try:
                self._live = ~dele
            finally:
                dele.close()
        return compile_where(w, self.facets, self.geo, self.nbits, self._live)

    def sort_fields(self) -> Dict[str, object]:
        """The mapping resolve_sort_by takes: every number, date and bool property to a SortField of the version the
        last refresh_facets() / commit() published (built on the device the first time it is asked for after a
        refresh), and every string, string_filter and geopoint property to its kind name.  Values queued since that
        refresh do not move a sort.  A SortField is valid until the next refresh_facets() / commit(), which closes it."""
        out: Dict[str, object] = {f: "string" for f in self.string_fields}
        out.update({f: "string_filter" for f in self._strf})
        out.update({f: "geopoint" for f in self._geo})
        for f in self._bool + self._num + self._date:
            if f not in self._sorts:
                self._sorts[f] = SortField.from_facets(self.facets, f)
            out[f] = self._sorts[f]
        return out

    def group_by(self, properties: Sequence[str]) -> Optional[GroupBy]:
        """The GroupBy of `properties` over the version the last commit() published (built the first time it is asked
        for after a commit, closed by the next), or None when the index lacks one of them (it adds no groups,
        group.rs:104-168).  A date or geopoint property raises ValueError."""
        for p in properties:
            if p in self._date or p in self._geo:
                raise ValueError(f"{p!r} is a {'date' if p in self._date else 'geopoint'} field: it cannot group")
        key = tuple(properties)
        if self.facets is None or not all(p in self.facets.fields for p in key):
            return None
        if key not in self._groups:   # closed with the retired handles at the next commit
            self._groups[key] = GroupBy(self.facets, list(key))
            self._retired.append(self._groups[key])
        return self._groups[key]

    def sort_by(self, sort_by: SortBy):
        """resolve_sort_by over sort_fields(): the (SortField, order) pair the sorted searches take.  Raises
        SortFieldNotFound / InvalidSortField as the reference does (read/index/sort.rs:186-265)."""
        return resolve_sort_by(self.sort_fields(), sort_by)

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
        for x in list(self._sorts.values()) + [self.facets, self.emb, self.strs, self.dict, self._live, self.omc_store] + list(self.geo.values()) + self._retired:
            if x is not None:
                x.close()


def search_collection(loaders: Sequence[IndexLoader], texts: Optional[Sequence[str]], params: TokenScoreParams, where=None,
                      sort_by: Optional[SortBy] = None, q_vecs: Optional[np.ndarray] = None, promote=None,
                      **resolve_kw) -> Tuple[List[SearchHits], np.ndarray]:
    """search_on_indexes (read/search.rs:283-501) over the indexes of one collection, all on one ctx, in one
    oc_search_indexes call: each index resolves the texts with its own dictionary, compiles `where` over its own filter
    fields (a key that is a filter field of no index raises FilterFieldNotFound, search.rs:434-450; a key only some
    indexes have filters out everything on the others), sorts by its own `sort_by` field and scores with its own OMC
    map.  `params` holds the request (mode, limit_hint, offset, similarity, threshold, query_params) and is shared by
    every index.  Returns (one SearchHits per query, the sort values [B, limit])."""
    res = search_collection_ex(loaders, texts, params, where, sort_by, q_vecs, promote, **resolve_kw)
    return [r["hits"] for r in res], np.stack([r["sort_values"] for r in res]) if res else np.zeros((0, 0))


def search_collection_ex(loaders: Sequence[IndexLoader], texts: Optional[Sequence[str]], params: TokenScoreParams, where=None,
                         sort_by: Optional[SortBy] = None, q_vecs: Optional[np.ndarray] = None, promote=None, facets=None,
                         group_by=None, **resolve_kw) -> List[dict]:
    """search_collection with the reference's `facets` and `group_by` (GroupByConfig: {"properties": [...],
    "max_results": n}), one request for every query, in one oc_search_indexes_ex call.  Per query a dict: "hits"
    (SearchHits), "sort_values" [limit], "facets" ({field: {"count", "values"}}, None without facets) and "groups" (a
    list of {"values", "result": [(doc, score), ...]} in key order, None without group_by).
      - facets: the fields that no index has raise FacetFieldNotFound (search.rs:452-464); a definition of the wrong kind
        for an index's field, or a date field, raises ValueError (facet.rs:166-178).
      - group_by: an index that lacks one of the properties adds no groups (group.rs:104-168); a date or geopoint
        property raises ValueError.  Each index's GroupBy is built once per commit (IndexLoader.group_by)."""
    B = len(texts) if texts is not None else int(np.asarray(q_vecs).shape[0])
    w = None if where is None else (where if isinstance(where, WhereFilter) else parse_where(where))
    if w is not None:
        check_where_keys(w, [l.filter_fields() for l in loaders])
    parts, sorts = [], None if sort_by is None else []
    for l in loaders:
        fields = {"omc_store": l.omc()}
        if w is not None:
            fields["where_programs"] = [l._compile_where(w)] * B
        parts.append(IndexPart(l.context(), None if texts is None else l.resolve(texts, **resolve_kw), q_vecs, fields, l.facets))
        if sorts is not None:
            sorts.append([l.sort_by(sort_by)] * B)
    groups = None
    if group_by is not None:
        props = list(group_by["properties"])
        groups = [([l.group_by(props) for l in loaders], int(group_by.get("max_results", 1)))] * B
    if facets is not None:
        missing = [f for f in facets if not any(l.facets is not None and f in l.facets.fields for l in loaders)]
        if missing:
            raise FacetFieldNotFound(missing)
    got = search_indexes_arrays(loaders[0].ctx, parts, params, sorts, promote,
                                groups=groups, facets=None if facets is None else [facets] * B)
    docs, scores, sv, n, cnt = got[:5]
    out = []
    for b in range(B):
        r = {"hits": SearchHits(docs[b, :n[b]].copy(), scores[b, :n[b]].copy(), int(cnt[b])), "sort_values": sv[b],
             "facets": None, "groups": None}
        if len(got) > 7:
            gd, gs, _, gn, rows, keys, fc, foff, labels = got[7:]
            if groups is not None:
                r["groups"] = [{"values": list(keys[b][k]), "result": [(int(gd[row, j]), float(gs[row, j])) for j in range(int(gn[row]))]}
                               for k, row in enumerate(range(int(rows[b]), int(rows[b + 1])))]
            if facets is not None:
                r["facets"] = _facet_result(fc[foff[b]:foff[b + 1]], labels[b])
        out.append(r)
    return out
