"""Host-side mirror of the reference's read-side scoring interface over the C ABI.

Names and argument meaning follow the reference (oramasearch/oramacore @ 666ab48):
  * EmbeddingFieldStorage  — read/index/embedding_field.rs:29-34 (insert :232, delete :240,
                             search :250-278, info/stats :303-310)
  * VectorSearchParams     — read/index/committed_field/vector.rs:10-15
  * StringFieldStorage set — read/index/string_field.rs (one oc_str per Index)
  * TokenScoreParams / TokenScoreContext.execute — read/index/token_score.rs:31-41, 460-509
  * search()               — the CollectionManager search surface restricted to the hot path
                             (read/search.rs:283-501): mode = fulltext | vector | hybrid.
All compute happens in liboramacore_b200.so on the GPU; nothing here scores on the CPU.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import OcError, SearchParams, Timing, check, lib
from .types import (BM25_B, BM25_K, MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR, InvalidSortField, PromoteItem, SearchHits,
                    SortBy, SortFieldNotFound, StringIndexData, TextQuery)

# Model::dimensions / rescale_score (python/embeddings.rs:52-92)
MODEL_DIMS = {
    "BGESmall": 384, "BGEBase": 768, "BGELarge": 1024, "JinaEmbeddingsV2BaseCode": 768,
    "MultilingualE5Small": 384, "MultilingualE5Base": 768, "MultilingualE5Large": 1024,
    "MultilingualMiniLML12V2": 384,
}
E5_MODELS = {"MultilingualE5Small", "MultilingualE5Base", "MultilingualE5Large"}


def _p(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Context:
    """One GPU + stream + workspace (oc_ctx). One per process, like one rank per GPU."""

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        check(lib().oc_init(device, C.byref(self._h)))
        self.device = device

    def close(self):
        if self._h:
            lib().oc_shutdown(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def device_info(self):
        sm = C.c_int()
        mem = C.c_size_t()
        name = C.create_string_buffer(256)
        check(lib().oc_device_info(self._h, C.byref(sm), C.byref(mem), name, 256))
        return {"sm_count": sm.value, "hbm_bytes": mem.value, "name": name.value.decode()}

    def last_timing(self) -> dict:
        t = Timing()
        check(lib().oc_last_timing(self._h, C.byref(t)))
        return t.as_dict()

    def launch_count(self) -> int:
        return int(lib().oc_launch_count(self._h))

    # ---- document-sharded multi-GPU (SURVEY.md §8e)
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_uint8 * _lib.OC_COMM_ID_BYTES)()
        check(lib().oc_comm_unique_id(buf))
        return bytes(buf)

    def comm_init(self, world_size: int, rank: int, unique_id: bytes):
        buf = (C.c_uint8 * _lib.OC_COMM_ID_BYTES).from_buffer_copy(unique_id)
        check(lib().oc_comm_init(self._h, world_size, rank, buf))

    @staticmethod
    def comm_init_local(ctxs):
        """Join contexts of this process (e.g. several on one GPU) as ranks 0..len(ctxs)-1 of one group whose
        collectives run through host memory (oc_comm_init_local).  Each rank then calls the sharded search on its own
        thread."""
        arr = (C.c_void_p * len(ctxs))(*[c._h for c in ctxs])
        check(lib().oc_comm_init_local(arr, len(ctxs)))

    def comm_enable_p2p(self, all_gather):
        """Direct NVLink exchange of the shard records (oc_comm_p2p_*).  `all_gather(blob: bytes) -> list[bytes]`
        is the host runtime's all-gather in rank order (e.g. torch.distributed.all_gather_object)."""
        buf = (C.c_uint8 * 128)()
        check(lib().oc_comm_p2p_export(self._h, buf))
        blobs = all_gather(bytes(buf))
        cat = b"".join(blobs)
        arr = (C.c_uint8 * len(cat)).from_buffer_copy(cat)
        check(lib().oc_comm_p2p_import(self._h, arr))


def to_bf16(x: np.ndarray) -> np.ndarray:
    """fp32 -> bf16 bit patterns (uint16), round to nearest even."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    r = u + np.uint32(0x7fff) + ((u >> np.uint32(16)) & np.uint32(1))
    return (r >> np.uint32(16)).astype(np.uint16)


def from_bf16(b: np.ndarray) -> np.ndarray:
    """bf16 bit patterns -> the fp32 values they denote (exact)."""
    return (b.astype(np.uint32) << np.uint32(16)).view(np.float32)


def pinned_empty(shape, dtype=np.float32) -> np.ndarray:
    """numpy array backed by page-locked host memory (oc_pinned_alloc): inputs placed here are DMA'd
    directly by oc_search. The memory is intentionally never freed before interpreter exit."""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    p = C.c_void_p()
    check(lib().oc_pinned_alloc(n, C.byref(p)))
    buf = (C.c_uint8 * max(n, 1)).from_address(p.value)
    return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)


@dataclass
class VectorSearchParams:
    """committed_field/vector.rs:10-15"""
    target: np.ndarray
    similarity: float
    limit: int
    filtered_doc_ids: Optional[np.ndarray] = None  # bitmap over DocumentId (uint64 words)
    filter_nbits: int = 0


class EmbeddingFieldStorage:
    """embedding_field.rs:29-34 — cosine metric, device resident."""

    def __init__(self, ctx: Context, model: str = "BGEBase", dim: Optional[int] = None, dtype: str = "f32"):
        """dtype "f32" (what the reference stores, embedding_field.rs:232) or "bf16" (storage extension:
        rows are kept as bf16, scores are exact fp32 arithmetic on those values)."""
        self.ctx = ctx
        self.model = model
        self.dim = int(dim if dim is not None else MODEL_DIMS[model])
        self.dtype = dtype
        self._h = C.c_void_p()
        check(lib().oc_emb_create(ctx._h, self.dim, {"f32": 0, "bf16": 1}[dtype], 1 if model in E5_MODELS else 0,
                                  C.byref(self._h)))

    def close(self):
        if self._h:
            lib().oc_emb_destroy(self._h)
            self._h = C.c_void_p()

    def reserve(self, n_rows: int):
        check(lib().oc_emb_reserve(self._h, n_rows))

    def insert(self, doc_id: int, vectors: Sequence[Sequence[float]]):
        """insert(DocumentId, Vec<Vec<f32>>) — several chunks per document (embedding_field.rs:232-237)."""
        v = np.ascontiguousarray(np.asarray(vectors, np.float32).reshape(-1, self.dim))
        self.insert_batch(np.full(v.shape[0], doc_id, np.uint64), v)

    def insert_batch(self, doc_ids: np.ndarray, rows: np.ndarray):
        d = np.ascontiguousarray(doc_ids, np.uint64)
        if self.dtype == "bf16":   # fp32 input is rounded to bf16 (RNE); uint16 input is taken as bf16 bits
            r = np.ascontiguousarray(rows) if rows.dtype == np.uint16 else to_bf16(rows)
        else:
            r = np.ascontiguousarray(rows, np.float32)
        assert r.ndim == 2 and r.shape[1] == self.dim and r.shape[0] == d.shape[0]
        check(lib().oc_emb_insert(self._h, _p(d), _p(r), d.shape[0]))

    def delete(self, doc_id):
        """One DocumentId or a sequence of them."""
        d = np.ascontiguousarray(np.atleast_1d(np.asarray(doc_id, np.uint64)).ravel())
        check(lib().oc_emb_delete(self._h, _p(d), int(d.shape[0])))

    def compact(self, shrink: bool = False) -> dict:
        """compact() as Index::commit runs it (index/mod.rs:583-590): drop the deleted rows on the device, in place and
        order-preserving, so that searches return what they returned before.  shrink=True also gives the capacity
        beyond num_rows back.  Returns the call's statistics (oc_emb_compact_t)."""
        st = _lib.EmbCompact()
        check(lib().oc_emb_compact(self._h, _lib.OC_EMB_COMPACT_SHRINK if shrink else 0, C.byref(st)))
        return st.as_dict()

    def info(self) -> dict:
        i = _lib.EmbInfo()
        check(lib().oc_emb_info(self._h, C.byref(i)))
        return {"num_embeddings": i.num_embeddings, "num_rows": i.num_rows, "dimensions": i.dimensions,
                "device_bytes": i.device_bytes}

    def search_batch(self, targets: np.ndarray, limit: int, similarity: float,
                     filter_bits: Optional[np.ndarray] = None, filter_nbits: int = 0):
        q = np.ascontiguousarray(targets, np.float32).reshape(-1, self.dim)
        B = q.shape[0]
        docs = np.zeros((B, limit), np.uint64)
        scores = np.zeros((B, limit), np.float32)
        counts = np.zeros(B, np.uint32)
        fb = None if filter_bits is None else np.ascontiguousarray(filter_bits, np.uint64)
        check(lib().oc_emb_search(self._h, _p(q), B, limit, similarity, _p(fb), int(filter_nbits),
                                  _p(docs), _p(scores), _p(counts)))
        return docs, scores, counts

    def search(self, params: VectorSearchParams, output: Dict[int, float]) -> None:
        """EmbeddingFieldStorage::search(&VectorSearchParams, &mut HashMap) — `output[doc] += score`."""
        docs, scores, counts = self.search_batch(params.target, params.limit, params.similarity,
                                                 params.filtered_doc_ids, params.filter_nbits)
        for i in range(int(counts[0])):
            d = int(docs[0, i])
            output[d] = np.float32(output.get(d, np.float32(0.0)) + scores[0, i])


class StringFieldStorage:
    """All string fields of one Index on the device (string_field.rs:32-36); built from
    committed postings (`StringIndexData`)."""

    def __init__(self, ctx: Context, data: StringIndexData, global_df: Optional[List[np.ndarray]] = None):
        self.ctx = ctx
        self.data = data
        self._h = C.c_void_p()
        check(lib().oc_str_create(ctx._h, len(data.fields), C.byref(self._h)))
        rd = None if data.row_doc_ids is None else np.ascontiguousarray(data.row_doc_ids, np.uint64)
        check(lib().oc_str_set_rows(self._h, int(data.n_rows), _p(rd), int(data.document_count)))
        for i, f in enumerate(data.fields):
            f.validate()
            gdf = None if global_df is None else np.ascontiguousarray(global_df[i], np.uint32)
            check(lib().oc_str_load_field(self._h, i, float(f.avg_field_len), f.n_terms,
                                          _p(np.ascontiguousarray(f.term_offsets)), _p(np.ascontiguousarray(f.post_row)),
                                          _p(np.ascontiguousarray(f.post_tf)), _p(np.ascontiguousarray(f.post_len)),
                                          _p(gdf)))

    @classmethod
    def empty(cls, ctx: Context, n_fields: int = 1) -> "StringFieldStorage":
        """StringFieldStorage::new (string_field.rs:72-82): no committed postings yet."""
        self = cls.__new__(cls)
        self.ctx, self.data = ctx, None
        self._h = C.c_void_p()
        check(lib().oc_str_create(ctx._h, n_fields, C.byref(self._h)))
        return self

    def close(self):
        if self._h:
            lib().oc_str_destroy(self._h)
            self._h = C.c_void_p()

    def insert(self, doc_id: int, field: int, field_length: int, terms: Dict[int, int]):
        """insert(DocumentId, IndexedValue{field_length, terms}) (string_field.rs:155-177) with terms
        resolved to term ids; visible after commit()."""
        t = np.asarray(list(terms.keys()), np.uint32)
        f = np.asarray([min(v, 65535) for v in terms.values()], np.uint16)
        check(lib().oc_str_insert(self._h, field, int(doc_id), min(int(field_length), 65535), t.shape[0], _p(t), _p(f)))

    def commit(self) -> dict:
        """compact(version) (string_field.rs:186-191), merged on the device.  Returns the call's statistics
        (oc_str_commit_t)."""
        st = _lib.StrCommit()
        check(lib().oc_str_commit_ex(self._h, C.byref(st)))
        return st.as_dict()

    def read_rows(self) -> dict:
        """The published snapshot's rows: {"row_doc_ids": uint64[n_rows], "document_count", "version"}."""
        n, dc, ver = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        check(lib().oc_str_read_rows(self._h, C.byref(n), None, None, None))
        rd = np.zeros(n.value, np.uint64)
        check(lib().oc_str_read_rows(self._h, C.byref(n), _p(rd), C.byref(dc), C.byref(ver)))
        return {"row_doc_ids": rd[:n.value], "document_count": dc.value, "version": ver.value}

    def read_field(self, field: int) -> dict:
        """One field of the published snapshot as oc_str_load_field takes it: {"avg_field_len", "n_terms",
        "term_offsets": uint64[n_terms + 1], "post_row": uint32[], "post_tf": uint16[], "post_len": uint16[]}."""
        nt, npost, avg = C.c_uint32(0), C.c_uint64(0), C.c_float(0)
        check(lib().oc_str_read_field(self._h, field, None, C.byref(nt), C.byref(npost), None, None, None, None))
        off = np.zeros(nt.value + 1, np.uint64)
        row, tf, ln = np.zeros(npost.value, np.uint32), np.zeros(npost.value, np.uint16), np.zeros(npost.value, np.uint16)
        check(lib().oc_str_read_field(self._h, field, C.byref(avg), C.byref(nt), C.byref(npost), _p(off), _p(row), _p(tf), _p(ln)))
        return {"avg_field_len": np.float32(avg.value), "n_terms": nt.value, "term_offsets": off[:nt.value + 1],
                "post_row": row[:npost.value], "post_tf": tf[:npost.value], "post_len": ln[:npost.value]}

    def delete(self, doc_id):
        """One DocumentId or a sequence of them."""
        d = np.ascontiguousarray(np.atleast_1d(np.asarray(doc_id, np.uint64)).ravel())
        check(lib().oc_str_delete(self._h, _p(d), int(d.shape[0])))

    def info(self) -> dict:
        i = _lib.StrInfo()
        check(lib().oc_str_info(self._h, C.byref(i)))
        return {"total_documents": i.total_documents, "total_postings": i.total_postings,
                "unique_terms_count": i.unique_terms_count, "n_fields": i.n_fields, "device_bytes": i.device_bytes,
                "version": i.version, "pending_postings": i.pending_postings}

    def set_global(self, document_count: int, avg_field_len: Optional[Sequence[float]] = None):
        """This store is one shard: N of the idf and the per-field avg_field_len are corpus-wide values
        owned by the caller (kept across commits)."""
        a = None if avg_field_len is None else np.ascontiguousarray(avg_field_len, np.float32)
        check(lib().oc_str_set_global(self._h, int(document_count), _p(a)))

    def sync_global(self) -> dict:
        """This store is one shard of a group (Context.comm_init / comm_init_local): rebuild the corpus-wide df tables
        and average field lengths from every rank's published snapshot (oc_str_sync_global).  A collective: every rank
        calls it, after its own commit() returned.  Returns the call's statistics (oc_str_sync_t)."""
        st = _lib.StrSync()
        check(lib().oc_str_sync_global(self._h, C.byref(st)))
        return st.as_dict()

    def read_global_df(self, field: int) -> Optional[np.ndarray]:
        """The corpus-wide df table installed for one field (uint32, the array global_df takes), or None."""
        n = C.c_uint32(0)
        check(lib().oc_str_read_global_df(self._h, field, C.byref(n), None))
        if n.value == 0:
            return None
        df = np.zeros(n.value, np.uint32)
        check(lib().oc_str_read_global_df(self._h, field, C.byref(n), _p(df)))
        return df[:n.value]


class DeviceFilter:
    """A FilterResult<DocumentId> evaluated to a bitmap that lives on the device (oc_filter_*): built once from
    the And / Or / Not tree of filters.py (filter.rs:344-392), reused by any number of searches."""

    def __init__(self, ctx: Context, handle, nbits: int):
        self.ctx, self._h, self.nbits = ctx, handle, int(nbits)

    @classmethod
    def of_handle(cls, ctx: Context, handle) -> "DeviceFilter":
        """A handle the library built, with its own nbits (a leaf takes the nbits of the field version it was built on)."""
        n = C.c_uint64()
        check(lib().oc_filter_nbits(handle, C.byref(n)))
        return cls(ctx, handle, n.value)

    @classmethod
    def from_ids(cls, ctx: Context, doc_ids, nbits: int) -> "DeviceFilter":
        ids = np.ascontiguousarray(np.asarray(list(doc_ids) if not isinstance(doc_ids, np.ndarray) else doc_ids, np.uint64))
        h = C.c_void_p()
        check(lib().oc_filter_from_ids(ctx._h, _p(ids), ids.shape[0], int(nbits), C.byref(h)))
        return cls(ctx, h, nbits)

    @classmethod
    def from_bits(cls, ctx: Context, bits: np.ndarray, nbits: int) -> "DeviceFilter":
        b = np.ascontiguousarray(bits, np.uint64)
        h = C.c_void_p()
        check(lib().oc_filter_from_bits(ctx._h, _p(b), int(nbits), C.byref(h)))
        return cls(ctx, h, nbits)

    @classmethod
    def from_expr(cls, ctx: Context, expr, nbits: int) -> "DeviceFilter":
        """filters.Ids / And / Or / Not tree -> device bitmap (leaves uploaded as id lists, combined on the device)."""
        from . import filters as F
        if isinstance(expr, F.Ids):
            return cls.from_ids(ctx, expr.doc_ids, nbits)
        if isinstance(expr, F.Not):
            a = cls.from_expr(ctx, expr.a, nbits)
            try:
                return ~a
            finally:
                a.close()
        if isinstance(expr, (F.And, F.Or)):
            a, b = cls.from_expr(ctx, expr.a, nbits), cls.from_expr(ctx, expr.b, nbits)
            try:
                return (a & b) if isinstance(expr, F.And) else (a | b)
            finally:
                a.close(); b.close()
        raise TypeError(f"not a filter expression: {expr!r}")

    def _bin(self, fn, other):
        h = C.c_void_p()
        check(fn(self._h, other._h, C.byref(h)))
        return DeviceFilter(self.ctx, h, self.nbits)

    def __and__(self, o): return self._bin(lib().oc_filter_and, o)
    def __or__(self, o): return self._bin(lib().oc_filter_or, o)

    def __invert__(self):
        h = C.c_void_p()
        check(lib().oc_filter_not(self._h, C.byref(h)))
        return DeviceFilter(self.ctx, h, self.nbits)

    def count(self) -> int:
        out = C.c_uint64()
        check(lib().oc_filter_count(self._h, C.byref(out)))
        return int(out.value)

    def read(self) -> np.ndarray:
        bits = np.zeros((self.nbits + 63) // 64, np.uint64)
        check(lib().oc_filter_read(self._h, _p(bits)))
        return bits

    def close(self):
        if self._h:
            lib().oc_filter_destroy(self._h)
            self._h = None


# GeoSearchRadiusValue::to_meter (types.rs:2159-2170): the value and the factor are f32, so is the product
GEO_UNIT_TO_METER = {"cm": 0.01, "m": 1.0, "km": 1000.0, "ft": 0.3048, "yd": 0.9144, "mi": 1609.344}


def geo_to_meter(value, unit: str = "m") -> float:
    """value.to_meter(unit) in f32, widened to f64 as geo_search_filter_to_op does (geopoint_field.rs:200)."""
    if unit not in GEO_UNIT_TO_METER:
        raise ValueError(f"radius unit {unit!r}: expected one of {tuple(GEO_UNIT_TO_METER)}")
    with np.errstate(over="ignore"):   # an f32 overflow is +inf, refused by the caller like any infinite radius
        return float(np.float32(value) * np.float32(GEO_UNIT_TO_METER[unit]))


def _geo_check(lat: float, lon: float, what: str):
    if not (np.isfinite(lat) and np.isfinite(lon) and -90.0 <= lat <= 90.0 and -180.0 <= lon <= 180.0):
        raise ValueError(f"{what}: invalid coordinates (lat {lat}, lon {lon})")


def _api_coord(p) -> Tuple[float, float]:
    """An API GeoPoint ({"lat", "lon"} or a (lat, lon) pair): f32 values widened to f64 (geopoint_field.rs:198, 216)."""
    lat, lon = (p["lat"], p["lon"]) if isinstance(p, Mapping) else p
    return float(np.float32(lat)), float(np.float32(lon))


class GeoPointField:
    """A geopoint filter field laid out for where-filter leaves on the device (oc_geo_field_*): one (doc_id, lat, lon)
    entry per point, degrees, so a document with several points repeats.  The points are taken as f64, as
    FilterGeoPoint2 carries them.  Ids >= nbits are ignored.  insert() / delete() queue changes that commit() merges.
    radius() / polygon() return a DeviceFilter over [0, nbits) that holds the documents with at least one point inside
    (inside=True) or outside (inside=False); semantics and assumptions in include/oramacore_b200.h."""

    def __init__(self, ctx: Context, nbits: int, doc_ids, lats, lons):
        d = np.ascontiguousarray(np.asarray(doc_ids, np.uint64).reshape(-1))
        la = np.ascontiguousarray(np.asarray(lats, np.float64).reshape(-1))
        lo = np.ascontiguousarray(np.asarray(lons, np.float64).reshape(-1))
        if not (d.shape == la.shape == lo.shape):
            raise ValueError(f"{d.shape[0]} doc ids for {la.shape[0]} latitudes and {lo.shape[0]} longitudes")
        bad = ~(np.isfinite(la) & np.isfinite(lo) & (np.abs(la) <= 90.0) & (np.abs(lo) <= 180.0))
        if bad.any():
            i = int(np.flatnonzero(bad)[0])
            _geo_check(la[i], lo[i], f"geopoint {i}")
        self.ctx, self.nbits, self.n = ctx, int(nbits), int(d.shape[0])
        self._h = C.c_void_p()
        check(lib().oc_geo_field_create(ctx._h, self.nbits, d.shape[0], _p(d), _p(la), _p(lo), C.byref(self._h)))

    def radius(self, lat, lon, value, unit: str = "m", inside: bool = True) -> DeviceFilter:
        """GeoSearchFilter::Radius: centre (lat, lon) as API f32 values, radius value.to_meter(unit) in f32."""
        clat, clon, r = self.radius_args(lat, lon, value, unit)
        h = C.c_void_p()
        check(lib().oc_filter_geo_radius(self._h, clat, clon, r, int(bool(inside)), C.byref(h)))
        return DeviceFilter.of_handle(self.ctx, h)

    @staticmethod
    def radius_args(lat, lon, value, unit: str = "m"):
        """The checked (lat, lon, radius_m) radius() passes to the library."""
        clat, clon = _api_coord((lat, lon))
        _geo_check(clat, clon, "radius centre")
        r = geo_to_meter(value, unit)
        if not (np.isfinite(r) and r >= 0.0):
            raise ValueError(f"radius {value} {unit}: must be finite and >= 0")
        return clat, clon, r

    def polygon(self, coords, inside: bool = True) -> DeviceFilter:
        """GeoSearchFilter::Polygon: `coords` = API GeoPoints ({"lat", "lon"} or (lat, lon) pairs), 3 to
        OC_GEO_MAX_VERTICES of them."""
        la, lo = self.polygon_args(coords)
        h = C.c_void_p()
        check(lib().oc_filter_geo_polygon(self._h, _p(la), _p(lo), la.shape[0], int(bool(inside)), C.byref(h)))
        return DeviceFilter.of_handle(self.ctx, h)

    @staticmethod
    def polygon_args(coords):
        """The checked vertex latitudes and longitudes (f64 arrays) polygon() passes to the library."""
        pts = [(p["lat"], p["lon"]) if isinstance(p, Mapping) else tuple(p) for p in coords]
        if not 3 <= len(pts) <= _lib.OC_GEO_MAX_VERTICES:
            raise ValueError(f"polygon of {len(pts)} vertices: 3 to {_lib.OC_GEO_MAX_VERTICES} are supported")
        a = np.asarray(pts, np.float32).astype(np.float64)   # API f32 values, widened
        la, lo = np.ascontiguousarray(a[:, 0]), np.ascontiguousarray(a[:, 1])
        bad = ~(np.isfinite(la) & np.isfinite(lo) & (np.abs(la) <= 90.0) & (np.abs(lo) <= 180.0))
        if bad.any():
            k = int(np.flatnonzero(bad)[0])
            _geo_check(la[k], lo[k], f"polygon vertex {k}")
        return la, lo

    def insert(self, doc_ids, lats, lons):
        """Queue points (doc_ids[i], lats[i], lons[i]), checked as the constructor checks them; visible after commit()."""
        d = np.ascontiguousarray(np.atleast_1d(np.asarray(doc_ids, np.uint64)).ravel())
        la = np.ascontiguousarray(np.atleast_1d(np.asarray(lats, np.float64)).ravel())
        lo = np.ascontiguousarray(np.atleast_1d(np.asarray(lons, np.float64)).ravel())
        if not (d.shape == la.shape == lo.shape):
            raise ValueError(f"{d.shape[0]} doc ids for {la.shape[0]} latitudes and {lo.shape[0]} longitudes")
        bad = ~(np.isfinite(la) & np.isfinite(lo) & (np.abs(la) <= 90.0) & (np.abs(lo) <= 180.0))
        if bad.any():
            i = int(np.flatnonzero(bad)[0])
            _geo_check(la[i], lo[i], f"geopoint {i}")
        check(lib().oc_geo_field_insert(self._h, d.shape[0], _p(d), _p(la), _p(lo)))

    def delete(self, doc_ids):
        """Queue the removal of every point of the documents (call order: a later insert stays)."""
        d = np.ascontiguousarray(np.atleast_1d(np.asarray(doc_ids, np.uint64)).ravel())
        check(lib().oc_geo_field_delete(self._h, d.shape[0], _p(d)))

    def commit(self, nbits: Optional[int] = None) -> dict:
        """Merge the queued ops into the next version on the device (oc_geo_field_commit_ex), over [0, nbits) (default:
        the current nbits; it may only grow).  Returns the call's statistics (oc_filter_commit_t)."""
        nb = self.nbits if nbits is None else int(nbits)
        st = _lib.FilterCommit()
        check(lib().oc_geo_field_commit_ex(self._h, nb, C.byref(st)))
        self.nbits, self.n = nb, int(st.rows_kept + st.rows_added)
        return st.as_dict()

    def read(self) -> dict:
        """The published points in their device order (ascending document): {"doc_ids", "lat", "lon"}."""
        n = C.c_uint64(0)
        check(lib().oc_geo_field_read(self._h, C.byref(n), None, None, None))
        d, la, lo = np.zeros(n.value, np.uint64), np.zeros(n.value, np.float64), np.zeros(n.value, np.float64)
        check(lib().oc_geo_field_read(self._h, C.byref(n), _p(d), _p(la), _p(lo)))
        return {"doc_ids": d, "lat": la, "lon": lo}

    def close(self):
        if self._h:
            lib().oc_geo_field_destroy(self._h)
            self._h = None


class FacetStore:
    """The filter fields of one Index laid out for facet counting on the device (oc_facets_*): per field the
    variants' document lists — bool true/false (bool_field.rs:182-208), string_filter keys
    (string_filter_field.rs:175-193), number and date fields sorted by value so a range is a slice
    (number_field.rs:368-387).  `leaf()` turns a where-filter leaf on one of these fields into a DeviceFilter."""

    def __init__(self, ctx: Context, nbits: int):
        self.ctx, self.nbits = ctx, int(nbits)
        self._h = C.c_void_p()
        check(lib().oc_facets_create(ctx._h, self.nbits, C.byref(self._h)))
        self.fields: Dict[str, dict] = {}

    def add_date_field(self, name: str, doc_ids, ms):
        """A date field: one millisecond timestamp per (document, value), kept as a number field of kind "date".  The
        doubles are exact: chrono's whole range is below 2^53 ms.  Dates have no facets and no groups
        (group.rs:234-236)."""
        fid = self.add_number_field(name, doc_ids, np.asarray(ms, np.int64).astype(np.float64))
        self.fields[name]["kind"] = "date"
        return fid

    def leaf(self, name: str, flt) -> DeviceFilter:
        """The documents of field `name` matched by the parsed where-filter leaf `flt` (where.Filter), as
        calculate_filter_for_fields does (filter.rs:49-124): a bool or string_filter value is one variant (an unknown
        key gives an empty leaf), a NumberFilter / DateFilter one value interval, compared in f64.  A filter of the
        wrong kind for the field gives an empty leaf."""
        spec = self.leaf_args(name, flt)
        if spec is None:
            return DeviceFilter.from_ids(self.ctx, [], self.nbits)
        h = C.c_void_p()
        if spec[0] == "variant":
            check(lib().oc_filter_facet_variant(self._h, spec[1], spec[2], C.byref(h)))
        else:
            check(lib().oc_filter_facet_range(self._h, spec[1], spec[2], spec[3], spec[4], C.byref(h)))
        return DeviceFilter.of_handle(self.ctx, h)

    def leaf_args(self, name: str, flt):
        """What leaf() asks of the library: ("variant", field id, variant), ("range", field id, lo, hi, flags), or None
        for an empty leaf."""
        from .where import DateFilter, NumberFilter
        f = self.fields[name]
        kind = f["kind"]
        if (kind == "bool" and isinstance(flt, bool)) or (kind == "string" and isinstance(flt, str)):
            key = ("true" if flt else "false") if kind == "bool" else flt
            if key not in f["variant"]:
                return None
            return "variant", f["id"], f["variant"][key]
        if (kind == "number" and isinstance(flt, NumberFilter)) or (kind == "date" and isinstance(flt, DateFilter)):
            # eq / gt / gte / lt / lte / between (number_field.rs:555-642, date_field.rs:271-280) as [lo, hi] + open ends
            b = flt.bounds()
            if flt.op == "between":
                lo, hi, flags = b[0], b[1], 0
            else:
                lo, hi, flags = {"eq": (b, b, 0), "gt": (b, np.inf, _lib.OC_RANGE_LO_OPEN), "gte": (b, np.inf, 0),
                                 "lt": (-np.inf, b, _lib.OC_RANGE_HI_OPEN), "lte": (-np.inf, b, 0)}[flt.op]
            return "range", f["id"], float(lo), float(hi), flags
        return None

    def add_bool_field(self, name: str, true_docs, false_docs):
        return self._add_variants(name, "bool", {"true": true_docs, "false": false_docs})

    def add_string_field(self, name: str, docs_by_key: Dict[str, Sequence[int]]):
        return self._add_variants(name, "string", docs_by_key)

    def _add_variants(self, name, kind, docs_by_key):
        keys = list(docs_by_key)
        lists = [np.sort(np.asarray(list(docs_by_key[k]), np.uint64)) for k in keys]
        offs = np.zeros(len(keys) + 1, np.uint64)
        offs[1:] = np.cumsum([l.shape[0] for l in lists])
        docs = np.ascontiguousarray(np.concatenate(lists) if lists else np.zeros(0, np.uint64))
        fid = C.c_uint32()
        check(lib().oc_facets_add_field(self._h, len(keys), _p(offs), _p(docs), C.byref(fid)))
        self.fields[name] = {"id": fid.value, "kind": kind, "keys": keys, "variant": {k: i for i, k in enumerate(keys)}}
        return fid.value

    def add_number_field(self, name: str, doc_ids, values):
        v = np.asarray(values, np.float64)
        d = np.asarray(doc_ids, np.uint64)
        o = np.argsort(v, kind="stable")
        v, d = np.ascontiguousarray(v[o]), np.ascontiguousarray(d[o])
        fid = C.c_uint32()
        check(lib().oc_facets_add_number_field(self._h, v.shape[0], _p(v), _p(d), C.byref(fid)))
        self.fields[name] = {"id": fid.value, "kind": "number", "values": np.unique(v)}   # distinct values, ascending
        return fid.value

    @staticmethod
    def _ids(doc_ids) -> np.ndarray:
        return np.ascontiguousarray(np.atleast_1d(np.asarray(doc_ids, np.uint64)).ravel())

    def add_key(self, name: str, key) -> int:
        """The variant of `key` in a bool or string_filter field; a new string_filter key gets the next variant
        (oc_facets_add_variant), listed in fields[name]["keys"] from the next commit() on."""
        f = self.fields[name]
        key = ("true" if key else "false") if f["kind"] == "bool" else key
        if key in f["variant"]:
            return f["variant"][key]
        pend = f.setdefault("pending_keys", {})
        if key not in pend:
            if f["kind"] != "string":
                raise ValueError(f"{name!r} is a {f['kind']} field: it has no key {key!r}")
            v = C.c_uint32()
            check(lib().oc_facets_add_variant(self._h, f["id"], C.byref(v)))
            pend[key] = v.value
        return pend[key]

    def insert_variants(self, name: str, doc_ids, keys):
        """Queue one (document, key) entry per pair of a bool (keys True / False, a set per document) or string_filter
        field (a document may list a key several times); visible after commit()."""
        f = self.fields[name]
        d = self._ids(doc_ids)
        v = np.ascontiguousarray([self.add_key(name, k) for k in keys], np.uint32)
        if v.shape != d.shape:
            raise ValueError(f"{d.shape[0]} doc ids for {v.shape[0]} keys")
        check(lib().oc_facets_insert_variants(self._h, f["id"], d.shape[0], _p(d), _p(v),
                                              _lib.OC_FACET_UNIQUE if f["kind"] == "bool" else 0))

    def insert_numbers(self, name: str, doc_ids, values):
        """Queue (document, value) entries of a number field, or of a date field with millisecond timestamps."""
        f = self.fields[name]
        d = self._ids(doc_ids)
        v = np.atleast_1d(np.asarray(values, np.int64 if f["kind"] == "date" else np.float64)).ravel()
        v = np.ascontiguousarray(v.astype(np.float64))
        if v.shape != d.shape:
            raise ValueError(f"{d.shape[0]} doc ids for {v.shape[0]} values")
        check(lib().oc_facets_insert_numbers(self._h, f["id"], d.shape[0], _p(d), _p(v)))

    def clear(self, name: str, doc_ids):
        """Queue the removal of every value of the documents in field `name` (a replaced value)."""
        d = self._ids(doc_ids)
        check(lib().oc_facets_clear(self._h, self.fields[name]["id"], d.shape[0], _p(d)))

    def delete(self, doc_ids):
        """Queue the removal of every value of the documents in every field."""
        d = self._ids(doc_ids)
        check(lib().oc_facets_delete(self._h, d.shape[0], _p(d)))

    def commit(self, nbits: Optional[int] = None) -> dict:
        """Merge the queued ops into the next version of every field on the device (oc_facets_commit_ex), over
        [0, nbits) (default: the current nbits; it may only grow).  Returns the call's statistics (oc_filter_commit_t)."""
        nb = self.nbits if nbits is None else int(nbits)
        st = _lib.FilterCommit()
        check(lib().oc_facets_commit_ex(self._h, nb, C.byref(st)))
        self.nbits = nb
        name_of = {f["id"]: n for n, f in self.fields.items()}
        for f in self.fields.values():
            for key, v in sorted(f.pop("pending_keys", {}).items(), key=lambda kv: kv[1]):
                f["keys"].append(key)
                f["variant"][key] = v
            if f["kind"] in ("number", "date"):
                f["values"] = None   # distinct_values() reads the new version back when asked
            elif f["kind"] == "string":   # the facets list the keys that hold documents, sorted
                off = self.read_offsets(name_of[f["id"]])
                f["listed"] = sorted(k for k, v in f["variant"].items() if off[v + 1] > off[v])
        return st.as_dict()

    def read_offsets(self, name: str) -> np.ndarray:
        """The published variant offsets of a bool or string_filter field (the host copy; no device read)."""
        fid = self.fields[name]["id"]
        nv, n = C.c_uint32(0), C.c_uint64(0)
        check(lib().oc_facets_read_field(self._h, fid, C.byref(nv), C.byref(n), None, None, None))
        off = np.zeros(nv.value + 1, np.uint64)
        check(lib().oc_facets_read_field(self._h, fid, C.byref(nv), C.byref(n), _p(off), None, None))
        return off

    def distinct_values(self, name: str) -> np.ndarray:
        """The distinct values of a number or date field, ascending."""
        f = self.fields[name]
        if f.get("values") is None:
            f["values"] = np.unique(self.read_field(name)["values"])
        return f["values"]

    def read_field(self, name: str) -> dict:
        """Field `name` of the published version as oc_facets_add_* take it: {"doc_ids"} plus {"offsets"} (bool /
        string_filter, one entry per variant + 1) or {"values"} (number / date, ascending)."""
        fid = self.fields[name]["id"]
        nv, n = C.c_uint32(0), C.c_uint64(0)
        check(lib().oc_facets_read_field(self._h, fid, C.byref(nv), C.byref(n), None, None, None))
        d = np.zeros(n.value, np.uint64)
        if self.fields[name]["kind"] in ("number", "date"):
            v = np.zeros(n.value, np.float64)
            check(lib().oc_facets_read_field(self._h, fid, C.byref(nv), C.byref(n), None, _p(v), _p(d)))
            return {"doc_ids": d, "values": v}
        off = np.zeros(nv.value + 1, np.uint64)
        check(lib().oc_facets_read_field(self._h, fid, C.byref(nv), C.byref(n), _p(off), None, _p(d)))
        return {"doc_ids": d, "offsets": off}

    def close(self):
        if self._h:
            lib().oc_facets_destroy(self._h)
            self._h = None


class OmcStore:
    """The OMC map of one Index (omc_committed + its log, index/mod.rs:604-627, 1720-1739) kept on the device
    (oc_omc_*): a score multiplier per document, applied to every score map before count and top-N (search.rs:39-48).
    set() / delete() queue ops, which apply in call order at the next commit(); the last op for a document wins.  Pass
    the store as TokenScoreParams.omc_store: a search reads the published version on the device, with the results of
    the same search given that version as omc_doc_ids / omc_mult."""

    def __init__(self, ctx: Context):
        self.ctx = ctx
        self._h = C.c_void_p()
        check(lib().oc_omc_create(ctx._h, C.byref(self._h)))

    def set(self, doc_ids, mults):
        """Queue (doc_ids[i], mults[i]).  Any finite f32 is taken; NaN or +-inf raises and queues nothing."""
        d = np.ascontiguousarray(doc_ids, np.uint64).reshape(-1)
        m = np.ascontiguousarray(mults, np.float32).reshape(-1)
        if d.shape != m.shape:
            raise ValueError(f"{d.shape[0]} doc_ids for {m.shape[0]} multipliers")
        check(lib().oc_omc_set(self._h, _p(d), _p(m), d.shape[0]))

    def delete(self, doc_ids):
        """Queue the removal of the documents' multipliers."""
        d = np.ascontiguousarray(doc_ids, np.uint64).reshape(-1)
        check(lib().oc_omc_delete(self._h, _p(d), d.shape[0]))

    def commit(self) -> dict:
        """Merge the queued ops into the next version on the device (oc_omc_commit_ex).  Returns the call's
        statistics (oc_filter_commit_t)."""
        st = _lib.FilterCommit()
        check(lib().oc_omc_commit_ex(self._h, C.byref(st)))
        return st.as_dict()

    def read(self):
        """The published version: (doc_ids ascending, multipliers, version number)."""
        n, ver = C.c_uint64(0), C.c_uint64(0)
        check(lib().oc_omc_read(self._h, C.byref(n), None, None, C.byref(ver)))
        d, m = np.zeros(n.value, np.uint64), np.zeros(n.value, np.float32)
        check(lib().oc_omc_read(self._h, C.byref(n), _p(d), _p(m), C.byref(ver)))
        return d, m, int(ver.value)

    def close(self):
        if self._h:
            lib().oc_omc_destroy(self._h)
            self._h = None


def _number_label(x) -> str:
    return str(int(x)) if np.isfinite(x) and float(x) == int(x) else repr(float(x))


def facet_requests(store: FacetStore, facets: Dict[str, dict]):
    """The oc_facet_req tuples (field, variant, from, to) and (field name, label) pairs of one reference-style `facets`
    map: {"field": {"true": bool, "false": bool}} for a bool field, {"field": {"ranges": [{"from": a, "to": b}, ...]}}
    for a number field (labels "from-to", number_field.rs:382), {"field": {}} for a string_filter field (every key; after
    a commit() the keys that hold documents, sorted).
    Date fields have no facets, and ranges only apply to number fields."""
    reqs, labels = [], []
    for name, d in facets.items():
        f = store.fields[name]
        if f["kind"] == "date":
            raise ValueError(f"{name!r} is a date field: dates have no facets")
        if f["kind"] == "number":
            if "ranges" not in d:
                raise ValueError(f"{name!r} is a number field: its facets are ranges")
            for r in d["ranges"]:
                reqs.append((f["id"], 0, float(r["from"]), float(r["to"])))
                labels.append((name, f"{_number_label(r['from'])}-{_number_label(r['to'])}"))
        else:
            if "ranges" in d:
                raise ValueError(f"{name!r} is a {f['kind']} field: ranges apply to number fields")
            for key in f.get("listed", f["keys"]):
                if f["kind"] == "bool" and not d.get(key, False):
                    continue
                reqs.append((f["id"], f["variant"][key], 0.0, 0.0))
                labels.append((name, key))
    return reqs, labels


def _facet_result(counts, labels) -> Dict[str, dict]:
    """FacetResult (types.rs:1508-1511) per field: {"count": n_values, "values": {label: count}}."""
    r: Dict[str, dict] = {}
    for j, (name, label) in enumerate(labels):
        r.setdefault(name, {"count": 0, "values": {}})["values"][label] = int(counts[j])
    for v in r.values():
        v["count"] = len(v["values"])
    return r


def search_facets(tsc: "TokenScoreContext", store: FacetStore, params: "TokenScoreParams", facets: Dict[str, dict], texts=None,
                  q_vecs: Optional[np.ndarray] = None) -> List[Dict[str, dict]]:
    """`facets` as in the reference's SearchParams (see facet_requests), one map for every query.  Returns, per query,
    {field: {"count": n_values, "values": {label: count}}}.  The where-filter of `params` is ignored, as in
    search.rs:361-396."""
    reqs, labels = facet_requests(store, facets)
    sp, keep, B = tsc._build_params(params, texts, q_vecs)
    arr = (_lib.FacetReq * len(reqs))(*[_lib.FacetReq(*r) for r in reqs])
    out = np.zeros((B, max(len(reqs), 1)), np.uint64)
    check(lib().oc_search_facets(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, store._h,
                                 C.byref(sp), arr, len(reqs), _p(out)))
    return [_facet_result(out[q], labels) for q in range(B)]


class GroupBy:
    """GroupByConfig.properties (types.rs:1367-1371) over the filter fields of a FacetStore (oc_group_by_*): one group per
    combination of the fields' variants, last property varying fastest (generate_group_combinations, read/index/group.rs).
    `values[g]` is group g's key: True / False for a bool field, the key for a string_filter field, the float value for a
    number field (its distinct values, ascending)."""

    def __init__(self, store: FacetStore, properties: Sequence[str]):
        self.ctx, self.properties = store.ctx, list(properties)
        fs = [store.fields[p] for p in self.properties]
        for p, f in zip(self.properties, fs):
            if f["kind"] == "date":
                raise ValueError(f"{p!r} is a date field: groups on dates are refused (group.rs:234-236)")
        ids = np.asarray([f["id"] for f in fs], np.uint32)
        self._h, n = C.c_void_p(), C.c_uint64()
        check(lib().oc_group_by_create(store._h, _p(ids), ids.shape[0], C.byref(self._h), C.byref(n)))
        self.n_groups = int(n.value)
        per_field = []
        for p, f in zip(self.properties, fs):
            if f["kind"] == "bool":
                per_field.append([k == "true" for k in f["keys"]])
            elif f["kind"] == "number":
                per_field.append([float(x) for x in store.distinct_values(p)])
            else:
                per_field.append(list(f["keys"]))
        self.values: List[list] = [[]]
        for vals in per_field:
            self.values = [v + [x] for v in self.values for x in vals]
        assert len(self.values) == self.n_groups

    def close(self):
        if self._h:
            lib().oc_group_by_destroy(self._h)
            self._h = None


def search_groups_arrays(tsc: "TokenScoreContext", group_by: GroupBy, params: "TokenScoreParams", max_results: int = 1, texts=None,
                         q_vecs: Optional[np.ndarray] = None, promote=None, sort_by: Optional[Tuple["SortField", str]] = None):
    """oc_search_groups as arrays: (docs [B,limit], scores, n [B], count [B], group docs [B,G,stride], group scores,
    group n [B,G]); stride = max_results.  With `promote` (see search_pinned_arrays) the call is oc_search_groups_pinned:
    a query with items gets pinned hits and every group's top 2 * max_results with its member items spliced in
    (apply_pin_rules_to_group), stride = 2 * max_results + the most items of one query.  With `sort_by` (a
    (SortField, order) pair, see resolve_sort_by) the call is oc_search_groups_sorted: hits and groups in field order,
    and two more arrays are returned, the hits' sort values [B,limit] and the groups' [B,G,stride]."""
    sp, keep, B = tsc._build_params(params, texts, q_vecs)
    L, G = params.limit_hint, group_by.n_groups
    pins = None if promote is None else _pins(promote, B)
    stride = max_results
    if pins is not None and pins[1]:
        stride = 2 * max_results + pins[1]
    docs, scores = np.zeros((B, L), np.uint64), np.zeros((B, L), np.float32)
    n, cnt = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    gd, gs = np.zeros((B, G, stride), np.uint64), np.zeros((B, G, stride), np.float32)
    gn = np.zeros((B, G), np.uint32)
    emb, strs = tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None
    if sort_by is not None:
        srt = _sort(*sort_by)
        sv, gsv = np.zeros((B, L), np.float64), np.zeros((B, G, stride), np.float64)
        check(lib().oc_search_groups_sorted(tsc.ctx._h, emb, strs, group_by._h, C.byref(sp), int(max_results), C.byref(srt),
                                            None if pins is None else C.byref(pins[0]), int(stride), _p(docs), _p(scores),
                                            _p(sv), _p(n), _p(cnt), _p(gd), _p(gs), _p(gsv), _p(gn)))
        return docs, scores, n, cnt, gd, gs, gn, sv, gsv
    if pins is None:
        check(lib().oc_search_groups(tsc.ctx._h, emb, strs, group_by._h, C.byref(sp), int(max_results), _p(docs), _p(scores), _p(n),
                                     _p(cnt), _p(gd), _p(gs), _p(gn)))
    else:
        check(lib().oc_search_groups_pinned(tsc.ctx._h, emb, strs, group_by._h, C.byref(sp), int(max_results), C.byref(pins[0]),
                                            int(stride), _p(docs), _p(scores), _p(n), _p(cnt), _p(gd), _p(gs), _p(gn)))
    return docs, scores, n, cnt, gd, gs, gn


def search_groups(tsc: "TokenScoreContext", group_by: GroupBy, params: "TokenScoreParams", max_results: int = 1, texts=None,
                  q_vecs: Optional[np.ndarray] = None, promote=None, sort_by: Optional[Tuple["SortField", str]] = None):
    """search() with groupBy (search.rs:415-429 + sort_groups, read/sort.rs:129-230): per query (hits, groups), groups a
    list in group order of {"values": [...], "result": [(doc_id, score), ...]} (GroupedResult, types.rs:1375), the
    top max_results documents of the group that are in the query's score map.  limit_hint 0 is allowed: no hits, and no
    vector search (the reference's limit_hint = 0).  `promote`: the pin rules' promote items per query (see
    search_pinned_arrays).  `sort_by`: a (SortField, order) pair; hits and group members then come in field order
    (sort_groups with sort_by, read/sort.rs:147-166)."""
    docs, scores, n, cnt, gd, gs, gn = search_groups_arrays(tsc, group_by, params, max_results, texts, q_vecs, promote, sort_by)[:7]
    out = []
    for q in range(cnt.shape[0]):
        hits = SearchHits(docs[q, :n[q]].copy(), scores[q, :n[q]].copy(), int(cnt[q]))
        groups = [{"values": list(group_by.values[g]),
                   "result": [(int(gd[q, g, i]), float(gs[q, g, i])) for i in range(int(gn[q, g]))]} for g in range(group_by.n_groups)]
        out.append((hits, groups))
    return out


def _pins(promote, B: int, apply: bool = True):
    """oc_pins for B queries from `promote` (per query a sequence of PromoteItem or (doc_id, position) pairs, in the
    order extract_pin_rules leaves the matched consequences' items).  Returns (struct, most items of one query, keep)."""
    if len(promote) != B:
        raise ValueError(f"promote has {len(promote)} entries for {B} queries")
    items = [[(int(it.doc_id), int(it.position)) if isinstance(it, PromoteItem) else (int(it[0]), int(it[1])) for it in q]
             for q in promote]
    off = np.zeros(B + 1, np.uint32)
    off[1:] = np.cumsum([len(q) for q in items])
    flat = [it for q in items for it in q]
    doc = np.ascontiguousarray([d for d, _ in flat] or [0], np.uint64)
    pos = np.ascontiguousarray([p for _, p in flat] or [0], np.uint32)
    pins = _lib.Pins(_p(off), _p(doc), _p(pos), 1 if apply else 0)
    pins._keep = (off, doc, pos)
    return pins, max((len(q) for q in items), default=0)


def search_pinned_arrays(tsc: "TokenScoreContext", params: "TokenScoreParams", promote, texts=None,
                         q_vecs: Optional[np.ndarray] = None, apply: bool = True):
    """oc_search_pinned: search() with pin rules (sort_token_scores + apply_pin_rules, read/sort.rs:17-46, 285-391).
    `promote`: per query the promote items (PromoteItem, or (doc_id, position)) of the consequences that matched it.
    Returns (docs [B,limit], scores, n [B], count [B], pin scores [items], pin present [items]): per item, in the
    concatenated order, the document's score-map value (0.0 when it is not a key) and whether it is a key.
    apply=False: oc_search's hits, only the per-item values (the per-index call of merge_index_results_pinned)."""
    sp, keep, B = tsc._build_params(params, texts, q_vecs)
    pins, _ = _pins(promote, B, apply)
    n_items = int(pins._keep[0][-1])
    L = params.limit_hint
    docs, scores = np.zeros((B, L), np.uint64), np.zeros((B, L), np.float32)
    n, cnt = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    ps, pp = np.zeros(max(n_items, 1), np.float32), np.zeros(max(n_items, 1), np.uint8)
    check(lib().oc_search_pinned(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, C.byref(sp),
                                 C.byref(pins), _p(docs), _p(scores), _p(n), _p(cnt), _p(ps), _p(pp)))
    return docs, scores, n, cnt, ps[:n_items], pp[:n_items]


def search_pinned(tsc: "TokenScoreContext", params: "TokenScoreParams", promote, texts=None,
                  q_vecs: Optional[np.ndarray] = None) -> List[SearchHits]:
    """search_pinned_arrays as one SearchHits per query."""
    docs, scores, n, cnt, _, _ = search_pinned_arrays(tsc, params, promote, texts, q_vecs)
    return [SearchHits(docs[i, :n[i]].copy(), scores[i, :n[i]].copy(), int(cnt[i])) for i in range(docs.shape[0])]


def merge_index_results(per_index, limit: int, offset: int = 0) -> List[SearchHits]:
    """search_on_indexes' union of the per-index score maps + top_n + skip/take (search.rs:304-338, 482-498):
    per_index = one (doc_ids [B, limit+offset], scores, n, count) tuple per index, each obtained with
    limit' = limit+offset, offset' = 0, vector_limit = limit."""
    k = len(per_index)
    B, stride = per_index[0][0].shape
    keep = [[np.ascontiguousarray(a) for a in r] for r in per_index]
    arr = lambda j: (C.c_void_p * k)(*[r[j].ctypes.data for r in keep])
    od, os_ = np.zeros((B, limit), np.uint64), np.zeros((B, limit), np.float32)
    on, oc = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    check(lib().oc_merge_results(k, B, limit, offset, stride, arr(0), arr(1), arr(2), arr(3), _p(od), _p(os_), _p(on), _p(oc)))
    return [SearchHits(od[i, :on[i]].copy(), os_[i, :on[i]].copy(), int(oc[i])) for i in range(B)]


def merge_index_results_pinned(per_index, promote, limit: int, offset: int = 0, apply: bool = True) -> List[SearchHits]:
    """The multi-index union with pin rules (oc_merge_pinned, host): per_index = one (doc_ids [B, 2*(limit+offset)],
    scores, n, count, pin scores, pin present) tuple per index, each from search_pinned_arrays with
    limit' = 2 * (limit + offset), offset' = 0, vector_limit = limit, apply=False; `promote` as there."""
    k = len(per_index)
    B, stride = per_index[0][0].shape
    keep = [[np.ascontiguousarray(a) for a in r] for r in per_index]
    arr = lambda j: (C.c_void_p * k)(*[r[j].ctypes.data for r in keep])  # noqa: E731
    pins, _ = _pins(promote, B, apply)
    od, os_ = np.zeros((B, limit), np.uint64), np.zeros((B, limit), np.float32)
    on, oc = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    check(lib().oc_merge_pinned(k, B, limit, offset, stride, arr(0), arr(1), arr(2), arr(3), C.byref(pins), arr(4), arr(5),
                                _p(od), _p(os_), _p(on), _p(oc)))
    return [SearchHits(od[i, :on[i]].copy(), os_[i, :on[i]].copy(), int(oc[i])) for i in range(B)]


class SortField:
    """A number, date or bool filter field laid out for sortBy on the device (oc_sort_field_*): one (doc_id, value)
    entry per value, so a multi-valued document repeats.  kind "number": any real value; "date": millisecond
    timestamps (integers or numpy datetime64); "bool": False / True.  Integers beyond 2^53 and NaN are refused: the
    values travel as doubles.  Immutable: build a new one when the field changes (from_facets builds one from a
    FacetStore field on the device)."""
    KINDS = ("number", "date", "bool")

    def __init__(self, ctx: Context, nbits: int, doc_ids, values, kind: str):
        if kind not in self.KINDS:
            raise ValueError(f"sort field kind {kind!r}: expected one of {self.KINDS}")
        d = np.ascontiguousarray(np.asarray(doc_ids, np.uint64).reshape(-1))
        v = np.asarray(values)
        if kind == "date" and np.issubdtype(v.dtype, np.datetime64):
            v = v.astype("datetime64[ms]").astype(np.int64)
        if kind == "bool":
            v = np.asarray(v, bool).astype(np.float64)
        elif np.issubdtype(v.dtype, np.integer):
            if v.size and int(np.max(np.abs(v.astype(object)))) > 2 ** 53:
                raise ValueError("sort value beyond 2^53: it does not round-trip through a double")
            v = v.astype(np.float64)
        else:
            v = v.astype(np.float64)
        v = np.ascontiguousarray(v.reshape(-1))
        if v.shape != d.shape:
            raise ValueError(f"{d.shape[0]} doc ids for {v.shape[0]} values")
        if np.isnan(v).any():
            raise ValueError("sort value is NaN")
        self.ctx, self.nbits, self.kind = ctx, int(nbits), kind
        self._h = C.c_void_p()
        check(lib().oc_sort_field_create(ctx._h, self.nbits, d.shape[0], _p(d), _p(v), C.byref(self._h)))

    @classmethod
    def from_facets(cls, store: "FacetStore", name: str) -> "SortField":
        """The sort field of field `name` of the store's published version, built on the device from the field's device
        arrays (oc_sort_field_from_facets) over the version's nbits: a number or date field sorts by its values, a bool
        field by true = 1.0, false = 0.0.  A string_filter field raises InvalidSortField(name, "StringFilter") before
        any device call, as resolve_sort_by does, and a name the store does not hold SortFieldNotFound(name).  The
        handle keeps the version it was built from: build a new one after the next commit() of the store."""
        if name not in store.fields:
            raise SortFieldNotFound(name)
        f = store.fields[name]
        vv = None
        if f["kind"] == "string":
            raise InvalidSortField(name, _NOT_SORTABLE["string_filter"])
        if f["kind"] == "bool":
            vv = np.zeros(len(f["keys"]), np.float64)
            vv[f["variant"]["true"]] = 1.0
        self = cls.__new__(cls)
        self.ctx, self.kind = store.ctx, f["kind"]
        self._h = C.c_void_p()
        check(lib().oc_sort_field_from_facets(store._h, f["id"], _p(vv), C.byref(self._h)))
        self.nbits = self._sizes()["nbits"]   # the version's, which a commit on another thread may have moved on from
        return self

    def _sizes(self, order: str = "ASC") -> dict:
        """{"nbits", "n" (documents with a value), "facets_version"} of one order, without reading the arrays."""
        nb, n, ver = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        check(lib().oc_sort_field_read(self._h, _order(order), C.byref(nb), C.byref(n), None, None, C.byref(ver)))
        return {"nbits": int(nb.value), "n": int(n.value), "facets_version": int(ver.value)}

    def read(self, order: str = "ASC") -> dict:
        """One order read back (oc_sort_field_read): {"nbits", "rank_doc" (documents in rank order), "rank_value" (the
        value each was placed by), "facets_version" (from_facets' store version, 0 for a handle built from values)}."""
        sz = self._sizes(order)
        d, v, n = np.zeros(sz["n"], np.uint64), np.zeros(sz["n"], np.float64), C.c_uint64(sz["n"])
        if sz["n"]:
            check(lib().oc_sort_field_read(self._h, _order(order), None, C.byref(n), _p(d), _p(v), None))
        return {"nbits": sz["nbits"], "rank_doc": d, "rank_value": v, "facets_version": sz["facets_version"]}

    def close(self):
        if self._h:
            lib().oc_sort_field_destroy(self._h)
            self._h = None


_NOT_SORTABLE = {"string": "String", "string_filter": "StringFilter", "geopoint": "GeoPoint"}


def resolve_sort_by(fields: Mapping[str, object], sort_by: SortBy) -> Tuple[SortField, str]:
    """The index's field lookup of IndexSortContext::execute (read/index/sort.rs:186-265): `fields` maps every filter
    property to its SortField, or to the kind name of a property that cannot be sorted ("string", "string_filter",
    "geopoint").  Returns the (SortField, order) pair the sorted searches take.  Raises SortFieldNotFound(name) for an
    unknown property and InvalidSortField(name, kind) for one that is not a number, date or bool field."""
    if sort_by.order not in ("ASC", "DESC"):
        raise ValueError(f"sort order {sort_by.order!r}: expected 'ASC' or 'DESC'")
    if sort_by.property not in fields:
        raise SortFieldNotFound(sort_by.property)
    f = fields[sort_by.property]
    if not isinstance(f, SortField):
        raise InvalidSortField(sort_by.property, _NOT_SORTABLE.get(str(f), str(f)))
    return f, sort_by.order


def _order(order: str) -> int:
    if order not in ("ASC", "DESC"):
        raise ValueError(f"sort order {order!r}: expected 'ASC' or 'DESC'")
    return 0 if order == "ASC" else 1


def _sort(field: SortField, order: str = "ASC"):
    return _lib.Sort(field._h, _order(order))


def search_sorted_arrays(tsc: "TokenScoreContext", params: "TokenScoreParams", field: SortField, order: str = "ASC", promote=None,
                         texts=None, q_vecs: Optional[np.ndarray] = None, apply: bool = True):
    """oc_search_sorted: search() with sortBy (sort_token_scores with sort_by, read/sort.rs:17-46, 48-126): the first
    limit + offset keys of the score map in field order, each with its score-map value (NaN kept), then pins and
    skip/take.  `promote` as in search_pinned_arrays (None: no pin rule).  Returns (docs [B,limit], scores, sort values
    [B,limit] (NaN for a promoted item), n [B], count [B], pin scores [items], pin present [items])."""
    sp, keep, B = tsc._build_params(params, texts, q_vecs)
    pins = None if promote is None else _pins(promote, B, apply)[0]
    n_items = 0 if pins is None else int(pins._keep[0][-1])
    L = params.limit_hint
    docs, scores, sv = np.zeros((B, L), np.uint64), np.zeros((B, L), np.float32), np.zeros((B, L), np.float64)
    n, cnt = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    ps, pp = np.zeros(max(n_items, 1), np.float32), np.zeros(max(n_items, 1), np.uint8)
    srt = _sort(field, order)
    check(lib().oc_search_sorted(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, C.byref(sp),
                                 C.byref(srt), None if pins is None else C.byref(pins), _p(docs), _p(scores), _p(sv), _p(n),
                                 _p(cnt), _p(ps), _p(pp)))
    return docs, scores, sv, n, cnt, ps[:n_items], pp[:n_items]


def search_sorted(tsc: "TokenScoreContext", params: "TokenScoreParams", field: SortField, order: str = "ASC", promote=None,
                  texts=None, q_vecs: Optional[np.ndarray] = None) -> List[SearchHits]:
    """search_sorted_arrays as one SearchHits per query."""
    docs, scores, _, n, cnt, _, _ = search_sorted_arrays(tsc, params, field, order, promote, texts, q_vecs)
    return [SearchHits(docs[i, :n[i]].copy(), scores[i, :n[i]].copy(), int(cnt[i])) for i in range(docs.shape[0])]


def _q_sorts(sorts, B: int):
    """oc_sort[B] from `sorts`: per query a (SortField, order) pair, or None for score order."""
    if len(sorts) != B:
        raise ValueError(f"sorts has {len(sorts)} entries for {B} queries")
    arr = (_lib.Sort * max(B, 1))()
    for i, s in enumerate(sorts):
        if s is not None:
            arr[i] = _sort(s[0], s[1])
    return arr


def search_q_sorted_arrays(tsc: "TokenScoreContext", params: "TokenScoreParams", sorts, promote=None, texts=None,
                           q_vecs: Optional[np.ndarray] = None):
    """oc_search_q_sorted: one batch in which every query has its own sort and pin rules, and (params.device_filters)
    its own where-filter.  `sorts[b]`: a (SortField, order) pair, or None for score order; `promote` as in
    search_pinned_arrays.  Query b gets what search_sorted_arrays (a sort) or search_pinned_arrays (None; sort values
    NaN) give it alone.  Returns what search_sorted_arrays returns."""
    sp, keep, B = tsc._build_params(params, texts, q_vecs)
    srt = _q_sorts(sorts, B)
    pins = None if promote is None else _pins(promote, B)[0]
    n_items = 0 if pins is None else int(pins._keep[0][-1])
    L = _stride(params)
    docs, scores, sv = np.zeros((B, L), np.uint64), np.zeros((B, L), np.float32), np.zeros((B, L), np.float64)
    n, cnt = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    ps, pp = np.zeros(max(n_items, 1), np.float32), np.zeros(max(n_items, 1), np.uint8)
    check(lib().oc_search_q_sorted(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, C.byref(sp),
                                   srt, None if pins is None else C.byref(pins), _p(docs), _p(scores), _p(sv), _p(n),
                                   _p(cnt), _p(ps), _p(pp)))
    return docs, scores, sv, n, cnt, ps[:n_items], pp[:n_items]


def _group_reqs(groups, B: int):
    """oc_group_req[B] and the group row of each query from `groups`: per query None (no groups, score order) or a
    (GroupBy or None, max_results[, (SortField, order)]) tuple."""
    if len(groups) != B:
        raise ValueError(f"groups has {len(groups)} entries for {B} queries")
    arr = (_lib.GroupReq * max(B, 1))()
    rows = np.zeros(B + 1, np.int64)
    for i, g in enumerate(groups):
        rows[i + 1] = rows[i]
        if g is None:
            continue
        if g[0] is not None:
            arr[i].groups, arr[i].max_results = g[0]._h, int(g[1])
            rows[i + 1] += g[0].n_groups
        if len(g) > 2 and g[2] is not None:
            arr[i].sort = _sort(*g[2])
    return arr, rows


def _group_need(g, k: int) -> int:
    """The group stride one request needs: 2 * max_results + its items when it has items, else max_results."""
    if g is None or g[0] is None:
        return 0
    return 2 * int(g[1]) + k if k else int(g[1])


def _q_outputs(B: int, L: int, n_items: int, R: int, S: int):
    """Zeroed outputs of oc_search_q_groups: docs, scores, sort values [B,L], n, count [B], pin scores, pin present
    [max(items, 1)], group docs, group scores, group sort values [R,S], group n [R]."""
    return (np.zeros((B, L), np.uint64), np.zeros((B, L), np.float32), np.zeros((B, L), np.float64), np.zeros(B, np.uint32),
            np.zeros(B, np.uint64), np.zeros(max(n_items, 1), np.float32), np.zeros(max(n_items, 1), np.uint8),
            np.zeros((R, S), np.uint64), np.zeros((R, S), np.float32), np.zeros((R, S), np.float64), np.zeros(R, np.uint32))


def search_q_groups_arrays(tsc: "TokenScoreContext", params: "TokenScoreParams", groups, promote=None, texts=None,
                           q_vecs: Optional[np.ndarray] = None, group_stride: Optional[int] = None):
    """oc_search_q_groups: one batch in which every query has its own groupBy, sortBy and pin rules, and
    (params.device_filters) its own where-filter.  `groups[b]`: None (no groups: the hits of search_q_sorted_arrays in
    score order), or (GroupBy, max_results) or (GroupBy, max_results, (SortField, order)); `promote` as in
    search_pinned_arrays.  (None, 0, (SortField, order)) is a query without groups in field order.  Query b gets what it
    gets alone from search_groups_arrays (with its sort and items) or, without groups, search_q_sorted_arrays.  group_stride: default the largest need of the batch.  Returns (docs [B,limit],
    scores, sort values [B,limit], n [B], count [B], pin scores [items], pin present [items], group docs [rows,stride],
    group scores, group sort values [rows,stride], group n [rows], rows [B+1]): query b's groups are the rows
    [rows[b], rows[b+1])."""
    sp, keep, B = tsc._build_params(params, texts, q_vecs)
    req, rows = _group_reqs(groups, B)
    pins = None if promote is None else _pins(promote, B)[0]
    n_items = 0 if pins is None else int(pins._keep[0][-1])
    if group_stride is None:
        k = [0] * B if promote is None else [len(x) for x in promote]
        group_stride = max([0] + [_group_need(g, k[b]) for b, g in enumerate(groups)])
    L, R, S = _stride(params), int(rows[-1]), int(group_stride)
    docs, scores, sv, n, cnt, ps, pp, gd, gs, gsv, gn = _q_outputs(B, L, n_items, R, S)
    check(lib().oc_search_q_groups(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, C.byref(sp),
                                   req, None if pins is None else C.byref(pins), S, _p(docs), _p(scores), _p(sv), _p(n),
                                   _p(cnt), _p(ps), _p(pp), _p(gd), _p(gs), _p(gsv), _p(gn)))
    return docs, scores, sv, n, cnt, ps[:n_items], pp[:n_items], gd, gs, gsv, gn, rows


def search_q_groups(tsc: "TokenScoreContext", params: "TokenScoreParams", groups, promote=None, texts=None,
                    q_vecs: Optional[np.ndarray] = None):
    """search_q_groups_arrays as search_groups returns it: per query (hits, groups), groups None for a query without
    groupBy."""
    docs, scores, _, n, cnt, _, _, gd, gs, _, gn, rows = search_q_groups_arrays(tsc, params, groups, promote, texts, q_vecs)
    out = []
    for q in range(cnt.shape[0]):
        hits = SearchHits(docs[q, :n[q]].copy(), scores[q, :n[q]].copy(), int(cnt[q]))
        res = None
        if groups[q] is not None and groups[q][0] is not None:
            gb = groups[q][0]
            res = [{"values": list(gb.values[g]), "result": [(int(gd[r, i]), float(gs[r, i])) for i in range(int(gn[r]))]}
                   for g, r in enumerate(range(int(rows[q]), int(rows[q + 1])))]
        out.append((hits, res))
    return out


def _q_facet_reqs(store: FacetStore, facets, B: int):
    """oc_facet_req[] in query order, q_facet_offsets [B+1] and each query's labels, from one facets map (or None) per
    query."""
    if len(facets) != B:
        raise ValueError(f"facets has {len(facets)} entries for {B} queries")
    reqs, labels, off = [], [], np.zeros(B + 1, np.uint32)
    for b, f in enumerate(facets):
        r, lab = facet_requests(store, f) if f else ([], [])
        reqs += r
        labels.append(lab)
        off[b + 1] = len(reqs)
    arr = (_lib.FacetReq * max(len(reqs), 1))(*[_lib.FacetReq(*r) for r in reqs])
    return arr, off, labels


def search_q_facets_arrays(tsc: "TokenScoreContext", store: FacetStore, params: "TokenScoreParams", facets, groups=None,
                           promote=None, texts=None, q_vecs: Optional[np.ndarray] = None, group_stride: Optional[int] = None):
    """oc_search_q_facets: search_q_groups_arrays with each query's own facets (`facets[b]`: a reference-style map, see
    facet_requests, or None) counted in the same call.  `groups` None: no query has groups.  Returns
    search_q_groups_arrays' tuple followed by (facet counts [requests], q_facet_offsets [B+1], labels per query): query b's
    counts are counts[off[b]:off[b+1]], what search_facets gives it alone (its where-filter ignored)."""
    sp, keep, B = tsc._build_params(params, texts, q_vecs)
    req, rows = _group_reqs(groups if groups is not None else [None] * B, B)
    farr, foff, labels = _q_facet_reqs(store, facets, B)
    pins = None if promote is None else _pins(promote, B)[0]
    n_items = 0 if pins is None else int(pins._keep[0][-1])
    if group_stride is None:
        k = [0] * B if promote is None else [len(x) for x in promote]
        group_stride = max([0] + [_group_need(g, k[b]) for b, g in enumerate(groups or [None] * B)])
    L, R, S = _stride(params), int(rows[-1]), int(group_stride)
    docs, scores, sv, n, cnt, ps, pp, gd, gs, gsv, gn = _q_outputs(B, L, n_items, R, S)
    fc = np.zeros(max(int(foff[-1]), 1), np.uint64)
    check(lib().oc_search_q_facets(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, C.byref(sp),
                                   req, None if pins is None else C.byref(pins), S, store._h, _p(foff), farr, _p(docs),
                                   _p(scores), _p(sv), _p(n), _p(cnt), _p(ps), _p(pp), _p(gd), _p(gs), _p(gsv), _p(gn), _p(fc)))
    return (docs, scores, sv, n, cnt, ps[:n_items], pp[:n_items], gd, gs, gsv, gn, rows, fc[:int(foff[-1])], foff, labels)


def search_q_facets(tsc: "TokenScoreContext", store: FacetStore, params: "TokenScoreParams", facets, groups=None, promote=None,
                    texts=None, q_vecs: Optional[np.ndarray] = None):
    """search_q_facets_arrays as search_q_groups returns it, plus the facets: per query (hits, groups, facets), groups
    None without groupBy, facets None without facets, else {field: FacetResult}."""
    got = search_q_facets_arrays(tsc, store, params, facets, groups, promote, texts, q_vecs)
    docs, scores, n, cnt, gd, gs, gn, rows, fc, foff, labels = got[0], got[1], got[3], got[4], got[7], got[8], got[10], got[11], \
        got[12], got[13], got[14]
    out = []
    for q in range(cnt.shape[0]):
        hits = SearchHits(docs[q, :n[q]].copy(), scores[q, :n[q]].copy(), int(cnt[q]))
        res = None
        if groups is not None and groups[q] is not None and groups[q][0] is not None:
            gb = groups[q][0]
            res = [{"values": list(gb.values[g]), "result": [(int(gd[r, i]), float(gs[r, i])) for i in range(int(gn[r]))]}
                   for g, r in enumerate(range(int(rows[q]), int(rows[q + 1])))]
        fr = _facet_result(fc[foff[q]:foff[q + 1]], labels[q]) if facets[q] else None
        out.append((hits, res, fr))
    return out


def merge_index_results_sorted(per_index, order: str, limit: int, offset: int = 0, promote=None, apply: bool = True):
    """The multi-index union in field order (oc_merge_sorted, host; MergeSortedIterator, read/sort.rs:491-559):
    per_index = one (doc_ids [B, limit'], scores, sort values, n, count[, pin scores, pin present]) tuple per index, each
    from search_sorted_arrays with limit' = limit + offset (2 * (limit + offset) and apply=False with pins), offset' = 0,
    vector_limit = limit.  On equal values the index listed first wins.  Returns (List[SearchHits], sort values
    [B, limit])."""
    k = len(per_index)
    B, stride = per_index[0][0].shape
    keep = [[np.ascontiguousarray(a) for a in r] for r in per_index]
    arr = lambda j: (C.c_void_p * k)(*[r[j].ctypes.data for r in keep])  # noqa: E731
    pins = None if promote is None else _pins(promote, B, apply)[0]
    od, os_, ov = np.zeros((B, limit), np.uint64), np.zeros((B, limit), np.float32), np.zeros((B, limit), np.float64)
    on, oc = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    if order not in ("ASC", "DESC"):
        raise ValueError(f"sort order {order!r}: expected 'ASC' or 'DESC'")
    check(lib().oc_merge_sorted(k, B, limit, offset, stride, 0 if order == "ASC" else 1, arr(0), arr(1), arr(2), arr(3), arr(4),
                                None if pins is None else C.byref(pins), arr(5) if pins is not None else None,
                                arr(6) if pins is not None else None, _p(od), _p(os_), _p(ov), _p(on), _p(oc)))
    return [SearchHits(od[i, :on[i]].copy(), os_[i, :on[i]].copy(), int(oc[i])) for i in range(B)], ov


@dataclass
class IndexPart:
    """One index of a search_indexes call: its TokenScoreContext (its embedding and string stores), its own query
    inputs (texts resolved with its own dictionary, q_vecs) and its index fields as TokenScoreParams fields of those
    names: device_filter / device_filters / where_programs / filtered_doc_ids + filter_nbits over its own filter fields,
    and omc_store or omc_doc_ids / omc_mult; store: its FacetStore, which facets across the indexes count over."""
    tsc: "TokenScoreContext"
    texts: object = None
    q_vecs: Optional[np.ndarray] = None
    fields: Optional[Mapping[str, object]] = None
    store: Optional[FacetStore] = None


def _group_value_key(v):
    """A group value as a dict key: a bool, a string or a float compared with == (so -0.0 is +0.0), kinds kept apart."""
    if isinstance(v, (bool, np.bool_)):
        return ("b", bool(v))
    if isinstance(v, str):
        return ("s", v)
    return ("f", float(v) + 0.0)


def collection_group_keys(group_bys: Sequence[Optional["GroupBy"]]):
    """The collection's groups over the indexes' GroupBy handles (None: the index adds no groups): the keys in order of
    first appearance, index by index, each a list of property values (GroupBy.values), and per index the key of each of
    its local groups (uint32 [n_groups], None without a handle).  Keys are compared as _group_value_key compares values."""
    index, keys, maps = {}, [], []
    for gb in group_bys:
        if gb is None:
            maps.append(None)
            continue
        m = np.zeros(max(gb.n_groups, 1), np.uint32)
        for g, vals in enumerate(gb.values):
            k = tuple(_group_value_key(v) for v in vals)
            if k not in index:
                index[k] = len(keys)
                keys.append(list(vals))
            m[g] = index[k]
        maps.append(m)
    return keys, maps


def collection_facet_requests(stores: Sequence[Optional[FacetStore]], facets: Dict[str, dict]):
    """The collection's facet slots of one reference-style `facets` map (see facet_requests) over the indexes' stores
    (None: an index without filter fields): the slot labels [(field, label)] and per index its (requests, slots).  A slot
    is labelled as facet_requests labels it; a string_filter field gets the union of the indexes' keys in order of first
    appearance, index by index.  Fields that no index has raise KeyError([fields]) (the caller's FacetFieldNotFound); a
    definition of the wrong kind for an index's field, or a date field, raises ValueError."""
    labels, slot_of, per_index = [], {}, []
    missing = [name for name in facets if not any(st is not None and name in st.fields for st in stores)]
    if missing:
        raise KeyError(missing)
    for st in stores:
        reqs, slots = [], []
        if st is not None:
            present = {k: v for k, v in facets.items() if k in st.fields}
            r, lab = facet_requests(st, present)
            for req, l in zip(r, lab):
                if l not in slot_of:
                    slot_of[l] = len(labels)
                    labels.append(l)
                reqs.append(req)
                slots.append(slot_of[l])
        per_index.append((reqs, slots))
    # slots in field order of the map, labels in order of first appearance inside a field
    order = sorted(range(len(labels)), key=lambda j: (list(facets).index(labels[j][0]), j))
    renum = {old: new for new, old in enumerate(order)}
    return [labels[j] for j in order], [(r, [renum[x] for x in sl]) for r, sl in per_index]


def search_indexes_arrays(ctx: Context, parts: Sequence[IndexPart], params: "TokenScoreParams", sorts=None, promote=None,
                          groups=None, facets=None, group_stride: Optional[int] = None):
    """oc_search_indexes_ex: search_on_indexes (read/search.rs:283-501) over the indexes of one collection in one call.
    `params` holds the request (mode, limit, offset, similarity, threshold, query_params; vector_limit must be 0) and is
    shared by every index; each part adds its index's inputs.  `sorts`: None (score order), or per index None or per
    query a (SortField, order) pair or None; query b is sorted when every index gives it a field in one order.
    `promote` as in search_pinned_arrays.  Returns (docs [B,limit], scores, sort values [B,limit], n [B], count [B],
    pin scores [items], pin present [items]), byte for byte the per-index searches merged by the host merges.
    `groups` (per query None or (per index a GroupBy or None, max_results)) and `facets` (per query None or a
    reference-style map, counted over each part's `store`) add, after those seven, (group docs [rows,stride], group
    scores, group sort values [rows,stride], group n [rows], rows [B+1], group keys per query (collection_group_keys),
    facet counts [slots], q_facet_offsets [B+1], slot labels per query (collection_facet_requests)): query b's groups
    are rows [rows[b], rows[b+1]), its counts counts[off[b]:off[b+1]]."""
    import dataclasses
    if not parts:
        raise ValueError("search_indexes needs at least one index")
    keep, built = [], []
    for part in parts:
        sp, k, B = part.tsc._build_params(dataclasses.replace(params, **dict(part.fields or {})), part.texts, part.q_vecs)
        keep += [sp, k]
        built.append((part.tsc, sp))
    B = built[0][1].n_queries
    ni = len(parts)
    ixs = (_lib.IndexQuery * ni)()
    for i, (tsc, sp) in enumerate(built):
        srt = None
        if sorts is not None and sorts[i] is not None:
            srt = _q_sorts(sorts[i], B)
            keep.append(srt)
        ixs[i] = _lib.IndexQuery(tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None, C.pointer(sp),
                                 None if srt is None else C.cast(srt, C.c_void_p))
    pins = None if promote is None else _pins(promote, B)[0]
    n_items = 0 if pins is None else int(pins._keep[0][-1])
    L = _stride(params)
    docs, scores, sv = np.zeros((B, L), np.uint64), np.zeros((B, L), np.float32), np.zeros((B, L), np.float64)
    n, cnt = np.zeros(B, np.uint32), np.zeros(B, np.uint64)
    ps, pp = np.zeros(max(n_items, 1), np.float32), np.zeros(max(n_items, 1), np.uint8)
    if groups is None and facets is None:
        check(lib().oc_search_indexes(ctx._h, ni, ixs, None if pins is None else C.byref(pins), _p(docs), _p(scores),
                                      _p(sv), _p(n), _p(cnt), _p(ps), _p(pp)))
        return docs, scores, sv, n, cnt, ps[:n_items], pp[:n_items]
    ex = (_lib.IndexExtras * ni)()
    # groups: one key union per distinct combination of handles, shared by the queries that ask for it
    groups = groups if groups is not None else [None] * B
    if len(groups) != B:
        raise ValueError(f"groups has {len(groups)} entries for {B} queries")
    n_keys, max_res, q_keys, combos = np.zeros(B, np.uint32), np.zeros(B, np.uint32), [], {}
    q_gb = [(C.c_void_p * max(B, 1))() for _ in range(ni)]
    q_km = [(C.c_void_p * max(B, 1))() for _ in range(ni)]
    for b, g in enumerate(groups):
        if g is None:
            q_keys.append(None)
            continue
        gbs, m = list(g[0]), int(g[1])
        if len(gbs) != ni:
            raise ValueError(f"groups[{b}] has {len(gbs)} handles for {ni} indexes")
        ck = tuple(id(x) for x in gbs)
        if ck not in combos:
            combos[ck] = collection_group_keys(gbs)
        keys, maps = combos[ck]
        n_keys[b], max_res[b] = len(keys), m
        q_keys.append(keys)
        for i, gb in enumerate(gbs):
            if gb is not None:
                q_gb[i][b], q_km[i][b] = gb._h, maps[i].ctypes.data
    keep += [combos, q_gb, q_km]
    rows = np.zeros(B + 1, np.int64)
    rows[1:] = np.cumsum(n_keys)
    if group_stride is None:
        k = [0] * B if promote is None else [len(x) for x in promote]
        group_stride = max([0] + [_group_need((True, max_res[b]), k[b]) for b in range(B) if n_keys[b]])
    R, S = int(rows[-1]), int(group_stride)
    gd, gs, gsv = np.zeros((R, S), np.uint64), np.zeros((R, S), np.float32), np.zeros((R, S), np.float64)
    gn = np.zeros(R, np.uint32)
    # facets: per query its collection slots, per index its requests and their slots
    facets = facets if facets is not None else [None] * B
    if len(facets) != B:
        raise ValueError(f"facets has {len(facets)} entries for {B} queries")
    stores = [getattr(p, "store", None) for p in parts]
    foff, labels, planned = np.zeros(B + 1, np.uint32), [], {}
    f_reqs, f_slots = [[] for _ in range(ni)], [[] for _ in range(ni)]
    for b, f in enumerate(facets):
        if f and id(f) not in planned:   # once per distinct map of the batch
            planned[id(f)] = collection_facet_requests(stores, f)
        lab, per = planned[id(f)] if f else ([], [([], [])] * ni)
        for i, (r, sl) in enumerate(per):
            f_reqs[i] += r
            f_slots[i] += [int(foff[b]) + x for x in sl]
        labels.append(lab)
        foff[b + 1] = foff[b] + len(lab)
    fc = np.zeros(max(int(foff[-1]), 1), np.uint64)
    for i in range(ni):
        ex[i].q_groups = C.cast(q_gb[i], C.c_void_p) if any(g is not None and g[0][i] is not None for g in groups) else None
        ex[i].q_group_keys = C.cast(q_km[i], C.c_void_p)
        if f_reqs[i]:
            arr = (_lib.FacetReq * len(f_reqs[i]))(*[_lib.FacetReq(*r) for r in f_reqs[i]])
            sl = np.asarray(f_slots[i], np.uint32)
            keep += [arr, sl]
            ex[i].facets, ex[i].n_facet_reqs = stores[i]._h, len(f_reqs[i])
            ex[i].facet_reqs, ex[i].facet_slots = C.cast(arr, C.c_void_p), sl.ctypes.data
    check(lib().oc_search_indexes_ex(ctx._h, ni, ixs, ex, None if pins is None else C.byref(pins), _p(n_keys), _p(max_res), S,
                                     _p(foff), _p(docs), _p(scores), _p(sv), _p(n), _p(cnt), _p(ps), _p(pp), _p(gd), _p(gs),
                                     _p(gsv), _p(gn), _p(fc)))
    return (docs, scores, sv, n, cnt, ps[:n_items], pp[:n_items], gd, gs, gsv, gn, rows, q_keys, fc[:int(foff[-1])], foff,
            labels)


def search_indexes(ctx: Context, parts: Sequence[IndexPart], params: "TokenScoreParams", sorts=None,
                   promote=None) -> List[SearchHits]:
    """search_indexes_arrays as one SearchHits per query."""
    docs, scores, _, n, cnt, _, _ = search_indexes_arrays(ctx, parts, params, sorts, promote)
    return [SearchHits(docs[i, :n[i]].copy(), scores[i, :n[i]].copy(), int(cnt[i])) for i in range(docs.shape[0])]


class TermDictionary:
    """Native term dictionaries of the string fields of one Index + batch query resolution (oc_dict_*,
    csrc/dict.h): tokenize (+ stem hook), then per field exact / prefix / Levenshtein expansion — what
    TextParser::tokenize_and_stem and the FST inside StringStorage do in the reference
    (token_score.rs:196-209, string_field.rs:208-225).  Works without a GPU; resolve_batch(ctx=...) expands typos
    on that ctx's device."""

    def __init__(self, n_fields: int = 1):
        self.n_fields = n_fields
        self._h = C.c_void_p()
        check(lib().oc_dict_create(n_fields, C.byref(self._h)))
        self._stem_cb = None

    def close(self):
        if self._h:
            lib().oc_dict_destroy(self._h)
            self._h = C.c_void_p()

    def add_terms(self, field: int, terms: Sequence[str]) -> np.ndarray:
        """Returns the (stable) ids of the terms; known terms keep their id, new ones get the next."""
        arr = (C.c_char_p * len(terms))(*[t.encode("utf-8") for t in terms])
        ids = np.zeros(len(terms), np.uint32)
        check(lib().oc_dict_add_terms(self._h, field, arr, len(terms), _p(ids)))
        return ids

    def lookup(self, field: int, term: str) -> Optional[int]:
        out = C.c_uint32()
        check(lib().oc_dict_lookup(self._h, field, term.encode("utf-8"), C.byref(out)))
        return None if out.value == 0xffffffff else int(out.value)

    def size(self, field: int) -> int:
        return int(lib().oc_dict_size(self._h, field))

    def set_stemmer(self, fn):
        """fn(token: str) -> Optional[str]; None / "" = no stem (test hook: a production binding passes a C function)."""
        def cb(tok, n, out, cap, _user):
            s = fn(C.string_at(tok, n).decode("utf-8"))
            if not s:
                return 0
            b = s.encode("utf-8")
            if len(b) > cap:
                return 0
            C.memmove(out, b, len(b))
            return len(b)
        self._stem_cb = _lib.STEM_FN(cb) if fn is not None else None
        check(lib().oc_dict_set_stemmer(self._h, C.cast(self._stem_cb, C.c_void_p) if fn is not None else None, None))

    def use_english_stemmer(self):
        """Install the built-in Snowball English (Porter2) stemmer (oc_stem_english)."""
        check(lib().oc_dict_set_stemmer(self._h, C.cast(lib().oc_stem_english, C.c_void_p), None))

    @staticmethod
    def stem_english(token: str) -> str:
        b = token.encode("utf-8")
        out = C.create_string_buffer(len(b) + 8)
        n = lib().oc_stem_english(b, len(b), out, len(b) + 8, None)
        return out.raw[:n].decode("utf-8") if n else token

    def _field_arrays(self, boost, properties):
        fb = None if boost is None else np.ascontiguousarray(boost, np.float32)
        if fb is not None and fb.size != self.n_fields:
            raise ValueError(f"boost has {fb.size} entries for {self.n_fields} fields")
        fm = None
        if properties is not None:
            fm = np.zeros(self.n_fields, np.uint8)
            fm[list(properties)] = 1
        return fb, fm

    def device_bytes(self, ctx: "Context") -> int:
        """Device memory of this dictionary's mirror on ctx (0 before the first resolve_batch(ctx=ctx) that needed it)."""
        return int(lib().oc_dict_device_bytes(self._h, ctx._h))

    def resolve_batch(self, texts: Sequence[str], exact=False, tolerance=None, boost=None, properties=None,
                      exact_match_boost: float = 0.0, ctx: Optional["Context"] = None) -> "TextQueryBatch":
        """SearchParams{tokens, exact_match, boost, tolerance} for B queries at once (token_score.rs:235-242)
        -> the packed CSR arrays oc_search takes.  exact (bool), tolerance (None or int), boost (None or one weight per
        field) and properties (None or field indexes) each take one value for the batch or a list of one per query.
        With a ctx, the tolerance >= 1 expansions run on its device (oc_dict_resolve_q); the output is the same."""
        B = len(texts)

        def per_query(v, single):
            if single(v):
                return None
            v = list(v)
            if len(v) != B:
                raise ValueError(f"{len(v)} per-query values for {B} queries")
            return v

        def flat(v):
            return v is None or all(isinstance(x, (int, float, np.integer, np.floating)) for x in v)
        qe = per_query(exact, lambda v: isinstance(v, (bool, int, np.bool_, np.integer)))
        qt = per_query(tolerance, lambda v: v is None or isinstance(v, (int, np.integer)))
        qb, qp = per_query(boost, flat), per_query(properties, flat)
        rp = _lib.ResolveParams()
        arr = (C.c_char_p * B)(*[t.encode("utf-8") for t in texts])
        rp.texts, rp.n_queries = arr, B
        rp.exact_match_boost = float(exact_match_boost)
        keep, q = [], None
        if qe is None and qt is None and qb is None and qp is None:
            rp.exact, rp.tolerance = int(bool(exact)), -1 if tolerance is None else int(tolerance)
            fb, fm = self._field_arrays(boost, properties)
            rp.field_boost, rp.field_mask = _p(fb), _p(fm)
        else:
            q = (_lib.ResolveQuery * B)()
            for b in range(B):
                t = qt[b] if qt is not None else tolerance
                fb, fm = self._field_arrays(qb[b] if qb is not None else boost, qp[b] if qp is not None else properties)
                keep += [fb, fm]
                q[b].exact = int(bool(qe[b] if qe is not None else exact))
                q[b].tolerance = -1 if t is None else int(t)
                q[b].field_boost, q[b].field_mask = _p(fb), _p(fm)
        res = C.c_void_p()
        if q is None and ctx is None:
            check(lib().oc_dict_resolve(self._h, C.byref(rp), C.byref(res)))
        else:
            check(lib().oc_dict_resolve_q(self._h, None if ctx is None else ctx._h, C.byref(rp), q, C.byref(res)))
        try:
            ptrs = [C.c_void_p() for _ in range(5)]
            nt, ne = C.c_uint32(), C.c_uint32()
            lib().oc_resolved_arrays(res, *[C.byref(x) for x in ptrs], C.byref(nt), C.byref(ne))
            B = len(texts)

            def arr_of(ptr, n, ct, dt):
                return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(ct)), shape=(max(n, 1),))[:n].astype(dt, copy=True)
            out = TextQueryBatch.__new__(TextQueryBatch)
            out.n_queries = B
            out.q_token_offsets = arr_of(ptrs[0], B + 1, C.c_uint32, np.uint32)
            out.token_term_offsets = arr_of(ptrs[1], nt.value + 1, C.c_uint32, np.uint32)
            out.term_field = arr_of(ptrs[2], ne.value, C.c_uint32, np.uint32)
            out.term_id = arr_of(ptrs[3], ne.value, C.c_uint32, np.uint32)
            out.term_weight = arr_of(ptrs[4], ne.value, C.c_float, np.float32)
            return out
        finally:
            lib().oc_resolved_free(res)


class TextQueryBatch:
    """B resolved queries packed as the CSR arrays oc_search takes (q -> tokens -> expanded terms)."""

    def query(self, i: int) -> TextQuery:
        """The i-th query as a TextQuery (tests: compare with a host-side resolution)."""
        t0, t1 = int(self.q_token_offsets[i]), int(self.q_token_offsets[i + 1])
        e0, e1 = int(self.token_term_offsets[t0]), int(self.token_term_offsets[t1])
        return TextQuery((self.token_term_offsets[t0:t1 + 1] - np.uint32(e0)).astype(np.uint32), self.term_field[e0:e1].copy(),
                         self.term_id[e0:e1].copy(), self.term_weight[e0:e1].copy())

    def __init__(self, texts: Sequence[TextQuery]):
        B = len(texts)
        self.n_queries = B
        qoff = np.zeros(B + 1, np.uint32)
        tto, tf_, tid, tw = [np.zeros(1, np.uint32)], [], [], []
        ntok = nterm = 0
        for i, t in enumerate(texts):
            ntok += t.n_tokens
            qoff[i + 1] = ntok
            tto.append(t.token_term_offsets[1:].astype(np.uint32) + np.uint32(nterm))
            nterm += int(t.token_term_offsets[-1])
            tf_.append(t.term_field); tid.append(t.term_id); tw.append(t.term_weight)
        self.q_token_offsets = qoff
        self.token_term_offsets = np.ascontiguousarray(np.concatenate(tto), np.uint32)
        self.term_field = np.ascontiguousarray(np.concatenate(tf_) if tf_ else np.zeros(0), np.uint32)
        self.term_id = np.ascontiguousarray(np.concatenate(tid) if tid else np.zeros(0), np.uint32)
        self.term_weight = np.ascontiguousarray(np.concatenate(tw) if tw else np.zeros(0), np.float32)


@dataclass
class QueryParams:
    """One query's own scalars in a batch (oc_query_params; SearchParams, types.rs:1381-1409): the TokenScoreParams
    fields of the same meaning, for one query."""
    mode: int
    limit: int = 10
    offset: int = 0
    similarity: float = 0.7
    threshold: Optional[float] = None
    vector_limit: int = 0            # 0 => limit


@dataclass
class TokenScoreParams:
    """token_score.rs:31-41 (mode already resolved; boost/properties are folded into the
    resolved TextQuery by the host-side term resolution)."""
    mode: int
    limit_hint: int = 10
    offset: int = 0
    similarity: float = 0.7          # types.rs:881-885
    threshold: Optional[float] = None
    filtered_doc_ids: Optional[np.ndarray] = None
    filter_nbits: int = 0
    device_filter: Optional["DeviceFilter"] = None   # device-resident bitmap (oc_filter_*); wins over filtered_doc_ids
    # one entry per query (None = unfiltered): query b is scored as if alone with device_filter = device_filters[b]
    # (oc_search_params.q_filters); not together with device_filter / filtered_doc_ids
    device_filters: Optional[Sequence[Optional["DeviceFilter"]]] = None
    # one entry per query (None = unfiltered): query b's where-clause as a program (where.WhereProgram, e.g. from
    # IndexLoader.where_program), evaluated inside the search call (oc_search_params.q_where); the same results as
    # device_filters holding the handles the programs stand for, and not together with them or device_filter
    where_programs: Optional[Sequence[Optional[object]]] = None
    vector_limit: int = 0            # 0 => limit_hint (search.rs:330-336); see oc_search_params.vector_limit
    omc_doc_ids: Optional[np.ndarray] = None   # ascending
    omc_mult: Optional[np.ndarray] = None
    # the index's OMC map on the device (oc_search_params.omc): the same results as omc_doc_ids / omc_mult set to its
    # published version (OmcStore.read); not together with them
    omc_store: Optional["OmcStore"] = None
    sharded: bool = False
    shard_tombstones: bool = False   # OC_SHARD_TOMBSTONES: some rank's string store holds uncommitted deletes
    shard_count_df: bool = False     # OC_SHARD_COUNT_DF: some rank's store lacks the corpus-wide df tables
    # one entry per query (oc_search_params.q_params): query b takes its mode, limit, offset, similarity, threshold and
    # vector_limit from query_params[b], and the fields above of those names are ignored; the hit arrays are sized by
    # the largest limit (_stride)
    query_params: Optional[Sequence[QueryParams]] = None


def _stride(params: TokenScoreParams) -> int:
    """The row stride of the hit arrays: limit_hint, or with query_params the largest entry's limit."""
    if params.query_params is None:
        return params.limit_hint
    return max([0] + [int(q.limit) for q in params.query_params])


def _modes(params: TokenScoreParams):
    """The modes of a batch: params.mode, or each entry's."""
    return {params.mode} if params.query_params is None else {int(q.mode) for q in params.query_params}


class TokenScoreContext:
    """token_score.rs:49-57 + execute :460-509, fused with OMC, count and top-N.

    execute_batch() is the GPU drop-in: it returns, per query, the top (limit) hits after
    offset and the total match count — what search_on_indexes derives from the score map
    (search.rs:482-498) — instead of materialising the whole HashMap on the host."""

    def __init__(self, ctx: Context, embedding_field: Optional[EmbeddingFieldStorage],
                 string_fields: Optional[StringFieldStorage]):
        self.ctx, self.emb, self.str = ctx, embedding_field, string_fields

    def execute_batch(self, params: TokenScoreParams, texts=None,
                      q_vecs: Optional[np.ndarray] = None) -> List[SearchHits]:
        docs, scores, n, cnt = self.execute_batch_arrays(params, texts, q_vecs)
        return [SearchHits(docs[i, :n[i]].copy(), scores[i, :n[i]].copy(), int(cnt[i])) for i in range(docs.shape[0])]

    def execute_batch_arrays(self, params: TokenScoreParams, texts=None, q_vecs: Optional[np.ndarray] = None):
        """Same call, results as arrays: (doc_ids [B,limit], scores [B,limit], n [B], count [B]).
        `texts` is a sequence of TextQuery or a pre-packed TextQueryBatch (term resolution happens
        before the hot path in the reference as well: token_score.rs:196-209)."""
        sp, keep, B = self._build_params(params, texts, q_vecs)
        docs = np.empty((B, _stride(params)), np.uint64)
        scores = np.empty((B, _stride(params)), np.float32)
        n = np.empty(B, np.uint32)
        cnt = np.empty(B, np.uint64)
        check(lib().oc_search(self.ctx._h, self.emb._h if self.emb else None, self.str._h if self.str else None,
                              C.byref(sp), _p(docs), _p(scores), _p(n), _p(cnt)))
        return docs, scores, n, cnt

    def _build_params(self, params: TokenScoreParams, texts=None, q_vecs: Optional[np.ndarray] = None):
        """oc_search_params for a batch; `keep` holds the arrays the struct points into."""
        if texts is not None and not isinstance(texts, TextQueryBatch):
            texts = TextQueryBatch(texts)
        B = texts.n_queries if texts is not None else int(np.asarray(q_vecs).reshape(-1, self.emb.dim).shape[0])
        sp = SearchParams()
        sp.mode = params.mode
        sp.n_queries = B
        sp.limit, sp.offset = params.limit_hint, params.offset
        sp.similarity = params.similarity
        sp.threshold = -1.0 if params.threshold is None else params.threshold
        sp.bm25_k, sp.bm25_b = BM25_K, BM25_B
        keep = []
        modes = _modes(params)
        if params.query_params is not None:
            qps = list(params.query_params)
            if len(qps) != B:
                raise ValueError(f"query_params has {len(qps)} entries for {B} queries")
            arr = (_lib.QueryParams * max(B, 1))(*[_lib.QueryParams(int(q.mode), int(q.limit), int(q.offset), float(q.similarity),
                                                                    -1.0 if q.threshold is None else float(q.threshold),
                                                                    int(q.vector_limit)) for q in qps])
            keep.append(arr)
            sp.q_params = C.cast(arr, C.c_void_p)
            sp.limit = _stride(params)
        if modes & {MODE_VECTOR, MODE_HYBRID}:
            qv = np.ascontiguousarray(q_vecs, np.float32).reshape(B, self.emb.dim)
            keep.append(qv)
            sp.q_vecs = _p(qv)
        if modes & {MODE_FULLTEXT, MODE_HYBRID}:
            keep.append(texts)
            sp.q_token_offsets, sp.token_term_offsets = _p(texts.q_token_offsets), _p(texts.token_term_offsets)
            sp.term_field, sp.term_id, sp.term_weight = _p(texts.term_field), _p(texts.term_id), _p(texts.term_weight)
        sp.vector_limit = int(params.vector_limit)
        if params.device_filters is not None:
            fl = list(params.device_filters)
            if len(fl) != B:
                raise ValueError(f"device_filters has {len(fl)} entries for {B} queries")
            arr = (C.c_void_p * B)(*[None if f is None else f._h.value for f in fl])
            keep += [arr, fl]   # the handles stay alive for the call
            sp.q_filters = C.cast(arr, C.c_void_p)
        if params.where_programs is not None:
            from .where import pack_programs
            wl = list(params.where_programs)
            if len(wl) != B:
                raise ValueError(f"where_programs has {len(wl)} entries for {B} queries")
            if any(w is not None for w in wl):
                w, wkeep = pack_programs(wl)
                keep += [w, wkeep]
                sp.q_where = C.cast(C.pointer(w), C.c_void_p)
        if params.device_filter is not None:
            keep.append(params.device_filter)
            sp.filter = params.device_filter._h
        elif params.filtered_doc_ids is not None:
            fb = np.ascontiguousarray(params.filtered_doc_ids, np.uint64)
            keep.append(fb)
            sp.filter_bits, sp.filter_nbits = _p(fb), int(params.filter_nbits)
        if params.omc_doc_ids is not None and len(params.omc_doc_ids):
            od = np.ascontiguousarray(params.omc_doc_ids, np.uint64)
            om = np.ascontiguousarray(params.omc_mult, np.float32)
            keep += [od, om]
            sp.omc_doc_ids, sp.omc_mult, sp.n_omc = _p(od), _p(om), od.shape[0]
        if params.omc_store is not None:
            keep.append(params.omc_store)
            sp.omc = params.omc_store._h
        sp.sharded = (1 | (2 if params.shard_tombstones else 0) | (4 if params.shard_count_df else 0)) if params.sharded else 0
        return sp, keep, B

    def execute(self, params: TokenScoreParams, results: Dict[int, float], text: Optional[TextQuery] = None,
                q_vec: Optional[np.ndarray] = None) -> int:
        """Reference-shaped call: `results.extend(scores)` for one query; returns the match count.
        limit and offset are passed through unchanged (the vector stage's candidate depth is limit_hint =
        limit, NOT limit + offset: search.rs:330-336), so `results` receives the rows [offset, offset+limit)
        of the ranking — the rest of the score map never leaves the GPU."""
        hits = self.execute_batch(params, None if text is None else [text], q_vec)[0]
        for d, s in zip(hits.doc_ids, hits.scores):
            results[int(d)] = np.float32(s)
        return hits.count


class SearchBatcher:
    """Micro-batching front (oc_batcher_*, csrc/batcher.h): many threads call search() with ONE query
    each — the way the reference's request tasks call TokenScoreContext::execute — and the library
    coalesces concurrent calls that share (mode, limit, offset, similarity, threshold) into one
    batched oc_search.  A request's device_filter (its where-filter) travels with it into the batch as
    that query's own filter, so filtered and unfiltered requests are coalesced together; requests with
    filtered_doc_ids (a host bitmap), OMC arrays or sharding run as their own oc_search.  Requests with the
    same omc_store batch together (in both batchers).  ctypes
    releases the GIL while a caller is blocked in the library.
    mixed=True (OC_BATCHER_MIXED): calls that differ in mode, limit, offset, similarity, threshold or vector_limit
    share a batch too (each request's scalars become its q_params entry), and so do calls with the same OMC arrays;
    each caller still gets what it gets alone."""

    def __init__(self, tsc: TokenScoreContext, max_batch: int = 256, max_wait_us: int = 200, mixed: bool = False):
        self.tsc = tsc
        h = C.c_void_p()
        check(lib().oc_batcher_create2(tsc.ctx._h, tsc.emb._h if tsc.emb else None, tsc.str._h if tsc.str else None,
                                       int(max_batch), int(max_wait_us), _lib.OC_BATCHER_MIXED if mixed else 0, C.byref(h)))
        self._h = h

    def _params(self, params: TokenScoreParams, text: Optional[TextQuery], q_vec: Optional[np.ndarray]):
        """oc_search_params of one query and the arrays they point into.  A request is one query with its scalars in
        TokenScoreParams' own fields: query_params (a batch's per-query scalars) is refused."""
        if params.query_params is not None:
            raise ValueError("SearchBatcher takes one query per call: set mode / limit_hint / offset / similarity / "
                             "threshold / vector_limit, not query_params")
        sp, keep, B = self.tsc._build_params(params, None if text is None else [text],
                                             None if q_vec is None else np.asarray(q_vec, np.float32).reshape(1, -1))
        assert B == 1
        return sp, keep

    def search(self, params: TokenScoreParams, text: Optional[TextQuery] = None,
               q_vec: Optional[np.ndarray] = None) -> SearchHits:
        sp, keep = self._params(params, text, q_vec)
        L = params.limit_hint
        docs, scores = np.empty(L, np.uint64), np.empty(L, np.float32)
        n, cnt = np.zeros(1, np.uint32), np.zeros(1, np.uint64)
        check(lib().oc_batcher_search(self._h, C.byref(sp), _p(docs), _p(scores), _p(n), _p(cnt)))
        k = int(n[0])
        return SearchHits(docs[:k].copy(), scores[:k].copy(), int(cnt[0]))

    def search_sorted(self, params: TokenScoreParams, sort=None, promote=None, text: Optional[TextQuery] = None,
                      q_vec: Optional[np.ndarray] = None):
        """One query with its own sortBy (a (SortField, order) pair, None: score order) and pin rules (`promote`: its
        promote items, None: no rule), coalesced with concurrent search() / search_sorted() calls.  Returns
        (SearchHits, sort values [n], pin scores [items], pin present [items]) as search_q_sorted_arrays gives them for
        this query alone."""
        sp, keep = self._params(params, text, q_vec)
        srt = None if sort is None else _sort(sort[0], sort[1])
        pins = None if promote is None else _pins([promote], 1)[0]
        n_items = 0 if pins is None else int(pins._keep[0][-1])
        L = params.limit_hint
        docs, scores, sv = np.zeros(L, np.uint64), np.zeros(L, np.float32), np.zeros(L, np.float64)
        n, cnt = np.zeros(1, np.uint32), np.zeros(1, np.uint64)
        ps, pp = np.zeros(max(n_items, 1), np.float32), np.zeros(max(n_items, 1), np.uint8)
        check(lib().oc_batcher_search_sorted(self._h, C.byref(sp), None if srt is None else C.byref(srt),
                                             None if pins is None else C.byref(pins), _p(docs), _p(scores), _p(sv), _p(n),
                                             _p(cnt), _p(ps), _p(pp)))
        k = int(n[0])
        return SearchHits(docs[:k].copy(), scores[:k].copy(), int(cnt[0])), sv[:k].copy(), ps[:n_items], pp[:n_items]

    def search_groups(self, params: TokenScoreParams, group=None, promote=None, text: Optional[TextQuery] = None,
                      q_vec: Optional[np.ndarray] = None, group_stride: Optional[int] = None):
        """One query with its own groupBy (`group`: None or (GroupBy, max_results[, (SortField, order)]), as an entry of
        search_q_groups_arrays' `groups`) and pin rules, coalesced with concurrent search_groups() calls.  Returns (docs
        [limit], scores, sort values [limit], n, count, pin scores [items], pin present [items], group docs
        [n_groups, stride], group scores, group sort values, group n [n_groups]) as search_q_groups_arrays gives them for
        this query alone."""
        sp, keep = self._params(params, text, q_vec)
        req, rows = _group_reqs([group], 1)
        pins = None if promote is None else _pins([promote], 1)[0]
        n_items = 0 if pins is None else int(pins._keep[0][-1])
        if group_stride is None:
            group_stride = _group_need(group, n_items)
        S = int(group_stride)
        docs, scores, sv, n, cnt, ps, pp, gd, gs, gsv, gn = _q_outputs(1, params.limit_hint, n_items, int(rows[-1]), S)
        check(lib().oc_batcher_search_groups(self._h, C.byref(sp), req, None if pins is None else C.byref(pins), S, _p(docs),
                                             _p(scores), _p(sv), _p(n), _p(cnt), _p(ps), _p(pp), _p(gd), _p(gs), _p(gsv), _p(gn)))
        return docs[0], scores[0], sv[0], n[0], cnt[0], ps[:n_items], pp[:n_items], gd, gs, gsv, gn

    def search_faceted(self, store: FacetStore, params: TokenScoreParams, facets, group=None, promote=None,
                       text: Optional[TextQuery] = None, q_vec: Optional[np.ndarray] = None, group_stride: Optional[int] = None):
        """One query with its own facets (a reference-style map, see facet_requests), groupBy (`group`, as for
        search_groups, or None) and pin rules, coalesced with concurrent search_faceted() calls on the same store.
        Returns search_groups()' tuple followed by the facet counts [requests] and their (field, label) pairs, as
        search_q_facets_arrays gives them for this query alone."""
        sp, keep = self._params(params, text, q_vec)
        req, rows = _group_reqs([group], 1)
        farr, foff, labels = _q_facet_reqs(store, [facets], 1)
        pins = None if promote is None else _pins([promote], 1)[0]
        n_items = 0 if pins is None else int(pins._keep[0][-1])
        if group_stride is None:
            group_stride = _group_need(group, n_items)
        S, F = int(group_stride), int(foff[-1])
        docs, scores, sv, n, cnt, ps, pp, gd, gs, gsv, gn = _q_outputs(1, params.limit_hint, n_items, int(rows[-1]), S)
        fc = np.zeros(max(F, 1), np.uint64)
        check(lib().oc_batcher_search_faceted(self._h, C.byref(sp), store._h, farr, F, None if group is None else req,
                                              None if pins is None else C.byref(pins), S, _p(docs), _p(scores), _p(sv), _p(n),
                                              _p(cnt), _p(ps), _p(pp), _p(gd), _p(gs), _p(gsv), _p(gn), _p(fc)))
        return docs[0], scores[0], sv[0], n[0], cnt[0], ps[:n_items], pp[:n_items], gd, gs, gsv, gn, fc[:F], labels[0]

    def stats(self) -> dict:
        q, b, d = C.c_uint64(), C.c_uint64(), C.c_uint64()
        check(lib().oc_batcher_stats(self._h, C.byref(q), C.byref(b), C.byref(d)))
        return {"queries": q.value, "batches": b.value, "direct": d.value}

    def close(self):
        if self._h:
            lib().oc_batcher_destroy(self._h)
            self._h = None


def search(ctx: Context, emb: Optional[EmbeddingFieldStorage], strs: Optional[StringFieldStorage], mode: str,
           texts: Optional[Sequence[TextQuery]] = None, q_vecs: Optional[np.ndarray] = None, limit: int = 10,
           offset: int = 0, similarity: float = 0.7, threshold: Optional[float] = None, **kw) -> List[SearchHits]:
    """search() surface of the hot path: mode = "fulltext" | "vector" | "hybrid" (types.rs:924-999;
    "default" == fulltext)."""
    m = {"fulltext": MODE_FULLTEXT, "default": MODE_FULLTEXT, "vector": MODE_VECTOR, "hybrid": MODE_HYBRID}[mode]
    p = TokenScoreParams(mode=m, limit_hint=limit, offset=offset, similarity=similarity, threshold=threshold, **kw)
    return TokenScoreContext(ctx, emb, strs).execute_batch(p, texts, q_vecs)
