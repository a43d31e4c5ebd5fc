//! Bindings for `include/oramacore_b200.h` (C ABI of the H100-native search hot path) and safe
//! wrappers shaped like the reference types they replace:
//!   * `EmbeddingField`  ~ `EmbeddingFieldStorage` (read/index/embedding_field.rs:29-34)
//!   * `StringFields`    ~ the `StringFieldStorage` set of an Index (read/index/string_field.rs:32-36)
//!   * `Ctx::search`     ~ `TokenScoreContext::execute` + OMC + count + top-N
//!                         (token_score.rs:460-509, search.rs:39-48, 482-498, sort.rs:260-279)
//! SOURCE ONLY: the build image has no Rust toolchain; the identical ABI is exercised by the
//! ctypes mirror (`oramacore_b200/_lib.py`) and the GPU parity tests.
use std::ffi::{c_char, c_int, c_void, CStr};

#[repr(C)] pub struct OcCtx { _p: [u8; 0] }
#[repr(C)] pub struct OcEmb { _p: [u8; 0] }
#[repr(C)] pub struct OcStr { _p: [u8; 0] }
#[repr(C)] pub struct OcBatcher { _p: [u8; 0] }
#[repr(C)] pub struct OcFilter { _p: [u8; 0] }
#[repr(C)] pub struct OcFacets { _p: [u8; 0] }
#[repr(C)] pub struct OcGroupBy { _p: [u8; 0] }
#[repr(C)] pub struct OcSortField { _p: [u8; 0] }
#[repr(C)] pub struct OcGeoField { _p: [u8; 0] }
#[repr(C)] pub struct OcOmc { _p: [u8; 0] }
#[repr(C)] pub struct OcDict { _p: [u8; 0] }
#[repr(C)] pub struct OcResolved { _p: [u8; 0] }

pub const OC_MODE_FULLTEXT: c_int = 0;
pub const OC_MODE_VECTOR: c_int = 1;
pub const OC_MODE_HYBRID: c_int = 2;
pub const OC_DTYPE_F32: c_int = 0;
pub const OC_DTYPE_BF16: c_int = 1;
/// `oc_emb_compact` flag: also give the capacity beyond `num_rows` back.
pub const OC_EMB_COMPACT_SHRINK: u32 = 1;
/// Statistics of one `oc_emb_compact` call (`oc_emb_compact_t`).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct OcEmbCompact {
    pub rows_before: u64,
    pub rows_after: u64,
    pub rows_moved: u64,
    pub device_bytes_before: u64,
    pub device_bytes_after: u64,
    pub workspace_bytes: u64,
    pub device_ms: f32,
}
/// Statistics of one `oc_str_commit_ex` call (`oc_str_commit_t`).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct OcStrCommit {
    pub rows_before: u64,
    pub rows_after: u64,
    pub postings_before: u64,
    pub postings_after: u64,
    pub pending_postings: u64,
    pub workspace_bytes: u64,
    pub device_ms: f32,
    pub wall_ms: f32,
}
/// Statistics of one `oc_str_sync_global` call (`oc_str_sync_t`).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct OcStrSync {
    pub version: u64,
    pub rows_global: u64,
    pub bytes_reduced: u64,
    pub device_ms: f32,
    pub wall_ms: f32,
}
/// Statistics of one `oc_facets_commit_ex` / `oc_geo_field_commit_ex` call (`oc_filter_commit_t`).
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct OcFilterCommit {
    pub version: u64,
    pub rows_kept: u64,
    pub rows_dropped: u64,
    pub rows_added: u64,
    pub workspace_bytes: u64,
    pub device_ms: f32,
    pub wall_ms: f32,
}
/// `oc_facets_insert_variants` flag: set semantics (a bool field).
pub const OC_FACET_UNIQUE: u32 = 1;
/// `OcSearchParams::sharded`: merge across `oc_comm` ranks; add `OC_SHARD_TOMBSTONES` on every rank while
/// any rank's string store holds uncommitted deletes (the df all-reduce must be entered by all ranks).
pub const OC_SHARDED: c_int = 1;
pub const OC_SHARD_TOMBSTONES: c_int = 2;
/// count corpus df across ranks instead of using replicated tables (a commit on a shard drops them)
pub const OC_SHARD_COUNT_DF: c_int = 4;
/// geopoint leaves: sphere radius of the great-circle distance (an assumption) and the polygon vertex cap
pub const OC_GEO_EARTH_RADIUS_M: f64 = 6371000.0;
pub const OC_GEO_MAX_VERTICES: u32 = 2048;
/// oc_filter_facet_range: open ends of the interval (closed when the flag is clear)
pub const OC_RANGE_LO_OPEN: u32 = 1;
pub const OC_RANGE_HI_OPEN: u32 = 2;
/// `OcTiming::scan_variant`: which embedding sweep served the last batch
pub const OC_SCAN_EXACT: u32 = 0;
pub const OC_SCAN_TC_TF32: u32 = 1;
pub const OC_SCAN_TC_BF16: u32 = 4;
/// wgmma .f16 on the fp16 copy of an fp32 store (`OC_EMB_F16=0` selects `OC_SCAN_TC_TF32`)
pub const OC_SCAN_TC_F16: u32 = 5;
pub const OC_BATCHER_MIXED: u32 = 1;

#[repr(C)]
pub struct OcSearchParams {
    pub mode: c_int,
    pub n_queries: u32,
    pub limit: u32,
    pub offset: u32,
    pub similarity: f32,
    pub threshold: f32, // < 0 => None
    pub bm25_k: f32,
    pub bm25_b: f32,
    pub q_vecs: *const f32,
    pub q_token_offsets: *const u32,
    pub token_term_offsets: *const u32,
    pub term_field: *const u32,
    pub term_id: *const u32,
    pub term_weight: *const f32,
    pub filter_bits: *const u64,
    pub filter_nbits: u64,
    pub omc_doc_ids: *const u64,
    pub omc_mult: *const f32,
    pub n_omc: u64,
    pub sharded: c_int,
    pub vector_limit: u32,          // 0 => limit (limit_hint of the vector stage, search.rs:330-336)
    pub filter: *const OcFilter,    // device-resident FilterResult bitmap; wins over filter_bits
    pub q_filters: *const *const OcFilter,  // NULL, or B entries: query b's own filter (NULL = none); oc_search only
    pub q_params: *const OcQueryParams,     // NULL, or B entries: query b's own mode / limit / offset / similarity /
                                            // threshold / vector_limit; `limit` is then the hit arrays' row stride
    pub q_where: *const OcWhere,            // NULL, or each query's where-clause as a program, evaluated in the call
    pub omc: *const OcOmc,                  // NULL, or the index's OMC store: the published version, read on the device
                                            // (not together with n_omc != 0)
}

/// Where-program node ops (oc_where_node.op) and bounds.
pub const OC_WHERE_NONE: u32 = 0;
pub const OC_WHERE_VARIANT: u32 = 1;
pub const OC_WHERE_RANGE: u32 = 2;
pub const OC_WHERE_GEO_RADIUS: u32 = 3;
pub const OC_WHERE_GEO_POLYGON: u32 = 4;
pub const OC_WHERE_FILTER: u32 = 5;
pub const OC_WHERE_AND: u32 = 6;
pub const OC_WHERE_OR: u32 = 7;
pub const OC_WHERE_NOT: u32 = 8;
pub const OC_WHERE_MAX_NODES: u32 = 4096;
pub const OC_WHERE_MAX_DEPTH: u32 = 32;

/// One node of a where program (oc_where_node): a leaf (src = the facet store, geo field or filter handle), or
/// AND / OR (arg = arity) / NOT over the values on the stack.
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct OcWhereNode {
    pub op: u32,
    pub field: u32,
    pub arg: u32,            // VARIANT: variant; RANGE: flags; GEO_*: inside; AND / OR: arity
    pub first_vertex: u32,   // GEO_POLYGON
    pub n_vertices: u32,
    pub a: f64,              // RANGE: lo, hi; GEO_RADIUS: lat, lon, radius_m
    pub b: f64,
    pub c: f64,
    pub src: *const c_void,
}

/// The programs of a batch (oc_where): query b's nodes are nodes[q_node_offsets[b] .. q_node_offsets[b + 1]).
#[repr(C)]
pub struct OcWhere {
    pub nbits: u64,
    pub q_node_offsets: *const u32,
    pub nodes: *const OcWhereNode,
    pub vertex_lat: *const f64,
    pub vertex_lon: *const f64,
}

/// One query's scalars (oc_query_params), the entry of OcSearchParams::q_params.
#[repr(C)]
#[derive(Clone, Copy, Debug)]
pub struct OcQueryParams {
    pub mode: c_int,
    pub limit: u32,
    pub offset: u32,
    pub similarity: f32,
    pub threshold: f32,     // < 0 => None
    pub vector_limit: u32,  // 0 => limit
}

#[repr(C)]
pub struct OcFacetReq { pub field: u32, pub variant: u32, pub from: f64, pub to: f64 }

/// the promote items of the pin rules that matched each query (extract_pin_rules, search.rs:257-281)
#[repr(C)]
pub struct OcPins {
    pub q_pin_offsets: *const u32,  // B+1
    pub doc_ids: *const u64,        // PromoteItem.doc_id
    pub positions: *const u32,      // PromoteItem.position
    pub apply: c_int,               // 0: hits as oc_search, only the per-item score-map values
}

/// sortBy: a sort field handle and its order (OC_SORT_ASC = 0, OC_SORT_DESC = 1)
#[repr(C)]
pub struct OcSort {
    pub field: *const OcSortField,
    pub order: c_int,
}

/// most indexes of one oc_search_indexes call
pub const OC_MAX_INDEXES: u32 = 32;
/// oc_index_query: one index of an oc_search_indexes call (its stores, inputs and per-query sorts; q_sorts may be NULL)
#[repr(C)]
pub struct OcIndexQuery {
    pub emb: *mut OcEmb,
    pub str_: *mut OcStr,
    pub p: *const OcSearchParams,
    pub q_sorts: *const OcSort,
}

/// oc_index_extras: one index's groups (local group -> collection key per query) and facet requests (each added to a
/// collection slot) in an oc_search_indexes_ex call
#[repr(C)]
pub struct OcIndexExtras {
    pub q_groups: *const *const OcGroupBy,
    pub q_group_keys: *const *const u32,
    pub facets: *mut OcFacets,
    pub n_facet_reqs: u32,
    pub facet_reqs: *const OcFacetReq,
    pub facet_slots: *const u32,
}

/// one query's groupBy in oc_search_q_groups: its handle (NULL: no groups), max_results and sort (field NULL: score order)
#[repr(C)]
pub struct OcGroupReq {
    pub groups: *const OcGroupBy,
    pub max_results: u32,
    pub sort: OcSort,
}

#[repr(C)]
pub struct OcResolveParams {
    pub texts: *const *const c_char,
    pub n_queries: u32,
    pub exact: c_int,
    pub tolerance: c_int,           // < 0 => None (prefix expansion)
    pub field_boost: *const f32,
    pub field_mask: *const u8,
    pub exact_match_boost: f32,
}
#[repr(C)]
pub struct OcResolveQuery {
    pub exact: c_int,
    pub tolerance: c_int,           // < 0 => None (prefix expansion)
    pub field_boost: *const f32,
    pub field_mask: *const u8,
}
pub type OcStemFn = unsafe extern "C" fn(tok: *const c_char, len: usize, out: *mut c_char, cap: usize, user: *mut c_void) -> usize;

extern "C" {
    pub fn oc_last_error() -> *const c_char;
    pub fn oc_abi_sizes(out: *mut usize);
    pub fn oc_init(device_id: c_int, out: *mut *mut OcCtx) -> c_int;
    pub fn oc_shutdown(ctx: *mut OcCtx);
    pub fn oc_comm_unique_id(out_id: *mut u8) -> c_int;
    pub fn oc_comm_init(ctx: *mut OcCtx, world: c_int, rank: c_int, id: *const u8) -> c_int;
    pub fn oc_comm_init_local(ctxs: *const *mut OcCtx, world: c_int) -> c_int;
    pub fn oc_emb_create(ctx: *mut OcCtx, dim: u32, dtype: c_int, rescale_e5: c_int, out: *mut *mut OcEmb) -> c_int;
    pub fn oc_emb_destroy(emb: *mut OcEmb);
    pub fn oc_emb_insert(emb: *mut OcEmb, doc_ids: *const u64, rows: *const c_void, n: u64) -> c_int;
    pub fn oc_emb_delete(emb: *mut OcEmb, doc_ids: *const u64, n: u64) -> c_int;
    pub fn oc_emb_compact(emb: *mut OcEmb, flags: u32, out: *mut OcEmbCompact) -> c_int;
    pub fn oc_emb_search(emb: *mut OcEmb, queries: *const f32, b: u32, limit: u32, similarity: f32,
                         filter_bits: *const u64, filter_nbits: u64, out_doc_ids: *mut u64,
                         out_scores: *mut f32, out_counts: *mut u32) -> c_int;
    pub fn oc_str_create(ctx: *mut OcCtx, n_fields: u32, out: *mut *mut OcStr) -> c_int;
    pub fn oc_str_destroy(s: *mut OcStr);
    pub fn oc_str_set_rows(s: *mut OcStr, n_rows: u64, row_doc_ids: *const u64, document_count: u64) -> c_int;
    pub fn oc_str_load_field(s: *mut OcStr, field: u32, avg_field_len: f32, n_terms: u32, term_offsets: *const u64,
                             post_row: *const u32, post_tf: *const u16, post_len: *const u16,
                             global_df: *const u32) -> c_int;
    pub fn oc_str_delete(s: *mut OcStr, doc_ids: *const u64, n: u64) -> c_int;
    /// StringFieldStorage::insert (string_field.rs:155-177): buffered until `oc_str_commit`
    pub fn oc_str_insert(s: *mut OcStr, field: u32, doc_id: u64, field_len: u16, n_terms: u32,
                         term_ids: *const u32, tfs: *const u16) -> c_int;
    /// compaction (string_field.rs:186-191): merges pending inserts / deletes into the device layout
    pub fn oc_str_commit(s: *mut OcStr) -> c_int;
    /// `oc_str_commit` that also reports its statistics (`out` may be null)
    pub fn oc_str_commit_ex(s: *mut OcStr, out: *mut OcStrCommit) -> c_int;
    /// read-back of the published snapshot (compact(), string_field.rs:186-191): null arrays return the sizes;
    /// otherwise `*n_rows` / `*n_terms` / `*n_postings` give the arrays' capacity on entry
    pub fn oc_str_read_rows(s: *mut OcStr, n_rows: *mut u64, row_doc_ids: *mut u64, document_count: *mut u64,
                            version: *mut u64) -> c_int;
    pub fn oc_str_read_field(s: *mut OcStr, field: u32, avg_field_len: *mut f32, n_terms: *mut u32, n_postings: *mut u64,
                             term_offsets: *mut u64, post_row: *mut u32, post_tf: *mut u16, post_len: *mut u16) -> c_int;
    /// page-locked host buffers: query vectors placed here are DMA'd without staging
    pub fn oc_pinned_alloc(bytes: usize, out: *mut *mut c_void) -> c_int;
    /// micro-batching front: one query per call from many threads, coalesced into batched `oc_search`
    pub fn oc_batcher_create(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, max_batch: u32, max_wait_us: u32,
                             out: *mut *mut OcBatcher) -> c_int;
    /// flags: 0 or OC_BATCHER_MIXED (requests with different mode / limit / offset / similarity / threshold share a batch)
    pub fn oc_batcher_create2(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, max_batch: u32, max_wait_us: u32, flags: u32,
                              out: *mut *mut OcBatcher) -> c_int;
    pub fn oc_batcher_destroy(b: *mut OcBatcher);
    pub fn oc_batcher_search(b: *mut OcBatcher, p: *const OcSearchParams, out_doc_ids: *mut u64, out_scores: *mut f32,
                             out_n: *mut u32, out_count: *mut u64) -> c_int;
    /// one query with its own sort (NULL: score order) and pin items, coalesced with oc_batcher_search calls
    pub fn oc_batcher_search_sorted(b: *mut OcBatcher, p: *const OcSearchParams, sort: *const OcSort, pins: *const OcPins,
                                    out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64, out_n: *mut u32,
                                    out_count: *mut u64, out_pin_scores: *mut f32, out_pin_present: *mut u8) -> c_int;
    pub fn oc_batcher_search_groups(b: *mut OcBatcher, p: *const OcSearchParams, req: *const OcGroupReq, pins: *const OcPins,
                                    group_stride: u32, out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64,
                                    out_n: *mut u32, out_count: *mut u64, out_pin_scores: *mut f32, out_pin_present: *mut u8,
                                    out_group_doc_ids: *mut u64, out_group_scores: *mut f32, out_group_sort_values: *mut f64,
                                    out_group_n: *mut u32) -> c_int;
    pub fn oc_batcher_search_faceted(b: *mut OcBatcher, p: *const OcSearchParams, f: *mut OcFacets, facet_reqs: *const OcFacetReq,
                                     n_facet_reqs: u32, req: *const OcGroupReq, pins: *const OcPins, group_stride: u32,
                                     out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64, out_n: *mut u32,
                                     out_count: *mut u64, out_pin_scores: *mut f32, out_pin_present: *mut u8,
                                     out_group_doc_ids: *mut u64, out_group_scores: *mut f32, out_group_sort_values: *mut f64,
                                     out_group_n: *mut u32, out_facet_counts: *mut u64) -> c_int;
    pub fn oc_batcher_stats(b: *mut OcBatcher, n_queries: *mut u64, n_batches: *mut u64, n_direct: *mut u64) -> c_int;
    pub fn oc_pinned_free(p: *mut c_void);
    pub fn oc_search(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, p: *const OcSearchParams,
                     out_doc_ids: *mut u64, out_scores: *mut f32, out_n: *mut u32, out_count: *mut u64) -> c_int;
    /// caller-owned N / average field lengths (shards; Index::document_count), kept across commits
    pub fn oc_str_set_global(s: *mut OcStr, document_count: u64, avg_field_len: *const f32) -> c_int;
    /// collective over the ctx's comm group: rebuild a shard's corpus-wide df tables and average field lengths
    /// after every rank's `oc_str_commit` returned (`out` may be null)
    pub fn oc_str_sync_global(s: *mut OcStr, out: *mut OcStrSync) -> c_int;
    /// one field's installed df table: null `df` returns its size in `*n_terms` (0: no table); otherwise `*n_terms`
    /// is the capacity on entry
    pub fn oc_str_read_global_df(s: *mut OcStr, field: u32, n_terms: *mut u32, df: *mut u32) -> c_int;
    // FilterResult (filter.rs:344-392) evaluated on the device
    pub fn oc_filter_from_ids(ctx: *mut OcCtx, doc_ids: *const u64, n: u64, nbits: u64, out: *mut *mut OcFilter) -> c_int;
    pub fn oc_filter_from_bits(ctx: *mut OcCtx, bits: *const u64, nbits: u64, out: *mut *mut OcFilter) -> c_int;
    pub fn oc_filter_and(a: *const OcFilter, b: *const OcFilter, out: *mut *mut OcFilter) -> c_int;
    pub fn oc_filter_or(a: *const OcFilter, b: *const OcFilter, out: *mut *mut OcFilter) -> c_int;
    pub fn oc_filter_not(a: *const OcFilter, out: *mut *mut OcFilter) -> c_int;
    pub fn oc_filter_count(f: *const OcFilter, out: *mut u64) -> c_int;
    pub fn oc_filter_nbits(f: *const OcFilter, out: *mut u64) -> c_int;
    pub fn oc_filter_read(f: *const OcFilter, out_bits: *mut u64) -> c_int;
    pub fn oc_filter_destroy(f: *mut OcFilter);
    // geopoint where-filter leaves (GeoPointFieldStorage::filter, geopoint_field.rs:179-229): an oc_filter over [0, nbits)
    pub fn oc_geo_field_create(ctx: *mut OcCtx, nbits: u64, n: u64, doc_ids: *const u64, lat: *const f64, lon: *const f64,
                               out: *mut *mut OcGeoField) -> c_int;
    pub fn oc_geo_field_destroy(g: *mut OcGeoField);
    pub fn oc_geo_field_insert(g: *mut OcGeoField, n: u64, doc_ids: *const u64, lat: *const f64, lon: *const f64) -> c_int;
    pub fn oc_geo_field_delete(g: *mut OcGeoField, n: u64, doc_ids: *const u64) -> c_int;
    pub fn oc_geo_field_commit_ex(g: *mut OcGeoField, new_nbits: u64, out: *mut OcFilterCommit) -> c_int;
    pub fn oc_geo_field_read(g: *mut OcGeoField, n: *mut u64, doc_ids: *mut u64, lat: *mut f64, lon: *mut f64) -> c_int;
    pub fn oc_filter_geo_radius(g: *const OcGeoField, lat: f64, lon: f64, radius_m: f64, inside: c_int,
                                out: *mut *mut OcFilter) -> c_int;
    pub fn oc_filter_geo_polygon(g: *const OcGeoField, lat: *const f64, lon: *const f64, n_vertices: u32, inside: c_int,
                                 out: *mut *mut OcFilter) -> c_int;
    // where programs: host-only checks, and one query's program as a handle in one call
    pub fn oc_where_check(w: *const OcWhere, n_queries: u32) -> c_int;
    pub fn oc_filter_from_where(ctx: *mut OcCtx, w: *const OcWhere, query: u32, out: *mut *mut OcFilter) -> c_int;
    // facets over the score set (facet.rs:147-209)
    pub fn oc_facets_create(ctx: *mut OcCtx, nbits: u64, out: *mut *mut OcFacets) -> c_int;
    pub fn oc_facets_destroy(f: *mut OcFacets);
    pub fn oc_facets_add_field(f: *mut OcFacets, n_variants: u32, variant_offsets: *const u64, doc_ids: *const u64, out_field: *mut u32) -> c_int;
    pub fn oc_facets_insert_variants(f: *mut OcFacets, field: u32, n: u64, doc_ids: *const u64, variants: *const u32, flags: u32) -> c_int;
    pub fn oc_facets_add_variant(f: *mut OcFacets, field: u32, variant_out: *mut u32) -> c_int;
    pub fn oc_facets_insert_numbers(f: *mut OcFacets, field: u32, n: u64, doc_ids: *const u64, values: *const f64) -> c_int;
    pub fn oc_facets_clear(f: *mut OcFacets, field: u32, n: u64, doc_ids: *const u64) -> c_int;
    pub fn oc_facets_delete(f: *mut OcFacets, n: u64, doc_ids: *const u64) -> c_int;
    pub fn oc_facets_commit_ex(f: *mut OcFacets, new_nbits: u64, out: *mut OcFilterCommit) -> c_int;
    pub fn oc_facets_read_field(f: *mut OcFacets, field: u32, n_variants: *mut u32, n_entries: *mut u64, offsets: *mut u64,
                                values: *mut f64, doc_ids: *mut u64) -> c_int;
    pub fn oc_facets_add_number_field(f: *mut OcFacets, n: u64, values_sorted: *const f64, doc_ids: *const u64, out_field: *mut u32) -> c_int;
    // the OMC map of an index (index/mod.rs:604-627, 1720-1739): queued sets / deletes, committed on the device
    pub fn oc_omc_create(ctx: *mut OcCtx, out: *mut *mut OcOmc) -> c_int;
    pub fn oc_omc_destroy(omc: *mut OcOmc);
    pub fn oc_omc_set(omc: *mut OcOmc, doc_ids: *const u64, mults: *const f32, n: u64) -> c_int;
    pub fn oc_omc_delete(omc: *mut OcOmc, doc_ids: *const u64, n: u64) -> c_int;
    pub fn oc_omc_commit_ex(omc: *mut OcOmc, out: *mut OcFilterCommit) -> c_int;
    pub fn oc_omc_read(omc: *mut OcOmc, n: *mut u64, doc_ids: *mut u64, mults: *mut f32, version: *mut u64) -> c_int;
    // where-filter leaves over a filter field (filter.rs:49-124): a variant's documents, or a number field's value interval
    pub fn oc_filter_facet_variant(f: *const OcFacets, field: u32, variant: u32, out: *mut *mut OcFilter) -> c_int;
    pub fn oc_filter_facet_range(f: *const OcFacets, field: u32, lo: f64, hi: f64, flags: u32, out: *mut *mut OcFilter) -> c_int;
    pub fn oc_search_facets(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, f: *mut OcFacets, p: *const OcSearchParams,
                            reqs: *const OcFacetReq, n_reqs: u32, out_counts: *mut u64) -> c_int;
    // groups over the score map (group.rs + sort_groups, sort.rs:129-230)
    pub fn oc_group_by_create(f: *mut OcFacets, fields: *const u32, n_fields: u32, out: *mut *mut OcGroupBy,
                              out_n_groups: *mut u64) -> c_int;
    pub fn oc_group_by_destroy(g: *mut OcGroupBy);
    pub fn oc_search_groups(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, g: *mut OcGroupBy, p: *const OcSearchParams,
                            max_results: u32, out_doc_ids: *mut u64, out_scores: *mut f32, out_n: *mut u32,
                            out_count: *mut u64, out_group_doc_ids: *mut u64, out_group_scores: *mut f32,
                            out_group_n: *mut u32) -> c_int;
    /// search_on_indexes' union of the per-index maps (search.rs:304-338, 482-498), host side
    pub fn oc_merge_results(n_indexes: u32, n_queries: u32, limit: u32, offset: u32, in_stride: u32,
                            doc_ids: *const *const u64, scores: *const *const f32, n: *const *const u32,
                            counts: *const *const u64, out_doc_ids: *mut u64, out_scores: *mut f32,
                            out_n: *mut u32, out_count: *mut u64) -> c_int;
    // pin rules (apply_pin_rules / apply_pin_rules_to_group, sort.rs:285-391)
    pub fn oc_search_pinned(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, p: *const OcSearchParams, pins: *const OcPins,
                            out_doc_ids: *mut u64, out_scores: *mut f32, out_n: *mut u32, out_count: *mut u64,
                            out_pin_scores: *mut f32, out_pin_present: *mut u8) -> c_int;
    pub fn oc_search_groups_pinned(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, g: *mut OcGroupBy, p: *const OcSearchParams,
                                   max_results: u32, pins: *const OcPins, group_stride: u32, out_doc_ids: *mut u64,
                                   out_scores: *mut f32, out_n: *mut u32, out_count: *mut u64, out_group_doc_ids: *mut u64,
                                   out_group_scores: *mut f32, out_group_n: *mut u32) -> c_int;
    pub fn oc_merge_pinned(n_indexes: u32, n_queries: u32, limit: u32, offset: u32, in_stride: u32,
                           doc_ids: *const *const u64, scores: *const *const f32, n: *const *const u32,
                           counts: *const *const u64, pins: *const OcPins, pin_scores: *const *const f32,
                           pin_present: *const *const u8, out_doc_ids: *mut u64, out_scores: *mut f32,
                           out_n: *mut u32, out_count: *mut u64) -> c_int;
    // sortBy (sort_token_scores / sort_groups with sort_by, MergeSortedIterator; sort.rs:17-201, 491-559)
    pub fn oc_sort_field_create(ctx: *mut OcCtx, nbits: u64, n: u64, doc_ids: *const u64, values: *const f64,
                                out: *mut *mut OcSortField) -> c_int;
    /// the sort field of one field of the facet store's published version, built on the device
    pub fn oc_sort_field_from_facets(f: *mut OcFacets, field: u32, variant_values: *const f64, out: *mut *mut OcSortField) -> c_int;
    pub fn oc_sort_field_read(f: *const OcSortField, order: c_int, nbits: *mut u64, n: *mut u64, rank_doc: *mut u64,
                              rank_value: *mut f64, facets_version: *mut u64) -> c_int;
    pub fn oc_sort_field_destroy(f: *mut OcSortField);
    pub fn oc_search_sorted(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, p: *const OcSearchParams, sort: *const OcSort,
                            pins: *const OcPins, out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64,
                            out_n: *mut u32, out_count: *mut u64, out_pin_scores: *mut f32, out_pin_present: *mut u8) -> c_int;
    /// per query its own sort (q_sorts[b].field NULL: score order), pins and (q_filters) where-filter
    pub fn oc_search_q_sorted(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, p: *const OcSearchParams, q_sorts: *const OcSort,
                              pins: *const OcPins, out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64,
                              out_n: *mut u32, out_count: *mut u64, out_pin_scores: *mut f32, out_pin_present: *mut u8) -> c_int;
    pub fn oc_search_groups_sorted(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, g: *mut OcGroupBy, p: *const OcSearchParams,
                                   max_results: u32, sort: *const OcSort, pins: *const OcPins, group_stride: u32,
                                   out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64, out_n: *mut u32,
                                   out_count: *mut u64, out_group_doc_ids: *mut u64, out_group_scores: *mut f32,
                                   out_group_sort_values: *mut f64, out_group_n: *mut u32) -> c_int;
    pub fn oc_group_by_n_groups(g: *const OcGroupBy) -> u64;
    pub fn oc_search_q_groups(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, p: *const OcSearchParams, q_groups: *const OcGroupReq,
                              pins: *const OcPins, group_stride: u32, out_doc_ids: *mut u64, out_scores: *mut f32,
                              out_sort_values: *mut f64, out_n: *mut u32, out_count: *mut u64, out_pin_scores: *mut f32,
                              out_pin_present: *mut u8, out_group_doc_ids: *mut u64, out_group_scores: *mut f32,
                              out_group_sort_values: *mut f64, out_group_n: *mut u32) -> c_int;
    // per-query facets in the batched grouped call
    pub fn oc_facets_check(f: *const OcFacets, reqs: *const OcFacetReq, n: u32) -> c_int;
    pub fn oc_search_q_facets(ctx: *mut OcCtx, emb: *mut OcEmb, s: *mut OcStr, p: *const OcSearchParams, q_groups: *const OcGroupReq,
                              pins: *const OcPins, group_stride: u32, f: *mut OcFacets, q_facet_offsets: *const u32,
                              facet_reqs: *const OcFacetReq, out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64,
                              out_n: *mut u32, out_count: *mut u64, out_pin_scores: *mut f32, out_pin_present: *mut u8,
                              out_group_doc_ids: *mut u64, out_group_scores: *mut f32, out_group_sort_values: *mut f64,
                              out_group_n: *mut u32, out_facet_counts: *mut u64) -> c_int;
    pub fn oc_merge_sorted(n_indexes: u32, n_queries: u32, limit: u32, offset: u32, in_stride: u32, order: c_int,
                           doc_ids: *const *const u64, scores: *const *const f32, sort_values: *const *const f64,
                           n: *const *const u32, counts: *const *const u64, pins: *const OcPins,
                           pin_scores: *const *const f32, pin_present: *const *const u8, out_doc_ids: *mut u64,
                           out_scores: *mut f32, out_sort_values: *mut f64, out_n: *mut u32, out_count: *mut u64) -> c_int;
    /// every index of a collection on one ctx in one call, merged on the device (search_on_indexes)
    pub fn oc_search_indexes(ctx: *mut OcCtx, n_indexes: u32, ix: *const OcIndexQuery, pins: *const OcPins,
                             out_doc_ids: *mut u64, out_scores: *mut f32, out_sort_values: *mut f64, out_n: *mut u32,
                             out_count: *mut u64, out_pin_scores: *mut f32, out_pin_present: *mut u8) -> c_int;
    /// oc_search_indexes with groups and facets across the indexes; ex NULL or n_indexes entries
    pub fn oc_search_indexes_ex(ctx: *mut OcCtx, n_indexes: u32, ix: *const OcIndexQuery, ex: *const OcIndexExtras,
                                pins: *const OcPins, q_n_keys: *const u32, q_max_results: *const u32, group_stride: u32,
                                q_facet_offsets: *const u32, out_doc_ids: *mut u64, out_scores: *mut f32,
                                out_sort_values: *mut f64, out_n: *mut u32, out_count: *mut u64, out_pin_scores: *mut f32,
                                out_pin_present: *mut u8, out_group_doc_ids: *mut u64, out_group_scores: *mut f32,
                                out_group_sort_values: *mut f64, out_group_n: *mut u32, out_facet_counts: *mut u64) -> c_int;
    // term dictionary + batch query resolution (tokenize_and_stem + FST expansion), host only
    pub fn oc_dict_create(n_fields: u32, out: *mut *mut OcDict) -> c_int;
    pub fn oc_dict_destroy(d: *mut OcDict);
    pub fn oc_dict_add_terms(d: *mut OcDict, field: u32, terms: *const *const c_char, n: u32, out_ids: *mut u32) -> c_int;
    pub fn oc_dict_lookup(d: *mut OcDict, field: u32, term: *const c_char, out_id: *mut u32) -> c_int;
    pub fn oc_dict_size(d: *mut OcDict, field: u32) -> u32;
    pub fn oc_dict_set_stemmer(d: *mut OcDict, f: Option<OcStemFn>, user: *mut c_void) -> c_int;
    pub fn oc_dict_resolve(d: *mut OcDict, p: *const OcResolveParams, out: *mut *mut OcResolved) -> c_int;
    /// per query its own exact / tolerance / boost / mask (q NULL: p's); ctx non-NULL: typo tolerance on its device
    pub fn oc_dict_resolve_q(d: *mut OcDict, ctx: *mut OcCtx, p: *const OcResolveParams, q: *const OcResolveQuery,
                             out: *mut *mut OcResolved) -> c_int;
    pub fn oc_dict_device_bytes(d: *mut OcDict, ctx: *mut OcCtx) -> u64;
    pub fn oc_resolved_fill(r: *const OcResolved, p: *mut OcSearchParams);
    pub fn oc_resolved_free(r: *mut OcResolved);
}

fn check(rc: c_int) -> anyhow::Result<()> {
    if rc == 0 { return Ok(()); }
    let msg = unsafe { CStr::from_ptr(oc_last_error()) }.to_string_lossy().into_owned();
    anyhow::bail!("oramacore_b200 error {rc}: {msg}")
}

pub struct Ctx(*mut OcCtx);
unsafe impl Send for Ctx {}
unsafe impl Sync for Ctx {}
impl Ctx {
    pub fn new(device: i32) -> anyhow::Result<Self> {
        let mut sizes = [0usize; 4];
        unsafe { oc_abi_sizes(sizes.as_mut_ptr()) };
        assert_eq!(sizes[0], std::mem::size_of::<OcSearchParams>(), "oc_search_params layout drift");
        let mut p = std::ptr::null_mut();
        check(unsafe { oc_init(device, &mut p) })?;
        Ok(Ctx(p))
    }
}
impl Drop for Ctx { fn drop(&mut self) { unsafe { oc_shutdown(self.0) } } }

/// `EmbeddingFieldStorage` (embedding_field.rs): same method shapes.
pub struct EmbeddingField { h: *mut OcEmb, dim: usize }
unsafe impl Send for EmbeddingField {}
unsafe impl Sync for EmbeddingField {}
impl EmbeddingField {
    pub fn new(ctx: &Ctx, dimensions: usize, is_e5: bool) -> anyhow::Result<Self> {
        let mut h = std::ptr::null_mut();
        check(unsafe { oc_emb_create(ctx.0, dimensions as u32, 0, is_e5 as c_int, &mut h) })?;
        Ok(Self { h, dim: dimensions })
    }
    /// insert(DocumentId, Vec<Vec<f32>>)  (embedding_field.rs:232-237)
    pub fn insert(&self, doc_id: u64, vectors: &[Vec<f32>]) -> anyhow::Result<()> {
        let flat: Vec<f32> = vectors.iter().flat_map(|v| v.iter().copied()).collect();
        debug_assert_eq!(flat.len(), vectors.len() * self.dim);
        let ids = vec![doc_id; vectors.len()];
        check(unsafe { oc_emb_insert(self.h, ids.as_ptr(), flat.as_ptr() as *const c_void, ids.len() as u64) })
    }
    /// delete(DocumentId)  (embedding_field.rs:240-242)
    pub fn delete(&self, doc_id: u64) -> anyhow::Result<()> { check(unsafe { oc_emb_delete(self.h, &doc_id, 1) }) }
    /// compact() as Index::commit runs it (index/mod.rs:583-590): drops the deleted rows on the device, in place
    pub fn compact(&self, shrink: bool) -> anyhow::Result<OcEmbCompact> {
        let mut st = OcEmbCompact::default();
        check(unsafe { oc_emb_compact(self.h, if shrink { OC_EMB_COMPACT_SHRINK } else { 0 }, &mut st) })?;
        Ok(st)
    }
    /// search(&VectorSearchParams, &mut HashMap)  (embedding_field.rs:250-278): `output[doc] += score`
    pub fn search(&self, target: &[f32], similarity: f32, limit: usize, filter: Option<(&[u64], u64)>,
                  output: &mut std::collections::HashMap<u64, f32>) -> anyhow::Result<()> {
        let (mut docs, mut scores, mut n) = (vec![0u64; limit], vec![0f32; limit], 0u32);
        let (fb, nb) = filter.map(|(b, n)| (b.as_ptr(), n)).unwrap_or((std::ptr::null(), 0));
        check(unsafe { oc_emb_search(self.h, target.as_ptr(), 1, limit as u32, similarity, fb, nb,
                                     docs.as_mut_ptr(), scores.as_mut_ptr(), &mut n) })?;
        for i in 0..n as usize { *output.entry(docs[i]).or_insert(0.0) += scores[i]; }
        Ok(())
    }
}
impl Drop for EmbeddingField { fn drop(&mut self) { unsafe { oc_emb_destroy(self.h) } } }
