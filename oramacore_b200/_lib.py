"""ctypes binding of liboramacore_b200.so (the C ABI in include/oramacore_b200.h).

The library is CUDA-only.  Loading succeeds on a CPU box (symbols resolve; used by the
`not gpu` tests), every compute call fails loudly with OcError when no sm_90 device is
present — there is no CPU fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("OC_SO_PATH") or os.path.join(_HERE, "liboramacore_b200.so")   # OC_SO_PATH: A/B builds (csrc/Makefile)
CSRC = os.path.join(_HERE, "csrc")

OC_OK = 0
OC_MAX_TOPK = 1024
OC_COMM_ID_BYTES = 128
OC_GEO_EARTH_RADIUS_M = 6371000.0
OC_GEO_MAX_VERTICES = 2048
OC_RANGE_LO_OPEN = 1
OC_RANGE_HI_OPEN = 2
OC_FACET_UNIQUE = 1   # oc_facets_insert_variants: set semantics (a bool field)
# Timing.scan_variant: which embedding sweep served the last batch (include/oramacore_b200.h OC_SCAN_*)
OC_SCAN_EXACT = 0
OC_SCAN_TC_TF32 = 1
OC_SCAN_TC_BF16 = 4
OC_SCAN_TC_F16 = 5   # wgmma .f16 on the fp16 copy of an fp32 store; OC_EMB_F16=0 selects OC_SCAN_TC_TF32
OC_EMB_COMPACT_SHRINK = 1   # oc_emb_compact: also give the capacity beyond num_rows back
OC_BATCHER_MIXED = 1   # oc_batcher_create2: requests with different scalars share a batch
# where-program node ops (oc_where_node.op) and bounds
OC_WHERE_NONE, OC_WHERE_VARIANT, OC_WHERE_RANGE, OC_WHERE_GEO_RADIUS, OC_WHERE_GEO_POLYGON = 0, 1, 2, 3, 4
OC_WHERE_FILTER, OC_WHERE_AND, OC_WHERE_OR, OC_WHERE_NOT = 5, 6, 7, 8
OC_WHERE_MAX_NODES = 4096
OC_WHERE_MAX_DEPTH = 32

EXPORTED_SYMBOLS = [
    "oc_last_error", "oc_version", "oc_abi_sizes", "oc_init", "oc_shutdown", "oc_device_info", "oc_comm_unique_id",
    "oc_comm_init", "oc_comm_init_local", "oc_comm_p2p_export", "oc_comm_p2p_import", "oc_emb_create", "oc_emb_destroy", "oc_emb_reserve", "oc_emb_insert", "oc_emb_delete", "oc_emb_compact",
    "oc_emb_info", "oc_emb_search", "oc_str_create", "oc_str_destroy", "oc_str_set_rows", "oc_str_load_field",
    "oc_str_insert", "oc_str_commit", "oc_str_commit_ex", "oc_str_read_rows", "oc_str_read_field", "oc_str_delete", "oc_str_info", "oc_str_set_global", "oc_str_sync_global", "oc_str_read_global_df", "oc_search", "oc_pinned_alloc", "oc_pinned_free", "oc_last_timing", "oc_launch_count",
    "oc_batcher_create", "oc_batcher_create2", "oc_batcher_destroy", "oc_batcher_search", "oc_batcher_search_sorted", "oc_batcher_search_groups",
    "oc_batcher_search_faceted", "oc_batcher_stats",
    "oc_filter_from_ids", "oc_filter_from_bits", "oc_filter_and", "oc_filter_or", "oc_filter_not", "oc_filter_count",
    "oc_filter_read", "oc_filter_nbits", "oc_filter_destroy", "oc_merge_results",
    "oc_geo_field_create", "oc_geo_field_destroy", "oc_filter_geo_radius", "oc_filter_geo_polygon",
    "oc_geo_field_insert", "oc_geo_field_delete", "oc_geo_field_commit_ex", "oc_geo_field_read",
    "oc_facets_create", "oc_facets_destroy", "oc_facets_add_field", "oc_facets_add_number_field", "oc_search_facets",
    "oc_facets_insert_variants", "oc_facets_add_variant", "oc_facets_insert_numbers", "oc_facets_clear", "oc_facets_delete",
    "oc_facets_commit_ex", "oc_facets_read_field",
    "oc_omc_create", "oc_omc_destroy", "oc_omc_set", "oc_omc_delete", "oc_omc_commit_ex", "oc_omc_read",
    "oc_filter_facet_variant", "oc_filter_facet_range", "oc_where_check", "oc_filter_from_where",
    "oc_group_by_create", "oc_group_by_destroy", "oc_search_groups",
    "oc_search_pinned", "oc_search_groups_pinned", "oc_merge_pinned",
    "oc_sort_field_create", "oc_sort_field_from_facets", "oc_sort_field_read", "oc_sort_field_destroy", "oc_search_sorted", "oc_search_q_sorted", "oc_search_groups_sorted", "oc_merge_sorted",
    "oc_search_indexes", "oc_search_indexes_ex",
    "oc_group_by_n_groups", "oc_search_q_groups", "oc_facets_check", "oc_search_q_facets",
    "oc_dict_create", "oc_dict_destroy", "oc_dict_add_terms", "oc_dict_lookup", "oc_dict_size", "oc_dict_set_stemmer", "oc_stem_english",
    "oc_dict_resolve", "oc_dict_resolve_q", "oc_dict_device_bytes", "oc_resolved_arrays", "oc_resolved_fill", "oc_resolved_free",
]


class OcError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"oramacore_b200 error {code}: {msg}")
        self.code = code


class EmbInfo(C.Structure):
    _fields_ = [("num_embeddings", C.c_uint64), ("num_rows", C.c_uint64), ("dimensions", C.c_uint32),
                ("dtype", C.c_int), ("device_bytes", C.c_uint64)]


class EmbCompact(C.Structure):   # oc_emb_compact_t
    _fields_ = [("rows_before", C.c_uint64), ("rows_after", C.c_uint64), ("rows_moved", C.c_uint64),
                ("device_bytes_before", C.c_uint64), ("device_bytes_after", C.c_uint64), ("workspace_bytes", C.c_uint64),
                ("device_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class StrCommit(C.Structure):   # oc_str_commit_t
    _fields_ = [("rows_before", C.c_uint64), ("rows_after", C.c_uint64), ("postings_before", C.c_uint64),
                ("postings_after", C.c_uint64), ("pending_postings", C.c_uint64), ("workspace_bytes", C.c_uint64),
                ("device_ms", C.c_float), ("wall_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class StrSync(C.Structure):   # oc_str_sync_t
    _fields_ = [("version", C.c_uint64), ("rows_global", C.c_uint64), ("bytes_reduced", C.c_uint64),
                ("device_ms", C.c_float), ("wall_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class FilterCommit(C.Structure):   # oc_filter_commit_t
    _fields_ = [("version", C.c_uint64), ("rows_kept", C.c_uint64), ("rows_dropped", C.c_uint64), ("rows_added", C.c_uint64),
                ("workspace_bytes", C.c_uint64), ("device_ms", C.c_float), ("wall_ms", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class StrInfo(C.Structure):
    _fields_ = [("total_documents", C.c_uint64), ("total_postings", C.c_uint64),
                ("unique_terms_count", C.c_uint64), ("n_fields", C.c_uint32), ("device_bytes", C.c_uint64),
                ("version", C.c_uint64), ("pending_postings", C.c_uint64)]


class SearchParams(C.Structure):
    _fields_ = [("mode", C.c_int), ("n_queries", C.c_uint32), ("limit", C.c_uint32), ("offset", C.c_uint32),
                ("similarity", C.c_float), ("threshold", C.c_float), ("bm25_k", C.c_float), ("bm25_b", C.c_float),
                ("q_vecs", C.c_void_p), ("q_token_offsets", C.c_void_p), ("token_term_offsets", C.c_void_p),
                ("term_field", C.c_void_p), ("term_id", C.c_void_p), ("term_weight", C.c_void_p),
                ("filter_bits", C.c_void_p), ("filter_nbits", C.c_uint64),
                ("omc_doc_ids", C.c_void_p), ("omc_mult", C.c_void_p), ("n_omc", C.c_uint64),
                ("sharded", C.c_int), ("vector_limit", C.c_uint32), ("filter", C.c_void_p),
                ("q_filters", C.c_void_p), ("q_params", C.c_void_p), ("q_where", C.c_void_p), ("omc", C.c_void_p)]


class QueryParams(C.Structure):   # oc_query_params: one entry of SearchParams.q_params
    _fields_ = [("mode", C.c_int), ("limit", C.c_uint32), ("offset", C.c_uint32), ("similarity", C.c_float),
                ("threshold", C.c_float), ("vector_limit", C.c_uint32)]


class WhereNode(C.Structure):   # oc_where_node: one node of a where program
    _fields_ = [("op", C.c_uint32), ("field", C.c_uint32), ("arg", C.c_uint32), ("first_vertex", C.c_uint32),
                ("n_vertices", C.c_uint32), ("a", C.c_double), ("b", C.c_double), ("c", C.c_double), ("src", C.c_void_p)]


class Where(C.Structure):   # oc_where: the programs of a batch (SearchParams.q_where)
    _fields_ = [("nbits", C.c_uint64), ("q_node_offsets", C.c_void_p), ("nodes", C.c_void_p), ("vertex_lat", C.c_void_p),
                ("vertex_lon", C.c_void_p)]


class FacetReq(C.Structure):
    _fields_ = [("field", C.c_uint32), ("variant", C.c_uint32), ("from_", C.c_double), ("to", C.c_double)]


class Pins(C.Structure):
    _fields_ = [("q_pin_offsets", C.c_void_p), ("doc_ids", C.c_void_p), ("positions", C.c_void_p), ("apply", C.c_int)]


class Sort(C.Structure):
    _fields_ = [("field", C.c_void_p), ("order", C.c_int)]


class IndexQuery(C.Structure):   # oc_index_query: one index of an oc_search_indexes call
    _fields_ = [("emb", C.c_void_p), ("str", C.c_void_p), ("p", C.POINTER(SearchParams)), ("q_sorts", C.c_void_p)]


class IndexExtras(C.Structure):   # oc_index_extras: one index's groups and facets in an oc_search_indexes_ex call
    _fields_ = [("q_groups", C.c_void_p), ("q_group_keys", C.c_void_p), ("facets", C.c_void_p), ("n_facet_reqs", C.c_uint32),
                ("facet_reqs", C.c_void_p), ("facet_slots", C.c_void_p)]


class GroupReq(C.Structure):
    _fields_ = [("groups", C.c_void_p), ("max_results", C.c_uint32), ("sort", Sort)]


class ResolveParams(C.Structure):
    _fields_ = [("texts", C.POINTER(C.c_char_p)), ("n_queries", C.c_uint32), ("exact", C.c_int), ("tolerance", C.c_int),
                ("field_boost", C.c_void_p), ("field_mask", C.c_void_p), ("exact_match_boost", C.c_float)]


class ResolveQuery(C.Structure):   # oc_resolve_query: one query's options for oc_dict_resolve_q
    _fields_ = [("exact", C.c_int), ("tolerance", C.c_int), ("field_boost", C.c_void_p), ("field_mask", C.c_void_p)]


STEM_FN = C.CFUNCTYPE(C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p)


class Timing(C.Structure):
    _fields_ = [("h2d_ms", C.c_float), ("device_ms", C.c_float), ("d2h_ms", C.c_float), ("scan_ms", C.c_float),
                ("bm25_ms", C.c_float), ("fuse_ms", C.c_float), ("comm_ms", C.c_float),
                ("kernel_launches", C.c_uint32), ("scan_launches", C.c_uint32), ("scan_bytes", C.c_uint64),
                ("bm25_postings", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("scan_tensor_core", C.c_uint32), ("scan_unproven", C.c_uint32),
                ("scan_variant", C.c_uint32), ("scan_sweep_ms", C.c_float), ("rerun_ms", C.c_float),
                ("scan_rescored", C.c_uint32), ("bm25_dense_items", C.c_uint32), ("bm25_dense_skipped", C.c_uint32)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


def build(force: bool = False) -> str:
    """Compile the shared library in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))]
    srcs.append(os.path.join(_HERE, "..", "include", "oramacore_b200.h"))
    stale = (not os.path.exists(SO_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(SO_PATH) for s in srcs)
    if force or stale:
        r = subprocess.run(["make", "-C", CSRC] + (["-B"] if force else []), capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc build failed:\n" + r.stdout + r.stderr)
    return SO_PATH


_lib = None


def lib():
    """Load the CUDA library; raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise OcError(-2, f"{SO_PATH} is missing: run __graft_entry__.build() (nvcc, sm_90a). "
                          "There is no CPU fallback.")
    L = C.CDLL(SO_PATH)
    vp, u32, u64, f32, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_float, C.c_int
    L.oc_last_error.restype = C.c_char_p
    L.oc_version.restype = i32
    L.oc_abi_sizes.argtypes = [C.POINTER(C.c_size_t)]
    L.oc_abi_sizes.restype = None
    L.oc_init.argtypes = [i32, C.POINTER(vp)]
    L.oc_shutdown.argtypes = [vp]
    L.oc_shutdown.restype = None
    L.oc_device_info.argtypes = [vp, C.POINTER(i32), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
    L.oc_comm_unique_id.argtypes = [vp]
    L.oc_comm_init.argtypes = [vp, i32, i32, vp]
    L.oc_comm_init_local.argtypes = [vp, i32]
    L.oc_comm_p2p_export.argtypes = [vp, vp]
    L.oc_comm_p2p_import.argtypes = [vp, vp]
    L.oc_emb_create.argtypes = [vp, u32, i32, i32, C.POINTER(vp)]
    L.oc_emb_destroy.argtypes = [vp]
    L.oc_emb_destroy.restype = None
    L.oc_emb_reserve.argtypes = [vp, u64]
    L.oc_emb_insert.argtypes = [vp, vp, vp, u64]
    L.oc_emb_delete.argtypes = [vp, vp, u64]
    L.oc_emb_info.argtypes = [vp, C.POINTER(EmbInfo)]
    L.oc_emb_compact.argtypes = [vp, u32, C.POINTER(EmbCompact)]
    L.oc_emb_search.argtypes = [vp, vp, u32, u32, f32, vp, u64, vp, vp, vp]
    L.oc_str_create.argtypes = [vp, u32, C.POINTER(vp)]
    L.oc_str_destroy.argtypes = [vp]
    L.oc_str_destroy.restype = None
    L.oc_str_set_rows.argtypes = [vp, u64, vp, u64]
    L.oc_str_load_field.argtypes = [vp, u32, f32, u32, vp, vp, vp, vp, vp]
    L.oc_str_insert.argtypes = [vp, u32, u64, C.c_uint16, u32, vp, vp]
    L.oc_str_commit.argtypes = [vp]
    L.oc_str_commit_ex.argtypes = [vp, C.POINTER(StrCommit)]
    L.oc_str_read_rows.argtypes = [vp, C.POINTER(u64), vp, C.POINTER(u64), C.POINTER(u64)]
    L.oc_str_read_field.argtypes = [vp, u32, C.POINTER(f32), C.POINTER(u32), C.POINTER(u64), vp, vp, vp, vp]
    L.oc_str_set_global.argtypes = [vp, u64, vp]
    L.oc_str_sync_global.argtypes = [vp, C.POINTER(StrSync)]
    L.oc_str_read_global_df.argtypes = [vp, u32, C.POINTER(u32), vp]
    L.oc_str_delete.argtypes = [vp, vp, u64]
    L.oc_str_info.argtypes = [vp, C.POINTER(StrInfo)]
    L.oc_search.argtypes = [vp, vp, vp, C.POINTER(SearchParams), vp, vp, vp, vp]
    L.oc_batcher_create.argtypes = [vp, vp, vp, u32, u32, C.POINTER(vp)]
    L.oc_batcher_create2.argtypes = [vp, vp, vp, u32, u32, u32, C.POINTER(vp)]
    L.oc_batcher_destroy.argtypes = [vp]
    L.oc_batcher_destroy.restype = None
    L.oc_batcher_search.argtypes = [vp, C.POINTER(SearchParams), vp, vp, vp, vp]
    L.oc_batcher_search_sorted.argtypes = [vp, C.POINTER(SearchParams), vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.oc_batcher_search_groups.argtypes = [vp, C.POINTER(SearchParams), C.POINTER(GroupReq), vp, u32] + [vp] * 11
    L.oc_batcher_search_faceted.argtypes = [vp, C.POINTER(SearchParams), vp, vp, u32, vp, vp, u32] + [vp] * 12
    L.oc_batcher_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.oc_filter_from_ids.argtypes = [vp, vp, u64, u64, C.POINTER(vp)]
    L.oc_filter_from_bits.argtypes = [vp, vp, u64, C.POINTER(vp)]
    L.oc_filter_and.argtypes = [vp, vp, C.POINTER(vp)]
    L.oc_filter_or.argtypes = [vp, vp, C.POINTER(vp)]
    L.oc_filter_not.argtypes = [vp, C.POINTER(vp)]
    L.oc_filter_count.argtypes = [vp, C.POINTER(u64)]
    L.oc_filter_read.argtypes = [vp, vp]
    L.oc_filter_nbits.argtypes = [vp, C.POINTER(u64)]
    L.oc_filter_destroy.argtypes = [vp]
    L.oc_filter_destroy.restype = None
    L.oc_geo_field_create.argtypes = [vp, u64, u64, vp, vp, vp, C.POINTER(vp)]
    L.oc_geo_field_destroy.argtypes = [vp]
    L.oc_geo_field_destroy.restype = None
    L.oc_filter_geo_radius.argtypes = [vp, C.c_double, C.c_double, C.c_double, i32, C.POINTER(vp)]
    L.oc_filter_geo_polygon.argtypes = [vp, vp, vp, u32, i32, C.POINTER(vp)]
    L.oc_facets_create.argtypes = [vp, u64, C.POINTER(vp)]
    L.oc_facets_destroy.argtypes = [vp]
    L.oc_facets_destroy.restype = None
    L.oc_facets_add_field.argtypes = [vp, u32, vp, vp, C.POINTER(u32)]
    L.oc_facets_add_number_field.argtypes = [vp, u64, vp, vp, C.POINTER(u32)]
    L.oc_facets_insert_variants.argtypes = [vp, u32, u64, vp, vp, u32]
    L.oc_facets_add_variant.argtypes = [vp, u32, C.POINTER(u32)]
    L.oc_facets_insert_numbers.argtypes = [vp, u32, u64, vp, vp]
    L.oc_facets_clear.argtypes = [vp, u32, u64, vp]
    L.oc_facets_delete.argtypes = [vp, u64, vp]
    L.oc_facets_commit_ex.argtypes = [vp, u64, C.POINTER(FilterCommit)]
    L.oc_facets_read_field.argtypes = [vp, u32, C.POINTER(u32), C.POINTER(u64), vp, vp, vp]
    L.oc_omc_create.argtypes = [vp, C.POINTER(vp)]
    L.oc_omc_destroy.argtypes = [vp]
    L.oc_omc_destroy.restype = None
    L.oc_omc_set.argtypes = [vp, vp, vp, u64]
    L.oc_omc_delete.argtypes = [vp, vp, u64]
    L.oc_omc_commit_ex.argtypes = [vp, C.POINTER(FilterCommit)]
    L.oc_omc_read.argtypes = [vp, C.POINTER(u64), vp, vp, C.POINTER(u64)]
    L.oc_geo_field_insert.argtypes = [vp, u64, vp, vp, vp]
    L.oc_geo_field_delete.argtypes = [vp, u64, vp]
    L.oc_geo_field_commit_ex.argtypes = [vp, u64, C.POINTER(FilterCommit)]
    L.oc_geo_field_read.argtypes = [vp, C.POINTER(u64), vp, vp, vp]
    L.oc_filter_facet_variant.argtypes = [vp, u32, u32, C.POINTER(vp)]
    L.oc_filter_facet_range.argtypes = [vp, u32, C.c_double, C.c_double, u32, C.POINTER(vp)]
    L.oc_where_check.argtypes = [C.POINTER(Where), u32]
    L.oc_filter_from_where.argtypes = [vp, C.POINTER(Where), u32, C.POINTER(vp)]
    L.oc_search_facets.argtypes = [vp, vp, vp, vp, C.POINTER(SearchParams), C.POINTER(FacetReq), u32, vp]
    L.oc_group_by_create.argtypes = [vp, vp, u32, C.POINTER(vp), C.POINTER(u64)]
    L.oc_group_by_destroy.argtypes = [vp]
    L.oc_group_by_destroy.restype = None
    L.oc_search_groups.argtypes = [vp, vp, vp, vp, C.POINTER(SearchParams), u32, vp, vp, vp, vp, vp, vp, vp]
    L.oc_merge_results.argtypes = [u32, u32, u32, u32, u32, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), vp, vp, vp, vp]
    L.oc_search_pinned.argtypes = [vp, vp, vp, C.POINTER(SearchParams), C.POINTER(Pins), vp, vp, vp, vp, vp, vp]
    L.oc_search_groups_pinned.argtypes = [vp, vp, vp, vp, C.POINTER(SearchParams), u32, C.POINTER(Pins), u32, vp, vp, vp, vp, vp, vp, vp]
    L.oc_merge_pinned.argtypes = [u32, u32, u32, u32, u32, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(Pins),
                                  C.POINTER(vp), C.POINTER(vp), vp, vp, vp, vp]
    L.oc_sort_field_create.argtypes = [vp, u64, u64, vp, vp, C.POINTER(vp)]
    L.oc_sort_field_from_facets.argtypes = [vp, u32, vp, C.POINTER(vp)]
    L.oc_sort_field_read.argtypes = [vp, C.c_int, C.POINTER(u64), C.POINTER(u64), vp, vp, C.POINTER(u64)]
    L.oc_sort_field_destroy.argtypes = [vp]
    L.oc_sort_field_destroy.restype = None
    L.oc_search_sorted.argtypes = [vp, vp, vp, C.POINTER(SearchParams), C.POINTER(Sort), vp, vp, vp, vp, vp, vp, vp, vp]
    L.oc_search_q_sorted.argtypes = [vp, vp, vp, C.POINTER(SearchParams), C.POINTER(Sort), vp, vp, vp, vp, vp, vp, vp, vp]
    L.oc_search_groups_sorted.argtypes = [vp, vp, vp, vp, C.POINTER(SearchParams), u32, C.POINTER(Sort), vp, u32, vp, vp, vp, vp,
                                          vp, vp, vp, vp, vp]
    L.oc_group_by_n_groups.argtypes = [vp]
    L.oc_group_by_n_groups.restype = u64
    L.oc_search_q_groups.argtypes = [vp, vp, vp, C.POINTER(SearchParams), C.POINTER(GroupReq), vp, u32] + [vp] * 11
    L.oc_facets_check.argtypes = [vp, vp, u32]
    L.oc_search_q_facets.argtypes = [vp, vp, vp, C.POINTER(SearchParams), vp, vp, u32, vp, vp, vp] + [vp] * 12
    L.oc_merge_sorted.argtypes = [u32, u32, u32, u32, u32, C.c_int, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                  C.POINTER(vp), vp, C.POINTER(vp), C.POINTER(vp), vp, vp, vp, vp, vp]
    L.oc_search_indexes.argtypes = [vp, u32, C.POINTER(IndexQuery), vp] + [vp] * 7
    L.oc_search_indexes_ex.argtypes = [vp, u32, C.POINTER(IndexQuery), vp, vp, vp, vp, u32, vp] + [vp] * 12
    L.oc_dict_create.argtypes = [u32, C.POINTER(vp)]
    L.oc_dict_destroy.argtypes = [vp]
    L.oc_dict_destroy.restype = None
    L.oc_dict_add_terms.argtypes = [vp, u32, C.POINTER(C.c_char_p), u32, vp]
    L.oc_dict_lookup.argtypes = [vp, u32, C.c_char_p, C.POINTER(u32)]
    L.oc_dict_size.argtypes = [vp, u32]
    L.oc_dict_size.restype = u32
    L.oc_dict_set_stemmer.argtypes = [vp, vp, vp]
    L.oc_stem_english.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, vp]
    L.oc_stem_english.restype = C.c_size_t
    L.oc_dict_resolve.argtypes = [vp, C.POINTER(ResolveParams), C.POINTER(vp)]
    L.oc_dict_resolve_q.argtypes = [vp, vp, C.POINTER(ResolveParams), vp, C.POINTER(vp)]
    L.oc_dict_device_bytes.argtypes = [vp, vp]
    L.oc_dict_device_bytes.restype = u64
    L.oc_resolved_arrays.argtypes = [vp] + [C.POINTER(vp)] * 5 + [C.POINTER(u32)] * 2
    L.oc_resolved_arrays.restype = None
    L.oc_resolved_fill.argtypes = [vp, C.POINTER(SearchParams)]
    L.oc_resolved_fill.restype = None
    L.oc_resolved_free.argtypes = [vp]
    L.oc_resolved_free.restype = None
    L.oc_pinned_alloc.argtypes = [C.c_size_t, C.POINTER(vp)]
    L.oc_pinned_free.argtypes = [vp]
    L.oc_pinned_free.restype = None
    L.oc_last_timing.argtypes = [vp, C.POINTER(Timing)]
    L.oc_launch_count.argtypes = [vp]
    L.oc_launch_count.restype = u64
    _lib = L
    return L


def check(rc: int):
    if rc != OC_OK:
        raise OcError(rc, lib().oc_last_error().decode("utf-8", "replace"))
