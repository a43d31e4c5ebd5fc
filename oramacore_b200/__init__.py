"""oramacore_b200 — H100-native (sm_90a) implementation of OramaCore's search hot path:
embedding scan + BM25F posting scorer + hybrid fusion/top-k behind the reference's
search() surface (mode = fulltext | vector | hybrid).  CUDA only; no CPU fallback."""
from .types import (FacetFieldNotFound, FieldPostings, FilterFieldNotFound, InvalidSortField, PromoteItem, SortBy, SortFieldNotFound, StringIndexData, TextQuery, SearchHits, MODE_FULLTEXT, MODE_VECTOR,
                    MODE_HYBRID, BM25_B, BM25_K)
from ._lib import OcError, build, lib, SO_PATH
from .engine import (Context, DeviceFilter, FacetStore, GeoPointField, GroupBy, OmcStore, geo_to_meter, merge_index_results, merge_index_results_pinned, merge_index_results_sorted, resolve_sort_by, IndexPart, search_indexes, search_indexes_arrays,
                     collection_facet_requests, collection_group_keys,
                     facet_requests, search_facets, search_q_facets, search_q_facets_arrays, search_pinned, search_q_groups, search_q_groups_arrays, search_q_sorted_arrays, search_sorted, search_sorted_arrays, SortField,
                     search_pinned_arrays, search_groups, search_groups_arrays, EmbeddingFieldStorage, SearchBatcher, StringFieldStorage, TermDictionary, TextQueryBatch, TokenScoreContext, TokenScoreParams,
                     QueryParams, VectorSearchParams, from_bf16, pinned_empty, search, to_bf16)
from .where import WhereFilter, evaluate_where, parse_where, where_keys

__all__ = ["FieldPostings", "StringIndexData", "TextQuery", "SearchHits", "MODE_FULLTEXT", "MODE_VECTOR",
           "MODE_HYBRID", "BM25_B", "BM25_K", "OcError", "build", "lib", "SO_PATH", "Context", "DeviceFilter", "FacetStore", "GeoPointField", "GroupBy", "OmcStore", "geo_to_meter", "merge_index_results", "merge_index_results_pinned", "PromoteItem",
           "InvalidSortField", "FilterFieldNotFound", "FacetFieldNotFound", "collection_facet_requests", "collection_group_keys", "WhereFilter", "evaluate_where", "parse_where", "where_keys", "SortBy", "SortFieldNotFound", "SortField", "merge_index_results_sorted", "resolve_sort_by", "IndexPart", "search_indexes", "search_indexes_arrays",
           "facet_requests", "search_q_facets", "search_q_facets_arrays", "search_q_groups", "search_q_groups_arrays", "search_q_sorted_arrays", "search_sorted", "search_sorted_arrays",
           "search_facets", "search_pinned", "search_pinned_arrays", "search_groups", "search_groups_arrays",
           "EmbeddingFieldStorage", "SearchBatcher", "StringFieldStorage", "TermDictionary", "TextQueryBatch", "TokenScoreContext", "TokenScoreParams",
           "QueryParams", "VectorSearchParams", "from_bf16", "pinned_empty", "search", "to_bf16"]
