"""Document sharding of the index data across the GPUs of one box (SURVEY.md §8e).

Shard g owns the contiguous doc-row range [g*N/G, (g+1)*N/G) of the embedding matrix AND
the postings restricted to those rows (so BM25 accumulators are shard-local).  The global
quantities BM25 needs — N (document_count), avg_field_len and per-term df — are replicated, so
there is no per-query collective for them.  For a loaded corpus they are computed here, at load
time.  A commit on a shard drops its df table: StringFieldStorage.sync_global() on every rank then
rebuilds the tables and the averages on the devices from all shards (IndexLoader(shard=...) does so
at the end of each commit); N stays the caller's.
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np

from .types import FieldPostings, StringIndexData


def shard_range(n_rows: int, rank: int, world: int) -> Tuple[int, int]:
    return (n_rows * rank) // world, (n_rows * (rank + 1)) // world


def shard_string_index(data: StringIndexData, lo: int, hi: int) -> Tuple[StringIndexData, List[np.ndarray]]:
    """Postings restricted to rows [lo, hi) re-based to shard-local rows; returns the shard and
    the per-field global df table (posting-list lengths of the whole corpus)."""
    fields, gdf = [], []
    for f in data.fields:
        df = np.diff(f.term_offsets.astype(np.int64))
        sel = (f.post_row >= lo) & (f.post_row < hi)
        term_of = np.repeat(np.arange(f.n_terms, dtype=np.int64), df)[sel]
        offs = np.zeros(f.n_terms + 1, np.uint64)
        offs[1:] = np.cumsum(np.bincount(term_of, minlength=f.n_terms)).astype(np.uint64)
        fields.append(FieldPostings(f.avg_field_len, offs, (f.post_row[sel] - np.uint32(lo)).astype(np.uint32),
                                    f.post_tf[sel].copy(), f.post_len[sel].copy()))
        gdf.append(df.astype(np.uint32))
    docs = np.arange(lo, hi, dtype=np.uint64) if data.row_doc_ids is None else data.row_doc_ids[lo:hi].copy()
    return StringIndexData(fields, hi - lo, data.document_count, docs), gdf
