"""Plain host-side data carriers shared by the C-ABI binding (and, in tests, by the oracle wrapper).

Names follow the reference's domain (SURVEY.md §8a):
  * `FieldPostings`   — one StringFieldStorage's committed postings
                        (read/index/string_field.rs:155-177: field_length u16, per-term tf).
  * `StringIndexData` — the string fields of one Index sharing a row space
                        (`row -> DocumentId(u64)`, types.rs:111-112).
  * `TextQuery`       — one query after host-side token -> index-term resolution
                        (token_score.rs:196-209 tokenise/stem; prefix / Levenshtein expansion
                        is done by the external StringStorage on the host).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np

MODE_FULLTEXT = 0  # ScoreMode::FullText / Default (types.rs:934-940)
MODE_VECTOR = 1    # ScoreMode::Vector
MODE_HYBRID = 2    # ScoreMode::Hybrid

BM25_B = 0.75      # bm25.rs:56-63
BM25_K = 1.2       # token_score.rs:283,291


@dataclass
class FieldPostings:
    avg_field_len: float
    term_offsets: np.ndarray  # uint64 [n_terms+1]
    post_row: np.ndarray      # uint32 [n_postings], ascending inside a term
    post_tf: np.ndarray       # uint16
    post_len: np.ndarray      # uint16

    @property
    def n_terms(self) -> int:
        return int(self.term_offsets.shape[0] - 1)

    def validate(self) -> None:
        assert self.term_offsets.dtype == np.uint64 and self.term_offsets.ndim == 1
        assert self.post_row.dtype == np.uint32 and self.post_tf.dtype == np.uint16
        assert self.post_len.dtype == np.uint16
        n = int(self.term_offsets[-1])
        assert self.post_row.shape[0] == n == self.post_tf.shape[0] == self.post_len.shape[0]


@dataclass
class StringIndexData:
    fields: List[FieldPostings]
    n_rows: int
    document_count: int                       # N for idf (token_score.rs:221)
    row_doc_ids: Optional[np.ndarray] = None  # uint64 ascending; None => doc_id == row


@dataclass
class TextQuery:
    token_term_offsets: np.ndarray  # uint32 [n_tokens+1]
    term_field: np.ndarray          # uint32 per expanded term
    term_id: np.ndarray             # uint32 per expanded term
    term_weight: np.ndarray         # float32: field boost * exact-match factor

    @property
    def n_tokens(self) -> int:
        return int(self.token_term_offsets.shape[0] - 1)

    @staticmethod
    def single_terms(term_ids, field: int = 0, weight: float = 1.0) -> "TextQuery":
        """One expanded term per token (exact resolution), all in `field`."""
        t = np.asarray(term_ids, dtype=np.uint32)
        n = t.shape[0]
        return TextQuery(np.arange(n + 1, dtype=np.uint32), np.full(n, field, np.uint32), t,
                         np.full(n, weight, np.float32))

    @staticmethod
    def from_tokens(tokens) -> "TextQuery":
        """tokens: list of lists of (field, term_id, weight)."""
        offs = [0]
        f, t, w = [], [], []
        for tok in tokens:
            for (fi, ti, wi) in tok:
                f.append(fi); t.append(ti); w.append(wi)
            offs.append(len(t))
        return TextQuery(np.asarray(offs, np.uint32), np.asarray(f, np.uint32),
                         np.asarray(t, np.uint32), np.asarray(w, np.float32))


@dataclass
class SearchHits:
    doc_ids: np.ndarray   # uint64 [n]
    scores: np.ndarray    # float32 [n]
    count: int            # search.rs:482 — all matching documents


@dataclass(frozen=True)
class PromoteItem:
    """oramacore_lib::pin_rules::PromoteItem: a pin rule's consequence places `doc_id` at `position`."""
    doc_id: int
    position: int


@dataclass(frozen=True)
class SortBy:
    """SortBy (types.rs:1350-1357, 1403-1404): order the hits by a number, date or bool field; order "ASC" (the
    default) or "DESC"."""
    property: str
    order: str = "ASC"


class SortFieldNotFound(KeyError):
    """ReadError::SortFieldNotFound: the sortBy property is not a filter field of the index."""

    def __init__(self, name: str):
        super().__init__(name)
        self.name = name


class FilterFieldNotFound(KeyError):
    """ReadError::FilterFieldNotFound: a key of the where-filter is not a filter field of any index (search.rs:435-449)."""

    def __init__(self, name: str):
        super().__init__(name)
        self.name = name


class FacetFieldNotFound(KeyError):
    """ReadError::FacetFieldNotFound: the facet fields that are not a filter field of any index (search.rs:452-464)."""

    def __init__(self, names):
        super().__init__(list(names))
        self.names = list(names)


class InvalidSortField(ValueError):
    """ReadError::InvalidSortField(name, kind): the sortBy property is a field that cannot be sorted by (string,
    string_filter, geopoint); `kind` is the reference's FieldType name, e.g. "GeoPoint"."""

    def __init__(self, name: str, kind: str):
        super().__init__(name, kind)
        self.name, self.kind = name, kind
