"""The rank rule of a sort field (oc_sort_field_create, oc_sort_field_from_facets), restated in numpy.

Per order, from (document, value) entries over DocumentId [0, nbits):
  * a value is normalised with + 0.0, so -0.0 and +0.0 are one value and the value written out is +0.0;
  * ASC sorts by ascending value, DESC by descending value; equal values go by ascending document in both orders;
  * a document appears once, at its first position in that order: its minimum value for ASC, its maximum for DESC
    (an entry repeated exactly counts once);
  * entries with a document >= nbits are dropped.
The result of one order is (rank_doc, rank_value): the documents in rank order and the value each was placed by, as
SortField.read returns them."""
from __future__ import annotations

from typing import Sequence, Tuple

import numpy as np


def rank_order(doc_ids, values, nbits: int, order: str) -> Tuple[np.ndarray, np.ndarray]:
    d = np.asarray(doc_ids, np.uint64).reshape(-1)
    v = np.asarray(values, np.float64).reshape(-1) + 0.0
    keep = d < np.uint64(nbits)
    d, v = d[keep], v[keep]
    o = np.lexsort((d, v if order == "ASC" else -v))   # last key first: value, then ascending document
    d, v = d[o], v[o]
    _, first = np.unique(d, return_index=True)
    first.sort()
    return d[first], v[first]


def variant_entries(layout: dict, variant_values: Sequence[float]) -> Tuple[np.ndarray, np.ndarray]:
    """The (document, value) entries of a bool or string_filter field read back by FacetStore.read_field ({"doc_ids",
    "offsets"}), each entry valued by its variant: variant_values[v] for the documents of variant v.  Entries before
    offsets[0] are in no variant and have no value."""
    off, docs = layout["offsets"].astype(np.int64), layout["doc_ids"]
    d = [docs[off[v]:off[v + 1]] for v in range(off.shape[0] - 1)]
    x = [np.full(off[v + 1] - off[v], float(variant_values[v])) for v in range(off.shape[0] - 1)]
    return (np.concatenate(d).astype(np.uint64) if d else np.zeros(0, np.uint64),
            np.concatenate(x) if x else np.zeros(0, np.float64))


def random_entries(rng: np.random.Generator, n: int, nbits: int) -> Tuple[np.ndarray, np.ndarray]:
    """n entries over documents [0, nbits + nbits // 8) (some dropped) with the awkward values: long runs of ties,
    -0.0 and +0.0, -inf and +inf, millisecond timestamps near 2^53, tiny and huge magnitudes; a tenth of them exact
    copies of earlier entries, and many documents with several values."""
    if n == 0:
        return np.zeros(0, np.uint64), np.zeros(0, np.float64)
    d = rng.integers(0, nbits + nbits // 8 + 1, size=n).astype(np.uint64)
    pick = rng.integers(0, 7, size=n)
    v = np.select([pick == 0, pick == 1, pick == 2, pick == 3, pick == 4, pick == 5],
                  [rng.integers(-5, 6, size=n).astype(np.float64),
                   np.where(rng.random(n) < 0.5, -0.0, 0.0),
                   np.where(rng.random(n) < 0.5, -np.inf, np.inf),
                   (2.0 ** 53 - rng.integers(0, 1000, size=n)) * np.where(rng.random(n) < 0.5, -1.0, 1.0),
                   rng.choice([5e-324, -5e-324, 1e308, -1e308, 1e-300], size=n),
                   rng.normal(0, 1e6, size=n)],
                  rng.normal(0, 1, size=n).round(2))
    dup = rng.random(n) < 0.1
    src = rng.integers(0, n, size=n)
    d[dup], v[dup] = d[src[dup]], v[src[dup]]
    return d, v
