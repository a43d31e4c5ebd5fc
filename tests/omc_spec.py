"""The OMC store's commit rule (oc_omc_commit_ex) and the index-level OMC rule it serves, restated in numpy.

Store (include/oramacore_b200.h, "OMC store"): a version is (doc ascending, mult f32).  Queued ops are ("set", doc,
mult) and ("delete", doc), applied in call order at the next commit; the last op for a document wins, a set writes the
entry and a delete removes it.

Index (read/index/mod.rs:604-627, 1566-1580, 1720-1739): Index2 appends (doc, omc) to an uncommitted log when omc is
not None; a search sees get_all_omc = the committed map with the log applied over it, last writer wins; commit merges
the log into the committed map, then removes every uncommitted delete from it."""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np


def commit(doc: np.ndarray, mult: np.ndarray, ops: Sequence[tuple]) -> Tuple[np.ndarray, np.ndarray]:
    """The next version: a stable sort of the ops by document, the last op per document, one merge with (doc, mult)."""
    doc = np.asarray(doc, np.uint64)
    mult = np.asarray(mult, np.float32)
    if not len(ops):
        return doc.copy(), mult.copy()
    q_doc = np.asarray([o[1] for o in ops], np.uint64)
    q_set = np.asarray([o[0] == "set" for o in ops], bool)
    q_mult = np.asarray([o[2] if o[0] == "set" else 0.0 for o in ops], np.float32)
    order = np.argsort(q_doc, kind="stable")
    b_doc, b_set, b_mult = q_doc[order], q_set[order], q_mult[order]
    last = np.ones(b_doc.shape[0], bool)
    last[:-1] = b_doc[1:] != b_doc[:-1]
    b_doc, b_set, b_mult = b_doc[last], b_set[last], b_mult[last]
    keep_a = ~np.isin(doc, b_doc)
    out_doc = np.concatenate([doc[keep_a], b_doc[b_set]])
    out_mult = np.concatenate([mult[keep_a], b_mult[b_set]])
    o = np.argsort(out_doc, kind="stable")
    return out_doc[o], out_mult[o]


def replay(ops: Sequence[tuple], start: Dict[int, float] = None) -> Dict[int, np.float32]:
    """The same rule as a dict replayed op by op."""
    m = {} if start is None else dict(start)
    for o in ops:
        if o[0] == "set":
            m[int(o[1])] = np.float32(o[2])
        else:
            m.pop(int(o[1]), None)
    return m


def as_arrays(m: Dict[int, float]) -> Tuple[np.ndarray, np.ndarray]:
    ks = sorted(m)
    return np.asarray(ks, np.uint64), np.asarray([m[k] for k in ks], np.float32)


class IndexOmc:
    """The reference's OMC state of one index: omc_committed, omc_uncommitted and uncommitted_deleted_documents."""

    def __init__(self):
        self.committed: Dict[int, np.float32] = {}
        self.log: List[Tuple[int, np.float32]] = []
        self.deleted: set = set()

    def index2(self, doc: int, omc) -> None:
        if omc is not None:
            self.log.append((int(doc), np.float32(omc)))

    def delete(self, docs) -> None:
        self.deleted |= {int(d) for d in docs}

    def all_omc(self) -> Dict[int, np.float32]:
        m = dict(self.committed)
        for d, x in self.log:
            m[d] = x
        return m

    def commit(self) -> None:
        self.committed = self.all_omc()
        for d in self.deleted:
            self.committed.pop(d, None)
        self.log, self.deleted = [], set()


def random_ops(rng: np.random.Generator, n: int, n_docs: int, p_delete: float = 0.25) -> List[tuple]:
    """n random ops over documents [0, n_docs), multipliers of a few exact and fractional kinds."""
    vals = np.asarray([0.5, 2.0, 3.0, 1.25, 0.1, 7.75, -1.5, 0.0], np.float32)
    out = []
    for _ in range(n):
        d = int(rng.integers(0, n_docs))
        if rng.random() < p_delete:
            out.append(("delete", d))
        else:
            out.append(("set", d, float(vals[rng.integers(0, vals.shape[0])] if rng.random() < 0.5 else np.float32(rng.random() * 4))))
    return out
