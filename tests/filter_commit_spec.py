"""The filter-field commit (oc_facets_commit_ex, oc_geo_field_commit_ex) restated in numpy.

A field's layout is one sorted list of entries:
  * bool / string_filter ("csr"):  offsets (n_variants + 1) and the documents of each variant, ascending;
  * number / date ("number"):      (value, doc) pairs, ascending value (-0.0 before +0.0), then ascending doc;
  * geopoint ("geo"):              (doc, lat, lon) triples, ascending doc; a document's points in the order they came.
Pending ops, in call order:
  ("ins", field, doc, payload, unique)  payload: the variant, the value, or (lat, lon); unique: set semantics
  ("clr", field, doc)                   every value of doc in field
  ("del", doc)                          every value of doc in every field
A removal applies to the committed entries and to the earlier inserts, never to a later insert.

The loader's per-kind rules (IndexLoader.apply) map onto these ops:
  * FilterBool replaces the document's value: ("clr", field, doc) then a unique insert of the variant;
  * FilterBool2 adds to the document's set of bools: unique inserts;
  * FilterNumber(2), FilterString(2), FilterDate(2) append: plain inserts (a repeated value is listed twice);
  * FilterGeoPoint2 appends its points; DeleteDocuments removes every value: ("del", doc)."""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np


def order_key(v: float) -> int:
    """The value order of a number field: a double's bits as an unsigned integer of the same order."""
    b = int(np.float64(v).view(np.uint64))
    return (~b & (2**64 - 1)) if b >> 63 else b | (1 << 63)


def empty(kind: str, n_variants: int = 0):
    if kind == "csr":
        return {"offsets": np.zeros(n_variants + 1, np.uint64), "docs": np.zeros(0, np.uint64)}
    if kind == "number":
        return {"values": np.zeros(0, np.float64), "docs": np.zeros(0, np.uint64)}
    return {"docs": np.zeros(0, np.uint64), "lat": np.zeros(0, np.float64), "lon": np.zeros(0, np.float64)}


def _entries(kind: str, lay) -> List[Tuple[tuple, tuple]]:
    """(key, payload) of each committed entry, in layout order."""
    if kind == "csr":
        off, d = lay["offsets"], lay["docs"]
        return [((v, int(d[i])), (int(d[i]),)) for v in range(len(off) - 1) for i in range(int(off[v]), int(off[v + 1]))]
    if kind == "number":
        return [((order_key(x), int(d)), (float(x), int(d))) for x, d in zip(lay["values"], lay["docs"])]
    return [((int(d), 0), (int(d), float(a), float(o))) for d, a, o in zip(lay["docs"], lay["lat"], lay["lon"])]


def commit(kind: str, field: int, prev, ops: Sequence[tuple], n_variants: int = 0):
    """The next layout of one field from the previous one and the pending ops of its handle, in call order.
    n_variants: a csr field's variant count after the commit (new keys append)."""
    last_kill: Dict[int, int] = {}
    for s, op in enumerate(ops):
        if op[0] == "del" or (op[0] == "clr" and op[1] == field):
            last_kill[op[-1] if op[0] == "del" else op[2]] = s
    survivors, seen = [], set()
    for s, op in enumerate(ops):
        if op[0] != "ins" or op[1] != field or last_kill.get(op[2], -1) > s:
            continue
        doc, pay = op[2], op[3]
        key = (pay, doc) if kind == "csr" else (order_key(pay), doc) if kind == "number" else (doc, 0)
        if key in seen and op[4]:
            continue
        seen.add(key)
        payload = (doc,) if kind == "csr" else (float(pay), doc) if kind == "number" else (doc, float(pay[0]), float(pay[1]))
        survivors.append((key, s, payload, op[4]))
    kept = [(k, p) for k, p in _entries(kind, prev) if k[1 if kind == "csr" else (1 if kind == "number" else 0)] not in last_kill]
    kept_keys = {k for k, _ in kept}
    new = [(k, p) for k, s, p, u in sorted(survivors, key=lambda t: (t[0], t[1])) if not (u and k in kept_keys)]
    merged = sorted(kept + new, key=lambda kp: kp[0])   # stable: committed entries before pending ones of equal key
    if kind == "csr":
        nv = max(n_variants, len(prev["offsets"]) - 1)
        counts = np.bincount(np.asarray([k[0] for k, _ in merged], np.int64), minlength=nv) if merged else np.zeros(nv, np.int64)
        off = np.zeros(nv + 1, np.uint64)
        off[1:] = np.cumsum(counts)
        return {"offsets": off, "docs": np.asarray([p[0] for _, p in merged], np.uint64)}
    if kind == "number":
        return {"values": np.asarray([p[0] for _, p in merged], np.float64), "docs": np.asarray([p[1] for _, p in merged], np.uint64)}
    return {"docs": np.asarray([p[0] for _, p in merged], np.uint64), "lat": np.asarray([p[1] for _, p in merged], np.float64),
            "lon": np.asarray([p[2] for _, p in merged], np.float64)}


def rebuild(kind: str, field: int, ops: Sequence[tuple], n_variants: int = 0):
    """The layout a from-scratch build gives after every op so far: a per-document record of the field's values, replayed
    as the loader keeps it, then laid out as FacetStore.add_* / GeoPointField lay it out."""
    per_doc: Dict[int, list] = {}
    for op in ops:
        if op[0] == "del":
            per_doc.pop(op[1], None)
        elif op[0] == "clr" and op[1] == field:
            per_doc.pop(op[2], None)
        elif op[0] == "ins" and op[1] == field:
            vals = per_doc.setdefault(op[2], [])
            if not (op[4] and op[3] in vals):
                vals.append(op[3])
    if kind == "csr":
        nv = n_variants
        lists = [sorted(d for d, vs in per_doc.items() for x in vs if x == v) for v in range(nv)]
        off = np.zeros(nv + 1, np.uint64)
        off[1:] = np.cumsum([len(l) for l in lists])
        return {"offsets": off, "docs": np.asarray([d for l in lists for d in l], np.uint64)}
    if kind == "number":
        pairs = sorted(((x, d) for d, vs in per_doc.items() for x in vs), key=lambda p: (order_key(p[0]), p[1]))
        return {"values": np.asarray([p[0] for p in pairs], np.float64), "docs": np.asarray([p[1] for p in pairs], np.uint64)}
    pts = [(d, p) for d in sorted(per_doc) for p in per_doc[d]]
    return {"docs": np.asarray([d for d, _ in pts], np.uint64), "lat": np.asarray([p[0] for _, p in pts], np.float64),
            "lon": np.asarray([p[1] for _, p in pts], np.float64)}


def same_up_to_ties(kind: str, a, b) -> bool:
    """Equal layouts, up to the order inside a run of equal keys (a set, for every consumer)."""
    if kind == "csr":
        return np.array_equal(a["offsets"], b["offsets"]) and np.array_equal(a["docs"], b["docs"])
    if kind == "number":
        ka = sorted(zip([order_key(x) for x in a["values"]], a["docs"].tolist()))
        kb = sorted(zip([order_key(x) for x in b["values"]], b["docs"].tolist()))
        return ka == kb and np.array_equal(a["values"], b["values"])
    return all(np.array_equal(a[k], b[k]) for k in ("docs", "lat", "lon"))
