"""A vectorised, independent host evaluation of a parsed where tree (where.parse_where's output): the rules of
calculate_filter / execute_filter (filter.rs:176-287, 344-392) as tests/test_where_host.py's `host_where` states them,
over numpy masks instead of Python sets, so it reaches millions of documents.  It calls no library entry point and
shares no code with compile_where or the device's planner.

Fields, per name:
  ("bool", docs, values)        one entry per (document, bool)
  ("string", docs, keys)        one entry per (document, key); keys a numpy array of str
  ("number", docs, values)      one entry per (document, f64 value); also "date" (millisecond timestamps as f64)
  ("geo", docs, (lat, lon))     one entry per point, degrees (f64)
A document is in a leaf when at least one of its entries passes; entries with a document id >= nbits pass no leaf.

Leaves:
  * bool / string_filter: the entries equal to the value.  An unknown key is an empty leaf.
  * number / date: the f64 comparison of every value with the bound(s) widened to f64: -0.0 == +0.0, bounds of
    +-inf, gt / lt open ends, `between` with lo > hi empty.  The bound is the parser's (an integer bound that does not
    fit i32 was rounded to f32 once, test_where_host.py::test_int_to_f32_rounds_once).
  * polygon: test_geo_host.pnpoly (the device's op order, so equal bit for bit), on the points whose latitude lies in
    the polygon's [min, max) latitude span: no edge of the even-odd test can cross a point outside it.
  * radius: test_geo_host.haversine_m in f64 against the radius in metres (the f32 product of value and unit).  A
    point within 1e-9 relative of the boundary, and at least within 1e-8 m of it, is undecided: the device's chord test
    carries an absolute error of a few ulp of the unit sphere, some nanometres, which the floor covers for the smallest
    radii.  Radius >= pi R takes every point and radius 0 takes the points exactly at the centre.
  * the wrong kind of filter for a field: an empty leaf.
So every value is a pair of masks over [0, nbits): (certainly in, certainly out).  Without radius leaves, or with no
point in a radius band, they are complements.  And / Or / Not combine them by three-valued logic."""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np

from oramacore_b200.where import DateFilter, GeoPolygon, GeoRadius, NumberFilter, WhereFilter
from test_geo_host import R, haversine_m, pnpoly

RADIUS_BAND = 1e-9         # relative; the band of tests/test_gpu_geo.py::test_radius_against_haversine
RADIUS_BAND_FLOOR_M = 1e-8  # absolute, in metres: above the device's chord error (~ulp(1) x R)
UNIT_TO_METER = {"cm": 0.01, "m": 1.0, "km": 1000.0, "ft": 0.3048, "yd": 0.9144, "mi": 1609.344}

Masks = Tuple[np.ndarray, np.ndarray]   # (certainly in, certainly out), bool[nbits] each


def radius_m(flt: GeoRadius) -> float:
    """GeoSearchRadiusValue::to_meter: the value and the unit factor in f32, their product rounded to f32."""
    return float(np.float32(np.float32(flt.value) * np.float32(UNIT_TO_METER[flt.unit])))


def _bound(x) -> float:
    return float(x.value) if hasattr(x, "value") else float(x)   # I32 / F32 (numbers), int (dates)


def range_hits(flt, v: np.ndarray) -> np.ndarray:
    """The entries of a number / date field that the filter passes, compared in f64."""
    v = np.asarray(v, np.float64)
    if flt.op == "between":
        lo, hi = _bound(flt.value[0]), _bound(flt.value[1])
        return (v >= lo) & (v <= hi)
    b = _bound(flt.value)
    return {"eq": v == b, "gt": v > b, "gte": v >= b, "lt": v < b, "lte": v <= b}[flt.op]


def polygon_points(flt: GeoPolygon, lat: np.ndarray, lon: np.ndarray) -> np.ndarray:
    """PNPOLY of every point, evaluated on the points inside the polygon's latitude span only."""
    vlat = np.array([p[0] for p in flt.coordinates], np.float64)
    vlon = np.array([p[1] for p in flt.coordinates], np.float64)
    out = np.zeros(lat.shape, bool)
    sel = np.flatnonzero((lat >= vlat.min()) & (lat < vlat.max()))
    if sel.size:
        out[sel] = pnpoly(vlat, vlon, lat[sel], lon[sel])
    return out


def radius_points(flt: GeoRadius, lat: np.ndarray, lon: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """(certainly within the radius, certainly beyond it) per point."""
    r = radius_m(flt)
    if r >= np.pi * R:
        return np.ones(lat.shape, bool), np.zeros(lat.shape, bool)
    d = haversine_m(lat, lon, flt.lat, flt.lon)
    band = np.abs(d - r) <= max(RADIUS_BAND * r, RADIUS_BAND_FLOOR_M)
    sure_in = (d <= r) & ~band
    if r == 0.0:
        sure_in = (lat == flt.lat) & (lon == flt.lon)
    return sure_in, (d > r) & ~band


def _docs_mask(docs: np.ndarray, hit: np.ndarray, nbits: int) -> np.ndarray:
    m = np.zeros(nbits, bool)
    d = np.asarray(docs, np.int64)[hit]
    m[d[(d >= 0) & (d < nbits)]] = True
    return m


def _exact(m: np.ndarray) -> Masks:
    return m, ~m


def _empty(nbits: int) -> Masks:
    return _exact(np.zeros(nbits, bool))


def leaf(field, flt, nbits: int) -> Masks:
    kind, docs, vals = field
    docs = np.asarray(docs, np.int64)
    if kind == "bool" and isinstance(flt, bool):
        return _exact(_docs_mask(docs, np.asarray(vals, bool) == flt, nbits))
    if kind == "string" and isinstance(flt, str):
        return _exact(_docs_mask(docs, np.asarray(vals) == flt, nbits))
    if (kind, type(flt)) in (("number", NumberFilter), ("date", DateFilter)):
        return _exact(_docs_mask(docs, range_hits(flt, vals), nbits))
    if kind == "geo" and isinstance(flt, GeoPolygon):
        p_in = polygon_points(flt, *vals)
        return _exact(_docs_mask(docs, p_in if flt.inside else ~p_in, nbits))
    if kind == "geo" and isinstance(flt, GeoRadius):
        p_in, p_out = radius_points(flt, *vals)
        if not flt.inside:
            p_in, p_out = p_out, p_in
        # a document is in when one point is surely in, out when every point is surely out
        some_unsure = _docs_mask(docs, ~(p_in | p_out), nbits)
        sure_in = _docs_mask(docs, p_in, nbits)
        return sure_in, ~sure_in & ~some_unsure
    return _empty(nbits)


def _and(parts, nbits) -> Masks:
    t, f = np.ones(nbits, bool), np.zeros(nbits, bool)
    for a, b in parts:
        t &= a
        f |= b
    return t, f


def _or(parts, nbits) -> Masks:
    t, f = np.zeros(nbits, bool), np.ones(nbits, bool)
    for a, b in parts:
        t |= a
        f &= b
    return t, f


def node(w: WhereFilter, fields, nbits: int, cache=None) -> Masks:
    """calculate_filter: the AND of the node's field leaves, of each `and` child, of the OR of its `or` children and of
    NOT its `not` child.  An unknown key empties the node; `or: []` and a node with no parts are empty.  `cache` (a
    dict, or None) keeps each distinct leaf's masks for the next time the tree names it."""
    parts = []
    for k, flt in w.filter_on_fields:
        if k not in fields:
            return _empty(nbits)
        if cache is None:
            parts.append(leaf(fields[k], flt, nbits))
            continue
        key = (k, type(flt), flt)
        if key not in cache:
            cache[key] = leaf(fields[k], flt, nbits)
        parts.append(cache[key])
    parts += [node(c, fields, nbits, cache) for c in w.and_ or []]
    if w.or_ is not None:
        if not w.or_:
            return _empty(nbits)
        parts.append(_or([node(c, fields, nbits, cache) for c in w.or_], nbits))
    if w.not_ is not None:
        t, f = node(w.not_, fields, nbits, cache)
        parts.append((f, t))
    if not parts:
        return _empty(nbits)
    return _and(parts, nbits)


def where_masks(w: WhereFilter, fields, nbits: int, deleted=(), cache=None) -> Optional[Masks]:
    """execute_filter: None when nothing is filtered, else (certainly in, certainly out) of tree AND NOT(deletes)."""
    dead = np.zeros(nbits, bool)
    d = np.asarray(list(deleted), np.int64)
    dead[d[(d >= 0) & (d < nbits)]] = True
    if w.is_empty():
        return None if len(d) == 0 else _exact(~dead)
    t, f = node(w, fields, nbits, cache)
    return t & ~dead, f | dead


def pack(mask: np.ndarray) -> np.ndarray:
    """bool[nbits] -> the uint64 words of a device bitmap, padding bits clear."""
    words = (mask.shape[0] + 63) // 64
    b = np.packbits(np.asarray(mask, bool), bitorder="little")
    out = np.zeros(words * 8, np.uint8)
    out[:b.shape[0]] = b
    return out.view(np.uint64)


def unpack(bits: np.ndarray, nbits: int) -> np.ndarray:
    return np.unpackbits(np.asarray(bits, np.uint64).view(np.uint8), bitorder="little")[:nbits].astype(bool)


def where_spec(w: WhereFilter, fields, nbits: int, deleted=(), cache=None) -> Optional[np.ndarray]:
    """The bitmap of w: None when nothing is filtered.  Every document must be decided (no radius band in the way)."""
    m = where_masks(w, fields, nbits, deleted, cache)
    if m is None:
        return None
    t, f = m
    undecided = ~(t | f)
    assert not undecided.any(), f"{int(undecided.sum())} documents on a radius boundary"
    return pack(t)


def from_host_fields(fields) -> dict:
    """test_where_host's field layout (bool {doc: {bools}}, string {doc: [keys]}, number / date (docs, values), geo
    (docs, lat, lon)) in this module's."""
    out = {}
    for name, (kind, data) in fields.items():
        if kind in ("bool", "string"):
            e = [(d, x) for d, xs in data.items() for x in xs]
            docs = np.array([d for d, _ in e], np.int64)
            vals = np.array([x for _, x in e], bool if kind == "bool" else object)
            out[name] = (kind, docs, vals)
        elif kind == "geo":
            d, la, lo = data
            out[name] = (kind, np.asarray(d, np.int64), (np.asarray(la, np.float64), np.asarray(lo, np.float64)))
        else:
            d, v = data
            out[name] = (kind, np.asarray(d, np.int64), np.asarray(v, np.float64))
    return out
