"""The reference's `where` clause: parsed as serde parses it, evaluated on the device.

parse_where(obj) restates the deserialisation of `WhereFilter` (types.rs:1173-1231) over a JSON object (as `json.loads`
gives it).  Every value of the map is tried, in this order, as
  * a `Filter` (untagged, types.rs:758-767), itself tried as Date, Number, Bool, String, GeoPoint;
  * a list of where-filters;
  * one where-filter;
and then `"and"` / `"or"` take a list, `"not"` takes a where-filter that is not a Filter, and any other key takes a
Filter.  Any other pairing is an error.  So `{"not": {"gt": 5}}` is a number filter on a field named `not`.
  * Number (types.rs:1861-1866): a JSON integer that fits i32 is I32, any other JSON number is F32 (rounded to f32, so
    `5.0` is F32(5.0) and `0.1` is f32(0.1)); a bool is not a number.
  * NumberFilter / DateFilter (types.rs:2068-2147): a map of exactly one of eq / gt / gte / lt / lte / between, the
    last taking a list of exactly two bounds.
  * A date bound is an RFC 3339 string, kept as its millisecond timestamp, floored as chrono's `timestamp_millis`
    does (also before 1970).  The reference parses with `dateparser`, which accepts more formats; those are refused
    here (assumption).
  * GeoSearchFilter (types.rs:2175-2221): {"radius": {coordinates, unit = "m", value, inside = true}} or
    {"polygon": {coordinates, inside = true}}, a GeoPoint being {"lat", "lon"}; unknown keys are ignored.

compile_where(...) restates calculate_filter + FilterContext::execute_filter (filter.rs:176-287, 344-392) as a postfix
program (include/oramacore_b200.h "where programs") over device leaves: variant and range leaves of bool / number /
date / string_filter fields, radius and polygon leaves of geopoint fields, and And / Or / Not.  A search call evaluates
it itself (oc_search_params.q_where); evaluate_where(...) evaluates it into a DeviceFilter with one call
(oc_filter_from_where).  A document is in a leaf when at least one of its values passes.
  * A node is the AND of its field leaves, of each `and` child, of the OR of its `or` children and of NOT its `not`
    child.
  * A key of a node that is not a filter field of the index makes the whole node empty.  The keys are checked in
    order as the leaves are compiled, so a leaf after such a key (an invalid polygon, say) is never checked.
  * A node with `or: []`, and a node with no parts at all (the `{}` of `{"and": [{}]}`), is empty.
  * At the top level an empty filter (`is_empty`, types.rs:1282-1287) means no filter: None, or NOT(deletes) when
    there are uncommitted deletes.  Otherwise the result is the tree AND NOT(uncommitted deletes).
Assumptions and deliberate differences (the oramacore_fields source is not available):
  * f64 comparisons follow IEEE, so -0.0 == 0.0; `between` with min > max is empty.
  * Number leaves compare every stored value with the bound widened to f64.  The reference converts F32 bounds for its
    integer store with ceil / floor and an EPSILON test; for integers |v| <= 2^53 that is the same selection, except
    that a nonzero F32 bound with |b| < 2^-52 counts as 0 there, so eq / gt / lt by such a bound differ at v = 0
    (tests/test_where_host.py shows this is the only difference).
  * The reference raises FilterFieldNotFound only when the search found nothing (search.rs:435-449); IndexLoader
    .where_filter checks the keys before any device work, so a clause naming an unknown field is always refused.
  * Bitmaps are exact, where the reference's sets may be Bloom-backed."""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, field
from typing import Dict, List, Mapping, Optional, Sequence, Tuple, Union

import ctypes as C

import numpy as np

from . import _lib
from ._lib import check
from .engine import Context, DeviceFilter, FacetStore, GeoPointField
from .types import FilterFieldNotFound

NUMBER_OPS = ("eq", "gt", "gte", "lt", "lte", "between")


@dataclass(frozen=True)
class I32:
    value: int


@dataclass(frozen=True)
class F32:
    value: float   # an f32 value, held exactly as a Python float


Number = Union[I32, F32]


@dataclass(frozen=True)
class NumberFilter:
    op: str
    value: Union[Number, Tuple[Number, Number]]

    def bounds(self):
        """The bound(s) widened to f64 (number_to_f64, number_field.rs:637-642)."""
        if self.op == "between":
            return tuple(float(x.value) for x in self.value)
        return float(self.value.value)


@dataclass(frozen=True)
class DateFilter:
    op: str
    value: Union[int, Tuple[int, int]]   # millisecond timestamps

    def bounds(self):
        if self.op == "between":
            return tuple(float(x) for x in self.value)
        return float(self.value)


@dataclass(frozen=True)
class GeoRadius:
    lat: float
    lon: float
    value: float   # f32
    unit: str = "m"
    inside: bool = True


@dataclass(frozen=True)
class GeoPolygon:
    coordinates: Tuple[Tuple[float, float], ...]   # (lat, lon), f32 values
    inside: bool = True


Filter = Union[DateFilter, NumberFilter, bool, str, GeoRadius, GeoPolygon]


@dataclass
class WhereFilter:
    filter_on_fields: List[Tuple[str, Filter]] = field(default_factory=list)
    and_: Optional[List["WhereFilter"]] = None
    or_: Optional[List["WhereFilter"]] = None
    not_: Optional["WhereFilter"] = None

    def is_empty(self) -> bool:
        return not self.filter_on_fields and not self.and_ and not self.or_ and self.not_ is None


class _NoMatch(ValueError):
    pass


# ---------------------------------------------------------------- parsing
def _int_to_f32(x: int) -> float:
    """`x as f32` for an integer that serde_json holds as u64 / i64: rounded once, to nearest even."""
    if not -(1 << 63) <= x < (1 << 64):
        return _float_to_f32(float(x))   # beyond u64 / i64 serde_json holds an f64
    a, sh = abs(x), max(abs(x).bit_length() - 24, 0)
    if sh:
        q, r = divmod(a, 1 << sh)
        half = 1 << (sh - 1)
        if r > half or (r == half and q & 1):
            q += 1
        a = q << sh
    return float(np.float32(math.copysign(a, x)))


def _float_to_f32(x: float) -> float:
    with np.errstate(over="ignore"):
        return float(np.float32(x))


def _number(x) -> Number:
    if isinstance(x, bool) or not isinstance(x, (int, float)):
        raise _NoMatch(f"not a number: {x!r}")
    if isinstance(x, int):
        return I32(x) if -(1 << 31) <= x < (1 << 31) else F32(_int_to_f32(x))
    return F32(_float_to_f32(x))


_RFC3339 = re.compile(r"(\d{4})-(\d{2})-(\d{2})[Tt ](\d{2}):(\d{2}):(\d{2})(?:\.(\d+))?(?:([Zz])|([+-])(\d{2}):(\d{2}))")


def _days_from_civil(y: int, m: int, d: int) -> int:
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    return era * 146097 + yoe * 365 + yoe // 4 - yoe // 100 + doy - 719468


def parse_date_ms(s) -> int:
    """An RFC 3339 date-time as OramaDate::as_i64: milliseconds since the epoch, floored (timestamp_millis)."""
    m = _RFC3339.fullmatch(s) if isinstance(s, str) else None
    if m is None:
        raise _NoMatch(f"not an RFC 3339 date: {s!r}")
    y, mo, d, hh, mi, ss = (int(m.group(i)) for i in range(1, 7))
    leap = y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)
    mdays = [31, 29 if leap else 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31]
    if not (1 <= mo <= 12 and 1 <= d <= mdays[mo - 1] and hh <= 23 and mi <= 59 and ss <= 60):
        raise _NoMatch(f"not a valid date: {s!r}")
    off = 0
    if m.group(9):
        oh, om = int(m.group(10)), int(m.group(11))
        if oh > 23 or om > 59:
            raise _NoMatch(f"not a valid offset: {s!r}")
        off = (oh * 60 + om) * 60 * (1 if m.group(9) == "+" else -1)
    frac_ms = int((m.group(7) or "").ljust(3, "0")[:3])
    secs = _days_from_civil(y, mo, d) * 86400 + hh * 3600 + mi * 60 + ss - off
    return secs * 1000 + frac_ms


def _tagged(obj, parse_value):
    """An externally tagged NumberFilter / DateFilter: a map of exactly one known op."""
    if not isinstance(obj, Mapping) or len(obj) != 1:
        raise _NoMatch("not a map of one op")
    (op, v), = obj.items()
    if op not in NUMBER_OPS:
        raise _NoMatch(f"unknown op {op!r}")
    if op == "between":
        if not isinstance(v, (list, tuple)) or len(v) != 2:
            raise _NoMatch("between takes two bounds")
        return op, (parse_value(v[0]), parse_value(v[1]))
    return op, parse_value(v)


def _geo_point(p) -> Tuple[float, float]:
    if not isinstance(p, Mapping) or "lat" not in p or "lon" not in p:
        raise _NoMatch("a GeoPoint is {lat, lon}")
    lat, lon = _number(p["lat"]), _number(p["lon"])
    return _float_to_f32(lat.value), _float_to_f32(lon.value)


def _inside(d) -> bool:
    v = d.get("inside", True)
    if not isinstance(v, bool):
        raise _NoMatch("inside is a bool")
    return v


def _geo(obj) -> Union[GeoRadius, GeoPolygon]:
    if not isinstance(obj, Mapping) or len(obj) != 1:
        raise _NoMatch("not a map of one geo op")
    (op, d), = obj.items()
    if not isinstance(d, Mapping):
        raise _NoMatch("a geo filter is a map")
    if op == "radius":
        if "coordinates" not in d or "value" not in d:
            raise _NoMatch("radius needs coordinates and value")
        lat, lon = _geo_point(d["coordinates"])
        unit = d.get("unit", "m")
        if unit not in ("cm", "m", "km", "ft", "yd", "mi"):
            raise _NoMatch(f"unknown unit {unit!r}")
        return GeoRadius(lat, lon, _float_to_f32(_number(d["value"]).value), unit, _inside(d))
    if op == "polygon":
        if not isinstance(d.get("coordinates"), list):
            raise _NoMatch("polygon needs a list of coordinates")
        return GeoPolygon(tuple(_geo_point(p) for p in d["coordinates"]), _inside(d))
    raise _NoMatch(f"unknown geo op {op!r}")


def parse_filter(v) -> Filter:
    """`Filter` (untagged): the first of Date, Number, Bool, String, GeoPoint that accepts `v`."""
    for attempt in (lambda: DateFilter(*_tagged(v, parse_date_ms)), lambda: NumberFilter(*_tagged(v, _number))):
        try:
            return attempt()
        except _NoMatch:
            pass
    if isinstance(v, (bool, str)):
        return v
    return _geo(v)


def parse_where(obj) -> WhereFilter:
    """A JSON where-clause -> WhereFilter, or ValueError where serde refuses it."""
    if not isinstance(obj, Mapping):
        raise ValueError(f"a where filter is a map, not {obj!r}")
    w = WhereFilter()
    for key, value in obj.items():
        kind, parsed = _value(key, value)
        if key in ("and", "or") and kind == "list":
            setattr(w, key + "_", parsed)
        elif key == "not" and kind == "where":
            w.not_ = parsed
        elif kind == "filter":
            w.filter_on_fields.append((key, parsed))
        else:
            raise ValueError(f"Invalid where filter for key {key}: {value!r}")
    return w


def _value(key, value):
    try:
        return "filter", parse_filter(value)
    except _NoMatch:
        pass
    if isinstance(value, list):
        try:
            return "list", [parse_where(x) for x in value]
        except ValueError:
            pass
    if isinstance(value, Mapping):
        try:
            return "where", parse_where(value)
        except ValueError:
            pass
    raise ValueError(f"where filter key {key!r}: {value!r} is neither a filter nor a where filter")


def where_keys(w: WhereFilter) -> List[str]:
    """get_all_keys (types.rs:1289-1310): the keys of the node, then of its and / or / not children."""
    keys = [k for k, _ in w.filter_on_fields]
    for c in (w.and_ or []) + (w.or_ or []) + ([w.not_] if w.not_ is not None else []):
        keys.extend(where_keys(c))
    return keys


def check_where_keys(w: WhereFilter, filter_fields_per_index: Sequence[Sequence[str]]) -> None:
    """search.rs:435-449: every key must be a filter field of at least one index, else FilterFieldNotFound(key)."""
    for k in where_keys(w):
        if not any(k in fs for fs in filter_fields_per_index):
            raise FilterFieldNotFound(k)


# ---------------------------------------------------------------- programs (oc_search_params.q_where)
def _node(b, w: WhereFilter):
    """The tree rules of calculate_filter (filter.rs:176-287) over the builder `b` (_Compile):
    the AND of the node's field leaves, of each `and` child, of the OR of its `or` children and of NOT its `not` child.
    A key that is not a filter field makes the node empty (leaves after it are never compiled); `or: []` and a node with
    no parts are empty."""
    parts = []
    for k, flt in w.filter_on_fields:
        if not b.has(k):
            return b.empty()
        parts.append(b.leaf(k, flt))
    parts += [_node(b, c) for c in w.and_ or []]
    if w.or_ is not None:
        if not w.or_:
            return b.empty()
        parts.append(b.or_([_node(b, c) for c in w.or_]))
    if w.not_ is not None:
        parts.append(b.not_(_node(b, w.not_)))
    return b.and_(parts) if parts else b.empty()


def _top_level(w: WhereFilter, has_deletes: bool) -> str:
    """execute_filter's top level (filter.rs:344-392): "none" (no filter), "live" (NOT deletes), "tree" or
    "tree_and_live"."""
    if w.is_empty():
        return "live" if has_deletes else "none"
    return "tree_and_live" if has_deletes else "tree"


@dataclass
class WhereProgram:
    """A where-clause compiled to the library's postfix program (include/oramacore_b200.h "where programs"): `nodes` are
    (op, field, arg, a, b, c, src, vertices) tuples, vertices = (lats, lons) for a polygon else None.  `keep` holds the
    handles the program points at (the deletes handle), `nbits` the DocumentId space of its leaves."""
    nbits: int
    nodes: List[tuple] = field(default_factory=list)
    keep: list = field(default_factory=list)


# Operands of one And / Or node that compile_where emits.  A list of parts costs up to _NARY - 1 stack slots above its
# deepest part, so 8 lets four nested wide lists fit the OC_WHERE_MAX_DEPTH = 32 slots, at one more node per 7 parts
# beyond the first 8 (a 300-part list: 300 leaves and 43 And / Or nodes).  Lists of up to 8 parts stay one node.
_NARY = 8


def _n(op, field_=0, arg=0, a=0.0, b=0.0, c=0.0, src=None, verts=None):
    return (op, field_, arg, a, b, c, src, verts)


class _Compile:
    """The builder `_node` runs over one index: which keys are filter fields, and the node list that pushes each value
    of the tree (a leaf, the empty set, And / Or / Not)."""

    def __init__(self, facets, geo_fields):
        self.facets, self.geo = facets, geo_fields

    def has(self, key) -> bool:
        return key in self.geo or (self.facets is not None and key in self.facets.fields)

    def leaf(self, key, flt):
        if key not in self.geo:
            return self.facet_leaf(key, flt)
        g = self.geo[key]
        if isinstance(flt, GeoRadius):
            return self.radius(g, flt)
        if isinstance(flt, GeoPolygon):
            return self.polygon(g, flt)
        return self.empty()   # wrong kind for a geopoint field

    def empty(self):
        return [_n(_lib.OC_WHERE_NONE)]

    def facet_leaf(self, key, flt):
        spec = self.facets.leaf_args(key, flt)
        if spec is None:
            return self.empty()
        src = self.facets._h.value
        if spec[0] == "variant":
            return [_n(_lib.OC_WHERE_VARIANT, spec[1], spec[2], src=src)]
        return [_n(_lib.OC_WHERE_RANGE, spec[1], spec[4], spec[2], spec[3], src=src)]

    def radius(self, g, flt):
        lat, lon, r = g.radius_args(flt.lat, flt.lon, flt.value, flt.unit)
        return [_n(_lib.OC_WHERE_GEO_RADIUS, 0, int(bool(flt.inside)), lat, lon, r, src=g._h.value)]

    def polygon(self, g, flt):
        la, lo = g.polygon_args(flt.coordinates)
        return [_n(_lib.OC_WHERE_GEO_POLYGON, 0, int(bool(flt.inside)), src=g._h.value, verts=(la, lo))]

    def _nary(self, parts, op):
        """One And / Or of `parts`, over at most _NARY operands per node: a wider list is folded, the first _NARY parts
        and then the running value with the next _NARY - 1, so it takes at most _NARY - 1 stack slots more than its
        deepest part.  Pushing every part before one node refused any list of more than OC_WHERE_MAX_DEPTH parts
        (tests/test_gpu_where_oracle.py::test_wide_and_or caught it)."""
        if len(parts) == 1:
            return parts[0]
        head, rest = parts[:_NARY], parts[_NARY:]
        out = [x for p in head for x in p] + [_n(op, arg=len(head))]
        for i in range(0, len(rest), _NARY - 1):
            chunk = rest[i:i + _NARY - 1]
            out += [x for p in chunk for x in p] + [_n(op, arg=len(chunk) + 1)]
        return out

    def and_(self, parts):
        return self._nary(parts, _lib.OC_WHERE_AND)

    def or_(self, parts):
        return self._nary(parts, _lib.OC_WHERE_OR)

    def not_(self, x):
        return x + [_n(_lib.OC_WHERE_NOT)]


def compile_where(w: WhereFilter, facets: Optional[FacetStore], geo_fields: Mapping[str, GeoPointField], nbits: int,
                  live: Optional[DeviceFilter] = None) -> Optional[WhereProgram]:
    """execute_filter's program over one index: None when nothing is filtered.  `live` is the NOT(uncommitted deletes)
    handle (None without deletes), passed as a FILTER node; leaves are checked as FacetStore.leaf_args and
    GeoPointField.radius_args / polygon_args check them."""
    top = _top_level(w, live is not None)
    if top == "none":
        return None
    prog = WhereProgram(int(nbits))
    if top != "live":
        prog.nodes = _node(_Compile(facets, dict(geo_fields)), w)
    if live is not None:
        prog.keep.append(live)
        prog.nodes = prog.nodes + [_n(_lib.OC_WHERE_FILTER, src=live._h.value)]
        if top == "tree_and_live":
            prog.nodes.append(_n(_lib.OC_WHERE_AND, arg=2))
    return prog


def pack_programs(programs: Sequence[Optional[WhereProgram]]):
    """The oc_where of a batch (query b: programs[b], None = unfiltered) and the arrays it points into."""
    progs = [p for p in programs if p is not None]
    if not progs:
        raise ValueError("pack_programs: no program")
    nbits = progs[0].nbits
    offs, nodes, vlat, vlon, keep = [0], [], [], [], []
    for p in programs:
        if p is not None:
            if p.nbits != nbits:
                raise ValueError(f"where programs over {p.nbits} and {nbits} documents in one batch")
            keep.append(p)
            for (op, fl, arg, a, b, c, src, verts) in p.nodes:
                first, nv = 0, 0
                if verts is not None:
                    first, nv = len(vlat), len(verts[0])
                    vlat.extend(verts[0]); vlon.extend(verts[1])
                nodes.append(_lib.WhereNode(op, fl, arg, first, nv, a, b, c, src))
        offs.append(len(nodes))
    off_a = np.asarray(offs, np.uint32)
    node_a = (_lib.WhereNode * max(len(nodes), 1))(*nodes)
    la, lo = np.asarray(vlat, np.float64), np.asarray(vlon, np.float64)
    w = _lib.Where(nbits, off_a.ctypes.data, C.cast(node_a, C.c_void_p).value, la.ctypes.data if len(la) else None,
                   lo.ctypes.data if len(lo) else None)
    return w, [off_a, node_a, la, lo, keep]


def filter_from_program(ctx: Context, prog: WhereProgram) -> DeviceFilter:
    """oc_filter_from_where: the program's bitmap as an ordinary handle, in one call."""
    w, keep = pack_programs([prog])
    h = C.c_void_p()
    check(_lib.lib().oc_filter_from_where(ctx._h, C.byref(w), 0, C.byref(h)))
    nbits = prog.nbits
    if len(prog.nodes) == 1 and prog.nodes[0][0] == _lib.OC_WHERE_FILTER:
        nbits = prog.keep[0].nbits   # a lone handle is taken as it is
    return DeviceFilter(ctx, h, nbits)


def evaluate_where(w: WhereFilter, facets: Optional[FacetStore], geo_fields: Mapping[str, GeoPointField], nbits: int,
                   uncommitted_deleted: Sequence[int] = (), ctx: Optional[Context] = None) -> Optional[DeviceFilter]:
    """FilterContext::execute_filter (filter.rs:344-392) over one index: None when nothing is filtered, else a
    DeviceFilter over [0, nbits), the program of compile_where evaluated in one call.  The NOT(uncommitted deletes)
    handle is built for this call and closed, unless it is the result.  `ctx` defaults to the context of the facet store
    or of a geopoint field."""
    if ctx is None:
        ctx = facets.ctx if facets is not None else next((g.ctx for g in geo_fields.values()), None)
    if ctx is None:
        raise ValueError("evaluate_where: no context (pass ctx= for an index without filter fields)")
    deleted = sorted({int(d) for d in uncommitted_deleted})
    top = _top_level(w, bool(deleted))
    if top == "none":
        return None
    live = None
    if deleted:
        dele = DeviceFilter.from_ids(ctx, deleted, nbits)
        try:
            live = ~dele
        finally:
            dele.close()
    if top == "live":
        return live
    try:
        return filter_from_program(ctx, compile_where(w, facets, geo_fields, nbits, live))
    finally:
        if live is not None:
            live.close()
