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

evaluate_where(...) restates calculate_filter + FilterContext::execute_filter (filter.rs:176-287, 344-392) with
device leaves: FacetStore.leaf for bool / number / date / string_filter fields, GeoPointField radius / polygon for
geopoint fields, and DeviceFilter and / or / not.  A document is in a leaf when at least one of its values passes.
  * A node is the AND of its field leaves, of each `and` child, of the OR of its `or` children and of NOT its `not`
    child.
  * A key of a node that is not a filter field of the index makes the whole node empty.  The keys are checked in
    order as the leaves are built, so a leaf after such a key (an invalid polygon, say) is never built.
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

import numpy as np

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


# ---------------------------------------------------------------- evaluation
class _Eval:
    """calculate_filter (filter.rs:176-287) over one index.  Every handle made while a tree is evaluated is kept in
    `owned` and closed when the evaluation ends, except the result."""

    def __init__(self, ctx, facets, geo_fields, nbits):
        self.ctx, self.facets, self.geo, self.nbits = ctx, facets, geo_fields, nbits
        self.owned: List[DeviceFilter] = []

    def evaluate(self, w: WhereFilter) -> DeviceFilter:
        try:
            res = self.node(w)
            self.owned.remove(res)
            return res
        finally:
            for f in self.owned:
                f.close()

    def keep(self, f: DeviceFilter) -> DeviceFilter:
        self.owned.append(f)
        return f

    def has(self, key) -> bool:
        return key in self.geo or (self.facets is not None and key in self.facets.fields)

    def leaf(self, key, flt) -> DeviceFilter:
        if key not in self.geo:
            return self.facets.leaf(key, flt)
        g = self.geo[key]
        if isinstance(flt, GeoRadius):
            return g.radius(flt.lat, flt.lon, flt.value, flt.unit, flt.inside)
        if isinstance(flt, GeoPolygon):
            return g.polygon(flt.coordinates, flt.inside)
        return DeviceFilter.from_ids(self.ctx, [], self.nbits)   # wrong kind for a geopoint field

    def fold(self, parts: List[DeviceFilter], op) -> DeviceFilter:
        acc = parts[0]
        for p in parts[1:]:
            acc = self.keep(op(acc, p))
        return acc

    def node(self, w: WhereFilter) -> DeviceFilter:
        empty = lambda: self.keep(DeviceFilter.from_ids(self.ctx, [], self.nbits))  # noqa: E731
        parts = []
        for k, flt in w.filter_on_fields:
            if not self.has(k):
                return empty()
            parts.append(self.keep(self.leaf(k, flt)))
        parts += [self.node(c) for c in w.and_ or []]
        if w.or_ is not None:
            if not w.or_:
                return empty()
            parts.append(self.fold([self.node(c) for c in w.or_], DeviceFilter.__or__))
        if w.not_ is not None:
            parts.append(self.keep(~self.node(w.not_)))
        return self.fold(parts, DeviceFilter.__and__) if parts else empty()


def evaluate_where(w: WhereFilter, facets: Optional[FacetStore], geo_fields: Mapping[str, GeoPointField], nbits: int,
                   uncommitted_deleted: Sequence[int] = (), ctx: Optional[Context] = None) -> Optional[DeviceFilter]:
    """FilterContext::execute_filter (filter.rs:344-392) over one index: None when nothing is filtered, else a
    DeviceFilter over [0, nbits).  `ctx` defaults to the context of the facet store or of a geopoint field."""
    if ctx is None:
        ctx = facets.ctx if facets is not None else next((g.ctx for g in geo_fields.values()), None)
    if ctx is None:
        raise ValueError("evaluate_where: no context (pass ctx= for an index without filter fields)")
    deleted = sorted({int(d) for d in uncommitted_deleted})
    if w.is_empty() and not deleted:
        return None
    live = None
    if deleted:
        dele = DeviceFilter.from_ids(ctx, deleted, nbits)
        try:
            live = ~dele
        finally:
            dele.close()
    if w.is_empty():
        return live
    tree = _Eval(ctx, facets, dict(geo_fields), int(nbits)).evaluate(w)
    if live is None:
        return tree
    try:
        return tree & live
    finally:
        tree.close()
        live.close()
