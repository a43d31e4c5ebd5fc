"""Host checks of the where-clause: the parser against serde's rules (types.rs:758-767, 1173-1231, 1861-1866,
2068-2221), the number-bound claim against a line-by-line restatement of number_filter_to_i64_filter_op /
number_filter_to_f64_filter_op (number_field.rs:555-642), and the tree rules of calculate_filter / execute_filter
(filter.rs:176-287, 344-392) on a restatement over Python sets.  The restatement (`host_where`) is also the oracle of
tests/test_gpu_where.py."""
import math

import numpy as np
import pytest

from oramacore_b200.where import (F32, I32, DateFilter, GeoPolygon, GeoRadius, NumberFilter, WhereFilter, parse_date_ms,
                                  parse_where, where_keys)
from test_geo_host import pnpoly

EPS = 2.0 ** -52   # f64::EPSILON
I64_MAX, I64_MIN = (1 << 63) - 1, -(1 << 63)


def f32(x):
    return float(np.float32(x))


# ---------------------------------------------------------------- parser
@pytest.mark.parametrize("json_value, expected", [
    (5, I32(5)), (-5, I32(-5)), (2**31 - 1, I32(2**31 - 1)), (-2**31, I32(-2**31)),
    (2**31, F32(2147483648.0)), (3000000000, F32(3000000000.0)), (5.0, F32(5.0)), (0.1, F32(f32(0.1))),
    (16777217, I32(16777217)), (2**33 + 1, F32(2.0**33)),
    (2**53 + 1, F32(f32(2.0**53))), (1e39, F32(math.inf)), (-0.0, F32(-0.0)),
])
def test_number_bounds(json_value, expected):
    got = parse_where({"n": {"eq": json_value}}).filter_on_fields[0][1]
    assert got == NumberFilter("eq", expected)
    if isinstance(expected, F32):
        assert math.copysign(1, got.value.value) == math.copysign(1, expected.value)


def test_int_to_f32_rounds_once():
    # an integer rounded straight to f32, as `u64 as f32` does, not through f64 first
    x = (1 << 60) + (1 << 36) + 1          # just above a tie at f32 precision: rounds up
    got = parse_where({"n": {"gt": x}}).filter_on_fields[0][1].value.value
    assert got == float((1 << 60) + (1 << 37))
    assert f32(float(x)) == float(1 << 60)  # the double-rounded value differs


@pytest.mark.parametrize("s, ms", [
    ("2023-01-01T00:00:00Z", 1672531200000), ("2023-01-01T01:00:00+01:00", 1672531200000),
    ("2022-12-31T19:00:00-05:00", 1672531200000), ("2023-01-01t00:00:00z", 1672531200000),
    ("2023-01-01T00:00:00.1239Z", 1672531200123), ("1970-01-01T00:00:00Z", 0),
    ("1969-12-31T23:59:59.9995Z", -1), ("1969-12-31T23:59:59Z", -1000), ("1900-03-01T00:00:00Z", -2203891200000),
    ("2000-02-29T12:00:00.5Z", 951825600500),
])
def test_dates(s, ms):
    assert parse_date_ms(s) == ms
    assert parse_where({"d": {"gte": s}}).filter_on_fields[0][1] == DateFilter("gte", ms)


@pytest.mark.parametrize("s", ["2023-01-01", "2023-02-30T00:00:00Z", "2023-01-01T00:00:00", "01/02/2023",
                               "2023-01-01T24:00:00Z", "2023-01-01T00:00:00+24:00"])
def test_dates_not_rfc3339_are_no_date(s):
    # not a DateFilter; as a Number it fails too, so the value is not a Filter at all
    with pytest.raises(ValueError):
        parse_where({"d": {"eq": s}})


def test_filter_kinds_and_order():
    w = parse_where({"a": True, "b": "x", "c": {"between": [1, 2.5]}, "d": {"lt": "2023-01-01T00:00:00Z"},
                     "e": {"polygon": {"coordinates": [{"lat": 1, "lon": 2}, {"lat": 3, "lon": 4}, {"lat": 5, "lon": 0.1}],
                                       "inside": False}},
                     "f": {"radius": {"coordinates": {"lat": 0.1, "lon": 2}, "unit": "km", "value": 1.5, "extra": 1}}})
    assert w.filter_on_fields == [
        ("a", True), ("b", "x"), ("c", NumberFilter("between", (I32(1), F32(2.5)))), ("d", DateFilter("lt", 1672531200000)),
        ("e", GeoPolygon(((1.0, 2.0), (3.0, 4.0), (5.0, f32(0.1))), False)), ("f", GeoRadius(f32(0.1), 2.0, 1.5, "km", True))]
    assert w.and_ is None and w.or_ is None and w.not_ is None


def test_combinators():
    assert parse_where({"not": {"gt": 5}}).filter_on_fields == [("not", NumberFilter("gt", I32(5)))]
    w = parse_where({"and": [{"a": True}], "or": [], "not": {"b": "x"}})
    assert w.and_ == [WhereFilter([("a", True)])] and w.or_ == [] and w.not_ == WhereFilter([("b", "x")])
    assert parse_where({"and": [{}]}).and_ == [WhereFilter()]
    assert parse_where({"not": {}}).not_ == WhereFilter()
    assert parse_where({"and": {"gt": 1}}).filter_on_fields == [("and", NumberFilter("gt", I32(1)))]
    assert parse_where({}).is_empty() and parse_where({"or": [], "and": []}).is_empty()
    assert not parse_where({"not": {}}).is_empty()


@pytest.mark.parametrize("bad", [
    {"a": [1]}, {"a": [{}]}, {"and": {"b": True}}, {"or": {"b": True}}, {"not": [{"b": True}]}, {"a": {"gt": 5, "lt": 9}},
    {"a": None}, {"a": 1}, {"a": {"eq": True}}, {"a": {"eq": "text"}}, {"a": {"between": [1]}}, {"a": {"between": [1, 2, 3]}},
    {"a": {"ne": 1}}, {"a": {"b": {"gt": 1}}}, {"a": {"radius": {"coordinates": {"lat": 1}, "value": 1}}},
    {"a": {"radius": {"coordinates": {"lat": 1, "lon": 2}, "value": 1, "unit": "au"}}},
    {"a": {"polygon": {"coordinates": [], "inside": "yes"}}}, [1], "x",
])
def test_refused(bad):
    with pytest.raises(ValueError):
        parse_where(bad)


def test_where_keys_order():
    w = parse_where({"a": True, "and": [{"b": "x", "or": [{"c": "y"}]}], "or": [{"d": "z"}], "not": {"e": "w"}})
    assert where_keys(w) == ["a", "b", "c", "d", "e"]


# ---------------------------------------------------------------- the number claim (number_field.rs:555-642)
def _as_i64(x):   # Rust `f64 as i64`: truncation, saturating
    return I64_MAX if x >= 2.0**63 else I64_MIN if x <= -2.0**63 else int(x)


def i64_op(op, n):
    """number_filter_to_i64_filter_op, line by line; None = no i64 interpretation."""
    if op == "between":
        lo = n[0].value if isinstance(n[0], I32) else _as_i64(math.ceil(n[0].value) if math.isfinite(n[0].value) else n[0].value)
        hi = n[1].value if isinstance(n[1], I32) else _as_i64(math.floor(n[1].value) if math.isfinite(n[1].value) else n[1].value)
        return None if lo > hi else ("between", (lo, hi))
    if isinstance(n, I32):
        return (op, n.value)
    f = n.value
    ceil = _as_i64(math.ceil(f) if math.isfinite(f) else f)
    floor = _as_i64(math.floor(f) if math.isfinite(f) else f)
    if op == "eq":
        r = _as_i64(f)
        return ("eq", r) if abs(float(r) - f) < EPS else None
    if op == "gt":
        return ("gt", ceil) if abs(float(ceil) - f) < EPS else ("gte", ceil)
    if op == "gte":
        return ("gte", ceil)
    if op == "lt":
        return ("lt", floor) if abs(float(floor) - f) < EPS else ("lte", floor)
    return ("lte", floor)


def apply_op(o, v):
    op, b = o
    return {"eq": lambda: v == b, "gt": lambda: v > b, "gte": lambda: v >= b, "lt": lambda: v < b, "lte": lambda: v <= b,
            "between": lambda: (v >= b[0]) & (v <= b[1])}[op]()


def interval(op, n, v):
    """The rule the device applies (FacetStore.leaf / oc_filter_facet_range): the f64 comparison with the bound(s)."""
    return apply_op((op, NumberFilter(op, n).bounds()), v)


def _bounds(rng):
    specials = [0.0, -0.0, 5.0, -5.0, 0.5, -0.5, 2.0**24, 2.0**53, -2.0**53, 2.0**63, -2.0**63, 1e30, -1e30, math.inf,
                -math.inf, 2.0**-149, -2.0**-149, 2.0**-126, -2.0**-126, 2.0**-53, -2.0**-60, 2.0**-52, 1 - 2.0**-24,
                f32(0.1), f32(-0.1), 16777217.0, 123456.5]
    out = [F32(f32(x)) for x in specials]
    out += [F32(f32(x)) for x in rng.standard_normal(60) * 10.0 ** rng.integers(-40, 20, 60)]
    out += [F32(f32(float(x))) for x in rng.integers(-2**40, 2**40, 20)]
    out += [I32(int(x)) for x in [0, 1, -1, 5, 2**31 - 1, -2**31]] + [I32(int(x)) for x in rng.integers(-2**31, 2**31, 20)]
    return out


def test_number_claim_i64_values():
    """For i64 values |v| <= 2^53 the reference's i64 op selects what the f64 interval selects, except for a nonzero F32
    bound with |b| < 2^-52: the EPSILON test then treats the bound as 0, so eq / gt / lt differ at v = 0 and only
    there.  The device keeps the interval (documented deviation)."""
    rng = np.random.default_rng(7)
    vals = np.concatenate([rng.integers(-2**53, 2**53 + 1, 3000), rng.integers(-20, 21, 41), [0, 1, -1, 2**53, -2**53, 5, -5],
                           rng.integers(-2**31, 2**31, 500)]).astype(np.int64)
    vals_obj = [int(x) for x in vals]
    bounds = _bounds(rng)
    diffs = set()
    for op in ("eq", "gt", "gte", "lt", "lte"):
        for n in bounds:
            o = i64_op(op, n)
            ref = np.array([o is not None and bool(apply_op(o, v)) for v in vals_obj])
            ours = interval(op, n, vals.astype(np.float64))
            for v in vals[ref != ours]:
                diffs.add((op, n, int(v)))
    pairs = [(a, b) for a in bounds for b in bounds[::3]]
    for a, b in pairs:
        o = i64_op("between", (a, b))
        ref = np.array([o is not None and bool(apply_op(o, v)) for v in vals_obj])
        ours = interval("between", (a, b), vals.astype(np.float64))
        assert np.array_equal(ref, ours), (a, b)
    expected = {(op, n, 0) for op in ("eq", "gt", "lt") for n in bounds
                if isinstance(n, F32) and 0 < abs(n.value) < EPS
                and ((op == "eq") or (op == "gt" and n.value < 0) or (op == "lt" and n.value > 0))}
    assert diffs == expected
    assert len(expected) >= 6   # the exception is exercised, not vacuous


def test_number_claim_f64_values():
    """The f64 store uses number_filter_to_f64_filter_op: the interval itself, including -0.0 == 0.0, subnormals, inf."""
    rng = np.random.default_rng(8)
    vals = np.concatenate([rng.standard_normal(2000) * 10.0 ** rng.integers(-45, 40, 2000),
                           [0.0, -0.0, 5.0, math.inf, -math.inf, 2.0**-149, -2.0**-149, f32(0.1), 0.1]])
    for op in ("eq", "gt", "gte", "lt", "lte"):
        for n in _bounds(rng):
            b = float(n.value)
            ref = apply_op((op, b), vals)
            assert np.array_equal(ref, interval(op, n, vals)), (op, n)
    assert not interval("eq", F32(f32(0.1)), np.array([0.1]))[0]        # {"eq": 0.1} does not match a stored f64 0.1
    assert interval("eq", F32(-0.0), np.array([0.0]))[0]
    assert not interval("between", (I32(5), I32(4)), np.array([4.0, 4.5, 5.0])).any()


# ---------------------------------------------------------------- tree rules on a host restatement
def host_leaf(field, flt, nbits):
    """A leaf as a set of documents < nbits.  `field` = (kind, data): bool {doc: {bools}}, string {doc: [keys]},
    number / date (docs, f64 values), geo (docs, lat, lon)."""
    kind, data = field
    if kind == "bool" and isinstance(flt, bool):
        docs = {d for d, bs in data.items() if flt in bs}
    elif kind == "string" and isinstance(flt, str):
        docs = {d for d, ks in data.items() if flt in ks}
    elif (kind, type(flt)) in (("number", NumberFilter), ("date", DateFilter)):
        d, v = data
        hit = apply_op((flt.op, flt.bounds()), v)
        docs = set(int(x) for x in d[hit])
    elif kind == "geo" and isinstance(flt, GeoPolygon):
        d, lat, lon = data
        vl, vo = np.array([p[0] for p in flt.coordinates]), np.array([p[1] for p in flt.coordinates])
        hit = pnpoly(vl, vo, lat, lon)
        hit = hit if flt.inside else ~hit
        docs = set(int(x) for x in d[hit])
    else:
        docs = set()
    return {x for x in docs if x < nbits}


def host_node(w, fields, nbits):
    """calculate_filter (filter.rs:176-287)."""
    parts = []
    for k, flt in w.filter_on_fields:
        if k not in fields:
            return set()
        parts.append(host_leaf(fields[k], flt, nbits))
    parts += [host_node(c, fields, nbits) for c in w.and_ or []]
    if w.or_ is not None:
        if not w.or_:
            return set()
        parts.append(set().union(*[host_node(c, fields, nbits) for c in w.or_]))
    if w.not_ is not None:
        parts.append(set(range(nbits)) - host_node(w.not_, fields, nbits))
    if not parts:
        return set()
    return set.intersection(*parts)


def host_where(w, fields, nbits, deleted=()):
    """execute_filter (filter.rs:344-392): None, or the set of documents that pass."""
    live = set(range(nbits)) - set(deleted)
    if w.is_empty():
        return None if not deleted else live
    return host_node(w, fields, nbits) & live


FIELDS = {"b": ("bool", {0: {True}, 1: {False}, 2: {True, False}}), "s": ("string", {0: ["x"], 1: ["y"], 3: ["x", "y"]}),
          "n": ("number", (np.array([0, 1, 2, 3, 3]), np.array([1.0, 2.0, 3.0, 4.0, -1.0])))}


# (where, deleted, the documents of host_where over FIELDS and 5 documents); also checked against tests/where_spec.py
TREE_RULE_CASES = [
    ({}, (), None), ({}, (1,), {0, 2, 3, 4}), ({"or": []}, (), None), ({"and": [], "or": []}, (2,), {0, 1, 3, 4}),
    ({"b": True}, (), {0, 2}), ({"b": True}, (2,), {0}), ({"b": False, "s": "x"}, (), set()),
    ({"unknown": True, "b": True}, (), set()), ({"b": True, "unknown": True}, (), set()),
    ({"or": [{"b": False}, {"unknown": True}]}, (), {1, 2}), ({"not": {"unknown": "z"}}, (), {0, 1, 2, 3, 4}),
    ({"and": [{}]}, (), set()), ({"not": {}}, (), {0, 1, 2, 3, 4}), ({"b": True, "or": []}, (), set()),
    ({"s": "y", "and": [{"n": {"gt": 1}}], "or": [{"b": False}, {"n": {"lt": 0}}], "not": {"s": "x"}}, (), {1}),
    ({"n": {"between": [3, 2]}}, (), set()), ({"n": True}, (), set()), ({"s": "nope"}, (), set()),
]


@pytest.mark.parametrize("where, deleted, expected", TREE_RULE_CASES)
def test_tree_rules(where, deleted, expected):
    assert host_where(parse_where(where), FIELDS, 5, deleted) == expected
