"""Geopoint where-filter leaves, host side (no GPU): the f32 unit conversion of GeoSearchRadiusValue::to_meter
(types.rs:2159-2170), the Python-side validation of GeoPointField, and the two restatements the GPU tests compare
against: the chord form of the radius test against the trigonometric haversine, and PNPOLY against hand-checked
cases.  The restatements here are the ones tests/test_gpu_geo.py uses."""
import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib

R = _lib.OC_GEO_EARTH_RADIUS_M


# ---------------------------------------------------------------- restatements
def unit(lat, lon):
    la, lo = np.asarray(lat, np.float64) * (np.pi / 180.0), np.asarray(lon, np.float64) * (np.pi / 180.0)
    return np.stack([np.cos(la) * np.cos(lo), np.cos(la) * np.sin(lo), np.sin(la)], -1)


def haversine_m(lat1, lon1, lat2, lon2):
    """Great-circle distance in f64 on the sphere of radius R."""
    p1, p2 = np.radians(lat1), np.radians(lat2)
    a = np.sin((p2 - p1) / 2) ** 2 + np.cos(p1) * np.cos(p2) * np.sin(np.radians(np.asarray(lon2) - lon1) / 2) ** 2
    return 2 * R * np.arcsin(np.sqrt(np.minimum(a, 1.0)))


def chord_inside(lat, lon, clat, clon, r):
    """The device's test: |u_p - u_c|^2 <= 4 sin^2(r / 2R), every point inside once r / 2R >= pi / 2."""
    half = r / (2 * R)
    if half >= np.pi / 2:
        return np.ones(np.shape(lat), bool)
    d = unit(lat, lon) - unit(clat, clon)
    return (d * d).sum(-1) <= 4 * np.sin(half) ** 2


def pnpoly(vlat, vlon, lat, lon):
    """Even-odd crossing test in planar (lon, lat), edges (v[i-1], v[i]), in f64 with the device's op order."""
    x, y = np.asarray(lon, np.float64), np.asarray(lat, np.float64)
    inside = np.zeros(x.shape, bool)
    n = len(vlat)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(n):
            j = i - 1 if i else n - 1
            xi, yi, xj, yj = float(vlon[i]), float(vlat[i]), float(vlon[j]), float(vlat[j])
            cross = ((yi > y) != (yj > y)) & (x < (xj - xi) * (y - yi) / (yj - yi) + xi)
            inside ^= cross
    return inside


def docs_of(doc_ids, pred, nbits):
    """The any-point rule: documents (< nbits) with at least one point where pred holds."""
    d = np.asarray(doc_ids, np.uint64)
    return np.unique(d[pred & (d < nbits)])


# ---------------------------------------------------------------- to_meter
@pytest.mark.parametrize("unit_name,factor", [("cm", 0.01), ("m", 1.0), ("km", 1000.0), ("ft", 0.3048), ("yd", 0.9144),
                                              ("mi", 1609.344)])
def test_to_meter_is_f32(unit_name, factor):
    for v in (0.0, 1.0, 7.0, 10.0, 0.1, 123.456, 3.3e4):
        got = ob.geo_to_meter(v, unit_name)
        assert got == float(np.float32(np.float32(v) * np.float32(factor)))
        assert got == float(np.float32(got))   # an f32 value, widened
    assert ob.geo_to_meter(10, "km") == 10000.0 and ob.geo_to_meter(1, "mi") == float(np.float32(1609.344))
    assert ob.geo_to_meter(5) == 5.0   # default unit: m (types.rs:2176-2178)


def test_to_meter_differs_from_f64():
    # 7 mi: 7 x f32(1609.344) rounded to f32 is not the f64 product 11265.408
    assert ob.geo_to_meter(7, "mi") == float(np.float32(7 * np.float32(1609.344))) != 7 * 1609.344
    assert ob.geo_to_meter(0.3, "ft") != 0.3 * 0.3048
    with pytest.raises(ValueError):
        ob.geo_to_meter(1, "furlong")


# ---------------------------------------------------------------- Python-side validation (no call reaches the library)
@pytest.mark.parametrize("lat,lon", [(np.nan, 0), (0, np.nan), (90.5, 0), (-91, 0), (0, 180.01), (0, -181), (np.inf, 0)])
def test_field_refuses_bad_coordinates(lat, lon):
    with pytest.raises(ValueError, match="invalid coordinates"):
        ob.GeoPointField(None, 10, [1, 2], [10.0, lat], [20.0, lon])


def test_field_refuses_mismatched_lengths():
    with pytest.raises(ValueError):
        ob.GeoPointField(None, 10, [1, 2], [10.0], [20.0, 21.0])


def _unbound():
    g = object.__new__(ob.GeoPointField)
    g.ctx, g.nbits, g._h = None, 10, None
    return g


def test_queries_refuse_bad_input():
    g = _unbound()
    for lat, lon in [(np.nan, 0), (91, 0), (0, -180.5)]:
        with pytest.raises(ValueError, match="centre"):
            g.radius(lat, lon, 10)
    for v, u in [(-1, "m"), (np.nan, "km"), (np.inf, "m"), (1e38, "mi")]:   # 1e38 mi overflows f32 -> inf
        with pytest.raises(ValueError, match="radius"):
            g.radius(0, 0, v, u)
    with pytest.raises(ValueError, match="unit"):
        g.radius(0, 0, 1, "parsec")
    with pytest.raises(ValueError, match="vertices"):
        g.polygon([(0, 0), (1, 1)])
    with pytest.raises(ValueError, match="vertices"):
        g.polygon([(0, k * 1e-3) for k in range(_lib.OC_GEO_MAX_VERTICES + 1)])
    with pytest.raises(ValueError, match="vertex 1"):
        g.polygon([{"lat": 0, "lon": 0}, {"lat": np.nan, "lon": 1}, {"lat": 1, "lon": 1}])


# ---------------------------------------------------------------- the chord test is the haversine test
def test_chord_equals_haversine_away_from_the_boundary():
    rng = np.random.default_rng(1)
    n = 200_000
    lat1, lat2 = np.degrees(np.arcsin(rng.uniform(-1, 1, (2, n))))
    lon1, lon2 = rng.uniform(-180, 180, (2, n))
    d = haversine_m(lat1, lon1, lat2, lon2)
    # radii on both sides of d, at least 1e-6 relative (and 1 mm) away from it
    r = d * np.where(rng.random(n) < 0.5, 1 - rng.uniform(1e-6, 0.5, n), 1 + rng.uniform(1e-6, 0.5, n))
    r = np.where(np.abs(r - d) < 1e-3, d + 1e-3, r)
    for i in range(0, n, 20_000):   # per-query centres: evaluate pairwise
        sl = slice(i, i + 20_000)
        u, c = unit(lat1[sl], lon1[sl]), unit(lat2[sl], lon2[sl])
        half = r[sl] / (2 * R)
        chord = ((u - c) ** 2).sum(-1) <= np.where(half >= np.pi / 2, np.inf, 4 * np.sin(np.minimum(half, np.pi / 2)) ** 2)
        assert np.array_equal(chord, d[sl] <= r[sl])


def test_chord_special_radii():
    lat, lon = np.array([0.0, 0.0, 89.0, -90.0]), np.array([0.0, 180.0, 10.0, 0.0])
    assert chord_inside(lat, lon, 0.0, 0.0, 0.0).tolist() == [True, False, False, False]       # r = 0: the centre itself
    assert chord_inside(lat, lon, 0.0, 0.0, np.pi * R).all()                                   # r >= pi R: everything
    assert chord_inside(lat, lon, 0.0, 0.0, 20_100_000.0).all()
    assert chord_inside(lat, lon, 0.0, 0.0, 10_007_600.0).tolist() == [True, False, True, True]  # quarter circle ~10 007 543 m


# ---------------------------------------------------------------- PNPOLY, hand-checked
def test_pnpoly_unit_square():
    vlat, vlon = [0, 0, 1, 1], [0, 1, 1, 0]
    pts = {  # (lat, lon): inside
        (0.5, 0.5): True, (0.5, 1.5): False, (1.5, 0.5): False, (-0.5, 0.5): False, (0.5, -0.5): False,
        # edges and vertices: PNPOLY's half-open rule puts the bottom and left edges inside, top and right outside
        (0.0, 0.5): True, (0.5, 0.0): True, (1.0, 0.5): False, (0.5, 1.0): False,
        (0.0, 0.0): True, (0.0, 1.0): False, (1.0, 0.0): False, (1.0, 1.0): False,
    }
    lat, lon = np.array([p[0] for p in pts], float), np.array([p[1] for p in pts], float)
    assert pnpoly(vlat, vlon, lat, lon).tolist() == list(pts.values())
    # a repeated closing vertex adds a zero-length edge that crosses nothing
    assert pnpoly(vlat + [0], vlon + [0], lat, lon).tolist() == list(pts.values())


def test_pnpoly_concave_and_triangle():
    # a "C" shape open to the east: the notch is outside
    vlat = [0, 0, 1, 1, 3, 3, 4, 4]
    vlon = [0, 4, 4, 1, 1, 4, 4, 0]
    # (2, 1) lies on the notch's west edge, which is the east edge of the bar: outside, as every east edge
    lat, lon = np.array([0.5, 2.0, 2.0, 3.5, 2.0, 5.0]), np.array([2.0, 0.5, 2.0, 2.0, 1.0, 2.0])
    assert pnpoly(vlat, vlon, lat, lon).tolist() == [True, True, False, True, False, False]
    tri_lat, tri_lon = [0, 0, 10], [0, 10, 0]
    assert pnpoly(tri_lat, tri_lon, np.array([1.0, 6.0, 4.0]), np.array([1.0, 6.0, 5.0])).tolist() == [True, False, True]
    # vertex order (clockwise / counter-clockwise) does not matter
    assert pnpoly(tri_lat[::-1], tri_lon[::-1], np.array([1.0, 6.0, 4.0]), np.array([1.0, 6.0, 5.0])).tolist() == [True, False, True]


def test_any_point_rule():
    d = np.array([1, 1, 2, 3, 3, 12], np.uint64)
    pred = np.array([False, True, False, False, False, True])
    assert docs_of(d, pred, 10).tolist() == [1]          # 12 >= nbits is ignored
    assert docs_of(d, ~pred, 10).tolist() == [1, 2, 3]   # outside: doc 1 has a point on each side
