"""Geopoint where-filter leaves on the GPU (oc_geo_field_*, oc_filter_geo_radius, oc_filter_geo_polygon) against
(1) the reference's own answers (src/tests/geosearch.rs:8-471), driven through IndexLoader op streams with
FilterGeoPoint2 values, deletes, commits and a re-insert, and (2) numpy restatements: an f64 haversine for radius
leaves (equal sets except for points within 1e-9 relative of the boundary) and PNPOLY with the device's op order for
polygon leaves (bit-identical), both under the any-point rule.  Also: a geo leaf combined with id leaves gives searches
byte-identical to the same bitmap passed as filter_bits, and every refused call creates nothing."""
import ctypes as C

import numpy as np
import pytest

import oramacore_b200 as ob
from oramacore_b200 import _lib
from oramacore_b200.hostindex import tokenize
from oramacore_b200.loader import IndexLoader
from oramacore_b200.types import MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR
from test_geo_host import docs_of, haversine_m, pnpoly
from test_gpu_pins import N, _inputs, _tsc, corpus  # noqa: F401  (corpus: fixture)

pytestmark = pytest.mark.gpu


def _bits_to_ids(bits, nbits):
    return np.flatnonzero(np.unpackbits(bits.view(np.uint8), bitorder="little")[:nbits]).astype(np.uint64)


def _leaf_ids(f):
    try:
        return _bits_to_ids(f.read(), f.nbits)
    finally:
        f.close()


# ---------------------------------------------------------------- the reference's answers (geosearch.rs)
class Collection:
    """One index with a string field "name" and a geopoint field "location", fed through IndexLoader.  External ids map
    to DocumentIds as in the reference: every insert takes the next id, so a re-insert is a new document.  This
    library's loader publishes inserts at commit; the reference's searches see them at once, so each scenario
    commits its inserts before searching and keeps the reference's order of deletes and commits otherwise."""

    def __init__(self, ctx):
        self.ctx, self.ops, self.ids, self.next, self.pending = ctx, [], {}, 1, set()
        self.ld = self._loader()

    def _loader(self):
        return IndexLoader(self.ctx, ["name"], geopoint_fields=["location"])

    def insert(self, docs):
        for ext, name, loc in docs:
            d, self.next = self.next, self.next + 1
            self.ids[ext] = d
            toks = tokenize(name)
            terms = {}
            for i, t in enumerate(toks):
                terms.setdefault(t, {"exact_positions": [], "positions": []})["exact_positions"].append(i)
            pts = [{"lat": la, "lon": lo} for la, lo in (loc if isinstance(loc, list) else [loc])]
            geo = {"Plain": pts[0]} if not isinstance(loc, list) else {"Array": pts}
            self._apply({"type": "Index", "doc_id": d, "indexed_values": [
                {"type": "ScoreString2", "field": "name", "field_length": len(toks), "terms": terms},
                {"type": "FilterGeoPoint2", "field": "location", "value": geo}]})

    def delete(self, exts):
        ds = [self.ids.pop(e) for e in exts]
        self._apply({"type": "DeleteDocuments", "doc_ids": ds})
        self.pending.update(ds)

    def _apply(self, op):
        self.ops.append(op)
        self.ld.apply(op)

    def commit(self):
        self.ld.commit()
        self.pending.clear()

    def publish(self):
        """Make the inserts searchable (string snapshot + field handles) while the deletes stay uncommitted."""
        self.ld.strs.commit()
        self.ld.refresh_facets()

    def reload(self):
        """A new reader over everything committed so far: the op stream replayed into a fresh loader."""
        self.ld.close()
        self.ld = self._loader()
        self.ld.apply_all(self.ops)
        self.ld.commit()

    def search(self, term, lat, lon, value, unit="km", inside=True):
        """The empty / given term under the geo leaf AND NOT(uncommitted deletes) (execute_filter, filter.rs:344-392)."""
        leaf = self.ld.geo["location"].radius(lat, lon, value, unit, inside)
        dele = ob.DeviceFilter.from_ids(self.ctx, sorted(self.pending), leaf.nbits)
        live = ~dele
        f = leaf & live
        try:
            hits = self.ld.context().execute_batch(ob.TokenScoreParams(mode=MODE_FULLTEXT, limit_hint=10, device_filter=f),
                                                   self.ld.resolve([term]))[0]
        finally:
            for x in (leaf, dele, live, f):
                x.close()
        back = {d: e for e, d in self.ids.items()}
        return hits.count, [back[int(d)] for d in hits.doc_ids]

    def close(self):
        self.ld.close()


@pytest.fixture
def coll(gpu_ctx):
    c = Collection(gpu_ctx)
    yield c
    c.close()


TWO_FAR = [("1", "T", (9.0814233, 45.2623823)), ("2", "T", (9.0979028, 45.1995182))]
Q_FAR = (9.1418481, 45.2324096, 10)
TWO_NEAR = [("1", "A", (10.0, 20.0)), ("2", "B", (10.1, 20.1))]
Q_NEAR = (10.05, 20.05, 10)


def test_geosearch(coll):   # :8-65
    coll.insert(TWO_FAR)
    coll.commit()
    assert coll.search("", *Q_FAR)[0] == 2


def test_geosearch_commit(coll):   # :67-139
    coll.insert(TWO_FAR)
    coll.commit()
    assert coll.search("", *Q_FAR)[0] == 2
    coll.commit()
    coll.reload()
    assert coll.search("", *Q_FAR)[0] == 2


def test_add_delete_search_no_commit(coll):   # :141-198
    coll.insert(TWO_NEAR)
    coll.delete(["1"])
    coll.publish()
    count, hits = coll.search("", *Q_NEAR)
    assert count == 1 and hits == ["2"]


def test_add_delete_commit_reload_search(coll):   # :200-271
    coll.insert(TWO_NEAR)
    coll.delete(["1"])
    coll.commit()
    coll.reload()
    count, hits = coll.search("", *Q_NEAR)
    assert count == 1 and hits == ["2"]


def test_add_commit_delete_search_no_commit(coll):   # :273-331
    coll.insert(TWO_NEAR)
    coll.commit()
    coll.delete(["1"])
    count, hits = coll.search("", *Q_NEAR)
    assert count == 1 and hits == ["2"]
    # the geo handle still holds document 1 until the next commit: only NOT(uncommitted deletes) removes it
    assert _leaf_ids(coll.ld.geo["location"].radius(*Q_NEAR, unit="km")).tolist() == [1, 2]


def test_add_commit_delete_commit_reload_search(coll):   # :333-403
    coll.insert(TWO_NEAR)
    coll.commit()
    coll.delete(["1"])
    coll.commit()
    assert _leaf_ids(coll.ld.geo["location"].radius(*Q_NEAR, unit="km")).tolist() == [2]
    coll.reload()
    count, hits = coll.search("", *Q_NEAR)
    assert count == 1 and hits == ["2"]


def test_add_delete_add_again_search(coll):   # :405-473
    coll.insert([("1", "Tommaso", (10.0, 20.0))])
    coll.delete(["1"])
    coll.insert([("1", "Tommaso", (10.0, 20.0))])
    coll.commit()
    count, hits = coll.search("Tommaso", 10.0, 20.0, 1)
    assert count == 1 and hits == ["1"] and coll.ids["1"] == 2


def test_array_values_and_outside(coll):
    # GeoPointIndexedValue::Array: a document with a point near Rome and one in Paris is inside both radii, and
    # outside both as well (each leaf only needs one point)
    coll.insert([("rome", "x", (41.9028, 12.4964)), ("both", "x", [(41.9028, 12.4964), (48.8566, 2.3522)]),
                 ("paris", "x", (48.8566, 2.3522))])
    coll.commit()
    g = coll.ld.geo["location"]
    name = {d: e for e, d in coll.ids.items()}
    ids = lambda f: sorted(name[int(d)] for d in _leaf_ids(f))  # noqa: E731
    assert ids(g.radius(41.9, 12.5, 50, "km")) == ["both", "rome"]
    assert ids(g.radius(48.85, 2.35, 50, "km")) == ["both", "paris"]
    assert ids(g.radius(41.9, 12.5, 50, "km", inside=False)) == ["both", "paris"]
    assert ids(g.polygon([(40, 10), (40, 15), (44, 15), (44, 10)])) == ["both", "rome"]
    assert ids(g.polygon([(40, 10), (40, 15), (44, 15), (44, 10)], inside=False)) == ["both", "paris"]
    coll.delete(["both"])
    coll.commit()
    assert ids(coll.ld.geo["location"].radius(41.9, 12.5, 50, "km")) == ["rome"]


# ---------------------------------------------------------------- radius leaves against an f64 haversine
NBITS = 300_000
DUP = (float(np.float32(12.345678)), float(np.float32(-98.7654321)))   # f32 values: a centre that hits them exactly


@pytest.fixture(scope="module")
def points(gpu_ctx):
    """~180 K points: uniform on the sphere, tight clusters, the poles, lon +-180, exact duplicates, documents with
    several points, sparse ids and ids >= nbits."""
    rng = np.random.default_rng(7)
    lat = [np.degrees(np.arcsin(rng.uniform(-1, 1, 150_000)))]
    lon = [rng.uniform(-180, 180, 150_000)]
    for clat, clon in [(45.0, 9.0), (-33.9, 151.2), (0.0, 179.9995), (64.1, -21.9)]:   # clusters of ~1 km
        lat.append(clat + rng.normal(0, 0.005, 8000)); lon.append(np.clip(clon + rng.normal(0, 0.005, 8000), -180, 180))
    lat.append(np.array([90.0, 90.0, 90.0, -90.0, -90.0])); lon.append(np.array([0.0, 77.0, -180.0, 180.0, 12.0]))
    lat.append(rng.uniform(-80, 80, 200)); lon.append(np.where(rng.random(200) < 0.5, -180.0, 180.0))
    lat.append(np.full(6, DUP[0])); lon.append(np.full(6, DUP[1]))   # duplicates, also a radius-0 centre below
    lat, lon = np.concatenate(lat), np.concatenate(lon)
    lat = np.clip(lat, -90, 90)
    n = lat.shape[0]
    # documents: sparse ids, ~1/8 of them with 2-4 points, a few ids >= nbits
    n_docs = n * 7 // 8
    doc_of_doc = np.sort(rng.choice(NBITS - 100, n_docs, replace=False)).astype(np.uint64) + 1
    docs = np.concatenate([doc_of_doc, doc_of_doc[rng.integers(0, n_docs, n - n_docs)]])
    docs[rng.choice(n, 50, replace=False)] = NBITS + rng.integers(0, 1000, 50).astype(np.uint64)
    perm = rng.permutation(n)   # the field sorts by document id itself
    lat, lon, docs = lat[perm], lon[perm], docs[perm]
    g = ob.GeoPointField(gpu_ctx, NBITS, docs, lat, lon)
    yield lat, lon, docs, g
    g.close()


CENTRES = [(90.0, 0.0), (-90.0, 37.0), (12.5, 180.0), (-33.0, -180.0), (45.0, 9.0), DUP,
           (0.0, 179.9995)]


@pytest.mark.parametrize("radius", [0.0, 1.0, 10_000.0, 1_000_000.0, 20_100_000.0])
@pytest.mark.parametrize("inside", [True, False], ids=["inside", "outside"])
def test_radius_against_haversine(points, radius, inside):
    lat, lon, docs, g = points
    rng = np.random.default_rng(int(radius) % 1000 + 3)
    centres = CENTRES + [(float(rng.uniform(-90, 90)), float(rng.uniform(-180, 180))) for _ in range(3)]
    band_total = 0
    for clat, clon in centres:
        flat, flon = float(np.float32(clat)), float(np.float32(clon))   # API values are f32, widened
        d = haversine_m(lat, lon, flat, flon)
        band = np.abs(d - radius) <= 1e-9 * max(radius, 1.0)
        band_total += int(band.sum())
        pred = (d <= radius) if inside else (d > radius)
        exp = set(docs_of(docs, pred, NBITS).tolist())
        got = set(_leaf_ids(g.radius(clat, clon, radius, "m", inside)).tolist())
        # documents whose answer may differ: a point in the band and no point that decides without the band
        sure = set(docs_of(docs, pred & ~band, NBITS).tolist())
        unsure = set(docs_of(docs, band, NBITS).tolist()) - sure
        assert got - unsure == exp - unsure, (clat, clon, sorted((got ^ exp) - unsure)[:10])
        if radius >= 20_000_000:
            assert got == (set(docs_of(docs, np.ones(len(docs), bool), NBITS).tolist()) if inside else set())
    # the poles, the radius-0 duplicates and nothing else of consequence sit on the boundary
    assert band_total <= 64, band_total


def test_radius_zero_keeps_the_exact_point(points):
    lat, lon, docs, g = points
    dup = (lat == DUP[0]) & (lon == DUP[1])
    assert dup.sum() == 6
    # boundary included: radius 0 takes exactly the documents of the points at the centre
    assert np.array_equal(_leaf_ids(g.radius(*DUP, 0.0)), docs_of(docs, dup, NBITS))
    # an f64 centre is narrowed to the API's f32 first: 12.345678 is not the stored f64 point 12.345678
    assert float(np.float32(12.345678)) != 12.345678


# ---------------------------------------------------------------- polygon leaves: bit-identical to PNPOLY
def _f32(a):
    return np.asarray(a, np.float32).astype(np.float64)


def _star(n, clat, clon, r1, r2, rot=0.0):
    a = np.linspace(0, 2 * np.pi, 2 * n, endpoint=False) + rot
    r = np.where(np.arange(2 * n) % 2 == 0, r1, r2)
    return _f32(clat + r * np.sin(a)), _f32(clon + r * np.cos(a))


def _blob(n, rng, clat, clon, r):
    a = np.sort(rng.uniform(0, 2 * np.pi, n))
    rr = r * (0.6 + 0.4 * rng.random(n))
    return _f32(np.clip(clat + rr * np.sin(a), -90, 90)), _f32(np.clip(clon + rr * np.cos(a), -180, 180))


POLYGONS = {
    "triangle": (_f32([0.0, 0.0, 10.0]), _f32([0.0, 10.0, 0.0])),
    "thin_triangle": (_f32([44.9, 45.0, 45.1]), _f32([8.9, 9.2, 8.95])),
    "star": _star(5, 45.0, 9.0, 0.02, 0.008),
    "star_closed": tuple(np.append(v, v[0]) for v in _star(7, -33.9, 151.2, 0.05, 0.01, 0.3)),
    "square_at_antimeridian": (_f32([-10.0, -10.0, 10.0, 10.0]), _f32([170.0, 180.0, 180.0, 170.0])),
    "blob_1000": _blob(1000, np.random.default_rng(11), 20.0, -40.0, 60.0),
}


@pytest.fixture(scope="module")
def poly_points(gpu_ctx):
    """Random points around every polygon plus each polygon's vertices, edge midpoints, points at vertex latitudes and
    points a few ulp off the vertices."""
    rng = np.random.default_rng(13)
    lat, lon = [np.degrees(np.arcsin(rng.uniform(-1, 1, 50_000)))], [rng.uniform(-180, 180, 50_000)]
    for vlat, vlon in POLYGONS.values():
        lo_lat, hi_lat, lo_lon, hi_lon = vlat.min(), vlat.max(), vlon.min(), vlon.max()
        m = 0.1 * max(hi_lat - lo_lat, hi_lon - lo_lon)
        lat.append(np.clip(rng.uniform(lo_lat - m, hi_lat + m, 20_000), -90, 90))
        lon.append(np.clip(rng.uniform(lo_lon - m, hi_lon + m, 20_000), -180, 180))
        nxt = np.roll(np.arange(len(vlat)), -1)
        lat += [vlat, (vlat + vlat[nxt]) / 2, vlat, np.nextafter(vlat, 100), np.nextafter(vlat, -100)]
        lon += [vlon, (vlon + vlon[nxt]) / 2, np.clip(vlon + rng.uniform(-m, m, len(vlon)), -180, 180),
                np.nextafter(vlon, -200).clip(-180, 180), np.nextafter(vlon, 200).clip(-180, 180)]
    lat, lon = np.clip(np.concatenate(lat), -90, 90), np.concatenate(lon)
    n = lat.shape[0]
    docs = (np.arange(n, dtype=np.uint64) // 2) * 3   # two points per document, sparse ids
    g = ob.GeoPointField(gpu_ctx, int(docs.max()) + 1, docs, lat, lon)
    yield lat, lon, docs, g
    g.close()


@pytest.mark.parametrize("name", list(POLYGONS))
@pytest.mark.parametrize("inside", [True, False], ids=["inside", "outside"])
def test_polygon_bit_identical(poly_points, name, inside):
    lat, lon, docs, g = poly_points
    vlat, vlon = POLYGONS[name]
    per_point = pnpoly(vlat, vlon, lat, lon)
    assert 0 < per_point.sum() < len(per_point)
    exp = docs_of(docs, per_point if inside else ~per_point, g.nbits)
    got = _leaf_ids(g.polygon(list(zip(vlat.tolist(), vlon.tolist())), inside))
    assert np.array_equal(got, exp), (name, np.setxor1d(got, exp)[:10])


# ---------------------------------------------------------------- composition with id leaves and every search entry point
@pytest.fixture(scope="module")
def corpus_geo(corpus):
    c = corpus
    rng = np.random.default_rng(21)
    has = np.flatnonzero(rng.random(N) < 0.8)
    two = has[rng.random(has.shape[0]) < 0.2]
    idx = np.concatenate([has, two])
    lat = np.degrees(np.arcsin(rng.uniform(-1, 1, idx.shape[0])))
    lon = rng.uniform(-180, 180, idx.shape[0])
    g = ob.GeoPointField(c["strs"].ctx, c["nbits"], c["ids"][idx], lat, lon)
    idl = ob.DeviceFilter.from_ids(c["strs"].ctx, c["ids"][rng.random(N) < 0.5], c["nbits"])
    sf = ob.SortField(c["strs"].ctx, c["nbits"], c["ids"], rng.random(N), "number")
    yield g, idl, sf
    g.close(); idl.close(); sf.close()


@pytest.mark.parametrize("mode", [MODE_FULLTEXT, MODE_HYBRID, MODE_VECTOR], ids=["fulltext", "hybrid", "vector"])
def test_composition_byte_identical_to_filter_bits(corpus, corpus_geo, mode):
    c = corpus
    g, idl, sf = corpus_geo
    tsc = _tsc(c, mode)
    texts, qv = _inputs(c, mode)
    radius = g.radius(30.0, 10.0, 6000, "km")
    poly = g.polygon([(-60, -120), (-60, 60), (70, 60), (10, -30), (70, -120)], inside=False)
    combos = {"geo_and_ids": radius & idl, "geo_or_ids": radius | idl, "not_geo": ~radius, "poly_and_not_ids": None}
    nid = ~idl
    combos["poly_and_not_ids"] = poly & nid
    try:
        for name, f in combos.items():
            bits = f.read()
            assert 0 < f.count() < c["nbits"]
            for limit, offset in [(10, 0), (50, 7)]:
                kw = dict(mode=mode, limit_hint=limit, offset=offset, similarity=0.0)
                a = tsc.execute_batch_arrays(ob.TokenScoreParams(device_filter=f, **kw), texts, qv)
                b = tsc.execute_batch_arrays(ob.TokenScoreParams(filtered_doc_ids=bits, filter_nbits=c["nbits"], **kw), texts, qv)
                for x, y in zip(a, b):
                    assert x.tobytes() == y.tobytes(), (name, mode, limit)
            kw = dict(mode=mode, limit_hint=10, similarity=0.0)
            a = ob.search_sorted_arrays(tsc, ob.TokenScoreParams(device_filter=f, **kw), sf, "DESC", texts=texts, q_vecs=qv)
            b = ob.search_sorted_arrays(tsc, ob.TokenScoreParams(filtered_doc_ids=bits, filter_nbits=c["nbits"], **kw), sf, "DESC",
                                        texts=texts, q_vecs=qv)
            for x, y in zip(a, b):
                assert x.tobytes() == y.tobytes(), (name, mode, "sorted")
    finally:
        for f in list(combos.values()) + [radius, poly, nid]:
            f.close()


# ---------------------------------------------------------------- refusals (through the C ABI: the Python layer refuses first)
def test_refusals_create_nothing(gpu_ctx):
    L = _lib.lib()
    d = lambda *a: np.ascontiguousarray(a, np.float64)  # noqa: E731
    ids = np.ascontiguousarray([1, 2], np.uint64)
    for la, lo in [(d(10, np.nan), d(20, 21)), (d(10, 91), d(20, 21)), (d(10, 11), d(20, -180.5)), (d(np.inf, 1), d(0, 0))]:
        h = C.c_void_p()
        assert L.oc_geo_field_create(gpu_ctx._h, 10, 2, ids.ctypes.data, la.ctypes.data, lo.ctypes.data, C.byref(h)) == -1
        assert not h.value
    g = ob.GeoPointField(gpu_ctx, 10, ids, [10.0, 10.1], [20.0, 20.1])
    try:
        for lat, lon, r in [(np.nan, 0, 1), (91, 0, 1), (0, 181, 1), (0, 0, -1.0), (0, 0, np.nan), (0, 0, np.inf)]:
            h = C.c_void_p()
            assert L.oc_filter_geo_radius(g._h, lat, lon, r, 1, C.byref(h)) == -1 and not h.value
        for nv in (0, 2, _lib.OC_GEO_MAX_VERTICES + 1):
            vla, vlo = np.zeros(max(nv, 1)), np.linspace(-1, 1, max(nv, 1))
            h = C.c_void_p()
            assert L.oc_filter_geo_polygon(g._h, vla.ctypes.data, vlo.ctypes.data, nv, 1, C.byref(h)) == -1 and not h.value
        vla, vlo = d(0, 1, np.nan), d(0, 1, 1)
        h = C.c_void_p()
        assert L.oc_filter_geo_polygon(g._h, vla.ctypes.data, vlo.ctypes.data, 3, 0, C.byref(h)) == -1 and not h.value
        # the cap itself is accepted
        big = np.linspace(0, 2 * np.pi, _lib.OC_GEO_MAX_VERTICES, endpoint=False)
        f = g.polygon(list(zip((10 + np.sin(big)).tolist(), (20 + np.cos(big)).tolist())))
        assert _leaf_ids(f).tolist() == [1, 2]
        with pytest.raises(ValueError):
            g.radius(0, 0, -5)
    finally:
        g.close()


def test_empty_field(gpu_ctx):
    g = ob.GeoPointField(gpu_ctx, 100, [], [], [])
    try:
        for inside in (True, False):
            assert _leaf_ids(g.radius(0, 0, 1e7, inside=inside)).tolist() == []
            assert _leaf_ids(g.polygon([(0, 0), (0, 1), (1, 1)], inside=inside)).tolist() == []
    finally:
        g.close()
