"""tests/where_spec.py (the vectorised host evaluation the GPU where tests compare with) against the set restatement of
tests/test_where_host.py, set for set, on random trees over small multi-valued fields of every kind but radius; and its
radius leaves against the hand-worked cases of tests/test_geo_host.py, with the undecided band and three-valued trees."""
import numpy as np
import pytest

from oramacore_b200.where import GeoRadius, parse_where
from test_geo_host import R
from test_where_host import FIELDS, TREE_RULE_CASES, host_where
from where_spec import from_host_fields, radius_m, radius_points, unpack, where_masks, where_spec

NB = 48


def _fields(rng):
    """test_where_host's layout over NB documents: multi-valued fields, values at -0.0 / +0.0 and +-inf, runs of equal
    values, ids >= NB, points on polygon vertices and horizontal edges."""
    docs = np.arange(NB + 6)
    bm, sm = {}, {}
    for d in docs[rng.random(docs.shape[0]) < 0.8].tolist():
        bm[d] = set(rng.choice([True, False], int(rng.integers(1, 3))).tolist())
    for d in docs[rng.random(docs.shape[0]) < 0.7].tolist():
        sm[d] = [f"k{int(k)}" for k in rng.integers(0, 4, int(rng.integers(1, 3)))]
    nd = np.concatenate([docs, docs[rng.random(docs.shape[0]) < 0.4]])
    nv = rng.choice([-0.0, 0.0, 1.0, 2.0, 2.0, 3.0, -5.0, np.inf, -np.inf, 2147483647.0, -2147483648.0, 16777217.0, 0.5],
                    nd.shape[0])
    dd = docs[rng.random(docs.shape[0]) < 0.9]
    dv = rng.choice([-1000.0, 0.0, 86400000.0, 1672531200000.0], dd.shape[0])
    gd = np.concatenate([docs, docs[rng.random(docs.shape[0]) < 0.5]])
    pts = np.array([(0, 0), (0, 1), (1, 1), (1, 0), (0.5, 0.5), (0.0, 0.5), (1.0, 0.5), (0.5, 0.0), (2, 2), (-1, 0.5),
                    (90, 0), (0, 180), (0, -180)], float)
    g = pts[rng.integers(0, len(pts), gd.shape[0])]
    return {"b": ("bool", bm), "s": ("string", sm), "n": ("number", (nd, nv)), "d": ("date", (dd, dv)),
            "g": ("geo", (gd, g[:, 0], g[:, 1]))}


POLYS = [[(0, 0), (0, 1), (1, 1), (1, 0)], [(0, 0), (1, 1), (0, 1), (1, 0)], [(0, 0), (2, 0), (2, 2), (1, 0.5), (0, 2)]]


def _leaf(rng):
    k = ["b", "s", "n", "d", "g", "zz"][int(rng.integers(0, 6))]
    op = ["eq", "gt", "gte", "lt", "lte", "between"][int(rng.integers(0, 6))]
    if k == "b":
        return k, bool(rng.random() < 0.5)
    if k == "s":
        return k, f"k{int(rng.integers(0, 5))}"
    if k == "n":
        pick = lambda: [0, -0.0, 2, 2.0, 3, 1e39, -1e39, 2**31, -2**31, 2**31 - 1, 16777217, 0.5][int(rng.integers(0, 12))]  # noqa: E731
        return k, {op: [pick(), pick()] if op == "between" else pick()}
    if k == "d":
        pick = lambda: ["1970-01-01T00:00:00Z", "1969-12-31T23:59:59Z", "1970-01-02T00:00:00Z", "2023-01-01T00:00:00Z"][int(rng.integers(0, 4))]  # noqa: E731
        return k, {op: [pick(), pick()] if op == "between" else pick()}
    if k == "g":
        p = POLYS[int(rng.integers(0, len(POLYS)))]
        return k, {"polygon": {"coordinates": [{"lat": a, "lon": b} for a, b in p], "inside": bool(rng.random() < 0.7)}}
    return k, True   # not a field


def _tree(rng, depth=1):
    w = {}
    for _ in range(int(rng.integers(0, 3))):
        k, v = _leaf(rng)
        w[k] = v
    if depth < 4:
        for key, p in (("and", 0.4), ("or", 0.4)):
            if rng.random() < p:
                w[key] = [_tree(rng, depth + 1) for _ in range(int(rng.integers(0, 4)))]
        if rng.random() < 0.3:
            w["not"] = _tree(rng, depth + 1)
    return w


def _ids(bits, nbits):
    return None if bits is None else set(np.flatnonzero(unpack(bits, nbits)).tolist())


@pytest.mark.parametrize("seed", range(6))
def test_random_trees_equal_host_where(seed):
    rng = np.random.default_rng(seed)
    hf = _fields(rng)
    sf = from_host_fields(hf)
    for i in range(150):
        w = parse_where(_tree(rng))
        deleted = rng.choice(NB + 4, int(rng.integers(1, 6)), replace=False).tolist() if i % 3 == 0 else ()
        assert _ids(where_spec(w, sf, NB, deleted), NB) == host_where(w, hf, NB, deleted), (seed, i)


@pytest.mark.parametrize("where, deleted, expected", TREE_RULE_CASES)
def test_tree_rules_cases(where, deleted, expected):
    assert _ids(where_spec(parse_where(where), from_host_fields(FIELDS), 5, deleted), 5) == expected


def test_padding_bits_clear():
    bits = where_spec(parse_where({"not": {"b": True}}), from_host_fields(FIELDS), 5)
    assert bits.tolist() == [0b11010]


# ---------------------------------------------------------------- radius: the cases of test_geo_host.py
LAT, LON = np.array([0.0, 0.0, 89.0, -90.0]), np.array([0.0, 180.0, 10.0, 0.0])


@pytest.mark.parametrize("r, inside", [(0.0, [True, False, False, False]), (20_100_000.0, [True] * 4),
                                       (2.5e7, [True] * 4), (10_007_600.0, [True, False, True, True]),
                                       (10_000_000.0, [True, False, True, False])])
def test_radius_hand_worked(r, inside):
    p_in, p_out = radius_points(GeoRadius(0.0, 0.0, r), LAT, LON)
    assert p_in.tolist() == inside and p_out.tolist() == [not x for x in inside]


def test_radius_band_and_centres():
    # a point exactly on the boundary is undecided; a point at the centre is in at radius 0, one a metre away is out
    q = 1e7 / R * 180 / np.pi   # 1e7 m north of (0, 0)
    p_in, p_out = radius_points(GeoRadius(0.0, 0.0, 1e7), np.array([q, q * 0.999, q * 1.001]), np.zeros(3))
    assert p_in.tolist() == [False, True, False] and p_out.tolist() == [False, False, True]
    p_in, p_out = radius_points(GeoRadius(12.5, 7.25, 0.0), np.array([12.5, 12.5 + 1e-5]), np.array([7.25, 7.25]))
    assert p_in.tolist() == [True, False] and p_out.tolist() == [False, True]
    # a centre at a pole: every longitude at the pole is within a metre; the other pole is not
    p_in, p_out = radius_points(GeoRadius(90.0, 0.0, 1.0), np.array([90.0, 90.0, -90.0]), np.array([0.0, -180.0, 33.0]))
    assert p_in.tolist() == [True, True, False] and p_out.tolist() == [False, False, True]
    # units are f32: 7 mi is f32(7 x f32(1609.344)) m, not 7 x 1609.344
    assert radius_m(GeoRadius(0.0, 0.0, 7.0, "mi")) == float(np.float32(7 * np.float32(1609.344))) != 7 * 1609.344


def test_radius_in_trees_is_three_valued():
    """Documents with a point in the band stay undecided through And / Or / Not unless another part decides them."""
    q = 1e7 / R * 180 / np.pi
    fields = {"g": ("geo", np.array([0, 1, 1, 2, 3]), (np.array([q, q, 0.0, 0.0, 0.0]), np.array([0.0, 0.0, 0.0, 0.0, 120.0]))),
              "b": ("bool", np.array([0, 1, 2, 3]), np.array([True, False, True, False]))}
    rad = {"radius": {"coordinates": {"lat": 0, "lon": 0}, "value": 1e7}}
    nb = 5
    cases = {   # where: (certainly in, certainly out)
        "leaf": ({"g": rad}, {1, 2}, {3, 4}),
        "outside": ({"g": dict(rad, radius=dict(rad["radius"], inside=False))}, {3}, {2, 4}),
        "not": ({"not": {"g": rad}}, {3, 4}, {1, 2}),
        "and": ({"g": rad, "b": True}, {2}, {1, 3, 4}),
        "or": ({"or": [{"g": rad}, {"b": True}]}, {0, 1, 2}, {3, 4}),
    }
    for name, (where, t, f) in cases.items():
        mt, mf = where_masks(parse_where(where), fields, nb)
        assert set(np.flatnonzero(mt).tolist()) == t and set(np.flatnonzero(mf).tolist()) == f, name
    with pytest.raises(AssertionError, match="boundary"):
        where_spec(parse_where({"g": rad}), fields, nb)
