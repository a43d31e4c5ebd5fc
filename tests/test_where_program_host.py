"""where.compile_where on the host: the postfix programs of the tree rules, checked (1) for their shape on the tree-rule
cases of test_where_host.py and (2) by a numpy interpreter of the programs over leaf id sets, against the host
restatement host_where, on a few hundred random trees with polygon leaves and deletes.  The stores are stand-ins that
carry the fields' layout and a handle value; no device is used."""
import ctypes as C
import types

import numpy as np
import pytest

from oramacore_b200 import _lib
from oramacore_b200.engine import FacetStore, GeoPointField
from oramacore_b200.where import _NARY, compile_where, parse_where
from test_geo_host import pnpoly
from test_where_host import FIELDS, host_where

NONE, VAR, RNG, RAD, POLY, FILT, AND, OR, NOT = (_lib.OC_WHERE_NONE, _lib.OC_WHERE_VARIANT, _lib.OC_WHERE_RANGE,
                                                 _lib.OC_WHERE_GEO_RADIUS, _lib.OC_WHERE_GEO_POLYGON, _lib.OC_WHERE_FILTER,
                                                 _lib.OC_WHERE_AND, _lib.OC_WHERE_OR, _lib.OC_WHERE_NOT)
STORE, GEO, LIVE = 0x1000, 0x2000, 0x3000


def _stores(fields):
    """A FacetStore / GeoPointField stand-in over host_where's `fields`, and a per-leaf id-set evaluator."""
    st = types.SimpleNamespace(fields={}, _h=C.c_void_p(STORE))
    st.leaf_args = types.MethodType(FacetStore.leaf_args, st)
    sets = {}
    for i, (name, (kind, data)) in enumerate((k, v) for k, v in fields.items() if v[0] != "geo"):
        if kind in ("bool", "string"):
            keys = ["true", "false"] if kind == "bool" else sorted({x for ks in data.values() for x in ks})
            st.fields[name] = {"id": i, "kind": kind, "variant": {k: j for j, k in enumerate(keys)}}
            for j, k in enumerate(keys):
                want = (k == "true") if kind == "bool" else k
                sets[(i, j)] = {d for d, vs in data.items() if want in vs}
        else:
            st.fields[name] = {"id": i, "kind": kind}
            sets[i] = data
    geo = {k: types.SimpleNamespace(_h=C.c_void_p(GEO), radius_args=GeoPointField.radius_args,
                                    polygon_args=GeoPointField.polygon_args, data=v[1])
           for k, v in fields.items() if v[0] == "geo"}
    return st, geo, sets


def run_program(nodes, sets, geo, nbits, live):
    """A numpy interpreter of a program: each node's id set, combined on a stack."""
    stack, everything = [], set(range(nbits))
    for (op, field, arg, a, b, c, src, verts) in nodes:
        if op == NONE:
            stack.append(set())
        elif op == VAR:
            stack.append({d for d in sets[(field, arg)] if d < nbits})
        elif op == RNG:
            d, v = sets[field]
            lo_ok = (v > a) if arg & _lib.OC_RANGE_LO_OPEN else (v >= a)
            hi_ok = (v < b) if arg & _lib.OC_RANGE_HI_OPEN else (v <= b)
            stack.append({int(x) for x in d[lo_ok & hi_ok] if x < nbits})
        elif op == POLY:
            d, lat, lon = next(iter(geo.values())).data
            hit = pnpoly(verts[0], verts[1], lat, lon)
            stack.append({int(x) for x in d[hit if arg else ~hit] if x < nbits})
        elif op == FILT:
            assert src == LIVE
            stack.append(live)
        elif op in (AND, OR):
            assert arg >= 2 and len(stack) >= arg
            parts = [stack.pop() for _ in range(arg)]
            stack.append(set.intersection(*parts) if op == AND else set.union(*parts))
        elif op == NOT:
            stack.append(everything - stack.pop())
        else:
            raise AssertionError(op)
        assert len(stack) <= _lib.OC_WHERE_MAX_DEPTH
    assert len(stack) == 1
    return stack[0]


def _program(where, fields, nbits, deleted):
    st, geo, sets = _stores(fields)
    live = C.c_void_p(LIVE) if deleted else None
    live_f = None if live is None else types.SimpleNamespace(_h=live, nbits=nbits)
    return compile_where(parse_where(where), st, geo, nbits, live_f), sets, geo


@pytest.mark.parametrize("where, deleted, shape", [
    ({}, (), None),
    ({}, (1,), [FILT]),
    ({"or": []}, (), None),
    ({"b": True}, (), [VAR]),
    ({"b": True}, (2,), [VAR, FILT, AND]),
    ({"b": False, "s": "x"}, (), [VAR, VAR, AND]),
    ({"unknown": True, "b": True}, (), [NONE]),
    ({"b": True, "unknown": True}, (), [NONE]),
    ({"or": [{"b": False}, {"unknown": True}]}, (), [VAR, NONE, OR]),
    ({"not": {"unknown": "z"}}, (), [NONE, NOT]),
    ({"and": [{}]}, (), [NONE]),
    ({"b": True, "or": []}, (), [NONE]),
    ({"n": {"between": [3, 2]}}, (), [RNG]),
    ({"n": True}, (), [NONE]),
    ({"s": "nope"}, (), [NONE]),
    ({"s": "y", "and": [{"n": {"gt": 1}}], "or": [{"b": False}, {"n": {"lt": 0}}], "not": {"s": "x"}}, (),
     [VAR, RNG, VAR, RNG, OR, VAR, NOT, AND]),
])
def test_tree_rule_shapes(where, deleted, shape):
    prog, sets, geo = _program(where, FIELDS, 5, deleted)
    if shape is None:
        assert prog is None
        return
    assert [n[0] for n in prog.nodes] == shape
    live = set(range(5)) - set(deleted)
    assert run_program(prog.nodes, sets, geo, 5, live) == host_where(parse_where(where), FIELDS, 5, deleted)
    # leaf parameters: a range carries [lo, hi] and its open ends, a FILTER the handle, the stores their handles
    for n in prog.nodes:
        if n[0] in (VAR, RNG):
            assert n[6] == STORE
        if n[0] == FILT:
            assert n[6] == LIVE


def _rand_fields(rng, nd):
    docs = np.arange(nd)
    bools = {int(d): {bool(x) for x in rng.random(int(rng.integers(1, 3))) < 0.5} for d in docs[rng.random(nd) < 0.8]}
    strs = {int(d): [f"k{int(x)}" for x in rng.integers(0, 5, int(rng.integers(1, 3)))] for d in docs[rng.random(nd) < 0.7]}
    nd_ = np.concatenate([docs, docs[rng.random(nd) < 0.3]])
    nv = rng.integers(-20, 20, nd_.shape[0]).astype(np.float64)
    gd = docs[rng.random(nd) < 0.8]
    return {"b": ("bool", bools), "s": ("string", strs), "n": ("number", (nd_, nv)),
            "g": ("geo", (gd, rng.uniform(-60, 60, gd.shape[0]), rng.uniform(-120, 120, gd.shape[0])))}


def _leaf(rng, key):
    if key == "b":
        return bool(rng.random() < 0.5)
    if key == "s":
        return f"k{int(rng.integers(0, 6))}"
    if key == "n":
        op = ["eq", "gt", "gte", "lt", "lte", "between"][int(rng.integers(0, 6))]
        return {op: [int(rng.integers(-25, 25)), int(rng.integers(-25, 25))] if op == "between" else int(rng.integers(-25, 25))}
    c, rr = rng.uniform(-40, 40, 2), rng.uniform(5, 50)
    a = np.linspace(0, 2 * np.pi, int(rng.integers(3, 8)), endpoint=False)
    return {"polygon": {"coordinates": [{"lat": float(c[0] + rr * np.sin(t)), "lon": float(c[1] + rr * np.cos(t))} for t in a],
                        "inside": bool(rng.random() < 0.7)}}


def _tree(rng, depth):
    w = {}
    for key in rng.choice(["b", "s", "n", "g", "zz"], int(rng.integers(0, 3)), replace=False):
        w[str(key)] = _leaf(rng, str(key)) if key != "zz" else True
    if depth < 4:
        if rng.random() < 0.4:
            w["and"] = [_tree(rng, depth + 1) for _ in range(int(rng.integers(0, 3)))]
        if rng.random() < 0.4:
            w["or"] = [_tree(rng, depth + 1) for _ in range(int(rng.integers(0, 3)))]
        if rng.random() < 0.3:
            w["not"] = _tree(rng, depth + 1)
    return w


def test_programs_agree_with_the_host_restatement():
    rng = np.random.default_rng(12)
    nd, nbits = 400, 380   # ids >= nbits are dropped by every leaf
    fields = _rand_fields(rng, nd)
    for i in range(300):
        where = _tree(rng, 1)
        deleted = sorted(rng.choice(nbits, 20, replace=False).tolist()) if i % 2 else []
        prog, sets, geo = _program(where, fields, nbits, deleted)
        ref = host_where(parse_where(where), fields, nbits, deleted)
        if ref is None:
            assert prog is None, where
            continue
        assert prog.nbits == nbits and len(prog.nodes) <= _lib.OC_WHERE_MAX_NODES
        assert run_program(prog.nodes, sets, geo, nbits, set(range(nbits)) - set(deleted)) == ref, where


def _peak(nodes):
    sp = top = 0
    for n in nodes:
        sp += 1 - n[2] if n[0] in (AND, OR) else 0 if n[0] == NOT else 1
        top = max(top, sp)
    return top


@pytest.mark.parametrize("op", ["and", "or"])
@pytest.mark.parametrize("n", [2, _NARY, _NARY + 1, 17, 31, 33, 300])
def test_wide_and_or_lists(op, n):
    """An And / Or of n parts is folded into nodes of at most _NARY operands: the stack holds at most _NARY - 1 values
    above the deepest part, and the program is the host restatement's set.  (A list of n > OC_WHERE_MAX_DEPTH parts
    pushed before one node was refused by the planner.)"""
    rng = np.random.default_rng(n)
    nd, nbits = 400, 380
    fields = _rand_fields(rng, nd)
    # And over NOT of narrow leaves, Or over narrow leaves: neither result is empty nor everything, and each part matters
    narrow = [{"n": {"eq": int(v)}} if i % 3 else {"s": f"k{int(v) % 3}"} for i, v in enumerate(rng.integers(-200, 200, n))]
    narrow[-1] = {"b": True}   # a broad last part, so the last node of the fold changes the result
    parts = [{"not": p} for p in narrow] if op == "and" else narrow
    prog, sets, geo = _program({op: parts}, fields, nbits, [])
    assert all(x[2] <= _NARY for x in prog.nodes if x[0] in (AND, OR))
    assert _peak(prog.nodes) <= _NARY - 1 + 2   # a part is a leaf, or a leaf and its Not
    got = run_program(prog.nodes, sets, geo, nbits, set(range(nbits)))
    assert got == host_where(parse_where({op: parts}), fields, nbits)
    assert 0 < len(got) < nbits
    if n > _NARY:   # the parts beyond the first node change the result
        assert got != host_where(parse_where({op: parts[:_NARY]}), fields, nbits)
    if n == _NARY:
        assert [x[0] for x in prog.nodes].count(AND if op == "and" else OR) == 1


def test_nested_wide_lists():
    """Four wide lists nested in each other (the inner one last) fit the stack; each costs _NARY - 1 slots."""
    rng = np.random.default_rng(4)
    nd, nbits = 400, 380
    fields = _rand_fields(rng, nd)
    leaves = [{"n": {"gt": int(v)}} if i % 2 else {"s": f"k{int(v) % 6}"} for i, v in enumerate(rng.integers(-20, 20, 200))]
    where = {"or": leaves[:40]}
    for level, op in enumerate(["and", "or", "and"]):
        part = leaves[40 * (level + 1): 40 * (level + 2)]
        where = {op: ([{"not": p} for p in part] if op == "and" else part) + [where]}
    prog, sets, geo = _program(where, fields, nbits, [])
    assert _peak(prog.nodes) <= 4 * (_NARY - 1) + 1 <= _lib.OC_WHERE_MAX_DEPTH
    assert run_program(prog.nodes, sets, geo, nbits, set(range(nbits))) == host_where(parse_where(where), fields, nbits)
