"""The filter-field commit on the device (oc_facets_commit_ex, oc_geo_field_commit_ex) through FacetStore and
GeoPointField: the read-back of every field kind after each commit of a random op stream equals
tests/filter_commit_spec.py, every where leaf equals the same leaf on a store built from scratch from the final state,
bit for bit, searches during a commit see one version or the other, and refused commits change nothing."""
import threading
import time

import numpy as np
import pytest

import filter_commit_spec as S
import oramacore_b200 as ob
from oramacore_b200 import _lib
from oramacore_b200._lib import check
from oramacore_b200.where import DateFilter

pytestmark = pytest.mark.gpu

FIELDS = {"b": "csr", "s": "csr", "n": "number", "d": "number"}   # field id order of the store below


def _store(ctx, nbits):
    st = ob.FacetStore(ctx, nbits)
    st.add_bool_field("b", [], [])
    st.add_string_field("s", {"k0": []})
    st.add_number_field("n", [], [])
    st.add_date_field("d", [], [])
    return st


class Stream:
    """Drives a FacetStore + GeoPointField with random ops and records them in the spec's form."""

    def __init__(self, ctx, seed, nbits=1):
        self.rng = np.random.default_rng(seed)
        self.st, self.geo = _store(ctx, nbits), ob.GeoPointField(ctx, nbits, [], [], [])
        self.ops = {f: [] for f in list(FIELDS) + ["g"]}   # per field, with deletes copied into every one
        self.n_var = {"b": 2, "s": 1}
        self.max_doc = -1

    def step(self, n_ops, n_docs):
        rng, st = self.rng, self.st
        for _ in range(n_ops):
            d = int(rng.integers(0, n_docs))
            r = rng.random()
            if r < 0.08:
                st.delete([d]); self.geo.delete([d])
                for f in self.ops:
                    self.ops[f].append(("del", d))
                continue
            self.max_doc = max(self.max_doc, d)
            if r < 0.2:   # FilterBool: replace
                v = bool(rng.random() < 0.5)
                st.clear("b", [d]); st.insert_variants("b", [d], [v])
                self.ops["b"] += [("clr", 0, d), ("ins", 0, d, 0 if v else 1, True)]
            elif r < 0.3:   # FilterBool2: add to the set
                v = bool(rng.random() < 0.5)
                st.insert_variants("b", [d], [v])
                self.ops["b"].append(("ins", 0, d, 0 if v else 1, True))
            elif r < 0.5:   # FilterString(2): new keys append
                k = f"k{int(rng.integers(0, 12))}"
                st.insert_variants("s", [d], [k])
                v = st.add_key("s", k)
                self.n_var["s"] = max(self.n_var["s"], v + 1)
                self.ops["s"].append(("ins", 0, d, v, False))
            elif r < 0.7:
                x = float(rng.choice([-0.0, 0.0, 1.0, 2.5, -3.0, np.inf, -np.inf, float(rng.integers(0, 50))]))
                st.insert_numbers("n", [d], [x])
                self.ops["n"].append(("ins", 0, d, x, False))
            elif r < 0.8:
                ms = int(rng.integers(0, 10**12))
                st.insert_numbers("d", [d], [ms])
                self.ops["d"].append(("ins", 0, d, float(ms), False))
            else:
                la, lo = float(rng.uniform(-60, 60)), float(rng.uniform(-120, 120))
                self.geo.insert([d], [la], [lo])
                self.ops["g"].append(("ins", 0, d, (la, lo), False))

    def commit(self):
        nbits = max(self.st.nbits, self.max_doc + 2)
        a, b = self.st.commit(nbits), self.geo.commit(nbits)
        return a, b

    def expected(self, f):
        kind = "geo" if f == "g" else FIELDS[f]
        return kind, S.rebuild(kind, 0, self.ops[f], self.n_var.get(f, 0))

    def scratch(self, ctx):
        """Stores built from scratch from the final state (FacetStore.add_* / GeoPointField)."""
        st = ob.FacetStore(ctx, self.st.nbits)
        for f in FIELDS:
            _, lay = self.expected(f)
            if FIELDS[f] == "csr":
                off = lay["offsets"]
                keys = self.st.fields[f]["keys"]
                by_key = {k: lay["docs"][int(off[i]):int(off[i + 1])] for i, k in enumerate(keys)}
                (st.add_bool_field(f, by_key["true"], by_key["false"]) if f == "b" else st.add_string_field(f, by_key))
            elif f == "n":
                st.add_number_field(f, lay["docs"], lay["values"])
            else:
                st.add_date_field(f, lay["docs"], lay["values"].astype(np.int64))
        _, g = self.expected("g")
        return st, ob.GeoPointField(ctx, self.geo.nbits, g["docs"], g["lat"], g["lon"])

    def close(self):
        self.st.close(); self.geo.close()


def _read(stream, f):
    if f == "g":
        r = stream.geo.read()
        return {"docs": r["doc_ids"], "lat": r["lat"], "lon": r["lon"]}
    r = stream.st.read_field(f)
    return {"offsets": r["offsets"], "docs": r["doc_ids"]} if FIELDS[f] == "csr" else {"values": r["values"], "docs": r["doc_ids"]}


def _leaves(st, geo):
    out = []
    for v in (True, False):
        out.append(st.leaf("b", v))
    for k in st.fields["s"]["keys"]:
        out.append(st.leaf("s", k))
    for lo, hi, fl in ((0.0, 0.0, 0), (-np.inf, 2.5, 0), (1.0, np.inf, _lib.OC_RANGE_LO_OPEN), (-3.0, 2.5, _lib.OC_RANGE_HI_OPEN),
                       (-np.inf, np.inf, 0), (5.0, 1.0, 0)):
        h = C_range(st, "n", lo, hi, fl)
        out.append(h)
    out.append(st.leaf("d", DateFilter("gt", 5 * 10**11)))
    out.append(st.leaf("d", DateFilter("between", (10**11, 6 * 10**11))))
    for inside in (True, False):
        out.append(geo.radius(10.0, 20.0, 3000, "km", inside))
        out.append(geo.polygon([(-30, -60), (-30, 60), (40, 60), (40, -60)], inside))
    return out


def C_range(st, name, lo, hi, flags):
    import ctypes as C
    h = C.c_void_p()
    check(ob.lib().oc_filter_facet_range(st._h, st.fields[name]["id"], lo, hi, flags, C.byref(h)))
    return ob.DeviceFilter.of_handle(st.ctx, h)


def _bytes(handles):
    try:
        return [h.read().tobytes() for h in handles]
    finally:
        for h in handles:
            h.close()


@pytest.mark.parametrize("seed", [1, 2])
def test_random_streams_read_back_and_leaves(gpu_ctx, seed):
    s = Stream(gpu_ctx, seed)
    try:
        for rnd in range(5):
            s.step(int(s.rng.integers(0, 400)), 50 + 60 * rnd)
            a, b = s.commit()
            assert a["version"] == b["version"] == rnd + 1
            for f in s.ops:
                kind, ref = s.expected(f)
                assert S.same_up_to_ties(kind, _read(s, f), ref), (seed, rnd, f)
            st2, g2 = s.scratch(gpu_ctx)
            try:
                assert _bytes(_leaves(s.st, s.geo)) == _bytes(_leaves(st2, g2)), (seed, rnd)
            finally:
                st2.close(); g2.close()
    finally:
        s.close()


def test_growth_from_empty_and_commit_without_ops(gpu_ctx):
    st = _store(gpu_ctx, 1)
    geo = ob.GeoPointField(gpu_ctx, 1, [], [], [])
    try:
        a = st.commit()
        assert a["version"] == 1 and a["rows_kept"] == a["rows_added"] == a["rows_dropped"] == 0
        assert geo.commit()["version"] == 1
        st.insert_variants("s", [5, 9], ["new", "k0"])
        st.insert_numbers("n", [9], [1.0])
        geo.insert([9], [1.0], [2.0])
        st.commit(11); geo.commit(11)
        assert st.nbits == 11 and st.fields["s"]["keys"] == ["k0", "new"]
        assert st.read_field("s")["offsets"].tolist() == [0, 1, 2]
        assert _bytes([st.leaf("s", "new")])[0] == _bytes([ob.DeviceFilter.from_ids(gpu_ctx, [5], 11)])[0]
        assert geo.read()["doc_ids"].tolist() == [9]
        a = st.commit(11)
        assert a["version"] == 3 and a["rows_kept"] == 3 and a["rows_added"] == 0   # every field: two strings, one number
    finally:
        st.close(); geo.close()


def test_refused_commit_changes_nothing_and_keeps_the_ops(gpu_ctx):
    st = _store(gpu_ctx, 10)
    geo = ob.GeoPointField(gpu_ctx, 10, [1], [0.0], [0.0])
    try:
        st.insert_numbers("n", [20], [4.0])
        geo.insert([20], [1.0], [1.0])
        with pytest.raises(ob.OcError):
            st.commit(5)                 # nbits only grows
        with pytest.raises(ob.OcError):
            st.commit(20)                # a queued document >= new_nbits
        with pytest.raises(ob.OcError):
            geo.commit(20)
        assert st.nbits == 10 and st.read_field("n")["doc_ids"].size == 0 and geo.read()["doc_ids"].tolist() == [1]
        with pytest.raises(ob.OcError):
            st.insert_numbers("n", [1], [np.nan])
        with pytest.raises(ValueError):
            geo.insert([1], [91.0], [0.0])
        with pytest.raises(ob.OcError):
            check(ob.lib().oc_facets_insert_variants(st._h, st.fields["n"]["id"], 0, None, None, 0))   # a number field
        a, b = st.commit(21), geo.commit(21)
        assert a["version"] == 1 and a["rows_added"] == 1 and b["rows_added"] == 1
        assert st.read_field("n")["doc_ids"].tolist() == [20] and geo.read()["doc_ids"].tolist() == [1, 20]
    finally:
        st.close(); geo.close()


def test_leaves_during_a_commit_see_one_version(gpu_ctx):
    s = Stream(gpu_ctx, 11)
    try:
        s.step(20000, 20000)
        s.commit()
        before = _bytes([s.st.leaf("s", "k3"), C_range(s.st, "n", 0.0, 10.0, 0), s.geo.radius(0.0, 0.0, 4000, "km")])
        s.step(5000, 30000)
        seen, spans, errors, stop = [], [], [], threading.Event()

        def reader():
            try:
                while not stop.is_set():
                    t0 = time.perf_counter()
                    seen.append(_bytes([s.st.leaf("s", "k3"), C_range(s.st, "n", 0.0, 10.0, 0),
                                        s.geo.radius(0.0, 0.0, 4000, "km")]))
                    spans.append((t0, time.perf_counter()))
            except Exception as e:   # noqa: BLE001 — reported below
                errors.append(e)

        t = threading.Thread(target=reader)
        t.start()
        while not spans and t.is_alive():   # the reader is running before the commit starts
            time.sleep(0.001)
        try:
            c0 = time.perf_counter()
            s.commit()
            c1 = time.perf_counter()
        finally:
            stop.set()
            t.join()
        after = _bytes([s.st.leaf("s", "k3"), C_range(s.st, "n", 0.0, 10.0, 0), s.geo.radius(0.0, 0.0, 4000, "km")])
        assert not errors, errors
        assert any(a < c1 and b > c0 for a, b in spans), "no read overlapped the commit"
        for x in seen:
            # each leaf is read under the ctx lock: it sees the facet store (or the geo field) before or after
            for k in range(3):
                assert x[k] in (before[k], after[k])
    finally:
        s.close()
