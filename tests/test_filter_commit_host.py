"""tests/filter_commit_spec.py (the filter-field commit restated in numpy) against a from-scratch rebuild of the final
state, on random op streams committed in several rounds.  No GPU."""
import numpy as np
import pytest

import filter_commit_spec as S

KINDS = ("csr", "number", "geo")


def _random_ops(rng, kind, n_ops, n_docs, n_var, p_del=0.1, p_clr=0.05, unique=False):
    ops = []
    for _ in range(n_ops):
        r, d = rng.random(), int(rng.integers(0, n_docs))
        if r < p_del:
            ops.append(("del", d))
        elif r < p_del + p_clr:
            ops.append(("clr", 0, d))
        elif kind == "csr":
            ops.append(("ins", 0, d, int(rng.integers(0, n_var)), unique))
        elif kind == "number":
            ops.append(("ins", 0, d, float(rng.choice([-0.0, 0.0, 1.5, -2.0, np.inf, -np.inf, float(rng.integers(0, 5))])), False))
        else:
            ops.append(("ins", 0, d, (float(rng.uniform(-90, 90)), float(rng.uniform(-180, 180))), False))
    return ops


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("seed", range(6))
def test_commits_equal_the_rebuild(kind, seed):
    rng = np.random.default_rng(seed)
    unique = kind == "csr" and seed % 2 == 0
    n_var = 1 + seed
    lay, history = S.empty(kind, 1 if kind == "csr" else 0), []
    for rnd in range(5):
        n_var += int(kind == "csr" and rnd % 2)   # new string_filter keys append
        ops = _random_ops(rng, kind, int(rng.integers(0, 60)), 20 + 10 * rnd, n_var, unique=unique)
        lay = S.commit(kind, 0, lay, ops, n_var)
        history += ops
        ref = S.rebuild(kind, 0, history, n_var)
        assert S.same_up_to_ties(kind, lay, ref), (kind, seed, rnd)


def test_delete_then_reinsert_keeps_the_insert():
    lay = S.commit("number", 0, S.empty("number"), [("ins", 0, 4, 1.0, False)])
    lay = S.commit("number", 0, lay, [("ins", 0, 4, 2.0, False), ("del", 4), ("ins", 0, 4, 3.0, False)])
    assert lay["values"].tolist() == [3.0] and lay["docs"].tolist() == [4]
    lay = S.commit("number", 0, lay, [("ins", 0, 4, 3.0, False)])   # append: a repeated value is listed twice
    assert lay["values"].tolist() == [3.0, 3.0]


def test_filter_bool_replaces_and_filter_bool2_adds():
    T, F = 0, 1
    # FilterBool(true) then FilterBool(false): a clear before each unique insert leaves {false}
    ops = [("clr", 0, 7), ("ins", 0, 7, T, True)]
    lay = S.commit("csr", 0, S.empty("csr", 2), ops, 2)
    lay = S.commit("csr", 0, lay, [("clr", 0, 7), ("ins", 0, 7, F, True)], 2)
    assert lay["offsets"].tolist() == [0, 0, 1] and lay["docs"].tolist() == [7]
    # FilterBool2 adds to the set, once per value however often it comes
    lay = S.commit("csr", 0, lay, [("ins", 0, 7, T, True), ("ins", 0, 7, F, True), ("ins", 0, 7, T, True)], 2)
    assert lay["offsets"].tolist() == [0, 1, 2] and lay["docs"].tolist() == [7, 7]
    # a string_filter key listed twice by one document is listed twice
    s = S.commit("csr", 0, S.empty("csr", 1), [("ins", 0, 3, 0, False), ("ins", 0, 3, 0, False)], 1)
    assert s["docs"].tolist() == [3, 3]


def test_empty_fields_and_fields_that_become_empty():
    for kind in KINDS:
        e = S.empty(kind, 2 if kind == "csr" else 0)
        assert S.same_up_to_ties(kind, S.commit(kind, 0, e, [], 2), e)
        pay = {"csr": 1, "number": 5.0, "geo": (1.0, 2.0)}[kind]
        lay = S.commit(kind, 0, e, [("ins", 0, 9, pay, False)], 2)
        assert lay["docs"].tolist() == [9]
        lay = S.commit(kind, 0, lay, [("del", 9)], 3)
        assert lay["docs"].shape[0] == 0
        if kind == "csr":
            assert lay["offsets"].tolist() == [0, 0, 0, 0]   # a new key with nothing in it yet


def test_other_fields_ops_do_not_apply():
    lay = S.commit("number", 0, S.empty("number"), [("ins", 0, 1, 1.0, False), ("ins", 1, 2, 2.0, False), ("clr", 1, 1)])
    assert lay["docs"].tolist() == [1]
