"""The fp16 sweep of an fp32 store (emb_gemm.cuh, GEMM_F16) reads a copy of every row scaled by a power of two that puts
its largest |x_i| in [2^14, 2^15), rounded to nearest fp16, and a query scaled the same way.  These CPU tests pin the
error bound GEMM_EPS_F16 the selection rule relies on: the scaling keeps every component of every finite row inside
fp16's range (rows with norms from 1e-30 to 1e30, components spanning 40 binades, values at rounding midpoints, values
above fp16's largest finite 65504), the per-operand residual stays within 2^-11 + 2^-34, and the 2*eps rule returns
the exact top-k on clustered data."""
import numpy as np
import pytest

from test_proof_bounds import ACC_RESCORE, ACC_TC, _constants, _select_exact_topk, tf32_trunc

RHO_F16 = 2.0 ** -11 + 2.0 ** -34    # per operand: round to nearest (11 bits) + the fp16-subnormal components


def f16_exponent(a):
    """s per row: largest |a_i| * 2^s in [2^14, 2^15); 0 for an all-zero row (f16_scaled_copy_warp)."""
    a = np.atleast_2d(np.asarray(a, np.float32))
    m = np.abs(a).max(axis=1).astype(np.float64)
    _, e = np.frexp(np.where(m > 0, m, 1.0))    # m = f 2^e, f in [0.5, 1): floor(log2 m) = e - 1
    return np.where(m > 0, 14 - (e - 1), 0).astype(np.int64)


def f16_operand(a):
    """-> (fp16 copy [n][d], s [n]): the bits the sweep reads and the power of two they were scaled by.  The scaling
    is exact in float64, so the cast rounds the exact product once, to nearest even (as __float2half_rn)."""
    a = np.atleast_2d(np.asarray(a, np.float32))
    s = f16_exponent(a)
    with np.errstate(over="ignore"):
        h = np.ldexp(a.astype(np.float64), s[:, None]).astype(np.float16)
    return h, s


def f16_value(a):
    """what the fp16 operand stands for, in the units of a (float64)"""
    h, s = f16_operand(a)
    return np.ldexp(h.astype(np.float64), -s[:, None])


def rho64(a, approx):
    a64 = np.atleast_2d(a).astype(np.float64)
    return np.linalg.norm(a64 - approx, axis=-1) / np.linalg.norm(a64, axis=-1)


def test_compiled_constant_covers_the_rigorous_bound():
    c = _constants()
    acc = ACC_TC + 2 * ACC_RESCORE
    f16 = 2 * RHO_F16 + RHO_F16 ** 2 + acc         # (rho_x + rho_q + rho_x rho_q) + accumulation + re-score
    assert 2 * (2.0 ** -11 + 2.0 ** -34) + 2.0 ** -22 + acc <= f16
    assert f16 <= c["EPS_F16"] <= f16 * 1.05
    assert c["EPS_F16"] < c["EPS_TF32"]             # tighter than tf32: fewer rows inside the 2 eps window


def _extreme_rows(rng, dim):
    rows = []
    for lg in range(-30, 31, 5):                     # norms 1e-30 .. 1e30
        v = rng.standard_normal(dim)
        rows.append(v / np.linalg.norm(v) * 10.0 ** lg)
    rows.append(2.0 ** (-np.arange(dim) % 40) * rng.choice([-1.0, 1.0], dim))   # 40 binades in one row
    rows.append(2.0 ** (np.arange(dim) % 40 - 20.0) * 1e-17)
    mid = np.full(dim, 1.0 + 2.0 ** -11)             # midway between two fp16 values once scaled (ties to even)
    mid[1::2] = 1.0 + 3 * 2.0 ** -11
    rows.append(mid)
    big = rng.uniform(65504.0, 3e38, dim)             # above fp16's largest finite value
    rows.append(big)
    rows.append(np.full(dim, 3e38))
    sub = rng.standard_normal(dim) * 1e-39            # fp32 subnormal components
    rows.append(sub)
    return np.asarray(rows, np.float64).astype(np.float32)


@pytest.mark.parametrize("dim", [300, 384, 768, 1024])
def test_scaling_keeps_every_row_in_range_and_within_rho(dim):
    rng = np.random.default_rng(dim)
    x = _extreme_rows(rng, dim)
    assert np.all(np.isfinite(x)) and np.all(np.abs(x).max(axis=1) > 0)
    h, s = f16_operand(x)
    hm = np.abs(h.astype(np.float64)).max(axis=1)
    assert np.all(np.isfinite(h.astype(np.float64)))
    assert np.all((hm >= 2.0 ** 14) & (hm <= 2.0 ** 15)), hm          # the largest component: fp16 normal, no overflow
    r = rho64(x, f16_value(x))
    assert np.all(r <= RHO_F16), (r.max(), RHO_F16)


def test_midpoints_round_to_even_and_reach_the_bound():
    v = np.full((1, 768), np.float32(1.0 + 2.0 ** -11))              # scaled by 2^14: exactly half an fp16 ulp
    h, s = f16_operand(v)
    assert s[0] == 14 and np.all(h.astype(np.float64) == 2.0 ** 14)  # ties to even: down
    r = rho64(v, f16_value(v))[0]
    assert 2.0 ** -11 * 0.99 <= r <= RHO_F16


def test_zero_row_and_subnormal_tail():
    z = np.zeros((1, 384), np.float32)
    h, s = f16_operand(z)
    assert s[0] == 0 and not np.any(h)
    x = np.zeros((1, 1024), np.float32)
    x[0, 0] = 1.0
    x[0, 1:] = 2.0 ** -40                             # 2^-26 once scaled: below half of fp16's smallest subnormal
    h, s = f16_operand(x)
    assert s[0] == 14 and np.count_nonzero(h) == 1
    assert rho64(x, f16_value(x))[0] <= 2.0 ** -34     # sqrt(1023) 2^-40: inside the subnormal term of RHO_F16


@pytest.mark.parametrize("dim", [384, 768, 1024])
def test_cosine_error_bound_holds_on_random_and_scaled_rows(dim):
    rng = np.random.default_rng(dim + 1)
    x = (rng.standard_normal((3000, dim)) * np.exp(3 * rng.standard_normal((3000, 1)))).astype(np.float32)
    q = (rng.standard_normal((4, dim)) * np.array([[1e-6], [1.0], [1e6], [3e20]])).astype(np.float32)
    xa, qa = f16_value(x), f16_value(q)
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    err = np.abs(qa @ xa.T - q64 @ x64.T) / (np.linalg.norm(q64, axis=1)[:, None] * np.linalg.norm(x64, axis=1)[None, :])
    assert err.max() <= 2 * RHO_F16 + RHO_F16 ** 2
    # the measured error is well below tf32's (the fp32 sweep without the copy)
    xt, qt = tf32_trunc(x).astype(np.float64), tf32_trunc(q).astype(np.float64)
    err_t = np.abs(qt @ xt.T - q64 @ x64.T) / (np.linalg.norm(q64, axis=1)[:, None] * np.linalg.norm(x64, axis=1)[None, :])
    assert err.max() < err_t.max()


def test_selection_rule_is_exact_on_near_duplicate_clusters():
    """400 rows within ~1e-3 of each other around the query: the whole cluster falls inside the 2 eps window and is
    re-scored; the rule returns the exact top-10, and fewer rows are re-scored than with the tf32 bound."""
    rng = np.random.default_rng(7)
    d, n = 768, 20000
    cent = rng.standard_normal(d).astype(np.float32)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[:400] = cent + 0.1 * rng.standard_normal((400, d)).astype(np.float32)
    q = (cent + 0.3 * rng.standard_normal(d)).astype(np.float32)[None, :]
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    norms = np.linalg.norm(x64, axis=1) * np.linalg.norm(q64)
    exact = (x64 @ q64.T)[:, 0] / norms
    approx = (f16_value(x) @ f16_value(q).T)[:, 0] / norms
    c = _constants()
    eps = c["EPS_F16"]
    assert np.abs(approx - exact).max() <= eps
    top, n_cand = _select_exact_topk(approx, exact, 10, eps)
    assert set(top.tolist()) == set(np.argsort(-exact)[:10].tolist())
    assert 100 <= n_cand <= 400
    approx_t = (tf32_trunc(x).astype(np.float64) @ tf32_trunc(q).astype(np.float64).T)[:, 0] / norms
    _, n_cand_t = _select_exact_topk(approx_t, exact, 10, c["EPS_TF32"])
    assert n_cand <= n_cand_t
    top, n_cand = _select_exact_topk(approx[400:], exact[400:], 10, eps)
    assert set(top.tolist()) == set(np.argsort(-exact[400:])[:10].tolist()) and n_cand < 200
