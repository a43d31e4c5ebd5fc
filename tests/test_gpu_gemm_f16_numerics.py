"""The fp16 sweep of an fp32 store (emb_gemm_kernel<GEMM_F16>) one kernel at a time, through the fp16 kernel test
harness (tests/kernels/libgemm_f16_harness.so, next to libgemm_harness.so for the query preparation):

* the operands: emb_f16_rows_kernel / emb_f16_queries_kernel produce, bit for bit, the power-of-two scaled,
  round-to-nearest fp16 copy that test_proof_bounds_f16 restates in numpy, with the same scales;
* the sweep's approximate scores equal the float64 emulation of those operands within the accumulation bound;
* |approx - exact| <= eps_v for every (query, row), eps_v as gemm_thr_kernel computes it for the fp16 sweep (in the
  sweep's units, cos * |q| * 2^e_q), on adversarial inputs and on rows of extreme norm; the worst ratio is printed."""
import ctypes as C
import os

import numpy as np
import pytest

from test_gpu_gemm_numerics import (ADVERSARIAL, CONST, HARNESS, ROOT, SENTINEL, Harness, _adversarial, _p, check_dump,
                                    inv_norms, pad_rows, stride_of)
from test_proof_bounds import ACC_TC
from test_proof_bounds_f16 import f16_operand

pytestmark = pytest.mark.gpu

HARNESS_F16 = os.path.join(ROOT, "tests", "kernels", "libgemm_f16_harness.so")


class HarnessF16(Harness):
    def __init__(self, path, path_f16):
        super().__init__(path)
        if not os.path.exists(path_f16):
            raise RuntimeError(f"{path_f16} is missing: run __graft_entry__.build()")
        L = C.CDLL(path_f16)
        vp, u32, u64, f32, i32, sz = C.c_void_p, C.c_uint32, C.c_uint64, C.c_float, C.c_int, C.c_size_t
        L.h16_last_error.restype = C.c_char_p
        L.h16_operands.argtypes = [vp, u64, u32, i32, vp, vp]
        L.h16_gemm_dump.argtypes = [vp, vp, vp, u64, u32, vp, u32, u32, vp, sz]
        L.h16_gemm_thr.argtypes = [vp, u32, u32, u32, vp, f32, vp, vp, vp, vp]
        self.L16 = L

    def _check16(self, rc):
        assert rc == 0, self.L16.h16_last_error().decode()

    def operands(self, v, is_query):
        v = np.ascontiguousarray(v, np.float32)
        n, stride = v.shape
        out, scale = np.zeros((n, stride), np.uint16), np.zeros(n, np.float32)
        self._check16(self.L16.h16_operands(_p(v), n, stride, int(is_query), _p(out), _p(scale)))
        return out, scale

    def dump_f16(self, rows16, inv_norm, row_scale, q16, B, cpg=0):
        n, stride = rows16.shape
        buf = np.full(q16.shape[0] * n + 256, SENTINEL, np.uint32)
        self._check16(self.L16.h16_gemm_dump(_p(np.ascontiguousarray(rows16)), _p(np.ascontiguousarray(inv_norm, np.float32)),
                                             _p(np.ascontiguousarray(row_scale, np.float32)), n, stride,
                                             _p(np.ascontiguousarray(q16)), B, cpg, _p(buf), buf.size))
        return buf

    def thr_f16(self, gmax, limit, inv_qnorm, q_scale):
        gmax = np.ascontiguousarray(gmax, np.float32)
        B, lists = gmax.shape
        thr, eps, ovf = np.zeros(B, np.uint32), np.zeros(B, np.float32), np.zeros(B, np.uint32)
        self._check16(self.L16.h16_gemm_thr(_p(gmax), B, lists, limit, _p(np.ascontiguousarray(inv_qnorm, np.float32)),
                                            CONST["EPS_F16"], _p(np.ascontiguousarray(q_scale, np.float32)), _p(thr), _p(eps),
                                            _p(ovf)))
        return thr, eps, ovf


@pytest.fixture(scope="module")
def h16():
    return HarnessF16(HARNESS, HARNESS_F16)


def _extreme(rng, n, dim):
    x = rng.standard_normal((n, dim))
    x *= (10.0 ** rng.uniform(-30, 30, (n, 1)))                 # norms 1e-30 .. 1e30
    x[::7] *= 2.0 ** (np.arange(dim) % 40 - 20.0)                # components spanning 40 binades
    x[3::11] = 1.0 + 2.0 ** -11                                  # fp16 rounding midpoints once scaled
    x[5::13, ::3] = rng.uniform(65504.0, 1e6, x[5::13, ::3].shape)   # above fp16's largest finite value
    return x.astype(np.float32)


@pytest.mark.parametrize("dim", [300, 384, 768, 1024])
def test_f16_operands_match_numpy(h16, dim):
    rng = np.random.default_rng(dim)
    stride = stride_of(dim)
    x = pad_rows(_extreme(rng, 517, dim), stride)
    x[0] = 0.0
    x[1, 5] = np.inf
    x[2, 7] = np.nan
    for is_query in (0, 1):
        bits, scale = h16.operands(x, is_query)
        h, s = f16_operand(x[3:])
        assert np.array_equal(bits[3:], h.view(np.uint16)), "fp16 copy differs from the numpy restatement"
        want = np.ldexp(np.float64(1.0), s if is_query else -s)
        assert np.array_equal(scale[3:].astype(np.float64), want.astype(np.float32).astype(np.float64))
        assert not np.any(bits[0]) and scale[0] == 1.0                           # zero vector: scale 1, zeros
        assert np.all(np.isnan(bits[1:3].view(np.float16)))                     # non-finite: NaN operand ...
        assert np.all(np.isnan(scale[1:3])) if not is_query else np.all(scale[1:3] == 1.0)   # ... NaN row scale


def _run_f16(h, x, q, cpg=0, dead=()):
    """x [n][dim], q [B][dim] -> (approx [B][n] in the sweep's units, emulation, sum|p~| * inr, exact in the sweep's
    units, q_scale, raw dump)"""
    n, dim = x.shape
    B = q.shape[0]
    stride = stride_of(dim)
    Bpad = (B + h.M - 1) // h.M * h.M
    xs = pad_rows(x, stride)
    qp = np.zeros((Bpad, stride), np.float32)
    qp[:B] = pad_rows(q, stride)
    inv = inv_norms(xs.astype(np.float64))
    inv_dev = inv.copy()
    inv_dev[list(dead)] = np.nan
    rows16, row_scale = h.operands(xs, 0)
    q16, q_scale = h.operands(qp, 1)
    buf = h.dump_f16(rows16, inv_dev, row_scale, q16, B, cpg)
    approx = buf[:B * n].view(np.float32).reshape(B, n).astype(np.float64)
    inr = (inv.astype(np.float64) * row_scale.astype(np.float64))[None, :]
    xt, qt = rows16.view(np.float16).astype(np.float64), q16[:B].view(np.float16).astype(np.float64)
    emu = (qt @ xt.T) * inr
    mag = (np.abs(qt) @ np.abs(xt).T) * inr
    exact = (qp[:B].astype(np.float64) @ xs.astype(np.float64).T) * inv.astype(np.float64)[None, :] \
        * q_scale[:B].astype(np.float64)[:, None]
    return approx, emu, mag, exact, q_scale[:B], buf


@pytest.mark.parametrize("dim", [128, 300, 768, 1024])
@pytest.mark.parametrize("B", [8, 129, 300])
def test_f16_sweep_scores_match_the_emulated_tensor_core(h16, dim, B):
    rng = np.random.default_rng(dim * 1000 + B)
    n = 11 * 128 + 37
    x = rng.standard_normal((n, dim)).astype(np.float32) * np.exp(rng.standard_normal((n, 1))).astype(np.float32)
    q = rng.standard_normal((B, dim)).astype(np.float32)
    dead = rng.choice(n, 20, replace=False)
    for cpg in (4, 0):
        approx, emu, mag, _, _, buf = _run_f16(h16, x, q, cpg=cpg, dead=dead)
        live = check_dump(h16, buf, approx, B, n, dead)
        err = np.abs(approx - emu)[:, live]
        tol = ACC_TC * mag[:, live] + 4 * np.spacing(np.abs(emu[:, live]).astype(np.float32)).astype(np.float64)
        bad = np.argwhere(err > tol)
        assert bad.size == 0, (f"cpg={cpg}: {bad.shape[0]} scores off, first (q, live row) {bad[:5].tolist()}",
                               err[tuple(bad[0])], tol[tuple(bad[0])])


@pytest.mark.parametrize("case", ADVERSARIAL + ["extreme_norms"])
def test_f16_sweep_error_stays_within_eps(h16, case):
    """|approx - exact| <= eps_v (both in the sweep's cos * |q| * 2^e_q units) for every live (query, row)."""
    rng = np.random.default_rng(abs(hash((case, "f16"))) % 2 ** 32)
    if case == "extreme_norms":
        x = _extreme(rng, 1061, 768)
        q = _extreme(rng, 16, 768)
    else:
        x, q = _adversarial(case, "f16", rng)
    B, dim = q.shape
    _, iqn, _ = h16.prep(q, stride_of(dim))
    approx, emu, mag, exact, q_scale, _ = _run_f16(h16, x, q)
    _, eps_v, _ = h16.thr_f16(np.zeros((B, 4), np.float32), 1, iqn, q_scale)
    zero_q = iqn == 0
    assert np.all(np.isinf(eps_v[zero_q])) and np.all(np.isfinite(eps_v[~zero_q]))
    assert not np.any(np.isnan(approx))
    err = np.abs(approx - exact)
    ratio = (err / eps_v[:, None].astype(np.float64))[~zero_q]
    with np.errstate(invalid="ignore", divide="ignore"):
        acc = np.where(mag > 0, np.abs(approx - emu) / mag, 0.0)[~zero_q]
    print(f"\n[eps f16] {case:26s} max |approx-exact|/eps_v = {ratio.max():.4f}   "
          f"max |approx-emu|/(sum|p~| inr) = {acc.max():.3e} = {acc.max() / ACC_TC:.4f} x 1024*2^-23")
    assert ratio.max() <= 1.0, (case, ratio.max())
    assert acc.max() <= ACC_TC, (case, acc.max())
