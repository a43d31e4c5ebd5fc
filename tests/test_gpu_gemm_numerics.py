"""K2's kernels one at a time, through the test-only harness in tests/kernels (libgemm_harness.so, built by
__graft_entry__.build()), against numpy restatements.

* The sweep (emb_gemm_kernel<BF16, DUMP = true>) dumps every approximate score it computes.  Compared with a
  float64 emulation of the tensor core's operands, a wrong wgmma fragment mapping, smem descriptor, K-advance
  inside the swizzle atom, warpgroup offset or ring phase shows up as an O(1) error at some (query, row).
* The exactness proof of the merge rests on |approx - exact| <= eps_v for every (query, row); eps_v comes from
  gemm_thr_kernel.  That is checked here on the hardware, on inputs built to make the tensor core's rounding
  as large as possible, and the measured ratios are printed.
* The merge and threshold kernels run on candidate lists / group maxima built here, and are compared with
  the merge rule restated in numpy (test_proof_bounds._select_exact_topk, plus the fp32 window cut)."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import assert_topk_equal
from test_proof_bounds import ACC_TC, _constants, bf16_rn, tf32_trunc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "kernels", "libgemm_harness.so")
CONST = _constants()
SENTINEL = np.uint32(0xFFBADBAD)          # a NaN payload the kernels never produce


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class Harness:
    def __init__(self, path):
        if not os.path.exists(path):
            raise RuntimeError(f"{path} is missing: run __graft_entry__.build()")
        L = C.CDLL(path)
        vp, u32, u64, f32, i32, sz = C.c_void_p, C.c_uint32, C.c_uint64, C.c_float, C.c_int, C.c_size_t
        L.h_last_error.restype = C.c_char_p
        L.h_constants.argtypes = [vp]
        L.h_constants.restype = None
        L.h_prep_queries.argtypes = [vp, u32, u32, u32, vp, vp, vp]
        L.h_gemm_dump.argtypes = [vp, vp, u64, u32, i32, vp, u32, u32, vp, sz]
        L.h_gemm_thr.argtypes = [vp, u32, u32, u32, vp, f32, vp, vp, vp, vp]
        L.h_gemm_merge.argtypes = [vp, vp, u32, u32, u32, vp, vp, u32, vp, u32, vp, i32, u64, u32, vp, vp, vp, i32, f32,
                                   vp, vp, vp, vp, vp, vp, vp]
        self.L = L
        c = np.zeros(10, np.uint32)
        L.h_constants(_p(c))
        (self.M, self.N, self.KB, self.STAGES, self.LIST_CAP, self.OVF_CAP, self.MERGE_BUF, self.MAX_RESCORE,
         self.MAX_LIMIT, self.LISTS_PER_CTA) = (int(v) for v in c)

    def _check(self, rc):
        assert rc == 0, self.L.h_last_error().decode()

    def prep(self, q, stride):
        q = np.ascontiguousarray(q, np.float32)
        nq, dim = q.shape
        pad = np.zeros((nq, stride), np.float32)
        iqn, rho = np.zeros(nq, np.float32), np.zeros(nq, np.float32)
        self._check(self.L.h_prep_queries(_p(q), dim, stride, nq, _p(pad), _p(iqn), _p(rho)))
        return pad, iqn, rho

    def dump(self, rows, inv_norm, q_operand, B, bf16, cpg=0):
        """rows [n][stride] (float32, or uint16 bf16 bits), q_operand [Bpad][stride] of the same type.  Returns the
        whole dump buffer ([Bpad * n + 256] floats as uint32 bits, SENTINEL where nothing was written)."""
        n, stride = rows.shape
        assert q_operand.shape[0] % self.M == 0 and q_operand.shape[0] >= B
        buf = np.full(q_operand.shape[0] * n + 256, SENTINEL, np.uint32)
        self._check(self.L.h_gemm_dump(_p(np.ascontiguousarray(rows)), _p(np.ascontiguousarray(inv_norm, np.float32)), n,
                                       stride, int(bf16), _p(np.ascontiguousarray(q_operand)), B, cpg, _p(buf), buf.size))
        return buf

    def thr(self, gmax, limit, inv_qnorm, eps_const, rho_q=None):
        gmax = np.ascontiguousarray(gmax, np.float32)
        B, lists = gmax.shape
        thr, eps, ovf = np.zeros(B, np.uint32), np.zeros(B, np.float32), np.zeros(B, np.uint32)
        rq = None if rho_q is None else np.ascontiguousarray(rho_q, np.float32)
        self._check(self.L.h_gemm_thr(_p(gmax), B, lists, limit, _p(np.ascontiguousarray(inv_qnorm, np.float32)),
                                      eps_const, _p(rq), _p(thr), _p(eps), _p(ovf)))
        return thr, eps, ovf

    def merge(self, cand, cand_cnt, ovf, ovf_cnt, eps_v, limit, rows, inv_norm, q_pad, iqn, bf16=False, similarity=-2.0):
        B, n_lists, cap = cand.shape
        n, stride = rows.shape
        out = dict(doc=np.zeros((B, limit), np.uint64), score=np.zeros((B, limit), np.float32),
                   row=np.zeros((B, limit), np.uint32), raw=np.zeros((B, limit), np.float32),
                   count=np.zeros(B, np.uint32), unproven=np.zeros(B, np.uint8), rescored=np.zeros(B, np.uint32))
        a = [np.ascontiguousarray(x) for x in (cand, cand_cnt, ovf, ovf_cnt)]
        self._check(self.L.h_gemm_merge(
            _p(a[0]), _p(a[1]), B, n_lists, cap, _p(a[2]), _p(a[3]), ovf.shape[1],
            _p(np.ascontiguousarray(eps_v, np.float32)), limit, _p(np.ascontiguousarray(rows)), int(bf16), n, stride,
            _p(np.ascontiguousarray(inv_norm, np.float32)), _p(np.ascontiguousarray(q_pad, np.float32)),
            _p(np.ascontiguousarray(iqn, np.float32)), 0, similarity,
            _p(out["doc"]), _p(out["score"]), _p(out["row"]), _p(out["raw"]), _p(out["count"]), _p(out["unproven"]),
            _p(out["rescored"])))
        return out


@pytest.fixture(scope="session")
def harness():
    return Harness(HARNESS)


# ---------------------------------------------------------------- numpy restatements
def f32_ordered(s):
    u = np.ascontiguousarray(np.asarray(s, np.float32) + np.float32(0)).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def f32_unordered(o):
    o = np.asarray(o, np.uint32)
    u = np.where(o & np.uint32(0x80000000), o & np.uint32(0x7FFFFFFF), ~o).astype(np.uint32)
    return u.view(np.float32)


def make_key(score, idx):
    return (f32_ordered(score).astype(np.uint64) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - np.asarray(idx, np.uint64))


def key_score(k):
    return f32_unordered((np.asarray(k, np.uint64) >> np.uint64(32)).astype(np.uint32))


def key_idx(k):
    return (np.uint64(0xFFFFFFFF) - (np.asarray(k, np.uint64) & np.uint64(0xFFFFFFFF))).astype(np.int64)


def inv_norms(rows64):
    """1 / |x| as fp32, 0 where |x|^2 is 0 in fp32 (as emb_inv_norm_kernel: a subnormal row has no direction)"""
    s = np.float32((rows64 * rows64).sum(1)).astype(np.float64)
    return np.where(s > 0, 1.0 / np.sqrt(np.where(s > 0, s, 1.0)), 0.0).astype(np.float32)


def tf32_rne(a):
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = (u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000
    return r.astype(np.uint32).view(np.float32)


def tf32_rna(a):
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x1000) & 0xFFFFE000).astype(np.uint32).view(np.float32)


TF32_MODES = {"truncate": tf32_trunc, "round-nearest-even": tf32_rne, "round-nearest-away": tf32_rna}


def pad_rows(x, stride):
    out = np.zeros((x.shape[0], stride), np.float32)
    out[:, :x.shape[1]] = x
    return out


def stride_of(dim):
    s = (dim + 127) // 128
    return 128 * (s + 1 if s in (5, 7) else s)


def run_sweep(h, x, q, bf16, tf32_op, cpg=0, dead=()):
    """x [n][dim], q [B][dim] float32 -> (approx [B][n], emulation [B][n], sum|p~| * inv_norm [B][n], exact64 [B][n],
    inv_norm, raw dump bits).  Dead rows get a NaN inverse norm (a tombstone)."""
    n, dim = x.shape
    B = q.shape[0]
    stride = stride_of(dim)
    Bpad = (B + h.M - 1) // h.M * h.M
    xs = pad_rows(bf16_rn(x) if bf16 else x, stride)
    inv = inv_norms(xs.astype(np.float64))
    inv_dev = inv.copy()
    inv_dev[list(dead)] = np.nan
    qp = np.zeros((Bpad, stride), np.float32)
    qp[:B] = pad_rows(q, stride)
    if bf16:
        rows_op = (xs.view(np.uint32) >> 16).astype(np.uint16)
        q_op = (bf16_rn(qp).view(np.uint32) >> 16).astype(np.uint16)
        xt, qt = xs.astype(np.float64), bf16_rn(qp[:B]).astype(np.float64)
    else:
        rows_op, q_op = xs, qp
        xt, qt = tf32_op(xs).astype(np.float64), tf32_op(qp[:B]).astype(np.float64)
    buf = h.dump(rows_op, inv_dev, q_op, B, bf16, cpg)
    approx = buf[:B * n].view(np.float32).reshape(B, n).astype(np.float64)
    inv64 = inv.astype(np.float64)[None, :]
    emu = (qt @ xt.T) * inv64
    mag = (np.abs(qt) @ np.abs(xt).T) * inv64
    exact = (qp[:B].astype(np.float64) @ xs.astype(np.float64).T) * inv64
    return approx, emu, mag, exact, inv, buf


def check_dump(h, buf, approx, B, n, dead):
    bits = buf.view(np.uint32)
    assert np.all(bits[B * n:] == SENTINEL), "the sweep wrote past the live (query, row) range"
    written = bits[:B * n].reshape(B, n)
    assert not np.any(written == SENTINEL), "some live (query, row) score was never written"
    live = np.ones(n, bool)
    live[list(dead)] = False
    assert np.all(np.isnan(approx[:, ~live])), "tombstoned rows must come out as NaN"
    assert not np.any(np.isnan(approx[:, live]))
    return live


# ---------------------------------------------------------------- 1. layout and tf32 rounding
@pytest.fixture(scope="session")
def tf32_mode(harness):
    """Which rounding the tensor core applies to fp32 operands of a .tf32 wgmma: a probe whose every row holds one
    value whose low 13 mantissa bits sit just below, at and just above the rounding midpoint, in either operand."""
    lows = np.array([0x0FFF, 0x1000, 0x1001, 0x1FFF, 0x3000, 0x2FFF], np.uint32)
    vals = ((np.uint32(0x3F800000) | lows).view(np.float32)).astype(np.float32)
    vals = np.concatenate([vals, -vals])
    n = 128
    x = np.zeros((n, 128), np.float32)
    x[:vals.size, 0] = vals
    x[vals.size:, 0] = 1.0
    qpad = np.zeros((harness.M, 128), np.float32)
    qpad[:8, 0] = 1.0
    # rows carry the pattern (B operand)
    b = harness.dump(x, np.ones(n, np.float32), qpad, 8, False)[:8 * n].view(np.float32).reshape(8, n)[0, :vals.size]
    # the query carries the pattern (A operand): query i = vals[i] in element 0, every row = 1.0
    qa = np.zeros((harness.M, 128), np.float32)
    qa[:vals.size, 0] = vals
    xa = np.zeros((n, 128), np.float32)
    xa[:, 0] = 1.0
    a = harness.dump(xa, np.ones(n, np.float32), qa, vals.size, False)[:vals.size * n].view(np.float32).reshape(vals.size, n)[:, 0]
    found = [m for m, f in TF32_MODES.items() if np.array_equal(f(vals), b) and np.array_equal(f(vals), a)]
    print(f"\n[tf32] tensor core operand rounding: {found or 'unknown'}; "
          f"inputs {[hex(v) for v in vals.view(np.uint32)]} -> B {[hex(v) for v in b.view(np.uint32)]} "
          f"A {[hex(v) for v in a.view(np.uint32)]}")
    assert len(found) == 1, (vals, a, b)
    return found[0]


def test_tf32_operand_rounding_is_known_and_covered_by_eps(tf32_mode):
    """GEMM_EPS_TF32 takes rho <= 2^-10 per operand: truncation's worst case, which bounds rounding to nearest too."""
    assert tf32_mode in TF32_MODES
    v = np.full(768, np.uint32(0x3F801FFF)).view(np.float32)
    f = TF32_MODES[tf32_mode]
    assert np.abs(f(v).astype(np.float64) - v).max() / np.abs(v).max() <= 2.0 ** -10


LAYOUT_DIMS = [100, 128, 256, 384, 512, 640, 768, 896, 1024]


@pytest.mark.parametrize("dim", LAYOUT_DIMS)
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("B", [8, 64, 128, 129, 300])
def test_sweep_scores_match_the_emulated_tensor_core(harness, tf32_mode, dim, dtype, B):
    """Every approximate score of the sweep equals the float64 emulation of the tensor core's operands within the
    accumulation bound.  4 CTAs per query group: each sweeps 3 row tiles, so the ring's phases cross tile
    boundaries (bf16 stride 128 has 2 K-blocks per tile for 4 stages); the last tile is partial."""
    bf16 = dtype == "bf16"
    rng = np.random.default_rng(dim * 1000 + B + bf16)
    n = 11 * 128 + 37
    x = rng.standard_normal((n, dim)).astype(np.float32) * np.exp(rng.standard_normal((n, 1))).astype(np.float32)
    q = rng.standard_normal((B, dim)).astype(np.float32)
    dead = rng.choice(n, 20, replace=False)
    for cpg in (4, 0):
        approx, emu, mag, _, _, buf = run_sweep(harness, x, q, bf16, TF32_MODES[tf32_mode], cpg=cpg, dead=dead)
        live = check_dump(harness, buf, approx, B, n, dead)
        err = np.abs(approx - emu)[:, live]
        tol = ACC_TC * mag[:, live] + 4 * np.spacing(np.abs(emu[:, live]).astype(np.float32)).astype(np.float64)
        bad = np.argwhere(err > tol)
        assert bad.size == 0, (f"cpg={cpg}: {bad.shape[0]} scores off, first (q, live row) {bad[:5].tolist()}",
                               err[tuple(bad[0])], tol[tuple(bad[0])])


# ---------------------------------------------------------------- 2. the proof's premise on adversarial inputs
def _adversarial(case, dtype, rng):
    """-> (rows [n][dim], queries [B][dim]) float32"""
    n, B = 1061, 16
    if case == "aligned_truncation":
        dim = 768
        v = np.full(dim, np.uint32(0x3F801FFF)).view(np.float32)
        x = np.tile(v, (n, 1))
        x[1::2] *= -1.0
        x[::3, ::2] = np.full(dim // 2, np.uint32(0x3FFFFFFF)).view(np.float32)   # 2 - 2^-23: low bits all set
        q = np.tile(v, (B, 1))
        q[1::2, ::3] = np.full(q[1::2, ::3].shape, np.uint32(0x3F9FFFFF)).view(np.float32)
        return x, q
    if case == "cancellation":
        dim = 1024
        q = (rng.choice([-1.0, 1.0], (B, dim)) * 2.0 ** rng.uniform(-20, 20, (B, dim)) *
             (1 + rng.random((B, dim)))).astype(np.float32)
        x = (q[rng.integers(0, B, n)] * rng.choice([-1.0, 1.0], (n, dim))).astype(np.float32)
        return x, q
    if case == "dominant_per_k_group":
        dim = 1024
        g = 16 if dtype == "bf16" else 8
        x = rng.uniform(0.5, 1.0, (n, dim)).astype(np.float32)
        q = rng.uniform(0.5, 1.0, (B, dim)).astype(np.float32)
        pos = np.arange(0, dim, g) + rng.integers(0, g, dim // g)
        x[:, pos] = 2.0 ** 12 * (1 + rng.random((n, pos.size))).astype(np.float32)
        x[:, pos[1::2]] = -x[:, pos[::2]]                   # the dominant products cancel pairwise
        q[:, pos] = 1.0
        return x, q
    if case == "all_positive":
        dim = 1024
        return rng.random((n, dim)).astype(np.float32) + 0.01, rng.random((B, dim)).astype(np.float32) + 0.01
    if case == "worst_case_rho_query":
        dim = 768
        x = rng.standard_normal((n, dim)).astype(np.float32)
        q = np.full((B, dim), np.float32(1.0 + 2.0 ** -8 - 2.0 ** -20), np.float32)
        q[:, 1::2] *= -1.0
        q[1::2] *= np.float32(3.0)
        return x, q
    if case == "zero_query_and_subnormals":
        dim = 384
        x = rng.standard_normal((n, dim)).astype(np.float32)
        x[::5, ::7] = np.float32(3e-39)                      # subnormal components
        x[7] = np.float32(1e-40)                             # a whole subnormal row: |x|^2 underflows -> inv norm 0
        q = rng.standard_normal((B, dim)).astype(np.float32)
        q[0] = 0.0
        q[1, ::2] = np.float32(2e-39)
        q[2] = np.float32(5e-41)                             # |q|^2 underflows: treated like the zero query
        return x, q
    raise KeyError(case)


ADVERSARIAL = ["aligned_truncation", "cancellation", "dominant_per_k_group", "all_positive", "worst_case_rho_query",
               "zero_query_and_subnormals"]


@pytest.mark.parametrize("case", ADVERSARIAL)
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_sweep_error_stays_within_eps(harness, tf32_mode, case, dtype):
    """|approx - exact| <= eps_v for every (query, row): eps_v as gemm_thr_kernel computes it from the library's
    own query preparation, exact in float64 from the unrounded operands (the stored rows, the fp32 query)."""
    bf16 = dtype == "bf16"
    rng = np.random.default_rng(abs(hash((case, dtype))) % 2 ** 32)
    x, q = _adversarial(case, dtype, rng)
    B, dim = q.shape
    stride = stride_of(dim)
    _, iqn, rho = harness.prep(q, stride)
    eps_const = CONST["EPS_ACC"] if bf16 else CONST["EPS_TF32"]
    _, eps_v, _ = harness.thr(np.zeros((B, 4), np.float32), 1, iqn, eps_const, rho if bf16 else None)
    approx, emu, mag, exact, inv, _ = run_sweep(harness, x, q, bf16, TF32_MODES[tf32_mode])
    zero_q = iqn == 0
    assert np.all(np.isinf(eps_v[zero_q])) and np.all(np.isfinite(eps_v[~zero_q]))
    if case == "zero_query_and_subnormals":
        assert zero_q[0] and zero_q[2]
    assert not np.any(np.isnan(approx))
    err = np.abs(approx - exact)
    ratio = (err / eps_v[:, None].astype(np.float64))[~zero_q]
    with np.errstate(invalid="ignore", divide="ignore"):
        # queries whose |q|^2 underflows are left out: eps_v = inf sends them to the exact sweep whatever the sweep does
        acc = np.where(mag > 0, np.abs(approx - emu) / mag, 0.0)[~zero_q]
    print(f"\n[eps] {case:26s} {dtype:4s} max |approx-exact|/eps_v = {ratio.max():.4f}   "
          f"max |approx-emu|/(sum|p~| inv_norm) = {acc.max():.3e} = {acc.max() / ACC_TC:.4f} x 1024*2^-23")
    assert ratio.max() <= 1.0, (case, dtype, ratio.max())
    assert acc.max() <= ACC_TC, (case, dtype, acc.max())


# ---------------------------------------------------------------- 3. the merge kernel
@pytest.fixture(scope="module")
def store():
    """8000 fp32 rows (dim 128; rows 100..139 are copies of row 7), 2 queries (query 1 = row 7)."""
    rng = np.random.default_rng(42)
    n, dim = 8000, 128
    x = rng.standard_normal((n, dim)).astype(np.float32)
    x[100:140] = x[7]
    q = rng.standard_normal((2, dim)).astype(np.float32)
    q[1] = x[7] * np.float32(2.0)
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    inv = inv_norms(x64)
    cos = (q64 @ x64.T) * inv[None, :].astype(np.float64) / np.linalg.norm(q64, axis=1)[:, None]
    return x, q, inv, cos


def _lists(keys_per_query, n_lists, cap, rng):
    """Spread each query's keys over n_lists lists (<= cap each) in random order."""
    B = len(keys_per_query)
    cand = np.zeros((B, n_lists, cap), np.uint64)
    cnt = np.zeros((B, n_lists), np.uint32)
    for b, keys in enumerate(keys_per_query):
        keys = rng.permutation(keys)
        assert keys.size <= n_lists * cap
        owner = np.sort(rng.integers(0, n_lists, keys.size))
        for l in range(n_lists):
            mine = keys[owner == l]
            assert mine.size <= cap, "unlucky spread"
            cand[b, l, :mine.size] = mine
            cnt[b, l] = mine.size
    return cand, cnt


def _merge_ref(keys, limit, eps_v, cos, lost=False):
    """The merge rule: a_lim = limit-th best gathered approximate score; every gathered row with
    approx >= a_lim - 2 eps (fp32) is re-scored exactly; the best `limit` exact scores win (ties: lower row)."""
    s = key_score(keys)
    if keys.size >= limit:
        a_lim = np.sort(s)[-limit]
        cut = np.float32(a_lim) - np.float32(2.0) * np.float32(eps_v)
    else:
        cut = np.float32(-np.inf)
    staged = key_idx(keys[s >= cut])
    order = staged[np.lexsort((staged, -cos[staged]))]
    unproven = lost or staged.size > 2048
    return order[:limit], staged.size, unproven


def _approx_keys(rows, cos_q, qn, eps_v, rng, spread=0.5):
    """Approximate keys (cos*|q| units) of the given rows, off the exact score by up to spread * eps_v."""
    a = (cos_q[rows] * qn + rng.uniform(-spread, spread, rows.size) * eps_v).astype(np.float32)
    return make_key(a, rows)


def _run_merge(harness, store, keys_q, limit, eps_cos, n_lists=64, ovf_keys=None, ovf_cnt=None, lost=False, seed=0):
    x, q, inv, cos = store
    rng = np.random.default_rng(seed)
    B = len(keys_q)
    q_pad, iqn, _ = harness.prep(q[:B], 128)
    qn = 1.0 / iqn.astype(np.float64)
    eps_v = (np.float32(eps_cos) / iqn).astype(np.float32)
    cand, cnt = _lists(keys_q, n_lists, harness.LIST_CAP, rng)
    ovf = np.zeros((B, harness.OVF_CAP), np.uint64)
    oc = np.zeros(B, np.uint32) if ovf_cnt is None else np.asarray(ovf_cnt, np.uint32)
    if ovf_keys is not None:
        for b, k in enumerate(ovf_keys):
            ovf[b, :k.size] = k
            if ovf_cnt is None:
                oc[b] = k.size
    out = harness.merge(cand, cnt, ovf, oc, eps_v, limit, x, inv, q_pad, iqn)
    return out, eps_v, qn


def _check_against_ref(out, b, gathered, limit, eps_v, cos, lost=False):
    top, n_staged, unproven = _merge_ref(gathered, limit, eps_v, cos, lost)
    assert bool(out["unproven"][b]) == unproven, (out["unproven"][b], unproven, n_staged)
    assert out["rescored"][b] == min(n_staged, 2048)
    if unproven:
        return n_staged
    c = int(out["count"][b])
    assert c == top.size
    got = out["row"][b, :c].astype(np.int64)
    assert np.array_equal(out["doc"][b, :c], got.astype(np.uint64))
    assert np.all(np.diff(out["score"][b, :c]) <= 0)
    assert_topk_equal(got, out["score"][b, :c], top, cos[top], atol=2e-6, tie_eps=2e-6)
    assert np.all(out["row"][b, c:] == 0xFFFFFFFF) and np.all(out["score"][b, c:] == 0)
    return n_staged


def test_merge_streams_more_than_the_shared_buffer_and_keeps_the_result(harness, store):
    """5120 listed + 300 spilled keys (> GEMM_MERGE_BUF): the streaming path; a few dozen inside the 2 eps window,
    so the query is proven and its result is the one returned."""
    x, q, inv, cos = store
    rng = np.random.default_rng(1)
    rows = rng.permutation(np.arange(140, 8000))[:5420]
    _, iqn, _ = harness.prep(q[:1], 128)
    qn = 1.0 / float(iqn[0])
    eps_v = np.float32(np.float32(0.02) / iqn[0])
    keys = _approx_keys(rows, cos[0], qn, float(eps_v), rng)
    assert keys.size > harness.MERGE_BUF
    out, ev, _ = _run_merge(harness, store, [keys[:5120]], 10, 0.02, n_lists=64, ovf_keys=[keys[5120:]], seed=1)
    n_staged = _check_against_ref(out, 0, keys, 10, ev[0], cos[0])
    assert 10 < n_staged <= 2048 and out["unproven"][0] == 0
    print(f"\n[merge] streaming path: {keys.size} gathered keys, {n_staged} re-scored")


def test_merge_flags_a_lost_spill(harness, store):
    x, q, inv, cos = store
    rng = np.random.default_rng(2)
    _, iqn, _ = harness.prep(q[:1], 128)
    rows = np.arange(200, 1200)
    keys = _approx_keys(rows, cos[0], 1.0 / float(iqn[0]), 0.02 / float(iqn[0]), rng)
    out, ev, _ = _run_merge(harness, store, [keys], 10, 0.02, ovf_keys=[keys[:10]], ovf_cnt=[harness.OVF_CAP + 1])
    assert out["unproven"][0] == 1


def test_merge_flags_a_window_larger_than_the_rescore_budget(harness, store):
    """3000 distinct rows with one approximate score: all inside the window -> more than GEMM_MAX_RESCORE."""
    x, q, inv, cos = store
    rows = np.arange(1000, 4000)
    keys = make_key(np.full(rows.size, 0.5, np.float32), rows)
    out, ev, _ = _run_merge(harness, store, [keys], 10, 1e-3, n_lists=64)
    _check_against_ref(out, 0, keys, 10, ev[0], cos[0])
    assert out["unproven"][0] == 1 and out["rescored"][0] == harness.MAX_RESCORE


def test_merge_with_fewer_keys_than_limit(harness, store):
    x, q, inv, cos = store
    rng = np.random.default_rng(3)
    _, iqn, _ = harness.prep(q[:1], 128)
    rows = np.array([5, 999, 3000, 7999, 4242])
    keys = _approx_keys(rows, cos[0], 1.0 / float(iqn[0]), 0.02 / float(iqn[0]), rng)
    out, ev, _ = _run_merge(harness, store, [keys], 10, 0.02, n_lists=8)
    _check_against_ref(out, 0, keys, 10, ev[0], cos[0])
    assert out["count"][0] == 5 and out["unproven"][0] == 0


def test_merge_resolves_exact_ties_to_the_lowest_rows(harness, store):
    """Query 1 is row 7 (x2); rows 100..139 are copies of row 7: 41 rows tie exactly at cos 1."""
    x, q, inv, cos = store
    rng = np.random.default_rng(4)
    rows = np.concatenate([[7], np.arange(100, 140), rng.choice(np.arange(140, 8000), 500, replace=False)])
    _, iqn, _ = harness.prep(q[:2], 128)
    keys = [_approx_keys(rows, cos[b], 1.0 / float(iqn[b]), 0.001 / float(iqn[b]), rng) for b in range(2)]
    out, ev, _ = _run_merge(harness, store, keys, 32, 0.001, n_lists=16)
    for b in range(2):
        _check_against_ref(out, b, keys[b], 32, ev[b], cos[b])
    assert out["row"][1, :32].tolist() == [7] + list(range(100, 131))
    assert np.all(out["score"][1, :32] == out["score"][1, 0])


def test_merge_gathers_512_lists(harness, store):
    x, q, inv, cos = store
    rng = np.random.default_rng(5)
    _, iqn, _ = harness.prep(q[:2], 128)
    keys = []
    for b in range(2):
        rows = rng.choice(np.arange(140, 8000), 3000, replace=False)
        keys.append(_approx_keys(rows, cos[b], 1.0 / float(iqn[b]), 0.005 / float(iqn[b]), rng))
    out, ev, _ = _run_merge(harness, store, keys, 128, 0.005, n_lists=512, seed=5)
    for b in range(2):
        _check_against_ref(out, b, keys[b], 128, ev[b], cos[b])
        assert out["unproven"][b] == 0 and out["count"][b] == 128


# ---------------------------------------------------------------- 4. the threshold kernel
def _fdiv_ru(a, b):
    r = np.float32(np.float64(a) / np.float64(b))
    return r if np.float64(r) >= np.float64(a) / np.float64(b) else np.nextafter(r, np.float32(np.inf))


def test_threshold_kernel(harness):
    rng = np.random.default_rng(6)
    B, lists, limit = 5, 96, 10
    gmax = rng.standard_normal((B, lists)).astype(np.float32)
    gmax[0, ::3] = -np.inf
    gmax[0, 1::7] = np.nan
    gmax[1, :] = -np.inf
    gmax[1, :limit - 1] = rng.standard_normal(limit - 1)           # fewer live lists than limit
    gmax[2, :] = np.nan
    gmax[2, 50:50 + limit] = 0.25                                   # exactly limit live lists, tied
    iqn = np.array([0.5, 0.5, 2.0, 0.0, 1.0 / 3.0], np.float32)     # query 3: the zero query
    rho = np.array([1e-3, 5e-3, 0.0, 0.0, 2e-3], np.float32)        # query 1: above the worst case (capped)
    for eps_const, rq in ((CONST["EPS_TF32"], None), (CONST["EPS_ACC"], rho)):
        thr, eps, ovf = harness.thr(gmax, limit, iqn, eps_const, rq)
        assert np.all(ovf == 0)
        for b in range(B):
            r = np.float32(0) if rq is None else np.minimum(rq[b], np.float32(CONST["RHO_BF16_WORST"]))
            e_cos = np.float32(eps_const) + r
            ev = _fdiv_ru(e_cos, iqn[b]) if iqn[b] > 0 else np.float32(np.inf)
            assert eps[b] == ev, (b, eps[b], ev)
            valid = np.sort(gmax[b][np.isfinite(gmax[b])])[::-1]
            if valid.size >= limit and np.isfinite(ev):
                t = np.float32(valid[limit - 1]) - np.float32(2.0) * ev
            else:
                t = np.float32(-np.inf)
            assert thr[b] == f32_ordered(t), (b, f32_unordered(thr[b]), t)
        assert f32_unordered(thr[1]) == -np.inf and f32_unordered(thr[3]) == -np.inf
        assert np.isfinite(f32_unordered(thr[2]))
