"""EmbeddingFieldStorage.search_batch against a float64 cosine at every shape the scan kernels are built for.

K1 (emb_scan_kernel<NCH, QB, T>) is instantiated for NCH in {1, 2, 3, 4, 6, 8} x QB in {1, 2, 4} x {fp32, bf16};
K2 (emb_gemm_kernel) runs 2..32 K-blocks per tile.  The dims below reach every NCH, both padded widths (stride
5 -> 6 and 7 -> 8 chunks of 128) and dims that are not a multiple of 4 or 32; the batch sizes reach every QB and
K2 with one, a full, a partial last and several query groups.  Every returned score must be within the rounding
bound of K1's fp32 arithmetic of the float64 cosine of that row (the reference rounds a bf16 store's rows to bf16
first), the hits must be the float64 top-k up to boundary ties within that bound, and wherever K2 ran its output
must equal the exact sweep (OC_DISABLE_GEMM=1) bit for bit."""
import os

import numpy as np
import pytest

import oramacore_b200 as ob
from helpers import assert_topk_equal

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SIM = -2.0                      # below every cosine: counts are min(limit, live rows)
GEMM_MAX_LIMIT = 128
DIMS = [1, 3, 100, 128, 129, 256, 300, 384, 385, 512, 513, 640, 700, 768, 769, 896, 1000, 1023, 1024]


def stride_of(dim):
    s = (dim + 127) // 128
    return 128 * (s + 1 if s in (5, 7) else s)


def uses_gemm(B, limit, n_rows):
    """run_vector_stage's routing rule for the tensor-core scan."""
    return B >= 8 and limit <= GEMM_MAX_LIMIT and n_rows >= max(4096, limit * 256)


def reference(rows, q):
    """float64 cosine [B][n] of the stored values and K1's rounding bound for each (query, row).
    K1: per lane a chain of stride/32 fp32 FMAs, a 5-level shuffle tree, |x| and |q| the same way (then sqrtf and
    a division), two multiplies by the inverse norms, then 1 - (1 - cos)."""
    x64, q64 = rows.astype(np.float64), q.astype(np.float64)
    nx, nq = np.linalg.norm(x64, axis=1), np.linalg.norm(q64, axis=1)
    inx = np.where(nx > 0, 1.0 / np.where(nx > 0, nx, 1.0), 0.0)
    inq = np.where(nq > 0, 1.0 / np.where(nq > 0, nq, 1.0), 0.0)
    cos = (q64 @ x64.T) * inq[:, None] * inx[None, :]
    rel = (np.abs(q64) @ np.abs(x64).T) * inq[:, None] * inx[None, :]      # sum |x_i q_i| / (|x||q|)
    k = stride_of(rows.shape[1]) // 32 + 5
    g = k * U / (1 - k * U)
    tol = (g * rel + (g + 6 * U) * np.abs(cos)) * 1.01 + 3 * U
    return cos, np.minimum(tol, 1e-5)


def check_hits(docs, scores, counts, cos, tol, limit, live=None):
    """counts, sortedness, per-score bound, doc set == float64 top-k up to boundary ties within the bound."""
    B, n = cos.shape
    if live is None:
        live = np.ones(n, bool)
    rows = np.flatnonzero(live)
    want = min(limit, rows.size)
    assert np.all(counts == want), (counts, want)
    for b in range(B):
        d = docs[b, :want].astype(np.int64)
        s = scores[b, :want].astype(np.float64)
        assert np.all(np.diff(s) <= 0), (b, s)
        assert np.all(live[d]), b
        err = np.abs(s - cos[b, d])
        assert np.all(err <= tol[b, d]), (b, d[err > tol[b, d]], err.max())
        c = cos[b, rows]
        top = rows[np.lexsort((rows, -c))[:want]]
        assert_topk_equal(d, s, top, cos[b, top], atol=2 * float(tol[b].max()), tie_eps=2 * float(tol[b].max()))


def search(emb, q, limit, fb=None, nb=0, exact=False):
    if exact:
        os.environ["OC_DISABLE_GEMM"] = "1"
    try:
        out = emb.search_batch(q, limit, SIM, fb, nb)
        t = emb.ctx.last_timing()
    finally:
        os.environ.pop("OC_DISABLE_GEMM", None)
    return out, t


def run_case(emb, q, limit, cos, tol, fb=None, nb=0, live=None):
    n = cos.shape[1]
    (docs, scores, counts), t = search(emb, q, limit, fb, nb)
    assert t["scan_tensor_core"] == int(uses_gemm(q.shape[0], limit, n)), (q.shape[0], limit, n, t)
    check_hits(docs, scores, counts, cos, tol, limit, live)
    if t["scan_tensor_core"]:
        (d2, s2, c2), t2 = search(emb, q, limit, fb, nb, exact=True)
        assert t2["scan_tensor_core"] == 0
        assert np.array_equal(docs, d2) and np.array_equal(scores.view(np.uint32), s2.view(np.uint32)) \
            and np.array_equal(counts, c2)
    return t


def make_store(ctx, dim, dtype, n, seed):
    rng = np.random.default_rng(seed)
    rows = rng.standard_normal((n, dim)).astype(np.float32) * np.exp(0.5 * rng.standard_normal((n, 1))).astype(np.float32)
    if dtype == "bf16":
        rows = ob.from_bf16(ob.to_bf16(rows))
    emb = ob.EmbeddingFieldStorage(ctx, "BGEBase", dim=dim, dtype=dtype)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    return emb, rows, rng


def queries(rows, B, rng):
    """half planted near stored rows, half random"""
    n, dim = rows.shape
    q = rng.standard_normal((B, dim)).astype(np.float32)
    h = B // 2
    q[:h] = rows[rng.integers(0, n, h)] + 0.1 * q[:h] * np.abs(rows).mean()
    return q


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("dim", DIMS)
def test_shape_matrix(gpu_ctx, dim, dtype):
    """n = 4133: not a multiple of 128 nor of any K1 rows-per-stage (a multiple of 8), and K2-eligible for
    limit <= 16.  B 1..7 reach QB 4 / 2 / 1 of K1; B 8..300 reach K2; limits 1, 10, 32, 33 reach both sides of
    the head-merge vs streaming switch of emb_scan_merge_kernel (K2 is not eligible for 32 / 33 at this n)."""
    n = 4133
    emb, rows, rng = make_store(gpu_ctx, dim, dtype, n, seed=dim * 7 + (dtype == "bf16"))
    q_all = queries(rows, 300, rng)
    cos, tol = reference(rows, q_all)
    ran_gemm = False
    for B, limit in [(1, 10), (2, 10), (3, 1), (4, 32), (5, 33), (7, 10),
                     (8, 10), (8, 1), (127, 16), (128, 10), (129, 10), (300, 10), (8, 33), (129, 32)]:
        t = run_case(emb, q_all[:B], limit, cos[:B], tol[:B])
        ran_gemm |= bool(t["scan_tensor_core"])
    assert ran_gemm
    emb.close()


@pytest.mark.parametrize("n,limit,dim", [(4095, 10, 128), (4096, 10, 128), (33 * 256 - 1, 33, 256), (33 * 256, 33, 256),
                                         (128 * 256 - 1, 128, 384), (128 * 256, 128, 384), (129 * 256, 129, 384)])
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_tensor_core_eligibility_edges(gpu_ctx, n, limit, dim, dtype):
    """The two sides of n >= 4096, n >= limit * 256 and limit <= GEMM_MAX_LIMIT (128)."""
    emb, rows, rng = make_store(gpu_ctx, dim, dtype, n, seed=n + limit)
    q = queries(rows, 8, rng)
    cos, tol = reference(rows, q)
    run_case(emb, q, limit, cos, tol)
    emb.close()


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
def test_max_topk_at_dim_1024(gpu_ctx, dtype):
    """limit = OC_MAX_TOPK (1024) at stride 1024: K1's warp buffers leave it only 3 ring stages."""
    n = 5000
    emb, rows, rng = make_store(gpu_ctx, 1024, dtype, n, seed=1024)
    q = queries(rows, 9, rng)
    cos, tol = reference(rows, q)
    for B in (1, 5, 9):
        run_case(emb, q[:B], 1024, cos[:B], tol[:B])
    emb.close()


@pytest.mark.parametrize("dim", [1, 2, 3])
@pytest.mark.parametrize("B", [3, 8])
def test_massive_ties_resolve_to_the_lowest_rows(gpu_ctx, orc, dim, B):
    """At dims 1..3 the rows take a handful of directions (scaled by powers of two, so every cosine of one
    direction is bitwise equal): thousands of rows tie and the hits are the lowest rows of the best direction,
    in row order, as the oracle returns them.  B = 8 at n = 4133 runs K2."""
    n, limit = 4133, 10
    rng = np.random.default_rng(dim * 10 + B)
    # dim 1 has two directions: +1 and -1 (two different positive values would score a few ulp apart)
    dirs = np.array([[1.0], [-1.0]] * 2, np.float32) if dim == 1 else rng.standard_normal((4, dim)).astype(np.float32)
    rows = (dirs[rng.integers(0, 4, n)] * 2.0 ** rng.integers(-3, 4, (n, 1))).astype(np.float32)
    q = np.concatenate([dirs[rng.integers(0, 4, B - 1)], np.zeros((1, dim), np.float32)])   # last: the zero query
    emb = ob.EmbeddingFieldStorage(gpu_ctx, "BGEBase", dim=dim)
    emb.insert_batch(np.arange(n, dtype=np.uint64), rows)
    cos, tol = reference(rows, q)
    t = run_case(emb, q, limit, cos, tol)
    assert t["scan_tensor_core"] == int(B >= 8)
    docs, scores, counts = emb.search_batch(q, limit, SIM)
    st = orc.EmbStore(rows)
    rows_idx = np.arange(n)
    for b in range(B):
        # the cosines of one direction are bitwise equal in float64 too: the float64 order is the key order
        want = np.lexsort((rows_idx, -cos[b]))[:limit]
        assert docs[b, :counts[b]].astype(np.int64).tolist() == want.tolist(), (b, docs[b], want)
        ed, es = orc.vector(st, q[b], limit, SIM)
        order = np.lexsort((ed, -es))
        assert docs[b, :counts[b]].tolist() == ed[order].astype(np.int64).tolist(), (b, docs[b], ed[order])
        assert np.allclose(scores[b, :counts[b]], es[order], rtol=0, atol=1e-6)
    emb.close()


@pytest.mark.parametrize("gemm", [False, True])
@pytest.mark.parametrize("left", ["zero", "limit-1", "limit", "limit+1"])
@pytest.mark.parametrize("how", ["filter", "delete"])
def test_few_live_rows(gpu_ctx, gemm, left, how):
    """A filter or deletes leave 0, limit - 1, limit or limit + 1 live rows (K2 still runs: it routes on the stored
    row count)."""
    n, dim, limit = 4133, 256, 10
    B = 8 if gemm else 4
    keep = {"zero": 0, "limit-1": limit - 1, "limit": limit, "limit+1": limit + 1}[left]
    emb, rows, rng = make_store(gpu_ctx, dim, "f32", n, seed=keep + 100 * gemm)
    q = queries(rows, B, rng)
    cos, tol = reference(rows, q)
    alive = rng.choice(n, keep, replace=False)
    live = np.zeros(n, bool)
    live[alive] = True
    fb, nb = None, 0
    if how == "filter":
        fb = np.zeros((n + 63) // 64, np.uint64)
        np.bitwise_or.at(fb, alive // 64, np.uint64(1) << (alive % 64).astype(np.uint64))
        nb = n
    else:
        emb.delete(np.flatnonzero(~live).astype(np.uint64))
    run_case(emb, q, limit, cos, tol, fb, nb, live)
    emb.close()


@pytest.mark.parametrize("dim", [0, 1025])
def test_unsupported_dims_are_rejected(gpu_ctx, dim):
    with pytest.raises(ob.OcError):
        ob.EmbeddingFieldStorage(gpu_ctx, "BGEBase", dim=dim)
