// oc_common.cuh — shared device helpers: ordered score keys, bitonic sorts, mbarrier /
// bulk-copy (TMA 1-D) PTX wrappers.  sm_90a only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "oramacore_b200.h"

namespace oc {

// ---------------------------------------------------------------------------------------
// 64-bit rank keys.  Larger key == better hit: (order-preserving score bits << 32) | ~idx,
// so ties on score resolve to the LOWER index (rows are stored in ascending DocumentId
// order, matching the oracle's "ties by ascending doc id").  Keys are unique per index.
// NaN scores never become keys (callers test `score == score`), mirroring
// NotNan::new(..) => continue in top_n (read/sort.rs:264-267).
// ---------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t f32_ordered(float f) {
#ifdef __CUDA_ARCH__
    uint32_t u = __float_as_uint(f);
#else
    union { float f; uint32_t u; } c; c.f = f; uint32_t u = c.u;
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float f32_unordered(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7fffffffu) : ~o;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    union { float f; uint32_t u; } c; c.u = u; return c.f;
#endif
}
__host__ __device__ __forceinline__ uint64_t make_key(float score, uint32_t idx) {
    score = score + 0.0f;  // -0.0 -> +0.0 so that it ties with +0.0 like a float compare
    return (uint64_t(f32_ordered(score)) << 32) | uint64_t(0xffffffffu - idx);
}
__host__ __device__ __forceinline__ float key_score(uint64_t k) { return f32_unordered(uint32_t(k >> 32)); }
__host__ __device__ __forceinline__ uint32_t key_idx(uint64_t k) { return 0xffffffffu - uint32_t(k); }

constexpr uint64_t KEY_NONE = 0ull;  // below every real key (f32_ordered(x) >= 0x007fffff for non-NaN)

__host__ __device__ __forceinline__ uint32_t next_pow2(uint32_t v) {
    uint32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------
// Bitonic sort, DESCENDING, of n (power of two) u64 keys in shared memory.
// ---------------------------------------------------------------------------------------
// by one warp; callers guarantee only this warp touches buf.
__device__ __forceinline__ void warp_bitonic_desc(uint64_t *buf, uint32_t n, uint32_t lane) {
    for (uint32_t k = 2; k <= n; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            __syncwarp();
            for (uint32_t i = lane; i < n; i += 32) {
                uint32_t ixj = i ^ j;
                if (ixj > i) {
                    uint64_t a = buf[i], b = buf[ixj];
                    bool desc = ((i & k) == 0);
                    if (desc ? (a < b) : (a > b)) { buf[i] = b; buf[ixj] = a; }
                }
            }
        }
    }
    __syncwarp();
}

// by `nthreads` threads that all call it (tid in [0,nthreads)); sync via named barrier `bar`.
__device__ __forceinline__ void named_bar_sync(uint32_t bar, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(bar), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void group_bitonic_desc(uint64_t *buf, uint32_t n, uint32_t tid,
                                                   uint32_t nthreads, uint32_t bar) {
    for (uint32_t k = 2; k <= n; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            named_bar_sync(bar, nthreads);
            for (uint32_t i = tid; i < n; i += nthreads) {
                uint32_t ixj = i ^ j;
                if (ixj > i) {
                    uint64_t a = buf[i], b = buf[ixj];
                    bool desc = ((i & k) == 0);
                    if (desc ? (a < b) : (a > b)) { buf[i] = b; buf[ixj] = a; }
                }
            }
        }
    }
    named_bar_sync(bar, nthreads);
}

// ---------------------------------------------------------------------------------------
// mbarrier + 1-D bulk async copy (TMA engine; SASS: UBLKCP / SYNCS).
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// global -> shared::cta bulk copy, completion signalled on `bar` as complete_tx(bytes).
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// same with an L2 evict-first policy: the matrix is streamed once per sweep.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void bulk_g2s_hint(void *dst_smem, const void *src_gmem, uint32_t bytes,
                                              uint64_t *bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], "
        "%4;" ::"r"(smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
        : "memory");
}

// ---------------------------------------------------------------------------------------
// Block-wide selection of the `keep` largest non-zero (non KEY_NONE) keys of buf[0, nv) into
// out[0, returned count) — UNSORTED; the caller sorts the (small) result.  Non-zero keys must be
// unique (rank keys carry the row index).  Radix select, most significant differing byte first,
// 8 bits per pass, one warp-aggregated shared atomic per distinct bin per warp; stops as soon as
// the boundary bin is taken whole.  O(nv) per pass instead of the O(nv log^2 nv) of a full sort.
// All threads of the block must call it (blockDim.x a multiple of 32); out must not alias buf.
// ---------------------------------------------------------------------------------------
__device__ inline uint32_t block_select_largest(const uint64_t *buf, uint32_t nv, uint32_t keep, uint64_t *out) {
    __shared__ uint32_t sl_hist[256];
    __shared__ unsigned long long sl_or, sl_and, sl_prefix;
    __shared__ uint32_t sl_need, sl_done, sl_n, sl_nz;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { sl_or = 0ull; sl_and = ~0ull; sl_n = 0; sl_nz = 0; }
    __syncthreads();
    {
        uint64_t o = 0, a = ~0ull; uint32_t nz = 0;
        for (uint32_t i = tid; i < nv; i += blockDim.x) { const uint64_t k = buf[i]; if (k) { o |= k; a &= k; nz++; } }
        const uint32_t ol = __reduce_or_sync(0xffffffffu, uint32_t(o)), oh = __reduce_or_sync(0xffffffffu, uint32_t(o >> 32));
        const uint32_t al = __reduce_and_sync(0xffffffffu, uint32_t(a)), ah = __reduce_and_sync(0xffffffffu, uint32_t(a >> 32));
        nz = __reduce_add_sync(0xffffffffu, nz);
        if (lane == 0 && nz) { atomicOr(&sl_or, (uint64_t(oh) << 32) | ol); atomicAnd(&sl_and, (uint64_t(ah) << 32) | al); atomicAdd(&sl_nz, nz); }
    }
    __syncthreads();
    const uint32_t nz = sl_nz;
    if (nz <= keep) {   // everything valid is kept
        for (uint32_t i = tid; i < nv; i += blockDim.x) { const uint64_t k = buf[i]; if (k) out[atomicAdd(&sl_n, 1u)] = k; }
        __syncthreads();
        return nz;
    }
    const uint64_t diff = sl_or ^ sl_and;   // bits on which the keys disagree (non-zero: nz >= 2 unique keys)
    int shift = ((63 - __clzll((long long)(diff | 1ull))) >> 3) << 3;
    uint64_t prefix = shift == 56 ? 0ull : (sl_and >> (shift + 8)) << (shift + 8);
    uint32_t need = keep;
    for (; shift >= 0; shift -= 8) {
        for (uint32_t i = tid; i < 256; i += blockDim.x) sl_hist[i] = 0;
        __syncthreads();
        for (uint32_t i0 = 0; i0 < nv; i0 += blockDim.x) {   // block-uniform trip count: match_any needs converged lanes
            const uint32_t i = i0 + tid;
            const uint64_t k = i < nv ? buf[i] : 0ull;
            const bool in = k != 0ull && (shift == 56 || (k >> (shift + 8)) == (prefix >> (shift + 8)));
            const uint32_t bin = in ? (uint32_t(k >> shift) & 255u) : 256u;
            const uint32_t peers = __match_any_sync(0xffffffffu, bin);
            if (in && lane == uint32_t(__ffs(peers) - 1)) atomicAdd(&sl_hist[bin], uint32_t(__popc(peers)));
        }
        __syncthreads();
        if (warp == 0) {   // lane l owns bins [255 - 8l - 7, 255 - 8l], walked from the top
            uint32_t mine = 0;
#pragma unroll
            for (uint32_t j = 0; j < 8; j++) mine += sl_hist[255 - 8 * lane - j];
            uint32_t above = mine;   // inclusive prefix over lanes (lane 0 = highest bins)
#pragma unroll
            for (uint32_t o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(0xffffffffu, above, o);
                if (lane >= o) above += v;
            }
            above -= mine;           // keys in bins above this lane's range
            if (above < need && above + mine >= need) {
                uint32_t cum = above;
                for (uint32_t j = 0; j < 8; j++) {
                    const uint32_t b = 255 - 8 * lane - j, h = sl_hist[b];
                    if (cum + h >= need) {
                        sl_prefix = prefix | (uint64_t(b) << shift);
                        sl_need = need - cum;
                        sl_done = (h == need - cum) ? 1u : 0u;
                        break;
                    }
                    cum += h;
                }
            }
        }
        __syncthreads();
        prefix = sl_prefix; need = sl_need;
        if (sl_done) break;
    }
    if (shift < 0) shift = 0;   // unique keys: the last byte always resolves
    // exactly `keep` keys have (key >> shift) >= (prefix >> shift)
    for (uint32_t i = tid; i < nv; i += blockDim.x) {
        const uint64_t k = buf[i];
        if (k != 0ull && (k >> shift) >= (prefix >> shift)) { const uint32_t s = atomicAdd(&sl_n, 1u); if (s < keep) out[s] = k; }
    }
    __syncthreads();
    return keep;
}

// exclusive prefix sum of one value per thread across the block (blockDim.x <= 1024, a multiple of 32);
// *total receives the block sum.  Every thread must call it.
__device__ inline uint32_t block_exclusive_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t bs_w[32];
    __shared__ uint32_t bs_tot;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) bs_w[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        const uint32_t w = lane < nw ? bs_w[lane] : 0u;
        uint32_t winc = w;
#pragma unroll
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += t;
        }
        bs_w[lane] = winc - w;
        if (lane == 31) bs_tot = winc;
    }
    __syncthreads();
    const uint32_t r = bs_w[warp] + inc - v;
    *total = bs_tot;
    __syncthreads();   // scratch may be reused by the next call
    return r;
}

__device__ __forceinline__ float warp_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 16);
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}
#endif  // __CUDACC__

}  // namespace oc
