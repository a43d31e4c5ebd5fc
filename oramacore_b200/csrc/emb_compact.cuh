// emb_compact.cuh — order-preserving, in-place removal of the dead rows of an embedding store (oc_emb_compact).
//
// The host knows which rows are dead (oc_emb_delete collects them) and uploads them as a bitmap, one bit per row.
//   1. compact_scan_words_kernel + compact_scan_blocks_kernel: dead rows below every 32-row word (popcount per word,
//      exclusive scan per block of COMPACT_SCAN_WORDS words, exclusive scan of the block totals).  The destination of
//      live row r is r - dead_below(r).
//   2. per window of source rows, ascending, on one stream:
//        compact_gather_kernel<ESZ>: the window's live rows, in order, into the staging buffer;
//        compact_store_kernel:     the staging buffer to rows [dst, dst + live) of the same array.
//      The staging buffer is what makes the move safe in place: a row's destination may be the source of a row
//      another CTA has not read yet, so no row is stored before its whole window is read.
//   3. compact_small_gather_kernel / compact_small_store_kernel: the same for inv_norm, row_doc and row_scale.
//
// Roofline: HBM.  Algorithmic bytes per moved row = 2 * stride * ESZ (one read, one write; the same again at
// 2 B per element for the fp16 copy of an fp32 store) + 2 * 16 B for the small arrays; dead rows are not read.  The
// staging buffer adds one write and one read of every moved row (from L2 for the part of a window that stays there).
// Rows are stride * ESZ bytes, a multiple of 256: they move as 16-byte vectors, a warp per row.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace oc {

constexpr uint32_t COMPACT_SCAN_WORDS = 1024;   // words (of 32 rows) per scan block == its threads
constexpr uint32_t COMPACT_THREADS = 256;

// set bits below bit r of a bitmap scanned by compact_scan_words_kernel + compact_scan_blocks_kernel (here: dead rows
// below row r; str_commit.cuh counts alive rows and surviving postings with it); word_pre: per word, within its scan
// block; block_pre: per scan block.  The sum wraps modulo 2^32, so a difference of two counts is exact whenever the
// bits between them number fewer than 2^32, however long the bitmap.
__device__ __forceinline__ uint32_t compact_bits_below(const uint32_t *bits, const uint32_t *word_pre,
                                                       const uint32_t *block_pre, uint64_t r) {
    const uint64_t w = r >> 5;
    return __ldg(block_pre + w / COMPACT_SCAN_WORDS) + __ldg(word_pre + w) +
           __popc(__ldg(bits + w) & ((1u << (r & 31)) - 1u));
}

// exclusive scan of one value per thread over a block of COMPACT_SCAN_WORDS threads; *total = the block's sum
template <typename T>
__device__ __forceinline__ T compact_block_exscan(T v, T *warp_sums, T *total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const T o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        const T s = warp_sums[lane];
        T si = s;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const T o = __shfl_up_sync(0xffffffffu, si, d);
            if (lane >= d) si += o;
        }
        warp_sums[lane] = si - s;
        if (lane == 31) *total = si;
    }
    __syncthreads();
    const T r = warp_sums[warp] + inc - v;
    __syncthreads();   // warp_sums is reused by the caller's next round
    return r;
}

// word_pre[w] = dead rows in the words of w's scan block below w; block_tot[b] = dead rows of scan block b
__global__ void __launch_bounds__(COMPACT_SCAN_WORDS)
compact_scan_words_kernel(const uint32_t *dead_bits, uint64_t n_words, uint32_t *word_pre, uint32_t *block_tot) {
    __shared__ uint32_t warp_sums[32];
    __shared__ uint32_t total;
    const uint64_t w = uint64_t(blockIdx.x) * COMPACT_SCAN_WORDS + threadIdx.x;
    const uint32_t ex = compact_block_exscan<uint32_t>(w < n_words ? __popc(dead_bits[w]) : 0u, warp_sums, &total);
    if (w < n_words) word_pre[w] = ex;
    if (threadIdx.x == 0) block_tot[blockIdx.x] = total;
}

// in place: block_tot -> exclusive prefix sums, i.e. dead rows below each scan block (one CTA; n_rows < 2^32 leaves at
// most 2^17 blocks).  T = uint64_t: str_commit.cuh's per-term posting counts.
template <typename T>
__global__ void __launch_bounds__(COMPACT_SCAN_WORDS)
compact_scan_blocks_kernel(T *block_tot, uint32_t n_blocks) {
    __shared__ T warp_sums[32];
    __shared__ T total;
    T carry = 0;
    for (uint32_t base = 0; base < n_blocks; base += COMPACT_SCAN_WORDS) {
        const uint32_t i = base + threadIdx.x;
        const T ex = compact_block_exscan<T>(i < n_blocks ? block_tot[i] : T(0), warp_sums, &total);
        if (i < n_blocks) block_tot[i] = carry + ex;
        carry += total;
        __syncthreads();   // every thread has read `total` before the next round overwrites it
    }
}

// Live rows of source rows [row_begin, row_end) -> stage[(r - dead_below(r)) - dst_begin], a warp per row.  ESZ is the
// element width of the array (4: fp32 rows, 2: bf16 rows or the fp16 copy); the bytes are not interpreted.
template <int ESZ>
__global__ void __launch_bounds__(COMPACT_THREADS)
compact_gather_kernel(const void *rows, uint32_t stride, uint64_t row_begin, uint64_t row_end, uint64_t dst_begin,
                      const uint32_t *dead_bits, const uint32_t *word_pre, const uint32_t *block_pre, uint4 *stage) {
    const uint32_t row_vec = stride * uint32_t(ESZ) / 16;   // a multiple of 16
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = uint64_t(gridDim.x) * (COMPACT_THREADS / 32);
    for (uint64_t r = row_begin + uint64_t(blockIdx.x) * (COMPACT_THREADS / 32) + (threadIdx.x >> 5); r < row_end; r += warps) {
        if ((__ldg(dead_bits + (r >> 5)) >> (r & 31)) & 1u) continue;   // warp-uniform: a dead row is not read
        const uint64_t d = r - compact_bits_below(dead_bits, word_pre, block_pre, r) - dst_begin;
        const uint4 *src = static_cast<const uint4 *>(rows) + r * row_vec;
        uint4 *dst = stage + d * row_vec;
        // the source is read once (streaming, evict-first); the staging buffer is read back by the next kernel
        uint32_t i = lane;
        for (; i + 96 < row_vec; i += 128) {
            const uint4 a = __ldcs(src + i), b = __ldcs(src + i + 32), c = __ldcs(src + i + 64), e = __ldcs(src + i + 96);
            dst[i] = a; dst[i + 32] = b; dst[i + 64] = c; dst[i + 96] = e;
        }
        for (; i < row_vec; i += 32) dst[i] = __ldcs(src + i);
    }
}

// stage[0, n_vec) -> dst[0, n_vec) in 16-byte vectors
__global__ void __launch_bounds__(COMPACT_THREADS)
compact_store_kernel(const uint4 *stage, uint4 *dst, uint64_t n_vec) {
    const uint64_t step = uint64_t(gridDim.x) * COMPACT_THREADS;
    uint64_t i = uint64_t(blockIdx.x) * COMPACT_THREADS + threadIdx.x;
    for (; i + 3 * step < n_vec; i += 4 * step) {
        const uint4 a = __ldcg(stage + i), b = __ldcg(stage + i + step), c = __ldcg(stage + i + 2 * step), e = __ldcg(stage + i + 3 * step);
        __stcs(dst + i, a); __stcs(dst + i + step, b); __stcs(dst + i + 2 * step, c); __stcs(dst + i + 3 * step, e);
    }
    for (; i < n_vec; i += step) __stcs(dst + i, __ldcg(stage + i));
}

// The per-row arrays of source rows [row_begin, row_end), a thread per row: live rows -> st_doc / st_inv / st_scale at
// (r - dead_below(r)) - dst_begin.  row_scale (and st_scale) NULL: the store has no fp16 copy.
__global__ void __launch_bounds__(COMPACT_THREADS)
compact_small_gather_kernel(const float *inv_norm, const uint64_t *row_doc, const float *row_scale, uint64_t row_begin,
                            uint64_t row_end, uint64_t dst_begin, const uint32_t *dead_bits, const uint32_t *word_pre,
                            const uint32_t *block_pre, uint64_t *st_doc, float *st_inv, float *st_scale) {
    const uint64_t r = row_begin + uint64_t(blockIdx.x) * COMPACT_THREADS + threadIdx.x;
    if (r >= row_end || ((__ldg(dead_bits + (r >> 5)) >> (r & 31)) & 1u)) return;
    const uint64_t d = r - compact_bits_below(dead_bits, word_pre, block_pre, r) - dst_begin;
    st_doc[d] = row_doc[r];
    st_inv[d] = inv_norm[r];
    if (row_scale) st_scale[d] = row_scale[r];
}

__global__ void __launch_bounds__(COMPACT_THREADS)
compact_small_store_kernel(const uint64_t *st_doc, const float *st_inv, const float *st_scale, uint64_t n,
                           uint64_t *row_doc, float *inv_norm, float *row_scale) {
    const uint64_t i = uint64_t(blockIdx.x) * COMPACT_THREADS + threadIdx.x;
    if (i >= n) return;
    row_doc[i] = st_doc[i];
    inv_norm[i] = st_inv[i];
    if (row_scale) row_scale[i] = st_scale[i];
}

}  // namespace oc
