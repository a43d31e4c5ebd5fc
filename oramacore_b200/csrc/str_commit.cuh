// str_commit.cuh — the device half of oc_str_commit: merges the pending postings of a string store into the next
// snapshot's CSR without a host copy of the committed postings.
//
// The host filters the pending ops (O(pending)) and uploads, in one copy: the sorted unique pending documents
// `pdoc`, for each of them the first old row whose document is not below it (`p_lbold`) and the number of pending
// documents before it that are not alive old documents (`p_newbelow`, one more entry at the end), the alive bitmap as
// it was when the commit started, and per field the old term offsets, the surviving pending postings (term, index
// into pdoc, tf, len) and the pending documents re-inserted in that field.  Then, on the store's load stream:
//   1. the alive bitmap is scanned (compact_scan_words_kernel + compact_scan_blocks_kernel, emb_compact.cuh); the
//      new rows are the alive old documents merged with the new pending ones, ascending:
//        new_row(doc) = alive old documents below doc + new pending documents below doc
//      sc_old_rows_kernel gives every old row its new row (remap, ~0u when dead), sc_pending_rows_kernel every
//      pending document (prow); both write the new row -> document map when it is not the identity.
//   2. per field: sc_replaced_kernel marks the rows re-inserted in the field; sc_survive_kernel sets a bit per old
//      posting whose row is alive and not re-inserted, and the bitmap is scanned like the alive bitmap;
//   3. sc_pending_keys_kernel keys the pending postings by (term, new row) and cub::DeviceRadixSort sorts them;
//      sc_duplicate_kernel flags two equal adjacent keys (a term listed twice in one insert of a document);
//   4. sc_term_counts_kernel: surviving + pending postings per term, scanned into the new term offsets (one block
//      exscan here, compact_scan_blocks_kernel<uint64_t> over the block totals, sc_add_block_kernel);
//   5. the host reads the new offsets back (they are also the snapshot's host copy), allocates the new posting array
//      at its exact size, and sc_scatter_old_kernel / sc_scatter_pending_kernel write every slot of it exactly once:
//        old posting:     new_off[t] + its rank among t's survivors + t's pending postings with a lower new row
//        pending posting: new_off[t] + its rank among t's pending postings + t's survivors with a lower new row
//      so the result does not depend on scheduling.  Both keep, per new row, the (term, len) of its posting with the
//      largest term id (atomicMax); sc_len_sum_kernel sums the non-zero lengths exactly in uint64 for avg_field_len.
// oc_str_sync_global takes the same sums of a published snapshot from its postings (sc_row_len_kernel).
//
// Roofline: HBM.  Algorithmic bytes per old posting: 8 (read for the survivor bit) + 8 (read again by the scatter)
// + 8 (written) + 4 (the remap entry of its row, mostly from L2) + 2 * 1/8 (survivor bit, written and read); per
// old row 4 B of remap written; per pending posting about 64 B (keys, sort passes, scatter).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "bm25.cuh"
#include "emb_compact.cuh"

namespace oc {

constexpr uint32_t SC_THREADS = 256;
constexpr uint32_t SC_ITEMS = 8;                               // old postings per thread in sc_scatter_old_kernel
constexpr uint32_t SC_TILE = SC_THREADS * SC_ITEMS;

// first index i in [lo, hi) with a[i] >= key (hi when none)
template <typename T>
__device__ __forceinline__ uint64_t sc_lower_bound(const T *a, uint64_t lo, uint64_t hi, T key) {
    while (lo < hi) {
        const uint64_t m = lo + (hi - lo) / 2;
        if (a[m] < key) lo = m + 1; else hi = m;
    }
    return lo;
}
// term of posting i: the last t in [lo, hi] with off[t] <= i (off ascending, off[lo] <= i < off[hi + 1])
__device__ __forceinline__ uint32_t sc_term_of(const uint64_t *off, uint32_t lo, uint32_t hi, uint64_t i) {
    while (lo < hi) {
        const uint32_t m = lo + (hi - lo + 1) / 2;
        if (__ldg(off + m) <= i) lo = m; else hi = m - 1;
    }
    return lo;
}
// alive old rows below old row r (r <= n_rows); alive == NULL: every row is alive
__device__ __forceinline__ uint32_t sc_alive_below(const uint32_t *alive, const uint32_t *a_pre, const uint32_t *a_blk, uint64_t r) {
    return alive ? compact_bits_below(alive, a_pre, a_blk, r) : uint32_t(r);
}

// remap[r] = new row of old row r (~0u: dead); new_doc[new row] = its document (new_doc NULL: the new map is the identity)
__global__ void __launch_bounds__(SC_THREADS)
sc_old_rows_kernel(uint64_t n_rows, const uint32_t *alive, const uint32_t *a_pre, const uint32_t *a_blk,
                   const uint64_t *old_doc, const uint64_t *pdoc, uint32_t n_pdoc, const uint32_t *p_newbelow,
                   uint32_t *remap, uint64_t *new_doc) {
    const uint64_t r = uint64_t(blockIdx.x) * SC_THREADS + threadIdx.x;
    if (r >= n_rows) return;
    if (alive && !((__ldg(alive + (r >> 5)) >> (r & 31)) & 1u)) { remap[r] = 0xffffffffu; return; }
    const uint64_t doc = old_doc ? old_doc[r] : r;
    const uint32_t nr = sc_alive_below(alive, a_pre, a_blk, r) + __ldg(p_newbelow + sc_lower_bound(pdoc, 0, n_pdoc, doc));
    remap[r] = nr;
    if (new_doc) new_doc[nr] = doc;
}

// prow[j] = new row of pending document j: the row of the alive old document it re-inserts, or a row of its own
__global__ void __launch_bounds__(SC_THREADS)
sc_pending_rows_kernel(uint32_t n_pdoc, const uint64_t *pdoc, const uint32_t *p_lbold, const uint32_t *p_newbelow,
                       const uint32_t *alive, const uint32_t *a_pre, const uint32_t *a_blk, const uint32_t *remap,
                       uint32_t *prow, uint64_t *new_doc) {
    const uint32_t j = blockIdx.x * SC_THREADS + threadIdx.x;
    if (j >= n_pdoc) return;
    const uint32_t lb = p_lbold[j];
    if (p_newbelow[j + 1] == p_newbelow[j]) { prow[j] = remap[lb]; return; }   // not new: lb is its alive old row
    const uint32_t nr = sc_alive_below(alive, a_pre, a_blk, lb) + p_newbelow[j];
    prow[j] = nr;
    if (new_doc) new_doc[nr] = pdoc[j];
}

// bit prow[j] of `bits` for every pending document j re-inserted in the field
__global__ void __launch_bounds__(SC_THREADS)
sc_replaced_kernel(uint32_t n, const uint32_t *repl, const uint32_t *prow, uint32_t *bits) {
    const uint32_t i = blockIdx.x * SC_THREADS + threadIdx.x;
    if (i >= n) return;
    const uint32_t r = prow[repl[i]];
    atomicOr(bits + (r >> 5), 1u << (r & 31));
}

// bit i of `keep` = old posting i survives: its row is alive and not re-inserted in this field.  A warp writes a word;
// n_words * 32 >= n_post + 1, so the bits past n_post are written as 0.
__global__ void __launch_bounds__(SC_THREADS)
sc_survive_kernel(uint64_t n_post, uint64_t n_words, const PostingRaw *raw, uint64_t n_rows, const uint32_t *remap,
                  const uint32_t *replaced, uint32_t *keep) {
    const uint64_t i = uint64_t(blockIdx.x) * SC_THREADS + threadIdx.x;
    bool k = false;
    if (i < n_post) {
        const uint32_t row = __ldcs(&raw[i].row);
        const uint32_t nr = row < n_rows ? __ldg(remap + row) : 0xffffffffu;
        k = nr != 0xffffffffu && !((__ldg(replaced + (nr >> 5)) >> (nr & 31)) & 1u);
    }
    const uint32_t w = __ballot_sync(0xffffffffu, k);
    if ((threadIdx.x & 31) == 0 && (i >> 5) < n_words) keep[i >> 5] = w;
}

// key of pending posting k = (term << 32) | new row; value = k
__global__ void __launch_bounds__(SC_THREADS)
sc_pending_keys_kernel(uint32_t n, const uint32_t *p_term, const uint32_t *p_doc, const uint32_t *prow,
                       uint64_t *keys, uint32_t *vals) {
    const uint32_t k = blockIdx.x * SC_THREADS + threadIdx.x;
    if (k >= n) return;
    keys[k] = (uint64_t(p_term[k]) << 32) | prow[p_doc[k]];
    vals[k] = k;
}

// flag[0] = 1 and flag[1] = the smallest such term when two sorted keys are equal (flag[1] starts at ~0u)
__global__ void __launch_bounds__(SC_THREADS)
sc_duplicate_kernel(uint32_t n, const uint64_t *keys, uint32_t *flag) {
    const uint32_t k = blockIdx.x * SC_THREADS + threadIdx.x;
    if (k == 0 || k >= n || keys[k] != keys[k - 1]) return;
    flag[0] = 1;
    atomicMin(flag + 1, uint32_t(keys[k] >> 32));
}

// Per term t < n_terms: surv_lo[t] = survivor bits below the term's first old posting, pend_lo[t] = its first sorted
// pending posting (pend_lo[n_terms] = n_pend), and new_off[t] = the exclusive prefix of (survivors + pending
// postings) within this block of COMPACT_SCAN_WORDS terms; blk[b] = the block's total.  new_off[n_terms] takes the
// grand total once the block prefixes are added.
__global__ void __launch_bounds__(COMPACT_SCAN_WORDS)
sc_term_counts_kernel(uint32_t n_terms, uint32_t n_terms_old, const uint64_t *old_off, const uint32_t *keep,
                      const uint32_t *k_pre, const uint32_t *k_blk, const uint64_t *keys, uint32_t n_pend,
                      uint32_t *surv_lo, uint32_t *pend_lo, uint64_t *new_off, uint64_t *blk) {
    __shared__ uint64_t warp_sums[32];
    __shared__ uint64_t total;
    const uint32_t t = blockIdx.x * COMPACT_SCAN_WORDS + threadIdx.x;
    uint64_t cnt = 0;
    if (t <= n_terms) {
        const uint32_t p0 = (uint32_t)sc_lower_bound(keys, 0, n_pend, uint64_t(t) << 32);
        pend_lo[t] = p0;
        if (t < n_terms) {
            cnt = (uint32_t)sc_lower_bound(keys, p0, n_pend, uint64_t(t + 1) << 32) - p0;
            uint32_t s0 = 0;
            if (t < n_terms_old) {
                s0 = compact_bits_below(keep, k_pre, k_blk, old_off[t]);
                cnt += compact_bits_below(keep, k_pre, k_blk, old_off[t + 1]) - s0;   // exact modulo 2^32 (emb_compact.cuh)
            }
            surv_lo[t] = s0;
        }
    }
    const uint64_t ex = compact_block_exscan<uint64_t>(cnt, warp_sums, &total);
    if (t <= n_terms) new_off[t] = ex;
    if (threadIdx.x == 0) blk[blockIdx.x] = total;
}

// new_off[t] += the postings of the term blocks below t's (blk: scanned by compact_scan_blocks_kernel<uint64_t>)
__global__ void __launch_bounds__(SC_THREADS)
sc_add_block_kernel(uint32_t n, const uint64_t *blk, uint64_t *new_off) {
    const uint32_t t = blockIdx.x * SC_THREADS + threadIdx.x;
    if (t < n) new_off[t] += blk[t / COMPACT_SCAN_WORDS];
}

// the (term, len) of the posting with the largest term id of each row (row_key == NULL: not wanted)
__device__ __forceinline__ void sc_note_len(unsigned long long *row_key, uint32_t row, uint32_t term, uint16_t len) {
    if (row_key) atomicMax(row_key + row, (unsigned long long)((uint64_t(term) << 16) | len));
}

// Surviving old postings -> out.  A CTA takes SC_TILE consecutive postings: two threads find the terms of the tile's
// first and last posting, and every posting then searches its term between them (a tile inside one long list
// searches nothing).
__global__ void __launch_bounds__(SC_THREADS)
sc_scatter_old_kernel(uint64_t n_post, const PostingRaw *raw, const uint32_t *remap, const uint32_t *keep,
                      const uint32_t *k_pre, const uint32_t *k_blk, uint32_t n_terms_old, const uint64_t *old_off,
                      const uint64_t *new_off, const uint32_t *surv_lo, const uint32_t *pend_lo, const uint64_t *keys,
                      PostingRaw *out, unsigned long long *row_key) {
    __shared__ uint32_t t_span[2];
    const uint64_t i0 = uint64_t(blockIdx.x) * SC_TILE;
    const uint64_t i1 = i0 + SC_TILE < n_post ? i0 + SC_TILE : n_post;
    if (threadIdx.x < 2) t_span[threadIdx.x] = sc_term_of(old_off, 0, n_terms_old - 1, threadIdx.x ? i1 - 1 : i0);
    __syncthreads();
    const uint32_t t_lo = t_span[0], t_hi = t_span[1];
#pragma unroll 2
    for (uint32_t it = 0; it < SC_ITEMS; it++) {
        const uint64_t i = i0 + it * SC_THREADS + threadIdx.x;
        if (i >= i1 || !((__ldg(keep + (i >> 5)) >> (i & 31)) & 1u)) continue;
        const PostingRaw p = raw[i];
        const uint32_t t = t_lo == t_hi ? t_lo : sc_term_of(old_off, t_lo, t_hi, i);
        const uint32_t nr = __ldg(remap + p.row);
        const uint32_t rank = compact_bits_below(keep, k_pre, k_blk, i) - __ldg(surv_lo + t);
        const uint32_t pb = __ldg(pend_lo + t), pe = __ldg(pend_lo + t + 1);
        const uint64_t below = pe > pb ? sc_lower_bound(keys, pb, pe, (uint64_t(t) << 32) | nr) - pb : 0;
        out[__ldg(new_off + t) + rank + below] = {nr, p.tf, p.len};
        sc_note_len(row_key, nr, t, p.len);
    }
}

// Sorted pending postings -> out.  The survivors of term t below new row nr are its old postings below the first old
// row whose document is not below the pending document (p_lbold), minus the dead and re-inserted ones among them.
__global__ void __launch_bounds__(SC_THREADS)
sc_scatter_pending_kernel(uint32_t n_pend, const uint64_t *keys, const uint32_t *vals, const uint32_t *p_doc,
                          const uint16_t *p_tf, const uint16_t *p_len, const uint32_t *p_lbold, const PostingRaw *raw,
                          uint32_t n_terms_old, const uint64_t *old_off, const uint32_t *keep, const uint32_t *k_pre,
                          const uint32_t *k_blk, const uint64_t *new_off, const uint32_t *surv_lo, const uint32_t *pend_lo,
                          PostingRaw *out, unsigned long long *row_key) {
    const uint32_t k = blockIdx.x * SC_THREADS + threadIdx.x;
    if (k >= n_pend) return;
    const uint64_t key = keys[k];
    const uint32_t t = uint32_t(key >> 32), nr = uint32_t(key), v = vals[k];
    uint32_t below = 0;
    if (t < n_terms_old) {
        const uint32_t lb = p_lbold[p_doc[v]];
        uint64_t lo = old_off[t], hi = old_off[t + 1];
        while (lo < hi) {   // first old posting of t with row >= lb
            const uint64_t m = lo + (hi - lo) / 2;
            if (raw[m].row < lb) lo = m + 1; else hi = m;
        }
        below = compact_bits_below(keep, k_pre, k_blk, lo) - surv_lo[t];
    }
    out[new_off[t] + (k - pend_lo[t]) + below] = {nr, p_tf[v], p_len[v]};
    sc_note_len(row_key, nr, t, p_len[v]);
}

// row_key[row] = the field length its postings carry (the largest, should they differ): the input sc_len_sum_kernel
// takes when a snapshot's length sums come from its postings (oc_str_sync_global) rather than from its commit
__global__ void __launch_bounds__(SC_THREADS)
sc_row_len_kernel(uint64_t n_post, const PostingRaw *raw, unsigned long long *row_key) {
    for (uint64_t i = uint64_t(blockIdx.x) * SC_THREADS + threadIdx.x; i < n_post; i += uint64_t(gridDim.x) * SC_THREADS) {
        const PostingRaw p = raw[i];
        if (p.len) atomicMax(row_key + p.row, (unsigned long long)p.len);
    }
}

// sum[0] += the non-zero lengths in row_key, sum[1] += their count
__global__ void __launch_bounds__(SC_THREADS)
sc_len_sum_kernel(uint32_t n_rows, const unsigned long long *row_key, unsigned long long *sum) {
    unsigned long long s = 0, c = 0;
    for (uint32_t r = blockIdx.x * SC_THREADS + threadIdx.x; r < n_rows; r += gridDim.x * SC_THREADS) {
        const uint32_t len = uint32_t(row_key[r] & 0xffffu);
        s += len; c += len != 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); c += __shfl_xor_sync(0xffffffffu, c, o); }
    if ((threadIdx.x & 31) == 0 && c) { atomicAdd(sum, s); atomicAdd(sum + 1, c); }
}

}  // namespace oc
