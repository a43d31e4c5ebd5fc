// omc.cuh — the device half of the OMC store (oc_omc_*): the commit of the queued ops into the next version, and the
// list of string rows the tile scorers read, derived from a version and a string-store snapshot.
//
// Commit (oc_omc_commit_ex).  A version is (doc[n] strictly ascending, mult[n]); the queue is n_b ops (document,
// multiplier or delete) in call order.
//   1. cub::DeviceRadixSort orders the ops by document; the sort is stable, so each document's ops stay in call order
//      and the last of a run is the one that wins;
//   2. om_keep_kernel marks each run's last op when it is a set (b_keep), and each committed entry whose document has
//      no op (a_keep);
//   3. cub::DeviceScan gives both sides their ranks among the kept entries;
//   4. om_scatter_a_kernel / om_scatter_b_kernel write every kept entry once, at its rank on its own side plus the
//      number of kept entries of the other side with a smaller document (a binary search): the merge is one pass and
//      deterministic.
// Row list (the first search after a commit or an oc_str_commit).  om_rows_kernel maps each entry to its string row
// (binary search over the snapshot's row_doc, or the identity), a scan compacts the entries that have a row, and
// om_rows_scatter_kernel writes (row, mult) ascending, as the tile scorers' omc_row / omc_mult.
// Roofline: HBM.  Commit: per committed entry 12 B read, a binary search over the sorted ops and 8 B of flags and
// ranks; per op 13 B uploaded and a radix sort of 12 B pairs.  Row list: per entry 12 B read, a binary search over
// row_doc, 12 B of flags and ranks and 8 B written.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace oc {

constexpr uint32_t OM_THREADS = 256;
constexpr uint32_t OM_NO_ROW = 0xffffffffu;

// first index i in [0, n) with a[i] >= x
__device__ __forceinline__ uint64_t om_lower_bound(const uint64_t *a, uint64_t n, uint64_t x) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) { const uint64_t m = (lo + hi) >> 1; if (a[m] < x) lo = m + 1; else hi = m; }
    return lo;
}

// b: the ops sorted by document (b_doc) with their call-order index (b_idx); b_del[index]: the op is a delete.
// a_keep[n_a] = b_keep[n_b] = 0, so the exclusive scans end with the totals.
__global__ void __launch_bounds__(OM_THREADS) om_keep_kernel(const uint64_t *a_doc, uint64_t n_a, const uint64_t *b_doc,
                                                             const uint32_t *b_idx, const uint8_t *b_del, uint64_t n_b,
                                                             uint32_t *a_keep, uint32_t *b_keep) {
    const uint64_t i = uint64_t(blockIdx.x) * OM_THREADS + threadIdx.x;
    if (i <= n_a) {
        bool keep = false;
        if (i < n_a) {
            const uint64_t j = om_lower_bound(b_doc, n_b, a_doc[i]);
            keep = j == n_b || b_doc[j] != a_doc[i];
        }
        a_keep[i] = keep ? 1u : 0u;
    }
    if (i <= n_b) {
        const bool last = i < n_b && (i + 1 == n_b || b_doc[i + 1] != b_doc[i]);
        b_keep[i] = last && !b_del[b_idx[i]] ? 1u : 0u;
    }
}

__global__ void __launch_bounds__(OM_THREADS) om_scatter_a_kernel(const uint64_t *a_doc, const float *a_mult, uint64_t n_a,
                                                                  const uint32_t *a_rank, const uint64_t *b_doc, uint64_t n_b,
                                                                  const uint32_t *b_rank, uint64_t *out_doc, float *out_mult) {
    const uint64_t i = uint64_t(blockIdx.x) * OM_THREADS + threadIdx.x;
    if (i >= n_a || a_rank[i + 1] == a_rank[i]) return;
    const uint64_t d = a_doc[i];
    const uint64_t o = uint64_t(a_rank[i]) + b_rank[om_lower_bound(b_doc, n_b, d)];
    out_doc[o] = d;
    out_mult[o] = a_mult[i];
}

__global__ void __launch_bounds__(OM_THREADS) om_scatter_b_kernel(const uint64_t *b_doc, const uint32_t *b_idx, const float *q_mult,
                                                                  uint64_t n_b, const uint32_t *b_rank, const uint64_t *a_doc,
                                                                  uint64_t n_a, const uint32_t *a_rank, uint64_t *out_doc,
                                                                  float *out_mult) {
    const uint64_t j = uint64_t(blockIdx.x) * OM_THREADS + threadIdx.x;
    if (j >= n_b || b_rank[j + 1] == b_rank[j]) return;
    const uint64_t d = b_doc[j];
    const uint64_t o = uint64_t(b_rank[j]) + a_rank[om_lower_bound(a_doc, n_a, d)];
    out_doc[o] = d;
    out_mult[o] = q_mult[b_idx[j]];
}

// row[i]: the string row of doc[i] (OM_NO_ROW: none); has[n] = 0 for the scan's total.  row_doc == NULL: identity.
__global__ void __launch_bounds__(OM_THREADS) om_rows_kernel(const uint64_t *doc, uint64_t n, const uint64_t *row_doc,
                                                             uint64_t n_rows, uint32_t *row, uint32_t *has) {
    const uint64_t i = uint64_t(blockIdx.x) * OM_THREADS + threadIdx.x;
    if (i > n) return;
    uint32_t r = OM_NO_ROW;
    if (i < n) {
        const uint64_t d = doc[i];
        if (!row_doc) {
            if (d < n_rows) r = uint32_t(d);
        } else {
            const uint64_t k = om_lower_bound(row_doc, n_rows, d);
            if (k < n_rows && row_doc[k] == d) r = uint32_t(k);
        }
        row[i] = r;
    }
    has[i] = r != OM_NO_ROW ? 1u : 0u;
}

__global__ void __launch_bounds__(OM_THREADS) om_rows_scatter_kernel(const uint32_t *row, const float *mult, uint64_t n,
                                                                     const uint32_t *pos, uint32_t *out_row, float *out_mult) {
    const uint64_t i = uint64_t(blockIdx.x) * OM_THREADS + threadIdx.x;
    if (i >= n || pos[i + 1] == pos[i]) return;
    out_row[pos[i]] = row[i];
    out_mult[pos[i]] = mult[i];
}

}  // namespace oc
