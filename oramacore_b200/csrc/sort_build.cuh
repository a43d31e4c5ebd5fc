// sort_build.cuh — the device build of a sort field (oc_sort_field_create, oc_sort_field_from_facets): from n entries
// (document, value) in device memory to the rank arrays of both orders that sort_walk_kernel reads (sort.cuh).
//
// The rank rule (oramacore_b200.h, sortBy deviations 1 and 2): a value is normalised with + 0.0 (-0.0 and +0.0 are one
// value); ASC orders by ascending value, DESC by descending value, equal values by ascending document in both; a
// document is placed once, at its first position in that order (its minimum for ASC, its maximum for DESC).  Entries
// whose document is >= nbits, or (variant fields) that lie in no variant, are dropped.
//   1. sf_keys_kernel gives every entry its document (SF_DROP when dropped) and the order-preserving key of its value
//      (fc_order, facet_commit.cuh); cub::DeviceRadixSort sorts the entries by document;
//   2. per order, a stable radix sort by key (ascending, or descending for DESC) keeps the document order inside a
//      value, so the entries are in rank order with repeats; sf_first_kernel puts each document's first position into
//      a [nbits] array with atomicMin (the minimum does not depend on scheduling);
//   3. cub::DeviceScan counts the entries that are their document's first position (the rank of each);
//   4. sf_scatter_kernel writes rank_doc[rank], doc_rank[doc] and the rank's value (decoded from its key): every
//      slot once, so the build is deterministic.
// Roofline: HBM.  Per entry about 12 B keyed, three radix sorts of 12 B pairs (8 passes of 8 B keys, 4 of 4 B keys)
// and per order 4 B atomics, 8 B of flags and ranks and 20 B scattered; per document id 4 B set and 4 B written per
// order.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "facet_commit.cuh"

namespace oc {

constexpr uint32_t SF_THREADS = 256;
constexpr uint32_t SF_DROP = 0xffffffffu;   // the document of a dropped entry (nbits < 2^32 - 1: never a real one)

// where an entry's value comes from: vals[i], or var_vals[v] for the variant v with off[v] <= i < off[v + 1]
struct SfSource {
    const double *vals;
    const uint64_t *off;       // [n_var + 1]; entries before off[0] are in no variant
    const double *var_vals;    // [n_var]
    uint32_t n_var;
};

__global__ void __launch_bounds__(SF_THREADS) sf_keys_kernel(const uint64_t *docs, uint64_t n, uint64_t nbits, const SfSource s,
                                                             uint32_t *doc, unsigned long long *key) {
    const uint64_t i = uint64_t(blockIdx.x) * SF_THREADS + threadIdx.x;
    if (i >= n) return;
    const uint64_t d = docs[i];
    bool ok = d < nbits;
    double v = 0.0;
    if (s.vals) {
        v = s.vals[i];
    } else if (i < s.off[0]) {
        ok = false;
    } else {
        uint32_t lo = 0, hi = s.n_var;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (s.off[mid] <= i) lo = mid; else hi = mid;
        }
        v = s.var_vals[lo];
    }
    doc[i] = ok ? uint32_t(d) : SF_DROP;
    key[i] = fc_order(v + 0.0);   // -0.0 ties with +0.0
}

__global__ void __launch_bounds__(SF_THREADS) sf_first_kernel(const uint32_t *doc, uint64_t n, uint32_t *first) {
    const uint64_t j = uint64_t(blockIdx.x) * SF_THREADS + threadIdx.x;
    if (j >= n || doc[j] == SF_DROP) return;
    atomicMin(&first[doc[j]], uint32_t(j));
}

// keep[n] = 0: the scan's last entry is the number of ranks
__global__ void __launch_bounds__(SF_THREADS) sf_keep_kernel(const uint32_t *doc, uint64_t n, const uint32_t *first, uint32_t *keep) {
    const uint64_t j = uint64_t(blockIdx.x) * SF_THREADS + threadIdx.x;
    if (j > n) return;
    keep[j] = (j < n && doc[j] != SF_DROP && first[doc[j]] == uint32_t(j)) ? 1u : 0u;
}

// the value of a key of fc_order (exact: the key holds all 64 bits)
__device__ __forceinline__ double sf_value(unsigned long long k) {
    const unsigned long long b = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
    double v;
    memcpy(&v, &b, 8);
    return v;
}

__global__ void __launch_bounds__(SF_THREADS) sf_scatter_kernel(const uint32_t *doc, const unsigned long long *key, const uint32_t *rank,
                                                                uint64_t n, uint64_t *rank_doc, uint32_t *doc_rank, double *rank_value) {
    const uint64_t j = uint64_t(blockIdx.x) * SF_THREADS + threadIdx.x;
    if (j >= n) return;
    const uint32_t r = rank[j];
    if (rank[j + 1] == r) return;   // not its document's first position
    const uint32_t d = doc[j];
    rank_doc[r] = d;
    doc_rank[d] = r;
    rank_value[r] = sf_value(key[j]);
}

}  // namespace oc
