// facet_commit.cuh — the device half of oc_facets_commit_ex and oc_geo_field_commit_ex: merges the pending values of a
// filter field into the next version of its device arrays without a host copy of the committed values.
//
// Every field kind is one sorted array of entries, each with a 128-bit key (hi, lo):
//   bool / string_filter (variant-major CSR):  (variant, doc)
//   number / date (sorted by value):           (fc_order(value), doc)  — ascending value, -0.0 before +0.0, then doc
//   geopoint (sorted by document):             (doc, 0)                — equal keys keep their order, committed first
// The host filters the pending ops (O(pending)): an insert survives when no later delete (or clear of its field)
// names its document, and a set-semantics insert (OC_FACET_UNIQUE) also when no earlier surviving insert has its key.
// It sorts the survivors by (key, call order) and uploads them with the sorted list of documents killed in the field.
// Then, on the handle's commit stream:
//   1. fc_keys_*_kernel gives every committed entry its key and a keep flag (its document is not in the kill list,
//      a binary search); fc_unique_kernel drops a set-semantics pending entry whose key a kept committed entry has;
//   2. cub::DeviceScan turns both flag arrays into ranks (one more entry at the end: the totals);
//   3. fc_scatter_*_kernel writes every output slot exactly once, so the result does not depend on scheduling:
//        committed entry i: rank_a[i] + rank_b[pending entries with a key <  key_a[i]]
//        pending entry j:   rank_b[j] + rank_a[committed entries with a key <= key_b[j]]
//      and fc_offsets_kernel gives a CSR field its new variant offsets the same way.
// Roofline: HBM.  Per committed entry about 8 B of payload read twice, its 16 B key written and read, 2 x 4 B of flag
// and rank, and the payload written once; per pending entry about 64 B.  The binary searches are log2(pending) and
// log2(committed) reads from L2.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace oc {

constexpr uint32_t FC_THREADS = 256;

struct FcKey { unsigned long long hi, lo; };

__host__ __device__ __forceinline__ bool fc_less(const FcKey &a, const FcKey &b) {
    return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo);
}
__host__ __device__ __forceinline__ bool fc_equal(const FcKey &a, const FcKey &b) { return a.hi == b.hi && a.lo == b.lo; }
// a double's bits mapped to an unsigned integer of the same order (no NaN)
__host__ __device__ __forceinline__ unsigned long long fc_order(double v) {
    unsigned long long b;
    memcpy(&b, &v, 8);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}

// number of k[0, n) below x (UPPER: not above x)
template <bool UPPER>
__device__ __forceinline__ uint64_t fc_bound(const FcKey *k, uint64_t n, FcKey x) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        const FcKey m = k[mid];
        if (UPPER ? !fc_less(x, m) : fc_less(m, x)) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ bool fc_killed(const uint64_t *kill, uint64_t n_kill, uint64_t d) {
    uint64_t lo = 0, hi = n_kill;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (kill[mid] < d) lo = mid + 1; else hi = mid;
    }
    return lo < n_kill && kill[lo] == d;
}

// keep[n] = 0: the scan's last entry is the total
__global__ void __launch_bounds__(FC_THREADS) fc_keys_csr_kernel(const uint64_t *docs, uint64_t n, const uint64_t *off, uint32_t n_var,
                                                                 const uint64_t *kill, uint64_t n_kill, FcKey *key, uint32_t *keep) {
    const uint64_t i = uint64_t(blockIdx.x) * FC_THREADS + threadIdx.x;
    if (i > n) return;
    if (i == n) { keep[n] = 0; return; }
    uint32_t lo = 0, hi = n_var;   // the variant v with off[v] <= i < off[v + 1]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (off[mid] <= i) lo = mid; else hi = mid;
    }
    const uint64_t d = docs[i];
    key[i] = FcKey{lo, d};
    keep[i] = (i >= off[0] && !fc_killed(kill, n_kill, d)) ? 1u : 0u;   // entries before off[0] are in no variant
}
__global__ void __launch_bounds__(FC_THREADS) fc_keys_num_kernel(const double *vals, const uint64_t *docs, uint64_t n, const uint64_t *kill,
                                                                 uint64_t n_kill, FcKey *key, uint32_t *keep) {
    const uint64_t i = uint64_t(blockIdx.x) * FC_THREADS + threadIdx.x;
    if (i > n) return;
    if (i == n) { keep[n] = 0; return; }
    const uint64_t d = docs[i];
    key[i] = FcKey{fc_order(vals[i]), d};
    keep[i] = fc_killed(kill, n_kill, d) ? 0u : 1u;
}
__global__ void __launch_bounds__(FC_THREADS) fc_keys_geo_kernel(const uint64_t *docs, uint64_t n, const uint64_t *kill, uint64_t n_kill,
                                                                 FcKey *key, uint32_t *keep) {
    const uint64_t i = uint64_t(blockIdx.x) * FC_THREADS + threadIdx.x;
    if (i > n) return;
    if (i == n) { keep[n] = 0; return; }
    const uint64_t d = docs[i];
    key[i] = FcKey{d, 0};
    keep[i] = fc_killed(kill, n_kill, d) ? 0u : 1u;
}
// b_keep[j] == 2 on entry: a set-semantics insert, kept (1) unless a kept committed entry has its key (0)
__global__ void __launch_bounds__(FC_THREADS) fc_unique_kernel(const FcKey *ka, const uint32_t *a_keep, uint64_t n_a, const FcKey *kb,
                                                               uint64_t n_b, uint32_t *b_keep) {
    const uint64_t j = uint64_t(blockIdx.x) * FC_THREADS + threadIdx.x;
    if (j >= n_b || b_keep[j] != 2) return;
    const FcKey x = kb[j];
    const uint64_t i = fc_bound<false>(ka, n_a, x);
    b_keep[j] = (i < n_a && fc_equal(ka[i], x) && a_keep[i]) ? 0u : 1u;   // a set-semantics field holds each key once
}

// W::a(i, slot) writes committed entry i, W::b(j, slot) pending entry j
template <class W>
__global__ void __launch_bounds__(FC_THREADS) fc_scatter_a_kernel(const FcKey *ka, const uint32_t *a_keep, const uint32_t *a_rank, uint64_t n_a,
                                                                  const FcKey *kb, const uint32_t *b_rank, uint64_t n_b, W w) {
    const uint64_t i = uint64_t(blockIdx.x) * FC_THREADS + threadIdx.x;
    if (i >= n_a || !a_keep[i]) return;
    w.a(i, uint64_t(a_rank[i]) + b_rank[fc_bound<false>(kb, n_b, ka[i])]);
}
template <class W>
__global__ void __launch_bounds__(FC_THREADS) fc_scatter_b_kernel(const FcKey *ka, const uint32_t *a_rank, uint64_t n_a, const FcKey *kb,
                                                                  const uint32_t *b_keep, const uint32_t *b_rank, uint64_t n_b, W w) {
    const uint64_t j = uint64_t(blockIdx.x) * FC_THREADS + threadIdx.x;
    if (j >= n_b || !b_keep[j]) return;
    w.b(j, uint64_t(b_rank[j]) + a_rank[fc_bound<true>(ka, n_a, kb[j])]);
}
// new_off[v] for v in [0, n_var]: kept committed entries of the variants below v + kept pending ones
__global__ void __launch_bounds__(FC_THREADS) fc_offsets_kernel(const uint64_t *old_off, uint32_t old_var, const uint32_t *a_rank,
                                                                const FcKey *kb, const uint32_t *b_rank, uint64_t n_b, uint32_t n_var,
                                                                uint64_t *new_off) {
    const uint32_t v = blockIdx.x * FC_THREADS + threadIdx.x;
    if (v > n_var) return;
    new_off[v] = uint64_t(a_rank[old_off[min(v, old_var)]]) + b_rank[fc_bound<false>(kb, n_b, FcKey{v, 0})];
}

struct FcCsrW {
    const uint64_t *docs; const FcKey *kb; uint64_t *out;
    __device__ void a(uint64_t i, uint64_t s) const { out[s] = docs[i]; }
    __device__ void b(uint64_t j, uint64_t s) const { out[s] = kb[j].lo; }
};
struct FcNumW {
    const double *vals; const uint64_t *docs; const double *b_vals; const FcKey *kb; double *out_v; uint64_t *out_d;
    __device__ void a(uint64_t i, uint64_t s) const { out_v[s] = vals[i]; out_d[s] = docs[i]; }
    __device__ void b(uint64_t j, uint64_t s) const { out_v[s] = b_vals[j]; out_d[s] = kb[j].lo; }
};
// geopoint: 5 f64 columns (x, y, z, lat, lon) then the doc column, n entries each (oc_geo_field's blob)
struct FcGeoW {
    const double *src; uint64_t n_src; const double *b_cols; uint64_t n_b; const FcKey *kb; double *out; uint64_t n_out;
    __device__ void a(uint64_t i, uint64_t s) const {
#pragma unroll
        for (int c = 0; c < 6; c++) out[c * n_out + s] = src[c * n_src + i];
    }
    __device__ void b(uint64_t j, uint64_t s) const {
#pragma unroll
        for (int c = 0; c < 5; c++) out[c * n_out + s] = b_cols[c * n_b + j];
        reinterpret_cast<unsigned long long *>(out)[5 * n_out + s] = kb[j].hi;
    }
};

}  // namespace oc
