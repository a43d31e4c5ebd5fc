// dict_dev.cuh — typo-tolerant query-term expansion on the device (oc_dict_resolve_q): a mirror of a term dictionary
// per ctx, and the kernels that test every sorted term of it against all fuzzy (token, field) pairs of a batch.
//
// A pair selects each sorted position whose term starts with the token or lies within byte-wise global Levenshtein
// distance t of it — the semantics of ocd::Dict::fuzzy.  The distance is the bit-parallel Myers/Hyyrö recurrence with
// the token as one 64-bit pattern word (ocd::FUZZY_RUN_MAX_TOK); a term whose length differs from the token's by more
// than t can only match as a prefix and skips it.  One CTA stages FZ_CHUNK sorted terms (the first stride - 4 bytes of
// each: the longest prefix test or recurrence of the batch reads no further) in shared memory and tests them against
// every pair of their field, so a batch reads the dictionary from HBM once; when the vocabulary has too few chunks to
// fill the GPU, a chunk's pairs are split over a few CTAs, which re-read the chunk from L2.  Output is an ordered compaction without atomics on
// the order: the count pass writes each (pair, chunk)'s matches, a scan turns them into offsets, and the emit pass
// re-tests only the (pair, chunk)s that matched and writes their terms in ascending position — Dict::fuzzy's order.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "dict.h"

namespace ocdd {

constexpr uint32_t FZ_CHUNK = 1024;     // sorted positions per CTA
constexpr uint32_t FZ_THREADS = 256;    // thread i tests positions i, i + 256, ...
constexpr uint32_t FZ_GROUP = 8;        // pairs whose match tables share shared memory in the count pass

struct FzField {                 // one field of the mirror as the kernels read it
    const uint8_t *bytes;        // term bytes in id order
    const uint64_t *off;         // term id -> bytes [off[id], off[id + 1])
    const uint32_t *sorted;      // sorted position -> term id
    uint32_t n;                  // sorted positions
    uint32_t chunk0, n_chunks;   // the field's CTAs (none when no pair reads the field)
    uint32_t p0, p1;             // its pairs: the pair list is ordered by field
};
struct FzPair {
    uint32_t m, t, field;        // token length (<= 64), tolerance (>= 1)
    uint32_t slot;               // counts[slot .. slot + n_chunks]: matches per chunk, then (scanned) offsets and total
    uint8_t tok[64];
};

// smem: the match tables of FZ_GROUP pairs, their tokens, the chunk's term ids, 32 reduction words, term lengths
// (clamped to 255: anything past the staged bytes only needs to be "longer"), then the term bytes at `stride`
inline size_t fuzzy_smem(uint32_t stride) {
    return size_t(FZ_GROUP) * 256 * 8 + FZ_GROUP * 64 + FZ_CHUNK * 4 + 32 * 4 + FZ_CHUNK + size_t(FZ_CHUNK) * stride;
}

// term (n bytes, the first min(n, staged) in shared memory) against token tok (m bytes) with match table peq
__device__ __forceinline__ bool fz_test(const uint8_t *term, uint32_t n, const uint8_t *tok, uint32_t m, uint32_t t,
                                        const uint64_t *peq, bool *exact) {
    bool pre = n >= m;
    for (uint32_t i = 0; pre && i < m; i++) pre = term[i] == tok[i];
    *exact = pre && n == m;
    if (pre) return true;
    if (n + t < m || n > m + t) return false;
    // each term byte that occurs nowhere in the token costs an edit of its own: more than t of them rule the term out
    uint32_t miss = 0;
    for (uint32_t i = 0; i < n; i++)
        if (!peq[term[i]] && ++miss > t) return false;
    // global edit distance (Hyyrö): row 0 of the DP grows by one per term byte, hence the carry-in of 1
    uint64_t vp = ~0ull, vn = 0;
    uint32_t d = m;
    const uint64_t hb = 1ull << (m - 1);
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t eq = peq[term[i]];
        const uint64_t d0 = (((eq & vp) + vp) ^ vp) | eq | vn;
        const uint64_t hp = vn | ~(d0 | vp), hn = vp & d0;
        d += (hp & hb) ? 1u : 0u;
        d -= (hn & hb) ? 1u : 0u;
        const uint64_t x = (hp << 1) | 1ull;
        vn = x & d0;
        vp = (hn << 1) | ~(x | d0);
    }
    return d <= t;
}

// EMIT = false: counts[slot + c] = matches of each pair in chunk c.  EMIT = true (counts scanned): writes each pair's
// matches of chunk c, ascending, at out0[pair] + counts[slot + c].  CTA b takes chunk b / split and the (b % split)-th
// of `split` slices of the chunk's pairs: a vocabulary of few chunks still fills the GPU.
template <bool EMIT>
__global__ void __launch_bounds__(FZ_THREADS) dict_fuzzy_kernel(const FzField *__restrict__ fields, uint32_t n_fields,
                                                                const FzPair *__restrict__ pairs, uint32_t stride, uint32_t split,
                                                                uint32_t *__restrict__ counts, const uint32_t *__restrict__ out0,
                                                                uint32_t *__restrict__ out_id, uint8_t *__restrict__ out_exact) {
    extern __shared__ __align__(16) uint8_t fz_smem[];
    uint64_t *peq = reinterpret_cast<uint64_t *>(fz_smem);
    uint8_t *tok = fz_smem + FZ_GROUP * 256 * 8;
    uint32_t *ids = reinterpret_cast<uint32_t *>(tok + FZ_GROUP * 64);
    uint32_t *red = ids + FZ_CHUNK;
    uint8_t *lens = reinterpret_cast<uint8_t *>(red + 32);
    uint8_t *bytes = lens + FZ_CHUNK;
    constexpr uint32_t G = EMIT ? 1 : FZ_GROUP;

    const uint32_t chunk = blockIdx.x / split, slice = blockIdx.x % split;
    uint32_t fi = 0;
    while (fi + 1 < n_fields && chunk >= fields[fi].chunk0 + fields[fi].n_chunks) fi++;
    const FzField F = fields[fi];
    const uint32_t c = chunk - F.chunk0, s0 = c * FZ_CHUNK, cnt = min(FZ_CHUNK, F.n - s0);
    const uint32_t pb = F.p0 + uint32_t(uint64_t(F.p1 - F.p0) * slice / split);
    const uint32_t pe = F.p0 + uint32_t(uint64_t(F.p1 - F.p0) * (slice + 1) / split);
    if (pb == pe) return;
    const uint32_t staged = stride - 4;
    for (uint32_t j = threadIdx.x; j < cnt; j += FZ_THREADS) {
        const uint32_t id = F.sorted[s0 + j];
        const uint64_t o = F.off[id], len = F.off[id + 1] - o;
        ids[j] = id;
        lens[j] = (uint8_t)(len < 255 ? len : 255);
        const uint32_t k = (uint32_t)(len < staged ? len : staged);
        for (uint32_t i = 0; i < k; i++) bytes[j * stride + i] = F.bytes[o + i];
    }
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t p = pb; p < pe; p += G) {
        const uint32_t g = min(G, pe - p);
        if (EMIT && counts[pairs[p].slot + c + 1] == counts[pairs[p].slot + c]) continue;
        __syncthreads();   // the staging, or the previous group's use of the tables, is done
        for (uint32_t i = threadIdx.x; i < g * 256; i += FZ_THREADS) peq[i] = 0;
        for (uint32_t i = threadIdx.x; i < g * 64; i += FZ_THREADS) tok[i] = pairs[p + i / 64].tok[i % 64];
        if (threadIdx.x < 32) red[threadIdx.x] = 0;
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < g * 64; i += FZ_THREADS)
            if (i % 64 < pairs[p + i / 64].m) atomicOr(reinterpret_cast<unsigned long long *>(&peq[(i / 64) * 256 + tok[i]]), 1ull << (i % 64));
        __syncthreads();
        for (uint32_t q = 0; q < g; q++) {
            const FzPair &P = pairs[p + q];
            const uint32_t m = P.m, t = P.t;
            if (!EMIT) {
                uint32_t hits = 0;
                for (uint32_t j = threadIdx.x; j < cnt; j += FZ_THREADS) {
                    bool ex;
                    hits += fz_test(bytes + j * stride, lens[j], tok + q * 64, m, t, peq + q * 256, &ex) ? 1u : 0u;
                }
                hits = __reduce_add_sync(0xffffffffu, hits);
                if (lane == 0 && hits) atomicAdd(&red[q], hits);
            } else {
                uint32_t base = out0[p] + counts[P.slot + c];
                for (uint32_t j0 = 0; j0 < cnt; j0 += FZ_THREADS) {
                    const uint32_t j = j0 + threadIdx.x;
                    bool ex = false;
                    const bool hit = j < cnt && fz_test(bytes + j * stride, lens[j], tok, m, t, peq, &ex);
                    const uint32_t bal = __ballot_sync(0xffffffffu, hit);
                    if (lane == 0) red[warp] = __popc(bal);
                    __syncthreads();
                    uint32_t before = 0, total = 0;
                    for (uint32_t v = 0; v < FZ_THREADS / 32; v++) {
                        const uint32_t x = red[v];
                        before += v < warp ? x : 0u;
                        total += x;
                    }
                    if (hit) {
                        const uint32_t at = base + before + __popc(bal & ((1u << lane) - 1u));
                        out_id[at] = ids[j];
                        out_exact[at] = ex ? 1 : 0;
                    }
                    base += total;
                    __syncthreads();
                }
            }
        }
        if (!EMIT) {
            __syncthreads();
            if (threadIdx.x < g) counts[pairs[p + threadIdx.x].slot + c] = red[threadIdx.x];
        }
    }
}

// one CTA per pair: its n_chunks counts become exclusive offsets, slot + n_chunks the total, totals[pair] = total
__global__ void __launch_bounds__(FZ_THREADS) dict_fuzzy_scan_kernel(const FzField *__restrict__ fields, const FzPair *__restrict__ pairs,
                                                                     uint32_t *__restrict__ counts, uint32_t *__restrict__ totals) {
    __shared__ uint32_t wsum[FZ_THREADS / 32];
    const FzPair &P = pairs[blockIdx.x];
    const uint32_t nch = fields[P.field].n_chunks;
    uint32_t *v = counts + P.slot;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t carry = 0;
    for (uint32_t c0 = 0; c0 < nch; c0 += FZ_THREADS) {
        const uint32_t i = c0 + threadIdx.x;
        const uint32_t x = i < nch ? v[i] : 0u;
        uint32_t s = x;
        for (uint32_t o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        if (lane == 31) wsum[warp] = s;
        __syncthreads();
        uint32_t before = 0, total = 0;
        for (uint32_t w = 0; w < FZ_THREADS / 32; w++) {
            before += w < warp ? wsum[w] : 0u;
            total += wsum[w];
        }
        if (i < nch) v[i] = carry + before + s - x;
        carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        v[nch] = carry;
        totals[blockIdx.x] = carry;
    }
}

// device memory that grows on demand and keeps a prefix of its content when it moves
struct DevArr {
    void *p = nullptr;
    size_t cap = 0;
    DevArr() = default;
    DevArr(const DevArr &) = delete;
    DevArr &operator=(const DevArr &) = delete;
    ~DevArr() { if (p) cudaFree(p); }
    cudaError_t reserve(size_t bytes, size_t keep, cudaStream_t st) {
        if (bytes <= cap) return cudaSuccess;
        size_t want = bytes + bytes / 4 + 256;
        void *q = nullptr;
        cudaError_t e = cudaMalloc(&q, want);
        if (e != cudaSuccess) { cudaGetLastError(); want = bytes; e = cudaMalloc(&q, want); }
        if (e != cudaSuccess) return e;
        if (keep && (e = cudaMemcpyAsync(q, p, keep, cudaMemcpyDeviceToDevice, st)) != cudaSuccess) { cudaFree(q); return e; }
        if (p) cudaFree(p);   // waits for the copy
        p = q; cap = want;
        return cudaSuccess;
    }
    template <typename T> T *as() const { return reinterpret_cast<T *>(p); }
};

// A dictionary's terms on one device.  Ids are stable and new terms append, so a refresh uploads the bytes of the terms
// indexed since the last one; the sorted permutation is uploaded again whenever a reindex changed it.  The ctx owns the
// mirror and watches the dictionary through `owner` (dense_cache.h's scheme): a mirror whose dictionary is gone is
// freed by the ctx's next device resolve, or by oc_shutdown; oc_dict_destroy never touches a ctx.
struct DictMirror {
    struct Field {
        DevArr bytes, off, sorted;
        uint64_t n_terms = 0, n_bytes = 0, n_sorted = 0;
    };
    std::weak_ptr<const uint64_t> owner;
    uint64_t gen = ~0ull;                  // Dict::generation() the mirror reflects
    std::unique_ptr<Field[]> f;
    size_t n_fields = 0;
    explicit DictMirror(size_t n) : f(new Field[n]), n_fields(n) {}
    uint64_t device_bytes() const {        // term bytes, 8 B of offset and 4 B of permutation per term
        uint64_t b = 0;
        for (size_t i = 0; i < n_fields; i++) b += f[i].n_bytes + (f[i].n_terms + (f[i].n_terms ? 1 : 0)) * 8 + f[i].n_sorted * 4;
        return b;
    }
    // fields and g under the dictionary's shared lock; uploads run on st and the host sources are copied before return
    cudaError_t sync(const std::vector<ocd::FieldDict> &fields, uint64_t g, cudaStream_t st) {
        if (g == gen) return cudaSuccess;
        cudaError_t e;
        for (size_t fi = 0; fi < n_fields; fi++) {
            const ocd::FieldDict &D = fields[fi];
            Field &M = f[fi];
            const uint64_t n = D.n_indexed;    // the ids `sorted` holds
            if (M.n_terms < n) {
                std::string blob;
                std::vector<uint64_t> off(1, M.n_bytes);   // off[M.n_terms .. n]
                for (uint64_t id = M.n_terms; id < n; id++) {
                    blob += D.terms[id];
                    off.push_back(M.n_bytes + blob.size());
                }
                if ((e = M.bytes.reserve(M.n_bytes + blob.size(), M.n_bytes, st)) != cudaSuccess) return e;
                if ((e = M.off.reserve((n + 1) * 8, M.n_terms ? (M.n_terms + 1) * 8 : 0, st)) != cudaSuccess) return e;
                if (!blob.empty() &&
                    (e = cudaMemcpyAsync(M.bytes.as<uint8_t>() + M.n_bytes, blob.data(), blob.size(), cudaMemcpyHostToDevice, st)) != cudaSuccess)
                    return e;
                if ((e = cudaMemcpyAsync(M.off.as<uint64_t>() + M.n_terms, off.data(), off.size() * 8, cudaMemcpyHostToDevice, st)) != cudaSuccess)
                    return e;
                M.n_terms = n;
                M.n_bytes += blob.size();
            }
            if (M.n_sorted != D.sorted.size()) {
                if ((e = M.sorted.reserve(D.sorted.size() * 4, 0, st)) != cudaSuccess) return e;
                if ((e = cudaMemcpyAsync(M.sorted.p, D.sorted.data(), D.sorted.size() * 4, cudaMemcpyHostToDevice, st)) != cudaSuccess) return e;
                M.n_sorted = D.sorted.size();
            }
        }
        gen = g;
        return cudaSuccess;
    }
};

}  // namespace ocdd
