// group.cuh — the group stage of oc_search_groups: for every (query, group) the top max_results documents of
// the group that are keys of the query's score map.
//
// Replaces GroupContext::execute (read/index/group.rs) + sort_groups (read/sort.rs:129-230, the branch without
// sort_by): per group, a capped heap of (NotNan score, doc) over the group's documents found in the score map.
//
// The score map never leaves the device.  Its fulltext part is the matched-row bitmap and the raw row scores the
// tile kernels emit in group mode (Bm25Params::matched_bits / row_ft); its vector part is the list of unique vector
// hits with their final scores that K4 exports (FuseParams::out_vdoc / out_vscore), together with the hybrid
// normalisation (out_gmin / out_den).  A document that is a vector hit takes the hit's score (in hybrid mode that
// score replaced the row's fulltext-only score, as in K4); any other document takes fused_ft_score() of its row.
#pragma once
#include "fuse.cuh"

namespace oc {

constexpr uint32_t GROUP_THREADS = 256;
constexpr uint32_t GROUP_CHUNK = GROUP_THREADS * 4;   // documents visited between two looks at the candidate buffer
constexpr uint32_t GROUP_BUF = 2048;                  // candidate keys in shared memory: >= OC_MAX_TOPK + GROUP_CHUNK

struct GroupParams {
    uint32_t n_groups, max_results;
    uint32_t kp2, vp2;              // selection scratch: max(32, next_pow2(max_results)); vector hits: next_pow2(v_stride)
    const uint64_t *g_off;          // [n_groups + 1] group CSR
    const uint64_t *g_doc;          // document ids, ascending inside each group
    const uint32_t *g_row;          // string row of each entry (0xffffffff = none); NULL without a fulltext map
    // fulltext part of the score map (has_ft)
    bool has_ft, hybrid;
    const uint32_t *mbits;          // [q][row_words]
    uint64_t row_words;
    const float *row_ft;            // [q][row_words * 32]
    const float *gmin, *den;        // [q]
    // vector part: unique hits, final scores
    const uint64_t *v_doc;
    const float *v_score;
    const uint32_t *v_n;            // [q]
    uint32_t v_stride;
    const uint64_t *omc_doc;
    const float *omc_mult;
    uint32_t n_omc;
    uint64_t *out_doc;              // [q][n_groups][max_results]
    float *out_score;
    uint32_t *out_n;                // [q][n_groups]
    // group_sort_topk_kernel: the sort field's rank of each document id (0xffffffff = no value)
    const uint32_t *doc_rank;
    uint64_t rank_nbits;
};

// SORT = false: the top max_results members by score (score desc, ties by ascending id, NaN dropped).
// SORT = true (sortBy, sort_groups with sort_by, read/sort.rs:147-166): the first max_results members in the sort
// field's rank order; the key is the rank instead of the score, NaN scores are kept and members with no value skipped.
template <bool SORT>
__device__ __forceinline__ void group_topk_body(const GroupParams &p) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *buf = reinterpret_cast<uint64_t *>(smem);   // [GROUP_BUF] candidate keys (score | position in group)
    uint64_t *sel = buf + GROUP_BUF;                       // [kp2]
    uint64_t *hdoc = sel + p.kp2;                          // [vp2] vector hits sorted by document id
    float *hsc = reinterpret_cast<float *>(hdoc + p.vp2);  // [vp2] their scores
    __shared__ uint32_t s_n;
    __shared__ unsigned long long s_tau;
    const uint32_t g = blockIdx.x, q = blockIdx.y, tid = threadIdx.x;
    const uint32_t m = p.max_results;
    const size_t og = size_t(q) * p.n_groups + g;
    if (m == 0) {
        if (tid == 0) p.out_n[og] = 0;
        return;
    }
    const uint64_t base = p.g_off[g], n = p.g_off[g + 1] - base;
    const uint64_t *gdoc = p.g_doc + base;
    const uint32_t *grow = p.g_row ? p.g_row + base : nullptr;

    const uint32_t vc = p.v_n[q];
    if (vc) {   // bitonic sort of the query's hits by document id (ascending, padding last)
        for (uint32_t i = tid; i < p.vp2; i += blockDim.x) {
            hdoc[i] = i < vc ? p.v_doc[size_t(q) * p.v_stride + i] : ~0ull;
            hsc[i] = i < vc ? p.v_score[size_t(q) * p.v_stride + i] : 0.f;
        }
        __syncthreads();
        for (uint32_t k = 2; k <= p.vp2; k <<= 1)
            for (uint32_t j = k >> 1; j > 0; j >>= 1) {
                for (uint32_t i = tid; i < p.vp2; i += blockDim.x) {
                    const uint32_t ixj = i ^ j;
                    if (ixj > i) {
                        const uint64_t a = hdoc[i], b = hdoc[ixj];
                        if (((i & k) == 0) ? (a > b) : (a < b)) {
                            hdoc[i] = b; hdoc[ixj] = a;
                            const float t = hsc[i]; hsc[i] = hsc[ixj]; hsc[ixj] = t;
                        }
                    }
                }
                __syncthreads();
            }
    }
    const float gmin = p.has_ft ? p.gmin[q] : 0.f, den = p.has_ft ? p.den[q] : 0.f;
    const uint32_t *mb = p.has_ft ? p.mbits + size_t(q) * p.row_words : nullptr;
    const float *rft = p.has_ft ? p.row_ft + size_t(q) * p.row_words * 32 : nullptr;

    // sort: the i-th member's score-map value; *present = 0 when it is not a key
    auto map_value = [&](uint64_t i, bool *present) -> float {
        *present = true;
        if (vc) {
            const uint64_t d = gdoc[i];
            uint32_t lo = 0, hi = vc;
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (hdoc[mid] < d) lo = mid + 1; else hi = mid; }
            if (lo < vc && hdoc[lo] == d) return hsc[lo];
        }
        const uint32_t row = p.has_ft ? grow[i] : 0xffffffffu;
        if (row == 0xffffffffu || !((mb[row >> 5] >> (row & 31)) & 1u)) { *present = false; return 0.f; }
        return fused_ft_score(rft[row], p.hybrid, gmin, den, p.omc_doc, p.omc_mult, p.n_omc, [&] { return gdoc[i]; });
    };
    // rank key of the i-th document of the group, KEY_NONE when it is not a key of the score map (or scores NaN)
    auto load = [&](uint64_t i) -> uint64_t {
        if constexpr (SORT) {   // larger key = smaller rank; ranks are unique, so the member index only decodes
            const uint64_t d = gdoc[i];
            const uint32_t r = d < p.rank_nbits ? p.doc_rank[d] : 0xffffffffu;
            if (r == 0xffffffffu) return KEY_NONE;
            bool present;
            map_value(i, &present);
            return present ? (uint64_t(0xffffffffu - r) << 32) | uint64_t(0xffffffffu - uint32_t(i)) : KEY_NONE;
        }
        if (vc) {
            const uint64_t d = gdoc[i];
            uint32_t lo = 0, hi = vc;
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (hdoc[mid] < d) lo = mid + 1; else hi = mid; }
            if (lo < vc && hdoc[lo] == d) {
                const float f = hsc[lo];
                return f == f ? make_key(f, uint32_t(i)) : KEY_NONE;
            }
        }
        if (!p.has_ft) return KEY_NONE;
        const uint32_t row = grow[i];
        if (row == 0xffffffffu || !((mb[row >> 5] >> (row & 31)) & 1u)) return KEY_NONE;
        const float f = fused_ft_score(rft[row], p.hybrid, gmin, den, p.omc_doc, p.omc_mult, p.n_omc, [&] { return gdoc[i]; });
        return f == f ? make_key(f, uint32_t(i)) : KEY_NONE;   // NaN dropped (NotNan, sort.rs:205-209)
    };

    // stream the group: keys above the running m-th best go to the buffer; a full buffer is cut back to its m best
    if (tid == 0) { s_n = 0; s_tau = KEY_NONE; }
    for (uint32_t i = tid; i < p.kp2; i += blockDim.x) sel[i] = KEY_NONE;
    __syncthreads();
    for (uint64_t c0 = 0; c0 < n; c0 += GROUP_CHUNK) {   // block-uniform trip count
        const unsigned long long tau = s_tau;
#pragma unroll
        for (uint32_t u = 0; u < GROUP_CHUNK / GROUP_THREADS; u++) {
            const uint64_t i = c0 + u * GROUP_THREADS + tid;
            if (i < n) {
                const uint64_t key = load(i);
                if (key > tau) buf[atomicAdd(&s_n, 1u)] = key;
            }
        }
        __syncthreads();
        const uint32_t cnt = s_n;   // snapshot, then barrier, so the branch is block-uniform
        __syncthreads();
        if (cnt + GROUP_CHUNK > GROUP_BUF && c0 + GROUP_CHUNK < n) {
            const uint32_t kept = block_select_largest(buf, cnt, m, sel);
            group_bitonic_desc(sel, p.kp2, tid, blockDim.x, 0);
            for (uint32_t i = tid; i < p.kp2; i += blockDim.x) {
                if (i < kept) buf[i] = sel[i];
                sel[i] = KEY_NONE;
            }
            __syncthreads();
            if (tid == 0) {
                s_n = kept;
                if (kept == m) s_tau = buf[m - 1];
            }
            __syncthreads();
        }
    }
    const uint32_t cnt = s_n;
    const uint32_t kept = block_select_largest(buf, cnt, m, sel);
    group_bitonic_desc(sel, p.kp2, tid, blockDim.x, 0);
    for (uint32_t i = tid; i < m; i += blockDim.x) {
        uint64_t doc = 0;
        float sc = 0.f;
        if (i < kept) {
            doc = gdoc[key_idx(sel[i])];
            if constexpr (SORT) {
                bool present;
                sc = map_value(key_idx(sel[i]), &present);   // NaN kept
            } else {
                sc = key_score(sel[i]);
            }
        }
        p.out_doc[og * m + i] = doc;
        p.out_score[og * m + i] = sc;
    }
    if (tid == 0) p.out_n[og] = kept;
}

// one CTA per (group, query): grid (n_groups, n_queries)
__global__ void __launch_bounds__(GROUP_THREADS) group_topk_kernel(const GroupParams p) { group_topk_body<false>(p); }
__global__ void __launch_bounds__(GROUP_THREADS) group_sort_topk_kernel(const GroupParams p) { group_topk_body<true>(p); }

}  // namespace oc
