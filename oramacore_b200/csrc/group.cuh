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

// One distinct (field, order) of a batch: its documents in rank order and the maps between ranks, ids and rows.  The
// entries of sort_walk_kernel (sort.cuh); group_sort_topk_kernel takes the rank of each document id from them.
struct SortEntry {
    uint64_t n_ranks;               // documents with a value
    const uint32_t *rank_row;       // [n_ranks] string row of each rank, RANK_NONE = none; NULL without a fulltext map
    const uint32_t *doc_rank;       // [nbits] rank of each document id, RANK_NONE = no value
    uint64_t nbits;
    const uint64_t *rank_doc;       // [n_ranks]
};

// One distinct oc_group_by of a batch: its CSR.
struct GroupHandle {
    const uint64_t *g_off;          // [n_groups + 1] group CSR
    const uint64_t *g_doc;          // document ids, ascending inside each group
    const uint32_t *g_row;          // string row of each entry (0xffffffff = none); NULL without a fulltext map
    uint32_t n_groups;
};
// One query's groups in a work list of (query, group) items, one CTA each: items [first, first + n_groups of its
// handle).  Query q's group g is output row row + g.
struct GroupSpan {
    uint32_t first;                 // its first item (the list's prefix sum of n_groups)
    uint32_t q, h;                  // query, index into the handle table
    uint32_t depth;                 // top list depth: max_results, 2 x max_results for an active pinned query
    uint32_t max_results;
    uint32_t ent;                   // group_sort_topk_kernel: index into the sort entries
    uint32_t row;
};
// The span that holds `item`, the local-th of the list's n_items: the last one with first <= item (every span of a list
// holds at least one item).  The first guess, local's share of the n spans, is exact when every span has as many items
// (one handle for the whole list), so the common case costs one round of loads instead of a binary search.
__device__ __forceinline__ GroupSpan group_span_of(const GroupSpan *s, uint32_t n, uint32_t item, uint32_t local, uint32_t n_items) {
    uint32_t lo = uint32_t(uint64_t(local) * n / n_items);
    const uint32_t next = lo + 1 < n ? s[lo + 1].first : 0xffffffffu;
    if (s[lo].first <= item && item < next) return s[lo];
    uint32_t hi = n;
    lo = 0;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (s[mid].first <= item) lo = mid; else hi = mid; }
    return s[lo];
}

struct GroupParams {
    const GroupHandle *handles;
    const GroupSpan *spans;         // this launch's work list: n_spans spans, items item0 + blockIdx.x
    uint32_t n_spans, item0;
    uint32_t top;                   // row stride of the top lists: the largest depth of the batch
    uint32_t kp2, vp2;              // selection scratch: max(32, next_pow2(top)); vector hits: next_pow2(v_stride)
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
    uint64_t *out_doc;              // [row][top]
    float *out_score;
    uint32_t *out_n;                // [row]
    // group_sort_topk_kernel: the batch's sort entries (sort.cuh); a span's entry gives the rank of each document id
    const SortEntry *ents;
    const QueryPlan *q_plan;        // NULL, or [q]: a query is hybrid when hybrid is set and its own mode is
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
    // this CTA's span, with `first` turned into its group and `row` into its output row; read from shared memory
    // wherever a value must outlive a call of block_select_largest (kept in registers, it would be saved to the stack
    // around every call)
    __shared__ GroupSpan s_sp;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) {
        const uint32_t item = p.item0 + blockIdx.x;
        GroupSpan sp = group_span_of(p.spans, p.n_spans, item, blockIdx.x, gridDim.x);
        sp.row += item - sp.first;
        sp.first = item - sp.first;
        s_sp = sp;
    }
    __syncthreads();
    const GroupHandle gh = p.handles[s_sp.h];
    const uint32_t g = s_sp.first, q = s_sp.q;
    if (s_sp.depth == 0) {
        if (tid == 0) p.out_n[s_sp.row] = 0;
        return;
    }
    const uint64_t base = gh.g_off[g], n = gh.g_off[g + 1] - base;
    const uint64_t *gdoc = gh.g_doc + base;
    const uint32_t *grow = gh.g_row ? gh.g_row + base : nullptr;

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
    const bool hybrid = p.hybrid && (!p.q_plan || p.q_plan[q].mode == OC_MODE_HYBRID);
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
        return fused_ft_score(rft[row], hybrid, gmin, den, p.omc_doc, p.omc_mult, p.n_omc, [&] { return gdoc[i]; });
    };
    // rank key of the i-th document of the group, KEY_NONE when it is not a key of the score map (or scores NaN)
    auto load = [&](uint64_t i) -> uint64_t {
        if constexpr (SORT) {   // larger key = smaller rank; ranks are unique, so the member index only decodes
            const uint64_t d = gdoc[i];
            const SortEntry &e = p.ents[s_sp.ent];
            const uint32_t r = d < e.nbits ? e.doc_rank[d] : 0xffffffffu;
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
        const float f = fused_ft_score(rft[row], hybrid, gmin, den, p.omc_doc, p.omc_mult, p.n_omc, [&] { return gdoc[i]; });
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
            const uint32_t kept = block_select_largest(buf, cnt, s_sp.depth, sel);
            group_bitonic_desc(sel, p.kp2, tid, blockDim.x, 0);
            for (uint32_t i = tid; i < p.kp2; i += blockDim.x) {
                if (i < kept) buf[i] = sel[i];
                sel[i] = KEY_NONE;
            }
            __syncthreads();
            if (tid == 0) {
                s_n = kept;
                if (kept == s_sp.depth) s_tau = buf[s_sp.depth - 1];
            }
            __syncthreads();
        }
    }
    const uint32_t cnt = s_n;
    const uint32_t kept = block_select_largest(buf, cnt, s_sp.depth, sel);
    group_bitonic_desc(sel, p.kp2, tid, blockDim.x, 0);
    const size_t og = s_sp.row;
    for (uint32_t i = tid; i < s_sp.depth; i += blockDim.x) {
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
        p.out_doc[og * p.top + i] = doc;
        p.out_score[og * p.top + i] = sc;
    }
    if (tid == 0) p.out_n[og] = kept;
}

// one CTA per (query, group) item of the work list: a 1-D grid over the list's items
__global__ void __launch_bounds__(GROUP_THREADS) group_topk_kernel(const GroupParams p) { group_topk_body<false>(p); }
__global__ void __launch_bounds__(GROUP_THREADS) group_sort_topk_kernel(const GroupParams p) { group_topk_body<true>(p); }

}  // namespace oc
