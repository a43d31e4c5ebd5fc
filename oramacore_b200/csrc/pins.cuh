// pins.cuh — pin rules (promoted documents) over the score map: oc_search_pinned / oc_search_groups_pinned.
//
// Replaces apply_pin_rules_internal (read/sort.rs:285-391) as called by sort_token_scores (:17-46) and, through
// apply_pin_rules_to_group, by sort_groups (:129-230).  Per query the caller passes the promote items of the
// consequences that matched it (rule matching stays on the host); a query with at least one item is "active".
//
//   pin_score_kernel        the score-map value of every promoted document: a vector hit takes the final score K4
//                           exported (FuseParams::out_vdoc / out_vscore), any other document the point lookup of its
//                           string row (bm25_point_kernel: same bits, presence under filter, tombstones and threshold)
//                           through fused_ft_score; a document that is not a key scores 0.0 and is "not present".
//   pin_splice_kernel       one CTA per query over K4's top 2 * (limit + offset) (or, sorted, the walk's list): remove
//                           the promoted ids, insert the items stably sorted by position, then skip(offset).take(limit).
//   group_pin_splice_kernel one CTA per (query, group) over group_topk_kernel's top 2 * max_results: the same splice
//                           with the items restricted to the group's members, not truncated afterwards.
#pragma once
#include "group.cuh"

namespace oc {

constexpr uint32_t PIN_THREADS = 256;

struct PinScoreParams {
    uint32_t n_queries, stride;     // items of query q: [q * stride, q * stride + cnt[q])
    const uint64_t *doc;            // [q][stride] promoted document of each item
    const uint32_t *cnt;            // [q]
    bool has_ft, hybrid;
    const float *ft;                // [q][stride] point-lookup fulltext score (has_ft)
    const uint8_t *ft_present;      // [q][stride]
    const float *gmin, *den;        // [q] hybrid normalisation (K4 export)
    const uint64_t *v_doc;          // [q][v_stride] unique vector hits, final scores (K4 export)
    const float *v_score;
    const uint32_t *v_n;
    uint32_t v_stride;
    const uint64_t *omc_doc;
    const float *omc_mult;
    uint32_t n_omc;
    float *out_score;               // [q][stride] score-map value, 0.0 when not a key
    uint8_t *out_present;           // [q][stride] 1 = the document is a key of the score map
    const QueryPlan *q_plan;        // NULL, or [q]: a query is hybrid when hybrid is set and its own mode is
};

// one warp per (query, item slot)
__global__ void __launch_bounds__(256) pin_score_kernel(const PinScoreParams p) {
    const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (wid >= p.n_queries * p.stride) return;
    const uint32_t q = wid / p.stride, j = wid % p.stride;
    if (j >= p.cnt[q]) return;
    const uint64_t d = p.doc[wid];
    const uint32_t vn = p.v_n[q];
    const uint64_t *vd = p.v_doc + size_t(q) * p.v_stride;
    int hit = -1;
    for (uint32_t i0 = 0; i0 < vn; i0 += 32) {   // warp-uniform trip count
        const uint32_t i = i0 + lane;
        const unsigned b = __ballot_sync(0xffffffffu, i < vn && vd[i] == d);
        if (b) { hit = int(i0 + __ffs(b) - 1); break; }
    }
    if (lane) return;
    float s = 0.f;
    uint8_t present = 0;
    if (hit >= 0) {
        s = p.v_score[size_t(q) * p.v_stride + hit];
        present = 1;
    } else if (p.has_ft && p.ft_present[wid]) {
        const bool hybrid = p.hybrid && (!p.q_plan || p.q_plan[q].mode == OC_MODE_HYBRID);
        s = fused_ft_score(p.ft[wid], hybrid, p.gmin[q], p.den[q], p.omc_doc, p.omc_mult, p.n_omc, [&] { return d; });
        present = 1;
    }
    p.out_score[wid] = s;   // NaN stays NaN: it is still the map's value
    p.out_present[wid] = present;
}

// Shared memory of pin_splice_block: kp2 = max(32, next_pow2(items)) item slots, n_top kept indices, n_slots output slots.
__host__ __device__ inline size_t pin_splice_smem(uint32_t kp2, uint32_t n_top, uint32_t n_slots) {
    return size_t(kp2) * (8 + 8 + 4 + 4) + size_t(n_top) * 4 + size_t(n_slots) * 4;
}

// apply_pin_rules_internal for one list, by the whole block.  top: n_top (doc, score) entries, best first.  Items j < k
// with member(j) take part (doc, position, score).  Writes the spliced list's slots [s0, s0 + n_take) to out_doc /
// out_score and returns how many it wrote.
//   1. drop from top every document some member item promotes;
//   2. sort the member items by position, stably (key = position << 32 | item index);
//   3. insert them in that order at min(position, current length).  The slot an item ends up in is its insertion
//      index plus one for every later item inserted at or before it; the other slots take the kept entries in order.
template <typename Member>
__device__ uint32_t pin_splice_block(const uint64_t *top_doc, const float *top_score, uint32_t n_top, const uint64_t *doc,
                                     const uint32_t *pos, const float *score, uint32_t k, uint32_t kp2, Member member,
                                     uint32_t s0, uint32_t n_take, uint64_t *out_doc, float *out_score, uint8_t *smem,
                                     uint32_t *out_src = nullptr) {
    uint64_t *ord = reinterpret_cast<uint64_t *>(smem);   // [kp2] ~(position << 32 | j), sorted descending
    uint64_t *ids = ord + kp2;                             // [kp2] ~doc, sorted descending
    uint32_t *ins = reinterpret_cast<uint32_t *>(ids + kp2);   // [kp2] insertion index
    uint32_t *fin = ins + kp2;                             // [kp2] final slot
    uint32_t *kidx = fin + kp2;                            // [n_top] kept entries of top
    uint32_t *slot = kidx + n_top;                         // [n_slots] item in each output slot, ~0 = a kept entry
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    uint32_t km = 0;
    for (uint32_t i0 = 0; i0 < kp2; i0 += nt) {   // block-uniform trip count (the scan has barriers)
        const uint32_t i = i0 + tid;
        const bool m = i < k && member(i);
        uint32_t n_m;
        block_exclusive_scan(m ? 1u : 0u, &n_m);
        if (i < kp2) {
            ord[i] = m ? ~((uint64_t(pos[i]) << 32) | i) : 0ull;
            ids[i] = m ? ~doc[i] : 0ull;
        }
        km += n_m;
    }
    if (km == 0) {   // nothing to splice (block-uniform): the page of top as it is
        const uint32_t n = n_top > s0 ? min(n_top - s0, n_take) : 0u;
        for (uint32_t i = tid; i < n; i += nt) {
            out_doc[i] = top_doc[s0 + i]; out_score[i] = top_score[s0 + i];
            if (out_src) out_src[i] = s0 + i;
        }
        return n;
    }
    group_bitonic_desc(ord, kp2, tid, nt, 0);   // ascending (position, j); non-members last
    group_bitonic_desc(ids, kp2, tid, nt, 0);   // ascending doc ids
    auto promoted = [&](uint64_t d) {
        uint32_t lo = 0, hi = km;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (~ids[mid] < d) lo = mid + 1; else hi = mid; }
        return lo < km && ~ids[lo] == d;
    };
    uint32_t L = 0;
    for (uint32_t t0 = 0; t0 < n_top; t0 += nt) {
        const uint32_t t = t0 + tid;
        const bool keep = t < n_top && !promoted(top_doc[t]);
        uint32_t n_k;
        const uint32_t at = block_exclusive_scan(keep ? 1u : 0u, &n_k);
        if (keep) kidx[L + at] = t;
        L += n_k;
    }
    for (uint32_t r = tid; r < km; r += nt) ins[r] = min(uint32_t(~ord[r] >> 32), L + r);
    __syncthreads();
    for (uint32_t r = tid; r < km; r += nt) {
        uint32_t f = ins[r];
        for (uint32_t i = r + 1; i < km; i++) f += ins[i] <= f ? 1u : 0u;
        fin[r] = f;
    }
    const uint32_t total = L + km;
    const uint32_t s_end = min(total, s0 + n_take);
    for (uint32_t s = tid; s < s_end; s += nt) slot[s] = 0xffffffffu;
    __syncthreads();
    for (uint32_t r = tid; r < km; r += nt)
        if (fin[r] < s_end) slot[fin[r]] = r;
    __syncthreads();
    uint32_t pins_before = 0;
    for (uint32_t s0b = 0; s0b < s_end; s0b += nt) {
        const uint32_t s = s0b + tid;
        const bool is_pin = s < s_end && slot[s] != 0xffffffffu;
        uint32_t n_p;
        const uint32_t pb = pins_before + block_exclusive_scan(is_pin ? 1u : 0u, &n_p);
        if (s < s_end && s >= s0) {
            uint64_t d;
            float sc;
            uint32_t src = 0xffffffffu;
            if (is_pin) {
                const uint32_t j = uint32_t(~ord[slot[s]]);
                d = doc[j]; sc = score[j];
            } else {
                src = kidx[s - pb];
                d = top_doc[src]; sc = top_score[src];
            }
            out_doc[s - s0] = d;
            out_score[s - s0] = sc;
            if (out_src) out_src[s - s0] = src;
        }
        pins_before += n_p;
    }
    return s_end > s0 ? s_end - s0 : 0u;
}

struct PinSpliceParams {
    uint32_t stride, kp2;           // item slots per query; max(32, next_pow2(stride))
    const uint64_t *doc;            // [q][stride]
    const uint32_t *pos;
    const float *score;             // pin_score_kernel's output
    const uint32_t *cnt;            // [q]
    // flat hits: K4's top n_top per query
    uint32_t n_top, limit, offset;
    const uint64_t *top_doc;        // [q][n_top]
    const float *top_score;
    const uint32_t *top_n;          // [q]
    uint64_t *out_doc;              // [q][limit]
    float *out_score;
    uint32_t *out_n;                // [q]
    // oc_search_q_sorted: the queries in score order (q_alt[q] != 0) take K4's list (alt_*) instead of the walk's
    const uint8_t *q_alt;           // [q], NULL: every query takes top_*
    uint32_t alt_n_top;
    const uint64_t *alt_doc;        // [q][alt_n_top]
    const float *alt_score;
    const uint32_t *alt_n;          // [q]
    const uint2 *q_page;            // NULL, or [q] each query's own (offset, limit); limit is then the output row stride
};

// one CTA per query: the flat hits of sort_token_scores with pins, then skip(offset).take(limit); a query without items
// gets top[offset, offset + limit), which is what K4 writes at n_keep = limit + offset
__global__ void __launch_bounds__(PIN_THREADS) pin_splice_kernel(const PinSpliceParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t q = blockIdx.x;
    const bool alt = p.q_alt && p.q_alt[q];
    const uint32_t n_top = alt ? p.alt_n_top : p.n_top;
    const uint64_t *top_doc = alt ? p.alt_doc : p.top_doc;
    const float *top_score = alt ? p.alt_score : p.top_score;
    const uint32_t top_n = alt ? p.alt_n[q] : p.top_n[q];
    const uint2 page = p.q_page ? p.q_page[q] : make_uint2(p.offset, p.limit);
    const size_t it = size_t(q) * p.stride, tp = size_t(q) * n_top, o = size_t(q) * p.limit;
    const uint32_t n = pin_splice_block(top_doc + tp, top_score + tp, top_n, p.doc + it, p.pos + it, p.score + it,
                                        p.cnt[q], p.kp2, [](uint32_t) { return true; }, page.x, page.y,
                                        p.out_doc + o, p.out_score + o, smem);
    for (uint32_t i = n + threadIdx.x; i < p.limit; i += blockDim.x) { p.out_doc[o + i] = 0; p.out_score[o + i] = 0.f; }
    if (threadIdx.x == 0) p.out_n[q] = n;
}

struct GroupPinParams {
    const GroupHandle *handles;
    const GroupSpan *spans;                               // the whole batch's work list, items 0 .. n_items - 1
    uint32_t n_spans;
    uint32_t stride, top, kp2;                            // output row stride; group_topk_kernel's row stride
    const uint64_t *doc;                                  // [q][item_stride] items, as PinSpliceParams
    const uint32_t *pos;
    const float *score;
    const uint32_t *cnt;                                  // NULL: the pins do not apply (every list is the top max_results)
    uint32_t item_stride;
    const uint64_t *top_doc;                              // [row][top]
    const float *top_score;
    const uint32_t *top_n;                                // [row]
    uint64_t *out_doc;                                    // [row][stride]
    float *out_score;
    uint32_t *out_n;                                      // [row]
};

// one CTA per (query, group) item of the work list.  An active query splices the items whose document is a member of
// the group into the group's top 2 * max_results and keeps the whole list; a query without items keeps the top
// max_results, exactly what group_topk_kernel computes at that depth.
__global__ void __launch_bounds__(PIN_THREADS) group_pin_splice_kernel(const GroupPinParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t item = blockIdx.x;
    const GroupSpan sp = group_span_of(p.spans, p.n_spans, item, item, gridDim.x);
    const GroupHandle gh = p.handles[sp.h];
    const uint32_t g = item - sp.first, q = sp.q;
    const size_t og = size_t(sp.row) + g, it = size_t(q) * p.item_stride;
    const uint32_t k = p.cnt ? p.cnt[q] : 0u;
    const uint64_t gb = gh.g_off[g], gn = gh.g_off[g + 1] - gb;
    const uint64_t *gdoc = gh.g_doc + gb;
    const uint64_t *idoc = p.doc + it;
    auto member = [&](uint32_t j) {
        const uint64_t d = idoc[j];
        uint64_t lo = 0, hi = gn;
        while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (gdoc[mid] < d) lo = mid + 1; else hi = mid; }
        return lo < gn && gdoc[lo] == d;
    };
    const uint32_t n = pin_splice_block(p.top_doc + og * p.top, p.top_score + og * p.top, p.top_n[og], idoc, p.pos + it,
                                        p.score + it, k, p.kp2, member, 0, k ? p.stride : sp.max_results,
                                        p.out_doc + og * p.stride, p.out_score + og * p.stride, smem);
    for (uint32_t i = n + threadIdx.x; i < p.stride; i += blockDim.x) { p.out_doc[og * p.stride + i] = 0; p.out_score[og * p.stride + i] = 0.f; }
    if (threadIdx.x == 0) p.out_n[og] = n;
}

}  // namespace oc
