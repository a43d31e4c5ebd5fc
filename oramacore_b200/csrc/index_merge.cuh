// index_merge.cuh — the multi-index union of oc_search_indexes on the device (search_on_indexes, read/search.rs:283-501).
//
// Every index of a collection has run its own search into a per-index top list; index_merge_kernel, one CTA per query,
// merges query q's lists into one page — what oc_merge_results / oc_merge_pinned / oc_merge_sorted compute on the host:
//   - score order: each list is sorted by (score desc, doc asc) under IEEE comparison (-0.0 == +0.0, ties to the doc).
//     The entry at position k of list i lands at merged position k plus, per other list j, the entries that come
//     before it: score greater, or equal with a lower doc (j > i) or a lower-or-equal doc (j < i: the host merge keeps
//     the lower index first on a full tie).  One binary search per other list (co-rank); score bits pass through.
//   - field order (MergeSortedIterator, read/sort.rs:491-559): merged by sort value, on equal values the lower index
//     first, each list in its own order.  ASC: k + #{value <= v in lists j < i} + #{value < v in lists j > i}; DESC
//     mirrored.  A hit's value is its rank value in that index's sort field (SortOrder.doc_rank / rank_value).
//   - then an active pinned query splices its items (pin_splice_block, pins.cuh) with each item's score taken from the
//     first index whose map holds the document (else 0.0), and every query takes skip(offset).take(limit).
#pragma once
#include "pins.cuh"
#include "sort.cuh"

namespace oc {

constexpr uint32_t IM_THREADS = 256;
constexpr uint8_t IM_BY_SCORE = 0, IM_ASC = 1, IM_DESC = 2;

struct ImSortSrc {                  // where index i's hits of query q find their sort values (field order)
    const uint32_t *doc_rank;       // [nbits] rank of each document id, RANK_NONE: no value
    const double *rank_value;       // [n] value of each rank
    uint64_t nbits;
};

struct IndexMergeParams {
    uint32_t n_idx, B, stride;      // indexes, queries, row stride of the per-index lists
    const uint64_t *doc;            // [n_idx][B][stride] per-index top lists
    const float *score;
    const uint32_t *n;              // [n_idx][B]
    const unsigned long long *count;   // [n_idx][B]
    double *value;                  // [n_idx][B][stride] workspace: the hits' sort values (field-order queries)
    const ImSortSrc *src;           // [n_idx][B] (NULL: no query is in field order)
    const uint8_t *q_sort;          // [B] IM_BY_SCORE / IM_ASC / IM_DESC
    const uint2 *q_page;            // [B] (offset, limit)
    // pins: the items [q][pin_stride] (cnt[q] each), the per-index score-map lookups, and which queries splice
    uint32_t pin_stride, kp2;
    const uint64_t *pin_doc;
    const uint32_t *pin_pos, *pin_cnt;
    const float *pin_score;         // [n_idx][B][pin_stride]
    const uint8_t *pin_present;
    const uint8_t *q_active;        // [B]
    uint32_t take_max;              // largest merged depth of a query (shared-memory size)
    uint32_t limit;                 // output row stride
    uint64_t *out_doc;              // [B][limit]
    float *out_score;
    double *out_value;              // [B][limit]: the value a hit was placed by; NaN for an item or in score order
    uint32_t *out_n;                // [B]
    unsigned long long *out_count;  // [B]
    float *out_pin_score;           // [B][pin_stride]
    uint8_t *out_pin_present;
};

__host__ __device__ inline size_t index_merge_smem(uint32_t take_max, uint32_t pin_stride, uint32_t kp2, uint32_t limit) {
    const size_t a = size_t(take_max) * 8 * 2 + size_t(take_max) * 4 + size_t(limit) * 4 + size_t(pin_stride) * 4;
    return ((a + 15) & ~size_t(15)) + pin_splice_smem(kp2, take_max, take_max);
}

// entries of list (doc, score, value)[0, n) that come before (s, d) / v in the merged order; `le`: ties count
__device__ __forceinline__ uint32_t im_rank_score(const uint64_t *doc, const float *score, uint32_t n, float s, uint64_t d, bool le) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const float sm = score[mid];
        const bool before = sm > s || (sm == s && (le ? doc[mid] <= d : doc[mid] < d));
        if (before) lo = mid + 1; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ uint32_t im_rank_value(const double *value, uint32_t n, double v, bool desc, bool le) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        const double vm = value[mid];
        const bool before = desc ? (vm > v || (le && vm == v)) : (vm < v || (le && vm == v));
        if (before) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// an item's score: the first index whose map holds its document, else 0.0
__device__ __forceinline__ float im_item_score(const float *score, const uint8_t *present, uint32_t ni, uint32_t B, uint32_t stride,
                                               uint32_t q, uint32_t j) {
    for (uint32_t i = 0; i < ni; i++) {
        const size_t o = (size_t(i) * B + q) * stride + j;
        if (present[o]) return score[o];
    }
    return 0.f;
}

// index_group_merge_kernel's merge (index_merge_kernel keeps its own copy of these steps inline, where the shared form
// costs it a spill).  Merges the ni sorted lists of L (L.doc(i), L.score(i), L.value(i) with L.len(i) entries) by the whole block into the
// first min(total, take) slots of m_doc / m_score / m_val, in score order or in field order (value, ASC or DESC).
// Returns min(total, take).  The caller synchronises before reading the slots.
template <typename Lists>
__device__ __forceinline__ uint32_t im_merge_block(const Lists &L, uint32_t ni, uint8_t mode, uint32_t take, uint64_t *m_doc, float *m_score,
                                   double *m_val) {
    const uint32_t tid = threadIdx.x, nt = blockDim.x;
    uint32_t total = 0;
    for (uint32_t i = 0; i < ni; i++) total += L.len(i);
    for (uint32_t i = 0; i < ni; i++) {
        const uint32_t n = L.len(i);
        const uint64_t *doc = L.doc(i);
        const float *score = L.score(i);
        const double *value = L.value(i);
        for (uint32_t k = tid; k < n; k += nt) {
            uint32_t pos = k;
            if (mode == IM_BY_SCORE) {
                const float s = score[k];
                const uint64_t d = doc[k];
                for (uint32_t j = 0; j < ni && pos < take; j++)
                    if (j != i) pos += im_rank_score(L.doc(j), L.score(j), L.len(j), s, d, j < i);
            } else {
                const double v = value[k];
                for (uint32_t j = 0; j < ni && pos < take; j++)
                    if (j != i) pos += im_rank_value(L.value(j), L.len(j), v, mode == IM_DESC, j < i);
            }
            if (pos < take) {
                m_doc[pos] = doc[k];
                m_score[pos] = score[k];
                m_val[pos] = mode == IM_BY_SCORE ? 0.0 : value[k];
            }
        }
    }
    return min(total, take);
}

// the sort values of one list's first n hits (in place), from its index's rank values
__device__ __forceinline__ void im_fill_values(const ImSortSrc sv, const uint64_t *doc, double *value, uint32_t n) {
    for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) {
        const uint64_t d = doc[k];
        const uint32_t r = d < sv.nbits ? sv.doc_rank[d] : RANK_NONE;
        value[k] = r == RANK_NONE ? __longlong_as_double(0x7ff8000000000000ll) : sv.rank_value[r];
    }
}

__global__ void __launch_bounds__(IM_THREADS) index_merge_kernel(const IndexMergeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t q = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, ni = p.n_idx;
    const uint2 page = p.q_page[q];
    const bool active = p.q_active[q] != 0;
    const uint8_t mode = p.q_sort[q];
    const uint32_t take = (page.x + page.y) * (active ? 2u : 1u);
    uint64_t *m_doc = reinterpret_cast<uint64_t *>(smem);        // [take_max] the merged top list
    double *m_val = reinterpret_cast<double *>(m_doc + p.take_max);
    float *m_score = reinterpret_cast<float *>(m_val + p.take_max);
    uint32_t *o_src = reinterpret_cast<uint32_t *>(m_score + p.take_max);   // [limit] source of each page slot
    float *i_score = reinterpret_cast<float *>(o_src + p.limit);            // [pin_stride] each item's score
    uint8_t *scratch = smem + ((size_t(p.take_max) * 20 + size_t(p.limit) * 4 + size_t(p.pin_stride) * 4 + 15) & ~size_t(15));
    const size_t qs = size_t(q) * p.stride;
    auto at = [&](uint32_t i) { return size_t(i) * p.B * p.stride + qs; };
    auto len = [&](uint32_t i) { return min(p.n[size_t(i) * p.B + q], take); };   // entries past take never land in it
    if (tid == 0) {
        unsigned long long c = 0;
        for (uint32_t i = 0; i < ni; i++) c += p.count[size_t(i) * p.B + q];
        p.out_count[q] = c;
    }
    // each item: the score of the first index whose map holds its document
    const uint32_t k_items = p.pin_cnt ? p.pin_cnt[q] : 0u;
    for (uint32_t j = tid; j < k_items; j += nt) {
        float s = 0.f;
        uint8_t present = 0;
        for (uint32_t i = 0; i < ni && !present; i++) {
            const size_t o = (size_t(i) * p.B + q) * p.pin_stride + j;
            if (p.pin_present[o]) { s = p.pin_score[o]; present = 1; }
        }
        i_score[j] = s;
        p.out_pin_score[size_t(q) * p.pin_stride + j] = s;
        p.out_pin_present[size_t(q) * p.pin_stride + j] = present;
    }
    if (mode != IM_BY_SCORE) {   // the hits' sort values, into the workspace the co-ranks read
        for (uint32_t i = 0; i < ni; i++) {
            const ImSortSrc sv = p.src[size_t(i) * p.B + q];
            const uint32_t n = len(i);
            for (uint32_t k = tid; k < n; k += nt) {
                const uint64_t d = p.doc[at(i) + k];
                const uint32_t r = d < sv.nbits ? sv.doc_rank[d] : RANK_NONE;
                p.value[at(i) + k] = r == RANK_NONE ? __longlong_as_double(0x7ff8000000000000ll) : sv.rank_value[r];
            }
        }
        __syncthreads();   // (global writes of this block are visible to it after the barrier)
    }
    uint32_t total = 0;
    for (uint32_t i = 0; i < ni; i++) total += len(i);
    const uint32_t M = min(total, take);
    for (uint32_t i = 0; i < ni; i++) {
        const uint32_t n = len(i);
        for (uint32_t k = tid; k < n; k += nt) {
            const size_t e = at(i) + k;
            uint32_t pos = k;
            if (mode == IM_BY_SCORE) {
                const float s = p.score[e];
                const uint64_t d = p.doc[e];
                for (uint32_t j = 0; j < ni && pos < take; j++)
                    if (j != i) pos += im_rank_score(p.doc + at(j), p.score + at(j), len(j), s, d, j < i);
            } else {
                const double v = p.value[e];
                for (uint32_t j = 0; j < ni && pos < take; j++)
                    if (j != i) pos += im_rank_value(p.value + at(j), len(j), v, mode == IM_DESC, j < i);
            }
            if (pos < take) {
                m_doc[pos] = p.doc[e];
                m_score[pos] = p.score[e];
                m_val[pos] = mode == IM_BY_SCORE ? 0.0 : p.value[e];
            }
        }
    }
    __syncthreads();
    const size_t o = size_t(q) * p.limit;
    uint32_t n_out;
    if (active && k_items) {
        n_out = pin_splice_block(m_doc, m_score, M, p.pin_doc + size_t(q) * p.pin_stride, p.pin_pos + size_t(q) * p.pin_stride,
                                 i_score, k_items, p.kp2, [](uint32_t) { return true; }, page.x, page.y, p.out_doc + o,
                                 p.out_score + o, scratch, o_src);
    } else {
        n_out = M > page.x ? min(M - page.x, page.y) : 0u;
        for (uint32_t s = tid; s < n_out; s += nt) {
            p.out_doc[o + s] = m_doc[page.x + s];
            p.out_score[o + s] = m_score[page.x + s];
            o_src[s] = page.x + s;
        }
    }
    __syncthreads();
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    for (uint32_t s = tid; s < p.limit; s += nt) {
        if (s < n_out) {
            p.out_value[o + s] = (mode == IM_BY_SCORE || o_src[s] == 0xffffffffu) ? nan : m_val[o_src[s]];
        } else {
            p.out_doc[o + s] = 0; p.out_score[o + s] = 0.f; p.out_value[o + s] = 0.0;
        }
    }
    if (tid == 0) p.out_n[q] = n_out;
}

// ---- groups across indexes (sort_groups over the union of the indexes' group maps, read/index/group.rs:104-168)
// The collection's group k of query q is the union of the local groups of every index that the caller's key maps send
// to k.  Each index has run its own group top lists (depth max_results, 2 x max_results for an active pinned query)
// into a slot of the workspace; index_group_merge_kernel merges the sources of one collection row, one CTA per
// (query, key) item of a work list of GroupSpans:
//   first: the span's first item; q; h: the offset of key 0 in the source table; ent: its handle set; max_results;
//   row: the query's first collection row (G_q).
// Score or field order as index_merge_kernel; an active query splices the items whose document is a member of any
// source group (apply_pin_rules_to_group, read/sort.rs:377-391) and keeps the whole spliced list; any other query keeps
// the top max_results.
constexpr uint32_t IM_NO_SRC = 0xffffffffu;
struct IndexGroupMergeParams {
    uint32_t n_idx, B;
    const GroupSpan *spans;
    uint32_t n_spans;
    const uint32_t *src_g;          // [offset + key * n_idx + i]: index i's local group, IM_NO_SRC: none
    const GroupHandle *set_h;       // [set * n_idx + i]: index i's handle in that set (members of the local groups)
    const uint32_t *q_lrow;         // [n_idx][B] the first local row of query q in index i's lists
    uint32_t rows, gtop;            // rows per index slot, row stride of the per-index lists
    const uint64_t *g_doc;          // [n_idx][rows][gtop]
    const float *g_score;
    const uint32_t *g_n;            // [n_idx][rows]
    double *g_val;                  // [n_idx][rows][gtop] workspace: sort values (field order)
    const ImSortSrc *src;           // [n_idx][B]
    const uint8_t *q_sort, *q_active;   // [B]
    uint32_t pin_stride, kp2;
    const uint64_t *pin_doc;
    const uint32_t *pin_pos, *pin_cnt;
    const float *pin_score;         // [n_idx][B][pin_stride]
    const uint8_t *pin_present;
    uint32_t take_max, n_slots;     // largest merged depth; spliced slots a row may need (<= stride)
    uint32_t stride;                // output row stride (group_stride)
    uint64_t *out_doc;              // [row][stride]
    float *out_score;
    double *out_value;
    uint32_t *out_n;                // [row]
};

__host__ __device__ inline size_t index_group_merge_smem(uint32_t take_max, uint32_t pin_stride, uint32_t kp2, uint32_t n_slots) {
    const size_t a = size_t(take_max) * 20 + size_t(n_slots) * 4 + size_t(pin_stride) * 4;
    return ((a + 15) & ~size_t(15)) + pin_splice_smem(kp2, take_max, n_slots);
}

__global__ void __launch_bounds__(IM_THREADS) index_group_merge_kernel(const IndexGroupMergeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t tid = threadIdx.x, nt = blockDim.x, ni = p.n_idx;
    const uint32_t item = blockIdx.x;
    const GroupSpan sp = group_span_of(p.spans, p.n_spans, item, item, gridDim.x);
    const uint32_t key = item - sp.first, q = sp.q;
    const size_t row = size_t(sp.row) + key;
    const bool active = p.q_active[q] != 0;
    const uint8_t mode = p.q_sort[q];
    const uint32_t take = sp.max_results * (active ? 2u : 1u);
    const uint32_t *gsrc = p.src_g + sp.h + size_t(key) * ni;
    uint64_t *m_doc = reinterpret_cast<uint64_t *>(smem);        // [take_max]
    double *m_val = reinterpret_cast<double *>(m_doc + p.take_max);
    float *m_score = reinterpret_cast<float *>(m_val + p.take_max);
    uint32_t *o_src = reinterpret_cast<uint32_t *>(m_score + p.take_max);   // [n_slots]
    float *i_score = reinterpret_cast<float *>(o_src + p.n_slots);          // [pin_stride]
    uint8_t *scratch = smem + ((size_t(p.take_max) * 20 + size_t(p.n_slots) * 4 + size_t(p.pin_stride) * 4 + 15) & ~size_t(15));
    struct Lists {   // the source rows of this collection row; an index without a source has an empty list
        const uint64_t *d; const float *s; double *v; const uint32_t *n, *lrow0, *gsrc; uint32_t rows, gtop, B, q, take;
        __device__ size_t lrow(uint32_t i) const { return size_t(i) * rows + lrow0[size_t(i) * B + q] + gsrc[i]; }
        __device__ size_t at(uint32_t i) const { return gsrc[i] == IM_NO_SRC ? 0 : lrow(i) * gtop; }
        __device__ uint32_t len(uint32_t i) const { return gsrc[i] == IM_NO_SRC ? 0u : min(n[lrow(i)], take); }
        __device__ const uint64_t *doc(uint32_t i) const { return d + at(i); }
        __device__ const float *score(uint32_t i) const { return s + at(i); }
        __device__ double *value(uint32_t i) const { return v + at(i); }
    } L{p.g_doc, p.g_score, p.g_val, p.g_n, p.q_lrow, gsrc, p.rows, p.gtop, p.B, q, take};
    const uint32_t k_items = active && p.pin_cnt ? p.pin_cnt[q] : 0u;
    for (uint32_t j = tid; j < k_items; j += nt) i_score[j] = im_item_score(p.pin_score, p.pin_present, ni, p.B, p.pin_stride, q, j);
    if (mode != IM_BY_SCORE) {
        for (uint32_t i = 0; i < ni; i++) im_fill_values(p.src[size_t(i) * p.B + q], L.doc(i), L.value(i), L.len(i));
        __syncthreads();
    }
    const uint32_t M = im_merge_block(L, ni, mode, take, m_doc, m_score, m_val);
    __syncthreads();
    const size_t o = row * p.stride;
    uint32_t n_out;
    if (k_items) {
        const uint64_t *idoc = p.pin_doc + size_t(q) * p.pin_stride;
        const GroupHandle *hs = p.set_h + size_t(sp.ent) * ni;
        auto member = [&](uint32_t j) {   // a member of some source group of this row
            const uint64_t d = idoc[j];
            for (uint32_t i = 0; i < ni; i++) {
                if (gsrc[i] == IM_NO_SRC) continue;
                const GroupHandle gh = hs[i];
                const uint64_t gb = gh.g_off[gsrc[i]], gn = gh.g_off[gsrc[i] + 1] - gb;
                const uint64_t *gdoc = gh.g_doc + gb;
                uint64_t lo = 0, hi = gn;
                while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (gdoc[mid] < d) lo = mid + 1; else hi = mid; }
                if (lo < gn && gdoc[lo] == d) return true;
            }
            return false;
        };
        n_out = pin_splice_block(m_doc, m_score, M, idoc, p.pin_pos + size_t(q) * p.pin_stride, i_score, k_items, p.kp2, member,
                                 0, p.n_slots, p.out_doc + o, p.out_score + o, scratch, o_src);
    } else {
        n_out = M;
        for (uint32_t s = tid; s < n_out; s += nt) {
            p.out_doc[o + s] = m_doc[s];
            p.out_score[o + s] = m_score[s];
            o_src[s] = s;
        }
    }
    __syncthreads();
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    for (uint32_t s = tid; s < p.stride; s += nt) {
        if (s < n_out) {
            p.out_value[o + s] = (mode == IM_BY_SCORE || o_src[s] == 0xffffffffu) ? nan : m_val[o_src[s]];
        } else {
            p.out_doc[o + s] = 0; p.out_score[o + s] = 0.f; p.out_value[o + s] = 0.0;
        }
    }
    if (tid == 0) p.out_n[row] = n_out;
}

}  // namespace oc
