// sort.cuh — sortBy over the score map: the flat hits of oc_search_sorted / oc_search_groups_sorted.
//
// Replaces sort_token_scores with sort_by (read/sort.rs:36-41, 48-126): walk the field's documents in sort order and
// keep the first top_count that are keys of the query's score map.  A sort field holds, per order, its documents in
// rank order (ties by ascending id, each document once, at its first value in that order), the string row of every
// rank (rebuilt per string-store snapshot) and the rank of every document id.
//
//   sort_walk_kernel   one CTA per query, each with its own (field, order) entry of the batch's table or none (score
//                      order: the query's hits are K4's, see pin_splice_kernel): streams the ranks in chunks of
//                      SORT_CHUNK, tests each rank's string row
//                      against the matched-row bitmap the tile scorers emit and its rank against the vector hits K4
//                      exports, and compacts the hits in rank order with a block-wide prefix sum.  It stops once
//                      top_count keys are found (in vector mode, once the last-ranked vector hit is passed).
// The selected documents are then scored like promoted documents (bm25_point_kernel + pin_score_kernel) and paged,
// with the pins spliced, by pin_splice_kernel (pins.cuh).  Groups take the rank key of group_topk_kernel<true>.
#pragma once
#include "pins.cuh"

namespace oc {

constexpr uint32_t SORT_THREADS = 256;
constexpr uint32_t SORT_PER_THREAD = 4;                      // consecutive ranks per thread and chunk
constexpr uint32_t SORT_CHUNK = SORT_THREADS * SORT_PER_THREAD;
constexpr uint32_t RANK_NONE = 0xffffffffu;

// SortEntry (group.cuh): one distinct (field, order) of a batch.
constexpr uint32_t SORT_BY_SCORE = 0xffffffffu;   // SortQuery::ent of a query in score order: no walk, no keys
struct SortQuery {
    uint32_t ent;                   // index into SortWalkParams::ents, or SORT_BY_SCORE
    uint32_t top;                   // top_count (<= SortWalkParams::top)
};

struct SortWalkParams {
    const SortEntry *ents;          // the batch's distinct (field, order) pairs
    const SortQuery *q;             // [q]
    const uint32_t *mbits;          // [q][row_words] matched rows (filter, deletes, threshold applied); NULL: none
    uint64_t row_words;
    const uint64_t *v_doc;          // [q][v_stride] unique vector hits (K4 export)
    const uint32_t *v_n;            // [q]
    uint32_t v_stride;
    uint32_t top;                   // row stride of the outputs: the largest top_count of the batch
    uint64_t *out_doc;              // [q][top] keys in rank order
    uint32_t *out_row;              // [q][top] their string rows (RANK_NONE past out_n, or without a row)
    uint32_t *out_n;                // [q]
};

// dynamic shared memory: v_stride ranks of the vector hits
__global__ void __launch_bounds__(SORT_THREADS) sort_walk_kernel(const SortWalkParams p) {
    extern __shared__ __align__(16) uint32_t vrank[];
    __shared__ uint32_t vmark[SORT_CHUNK / 32];   // vector hits among the ranks of the current chunk
    __shared__ uint32_t s_vmax;
    const uint32_t q = blockIdx.x, tid = threadIdx.x;
    const SortQuery sq = p.q[q];
    uint64_t *od = p.out_doc + size_t(q) * p.top;
    uint32_t *orow = p.out_row + size_t(q) * p.top;
    if (sq.ent == SORT_BY_SCORE) {   // (block-uniform) a score-order query takes K4's list: no key here
        for (uint32_t i = tid; i < p.top; i += blockDim.x) { od[i] = 0; orow[i] = RANK_NONE; }
        if (tid == 0) p.out_n[q] = 0;
        return;
    }
    const SortEntry e = p.ents[sq.ent];
    const uint32_t vn = p.v_n[q];
    if (tid == 0) s_vmax = 0;
    __syncthreads();
    for (uint32_t i = tid; i < vn; i += blockDim.x) {
        const uint64_t d = p.v_doc[size_t(q) * p.v_stride + i];
        const uint32_t r = d < e.nbits ? e.doc_rank[d] : RANK_NONE;
        vrank[i] = r;
        if (r != RANK_NONE) atomicMax(&s_vmax, r + 1);
    }
    __syncthreads();
    const uint32_t *mb = p.mbits ? p.mbits + size_t(q) * p.row_words : nullptr;
    // without a fulltext map the keys are the vector hits: nothing past the last-ranked one
    const uint64_t end = mb ? e.n_ranks : min(e.n_ranks, uint64_t(s_vmax));
    uint32_t found = 0;
    for (uint64_t c0 = 0; c0 < end && found < sq.top; c0 += SORT_CHUNK) {   // block-uniform trip count
        for (uint32_t w = tid; w < SORT_CHUNK / 32; w += blockDim.x) vmark[w] = 0;
        __syncthreads();
        for (uint32_t i = tid; i < vn; i += blockDim.x) {
            const uint32_t r = vrank[i];
            if (r != RANK_NONE && r >= c0 && r < c0 + SORT_CHUNK) atomicOr(&vmark[(r - c0) >> 5], 1u << ((r - c0) & 31));
        }
        __syncthreads();
        const uint64_t r0 = c0 + uint64_t(tid) * SORT_PER_THREAD;
        uint32_t row[SORT_PER_THREAD], hit = 0;
#pragma unroll
        for (uint32_t u = 0; u < SORT_PER_THREAD; u++) {
            const uint64_t r = r0 + u;
            row[u] = RANK_NONE;
            if (r >= end) continue;
            const uint32_t l = tid * SORT_PER_THREAD + u;
            bool key = (vmark[l >> 5] >> (l & 31)) & 1u;
            if (e.rank_row) {
                row[u] = e.rank_row[r];
                key = key || (mb && row[u] != RANK_NONE && ((mb[row[u] >> 5] >> (row[u] & 31)) & 1u));
            }
            hit |= (key ? 1u : 0u) << u;
        }
        uint32_t tot;
        uint32_t at = found + block_exclusive_scan(__popc(hit), &tot);
#pragma unroll
        for (uint32_t u = 0; u < SORT_PER_THREAD; u++)
            if ((hit >> u) & 1u) {
                if (at < sq.top) { od[at] = e.rank_doc[r0 + u]; orow[at] = row[u]; }
                at++;
            }
        found += tot;
    }
    const uint32_t n = min(found, sq.top);
    for (uint32_t i = n + tid; i < p.top; i += blockDim.x) { od[i] = 0; orow[i] = RANK_NONE; }
    if (tid == 0) p.out_n[q] = n;
}

}  // namespace oc
