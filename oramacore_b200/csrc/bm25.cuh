// bm25.cuh — K3: BM25F posting-list scorer over device-resident postings.
//
// Replaces, for a batch of queries, the hot loops of search_full_text
// (read/index/token_score.rs:186-303): the external
// StringStorage::collect_contributions posting walk (string_field.rs:208-225), the
// per-token corpus_df / add_precomputed_field accumulation (token_score.rs:257-276) and
// BM25Scorer::finalize_term / get_scores (bm25.rs:369-428, 484-524).
//
// Design (HBM-bound, postings read exactly once per (query, term)):
//   * the document-row space is cut into tiles of TILE rows; one CTA scores one
//     (query, tile) pair entirely in shared memory: score[TILE] (+ S[TILE] when a token
//     expands to several index terms, + mask[TILE] in threshold mode), so there is no
//     accumulator traffic to HBM and no atomics (rows are unique inside a posting list and
//     terms are processed one after another between barriers);
//   * a plan kernel binary-searches, once per batch, the posting sub-range of every
//     (expanded term, tile) pair;
//   * after accumulation the tile is scanned once: matched-doc count, pre-OMC min/max,
//     and threshold-gated insertion (against a per-query global threshold tau that earlier
//     tiles raise with atomicMax) into a small top-n buffer that is compressed by a
//     bitonic sort only when it overflows;
//   * arithmetic uses explicit round-to-nearest intrinsics in the reference's operation
//     order (no FMA contraction), idf is computed on the host with the same libm as the
//     oracle, so BM25 scores are bit-identical to the CPU restatement.
//
// Algorithmic bytes: 8 B per posting walked (u32 row, u16 tf, u16 field_len).
#pragma once
#include "oc_common.cuh"

namespace oc {

#ifndef OC_BM25_TILE_ROWS
#define OC_BM25_TILE_ROWS 8192
#endif
constexpr uint32_t BM25_TILE = OC_BM25_TILE_ROWS;   // rows per tile (8192: 32 KB of fp32 accumulators, 4 CTAs per SM); multiple of 1024
#ifndef OC_BM25_THREADS
#define OC_BM25_THREADS 256
#endif
constexpr uint32_t BM25_THREADS = OC_BM25_THREADS;   // threads per scorer CTA (1024 resident threads per SM either way)
constexpr uint32_t BM25_CHUNK = BM25_THREADS * 4;

struct PostingRaw {    // 8 bytes, as handed over by the host (string_field.rs:162: field_length is u16)
    uint32_t row;
    uint16_t tf, len;
};
struct Posting {       // 8 bytes, what the scorer streams: row + tf' = tf / (1 - b + b*len/avglen)
    uint32_t row;
    float ntf;         // bm25.rs:99-110, computed once per (field, b) at load time with the same rounded ops
};

struct TermDesc {      // one expanded index term of one token of one query
    const Posting *ptr;    // first posting of the term (device)
    uint32_t len;          // postings in the list (rows unique, ascending)
    float weight;          // field boost x exact-match factor
    float avg_len;         // the field's avg_field_length
    uint32_t flags;        // bit0: postings are batch-precomputed (row, c) records, see bm25_precompute_kernel
                           // bit1: DENSE: ptr is a float[n_tiles * TILE] array of per-row contributions (0 = absent)
};
constexpr uint32_t TD_PRE = 1u, TD_DENSE = 2u;

struct TokenDesc {
    uint32_t term_begin, term_end;  // into TermDesc[]
    float idf;                      // host-computed (libm log1pf), bm25.rs:78-82
    uint32_t bit;                   // 1 << (token_index & 31), token_score.rs:293
};

struct QueryDesc {
    uint32_t token_begin, token_end;  // into TokenDesc[]
    uint32_t required;                // floor(n_tokens * threshold), token_score.rs:211-218
    uint32_t flags;                   // bit0: threshold mode; bit1: some token has != 1 terms
};
constexpr uint32_t QF_THRESHOLD = 1u, QF_MULTI = 2u;

// ---- plan: seg[e][t] = first posting of term e with row >= t*TILE (relative to begin) ----
__global__ void bm25_plan_kernel(const TermDesc *terms, uint32_t n_terms, uint32_t n_tiles, uint32_t *seg) {
    const uint64_t gid = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const uint64_t per = uint64_t(n_tiles) + 1;
    if (gid >= uint64_t(n_terms) * per) return;
    const uint32_t e = uint32_t(gid / per), t = uint32_t(gid % per);
    const TermDesc td = terms[e];
    const uint64_t len = td.len;
    if (t == n_tiles) { seg[gid] = uint32_t(len); return; }
    const uint64_t target = uint64_t(t) * BM25_TILE;
    uint64_t lo = 0, hi = len;
    const Posting *pp = td.ptr;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (uint64_t(pp[mid].row) < target) lo = mid + 1; else hi = mid;
    }
    seg[gid] = uint32_t(lo);
}

// bm25.rs:99-110 with the boost baked in (token_score.rs:180-185):
//   ntf = w * (tf / (1 - b + b * (len / avglen)))   — every op rounded separately.
__device__ __forceinline__ float bm25_ntf(uint32_t tf, uint32_t len, float avg, float b, float one_minus_b,
                                          float w) {
    const float r = __fdiv_rn(float(len), avg);
    const float den = __fadd_rn(one_minus_b, __fmul_rn(b, r));
    return __fmul_rn(w, __fdiv_rn(float(tf), den));
}
// load-time derivation of the streamed posting format (re-run only if b or avg_field_len change)
__global__ void bm25_derive_postings_kernel(const PostingRaw *raw, uint64_t n, float avg, float b, Posting *out) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const PostingRaw r = raw[i];
    Posting o;
    o.row = r.row;
    o.ntf = bm25_ntf(r.tf, r.len, avg, b, __fsub_rn(1.0f, b), 1.0f);   // w = 1: x*1.0 is exact
    out[i] = o;
}

// bm25.rs:124-126: idf * (k + 1) * S / (k + S)
__device__ __forceinline__ float bm25_sat(float S, float k, float kp1, float idf) {
    return __fdiv_rn(__fmul_rn(__fmul_rn(idf, kp1), S), __fadd_rn(k, S));
}
struct PreDesc {        // one (term, weight) pair shared by several queries of the batch
    const Posting *src;
    Posting *dst;       // list form: (row, c) records; or
    float *dense;       // dense form (hot terms): c scattered into a zeroed float[rows] array, NULL = list form
    uint32_t len;
    float weight, idf;
    uint32_t n_tiles;   // dense form: tiles of the array (where its summary starts, bm25_dense_bits / bm25_dense_bound)
};
__device__ __forceinline__ bool f32_is_normal(float x) {
    const uint32_t e = (__float_as_uint(x) >> 23) & 0xffu;
    return e != 0u && e != 0xffu;
}

struct Bm25Params {
    const TermDesc *terms;
    const TokenDesc *tokens;
    const QueryDesc *queries;
    const uint32_t *term_token;   // [n_term_desc] token index of each expanded term
    const uint32_t *seg;          // [n_term_desc][n_tiles+1]
    uint32_t n_queries, n_tiles;  // (tile, query) items are numbered tile-major: item = tile * n_queries + q
    uint64_t n_rows;
    float k;                      // (b is applied by bm25_derive_postings_kernel before the scorers run)
    const uint32_t *row_ok_bits;  // NULL or bitmap over rows (alive AND filter)
    // OMC (search.rs:39-48), sorted by row
    const uint32_t *omc_row;
    const float *omc_mult;
    uint32_t n_omc;
    const float *min_hint;        // [n_queries] assumed global min for the rank proxy (0)
    // outputs per (query, tile)
    uint32_t n_keep;              // limit + offset
    uint32_t cap;                 // top buffer capacity, pow2 >= n_keep + BM25_CHUNK
    unsigned long long *tau;      // [n_queries] running global threshold keys
    uint64_t *cand_key;           // [n_queries][n_tiles][n_keep]
    float *cand_ft;               // raw fulltext score of each candidate
    uint32_t *cand_cnt;           // [n_queries][n_tiles]
    uint32_t *tile_count;         // matched docs
    float *tile_max, *tile_min;   // pre-OMC extrema (fold start 0.0, token_score.rs:398-401)
    uint32_t *matched_bits;       // NULL, or out: [n_queries][n_tiles * TILE/32] bitmap of the matched rows (the keys of the
                                  // score map) — what the facet counts run over (read/index/facet.rs:147-209)
    // Group mode (the ROWFT instantiations of K3 / K3b; set together with matched_bits): out, [n_queries][n_tiles * TILE]
    // raw fulltext score of every matched row, written where its matched bit is set — slots of unmatched rows are
    // never written and must be read through the bitmap.
    float *row_ft;
    // per-query where-filters (oc_search_params.q_filters): NULL, or [n_queries] slot of each query in row_ok_bits, which
    // then holds one bitmap of ok_words words per slot.  Only K3 and K3b read it (such a batch never runs K3c / K3d).
    const uint32_t *q_ok_slot;
    uint64_t ok_words;
    // NULL, or out: [2] (dense passes, dense passes replaced by a count pass) of the register-folded scorers — summed
    // over the items, for last_timing()
    uint32_t *dense_stat;
};
// the row bitmap of query q (or of token t in the df pre-pass): the shared one, or its slot's
__device__ __forceinline__ const uint32_t *row_ok_of(const uint32_t *bits, const uint32_t *slot, uint64_t words, uint32_t q) {
    return (bits && slot) ? bits + size_t(slot[q]) * words : bits;
}

__host__ __device__ inline size_t bm25_smem_bytes(bool multi, bool threshold, bool omc, uint32_t cap) {
    size_t b = size_t(BM25_TILE) * 4;                 // score
    if (multi || omc) b += size_t(BM25_TILE) * 4;     // S / omc multipliers
    if (threshold) b += size_t(BM25_TILE) * 4;        // token masks
    b += size_t(BM25_TILE) / 8;                       // row_ok bits
    b += size_t(cap) * 8;                             // top buffer keys (ft is re-read from score[])
    return b + 64;
}

// A dense array's summary, in the same allocation right after its float[rows_pad] (rows_pad = n_tiles * TILE):
//   * a presence bitmap, uint32[rows_pad / 32]: bit r = (c[r] != 0);
//   * tile_bound, float[n_tiles]: an upper bound of each tile's values — its largest positive c, or 0 (padded to
//     256 B, so arrays laid end to end keep the alignment of the float4 loads).
// The register-folded scorers use both to skip the dense scan of an item no dense-only row of which can reach the
// query's threshold (t3_count).  bm25_precompute_kernel sets them next to each value it stores (the allocation is zeroed
// first, as the array always was), so they follow every row it leaves at 0 and the "NaN is never stored" rule, and
// building them costs no launch of its own.
__host__ __device__ inline uint64_t bm25_dense_bytes(uint32_t n_tiles) {
    const uint64_t rows_pad = uint64_t(n_tiles) * BM25_TILE;
    return rows_pad * 4 + rows_pad / 8 + ((uint64_t(n_tiles) * 4 + 255) & ~uint64_t(255));
}
__host__ __device__ __forceinline__ const uint32_t *bm25_dense_bits(const float *arr, uint32_t n_tiles) {
    return reinterpret_cast<const uint32_t *>(arr + size_t(n_tiles) * BM25_TILE);
}
__host__ __device__ __forceinline__ const float *bm25_dense_bound(const float *arr, uint32_t n_tiles) {
    return reinterpret_cast<const float *>(bm25_dense_bits(arr, n_tiles) + size_t(n_tiles) * (BM25_TILE / 32));
}
// Zipf query terms repeat across the queries of a batch: the per-posting contribution
// c = idf*(k+1)*S/(k+S), S = w*tf' of a single-term token depends only on (term, weight), so it is
// computed ONCE per batch (same rounded ops => bit-identical scores) and the tile kernel only adds:
//   * list form: (row, c) records in posting order;
//   * DENSE form, for hot terms (a posting in at least every ~16th row): c scattered into a zeroed
//     float[rows] array.  A (query, tile) item then adds the tile's 8192 floats with 128-bit loads —
//     ~0.6 instructions per row instead of ~25 per posting of the scatter loop — and adding the 0.0 of an
//     absent row leaves every bit of the sum unchanged.  Rows failing the filter / tombstone bitmap are
//     left at 0 here, so the tile kernel needs no per-row check for a dense term.
// items[i] = (pre index, chunk of PRE_CHUNK postings).
constexpr uint32_t PRE_CHUNK = 4096;
__global__ void __launch_bounds__(256) bm25_precompute_kernel(const PreDesc *pre, const uint2 *items, float k,
                                                              const uint32_t *row_ok_bits) {
    const uint2 it = items[blockIdx.x];
    const PreDesc d = pre[it.x];
    const float kp1 = __fadd_rn(k, 1.0f);
    const uint32_t lo = it.y * PRE_CHUNK, hi = min(d.len, lo + PRE_CHUNK);
    const uint2 *src = reinterpret_cast<const uint2 *>(d.src);
    if (!d.dense) {
        uint2 *dst = reinterpret_cast<uint2 *>(d.dst);
        for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
            const uint2 r = __ldg(src + i);
            const float ntf = __fmul_rn(d.weight, __uint_as_float(r.y));
            float c = __int_as_float(0x7fc00000);              // NaN => skipped (bm25.rs:387,391)
            if (f32_is_normal(ntf)) c = bm25_sat(ntf, k, kp1, d.idf);
            dst[i] = make_uint2(r.x, __float_as_uint(c));
        }
        return;
    }
    // dense form, warp-uniform trip count (the summary's per-tile maximum is a warp reduction)
    uint32_t *bits = const_cast<uint32_t *>(bm25_dense_bits(d.dense, d.n_tiles));
    unsigned int *bound = reinterpret_cast<unsigned int *>(const_cast<float *>(bm25_dense_bound(d.dense, d.n_tiles)));
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t i0 = lo + (threadIdx.x - lane); i0 < hi; i0 += blockDim.x) {
        const uint32_t i = i0 + lane;
        uint32_t row = 0, v = 0;
        if (i < hi) {
            const uint2 r = __ldg(src + i);
            const float ntf = __fmul_rn(d.weight, __uint_as_float(r.y));
            float c = __int_as_float(0x7fc00000);              // NaN => never stored
            if (f32_is_normal(ntf)) c = bm25_sat(ntf, k, kp1, d.idf);
            const bool ok = !row_ok_bits || ((row_ok_bits[r.x >> 5] >> (r.x & 31)) & 1u);
            row = r.x;
            if (ok && c == c) {
                d.dense[row] = c;
                if (c != 0.f) atomicOr(bits + (row >> 5), 1u << (row & 31u));   // the row's presence bit
                if (c > 0.f) v = __float_as_uint(c);          // (positive floats order as their bits do)
            }
        }
        // the tile's bound: one atomic per tile the warp's postings fall in (rows ascend: nearly always one)
        const uint32_t tile = row / BM25_TILE;
        const uint32_t grp = __match_any_sync(0xffffffffu, tile);
        const uint32_t m = __reduce_max_sync(grp, v);
        if (m && lane == uint32_t(__ffs(grp) - 1)) atomicMax(bound + tile, m);
    }
}

// ---- df pre-pass (only when a filter / tombstones / multi-term tokens make df != list length):
// corpus_df = |union over the token's terms of docs passing the filter| (token_score.rs:262-275).
struct DfParams {
    const TermDesc *terms;
    const TokenDesc *tokens;
    uint32_t n_tokens, n_tiles;
    const uint32_t *seg;
    const uint32_t *row_ok_bits;
    unsigned int *df;  // [n_tokens]
    const uint32_t *tok_ok_slot;   // NULL, or [n_tokens] slot of each token's query (per-query where-filters)
    uint64_t ok_words;
};
__global__ void __launch_bounds__(BM25_THREADS) bm25_df_kernel(const DfParams p) {
    __shared__ uint8_t flag[BM25_TILE];
    __shared__ uint32_t okb[BM25_TILE / 32];
    __shared__ uint32_t s_sum;
    const uint32_t tile = blockIdx.x % p.n_tiles, tok = blockIdx.x / p.n_tiles;
    const uint32_t row0 = tile * BM25_TILE;
    const TokenDesc tk = p.tokens[tok];
    const uint32_t *okq = row_ok_of(p.row_ok_bits, p.tok_ok_slot, p.ok_words, tok);
    for (uint32_t i = threadIdx.x; i < BM25_TILE / 4; i += blockDim.x) reinterpret_cast<uint32_t *>(flag)[i] = 0;
    for (uint32_t i = threadIdx.x; i < BM25_TILE / 32; i += blockDim.x)
        okb[i] = okq ? okq[row0 / 32 + i] : 0xffffffffu;
    if (threadIdx.x == 0) s_sum = 0;
    __syncthreads();
    for (uint32_t e = tk.term_begin; e < tk.term_end; e++) {
        const TermDesc td = p.terms[e];
        const uint32_t *sg = p.seg + size_t(e) * (p.n_tiles + 1);
        const uint32_t lo = sg[tile], hi = sg[tile + 1];
        for (uint32_t pi = lo + threadIdx.x; pi < hi; pi += blockDim.x) {
            const uint32_t l = td.ptr[pi].row - row0;
            if ((okb[l >> 5] >> (l & 31)) & 1u) flag[l] = 1;
        }
    }
    __syncthreads();
    uint32_t c = 0;
    for (uint32_t i = threadIdx.x; i < BM25_TILE / 4; i += blockDim.x)
        c += __popc(reinterpret_cast<uint32_t *>(flag)[i] & 0x01010101u);
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(&s_sum, c);
    __syncthreads();
    if (threadIdx.x == 0 && s_sum) atomicAdd(&p.df[tok], s_sum);
}

// Keeps the best n keys of buf[0..count) (descending, in buf[0..n)).  For small n this is n
// rounds of a block-wide arg-max (cheap: <= 8 keys per thread per round) instead of a
// full bitonic sort of the whole buffer; large n falls back to the sort.
__device__ inline void block_keep_top(uint64_t *buf, uint32_t count, uint32_t cap, uint32_t n, uint32_t tid) {
    __shared__ uint64_t s_wk[BM25_THREADS / 32];
    __shared__ uint32_t s_wp[BM25_THREADS / 32];
    __shared__ uint64_t s_top[32];
    if (n > 32) {
        for (uint32_t i = count + tid; i < cap; i += BM25_THREADS) buf[i] = KEY_NONE;
        group_bitonic_desc(buf, cap, tid, BM25_THREADS, 0);
        return;
    }
    for (uint32_t r = 0; r < n; r++) {
        uint64_t best = KEY_NONE;
        uint32_t pos = 0;
        for (uint32_t i = tid; i < count; i += BM25_THREADS) {
            const uint64_t k = buf[i];
            if (k > best) { best = k; pos = i; }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const uint64_t ob = __shfl_xor_sync(0xffffffffu, best, o);
            const uint32_t op = __shfl_xor_sync(0xffffffffu, pos, o);
            if (ob > best) { best = ob; pos = op; }
        }
        if ((tid & 31) == 0) { s_wk[tid >> 5] = best; s_wp[tid >> 5] = pos; }
        __syncthreads();
        if (tid == 0) {
            uint64_t b = s_wk[0]; uint32_t bp = s_wp[0];
            for (uint32_t w = 1; w < BM25_THREADS / 32; w++) if (s_wk[w] > b) { b = s_wk[w]; bp = s_wp[w]; }
            s_top[r] = b;
            if (b != KEY_NONE) buf[bp] = KEY_NONE;
        }
        __syncthreads();
    }
    if (tid < n) buf[tid] = s_top[tid];
    __syncthreads();
}

// ---- the scorer: one CTA per (query, tile) ----
template <bool MULTI, bool THRESH, bool OMC, bool ROWFT = false>
__global__ void __launch_bounds__(BM25_THREADS) bm25_tile_kernel(const Bm25Params p) {
    extern __shared__ __align__(16) uint8_t smem[];
    float *score = reinterpret_cast<float *>(smem);
    float *aux = score + BM25_TILE;                                    // S, then OMC multipliers
    uint32_t *mask = reinterpret_cast<uint32_t *>(score + BM25_TILE * ((MULTI || OMC) ? 2 : 1));
    uint32_t *okb = mask + (THRESH ? BM25_TILE : 0);
    uint64_t *tbuf = reinterpret_cast<uint64_t *>(okb + BM25_TILE / 32);
    __shared__ uint32_t s_cnt, s_matched;
    __shared__ unsigned int s_maxo, s_mino;   // extrema in order-preserving uint space
    __shared__ unsigned long long s_tau;
    __shared__ uint32_t s_mbits[BM25_TILE / 32];

    const uint32_t q = blockIdx.x % p.n_queries;
    const uint32_t tile = blockIdx.x / p.n_queries;
    const uint32_t row0 = tile * BM25_TILE;
    const uint32_t tid = threadIdx.x;
    const QueryDesc qd = p.queries[q];
    const float kp1 = __fadd_rn(p.k, 1.0f);
    const bool use_ok = p.row_ok_bits != nullptr;

    for (uint32_t i = tid; i < BM25_TILE / 4; i += BM25_THREADS) {
        reinterpret_cast<float4 *>(score)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (MULTI) reinterpret_cast<float4 *>(aux)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (THRESH) reinterpret_cast<uint4 *>(mask)[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    if (use_ok) {
        const uint32_t *okq = row_ok_of(p.row_ok_bits, p.q_ok_slot, p.ok_words, q);
        for (uint32_t i = tid; i < BM25_TILE / 32; i += BM25_THREADS) okb[i] = okq[row0 / 32 + i];
    }
    if (tid == 0) { s_cnt = 0; s_matched = 0; s_maxo = f32_ordered(0.f); s_mino = f32_ordered(0.f); s_tau = p.tau[q]; }
    if (p.matched_bits && tid < BM25_TILE / 32) s_mbits[tid] = 0u;
    __syncthreads();

    // ------------------------------------------------ accumulate, token by token, term by term.
    // Warp 0 builds a per-CTA table of the query's term sub-ranges for this tile (up to
    // TERM_PASS terms per pass); every thread then walks the table with broadcast LDS.  Terms
    // with no posting in the tile cost nothing (no barrier); the first batch of the next
    // non-empty term is requested before the barrier that closes the current one.
    {
        constexpr uint32_t TERM_PASS = 96;
        __shared__ const uint2 *t_ptr[TERM_PASS];
        __shared__ uint32_t t_n[TERM_PASS], t_bit[TERM_PASS], t_flag[TERM_PASS];   // flag bit0: single, bit1: last term of its token
        __shared__ float t_w[TERM_PASS], t_idf[TERM_PASS];
        __shared__ uint32_t t_tok_begin[TERM_PASS];                                 // first term (table index space: global e) of the token
        const uint32_t e_begin = qd.token_begin < qd.token_end ? p.tokens[qd.token_begin].term_begin : 0;
        const uint32_t e_end = qd.token_begin < qd.token_end ? p.tokens[qd.token_end - 1].term_end : 0;
        for (uint32_t pass0 = e_begin; pass0 < e_end; pass0 += TERM_PASS) {
            const uint32_t nt = min(TERM_PASS, e_end - pass0);
            __syncthreads();   // previous pass fully consumed
            for (uint32_t j = tid; j < nt; j += BM25_THREADS) {
                const uint32_t e = pass0 + j;
                const TermDesc td = p.terms[e];
                const TokenDesc tk = p.tokens[p.term_token[e]];
                const uint32_t *sg = p.seg + size_t(e) * (p.n_tiles + 1);
                const uint32_t lo = sg[tile], hi = sg[tile + 1];
                t_ptr[j] = reinterpret_cast<const uint2 *>(td.ptr) + lo;
                t_n[j] = hi - lo;
                t_w[j] = td.weight; t_idf[j] = tk.idf; t_bit[j] = tk.bit;
                const bool single = !MULTI || (tk.term_end - tk.term_begin == 1);
                t_flag[j] = (single ? 1u : 0u) | ((e + 1 == tk.term_end) ? 2u : 0u) | ((td.flags & 1u) ? 4u : 0u);
                t_tok_begin[j] = tk.term_begin;
            }
            __syncthreads();
            uint2 rec[4];
            auto fetch = [&](uint32_t j, uint32_t base, uint2 (&r)[4]) {
                const uint2 *pp = t_ptr[j];
                const uint32_t n = t_n[j];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const uint32_t pi = base + tid + u * BM25_THREADS;
                    r[u] = pi < n ? __ldg(pp + pi) : make_uint2(0xffffffffu, 0u);
                }
            };
            // first non-empty term of the pass (multi-term tokens keep their empty terms: finalize needs the walk)
            auto next_nonempty = [&](uint32_t j) { while (j < nt && t_n[j] == 0 && (t_flag[j] & 1u)) j++; return j; };
            uint32_t j = next_nonempty(0);
            if (j < nt && (tid & ~31u) < t_n[j]) fetch(j, 0, rec);
            while (j < nt) {
                const uint32_t n = t_n[j], flag = t_flag[j];
                const bool single = flag & 1u;
                const float w = t_w[j], idf = t_idf[j];
                const uint32_t bit = t_bit[j];
                // request the next non-empty term's first batch now: its latency hides behind this term's work
                const uint32_t jn = next_nonempty(j + 1);
                uint2 nrec[4];
                const bool pre = jn < nt && (tid & ~31u) < t_n[jn];
                if (pre) fetch(jn, 0, nrec);
                for (uint32_t base = 0; base < n; base += BM25_THREADS * 4) {
                    if (base + (tid & ~31u) >= n) break;             // this warp has no posting in the batch
                    if (base != 0) fetch(j, base, rec);
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        if (rec[u].x == 0xffffffffu) continue;
                        const uint32_t l = rec[u].x - row0;
                        if (use_ok && !((okb[l >> 5] >> (l & 31)) & 1u)) continue;
                        if (flag & 4u) {   // contribution precomputed once per batch for this (term, weight): NaN = skip
                            const float c = __uint_as_float(rec[u].y);
                            if (c == c) {
                                score[l] = __fadd_rn(score[l], c);
                                if (THRESH) mask[l] |= bit;
                            }
                            continue;
                        }
                        const float ntf = __fmul_rn(w, __uint_as_float(rec[u].y));   // w * tf'
                        if (single) {
                            // S = 0.0 + 1.0*ntf; skip unless is_normal (bm25.rs:387,501)
                            if (f32_is_normal(ntf)) {
                                const float c = bm25_sat(ntf, p.k, kp1, idf);
                                if (c == c) {
                                    score[l] = __fadd_rn(score[l], c);
                                    if (THRESH) mask[l] |= bit;
                                }
                            }
                        } else {
                            aux[l] = __fadd_rn(aux[l], ntf);  // S += weight(1.0) * ntf, push order
                        }
                    }
                }
                __syncthreads();  // next term / token may touch the same rows
                if (MULTI && !single && (flag & 2u)) {
                    // finalize_term: drain S over the rows this token touched (second walk, L2-hot)
                    const uint32_t tb = t_tok_begin[j];
                    for (uint32_t fe = tb; fe <= pass0 + j; fe++) {
                        // terms of this token that fell into an earlier pass are re-read from the descriptors
                        const uint2 *fp; uint32_t fn;
                        if (fe >= pass0) { fp = t_ptr[fe - pass0]; fn = t_n[fe - pass0]; }
                        else {
                            const TermDesc fd = p.terms[fe];
                            const uint32_t *sg = p.seg + size_t(fe) * (p.n_tiles + 1);
                            fp = reinterpret_cast<const uint2 *>(fd.ptr) + sg[tile]; fn = sg[tile + 1] - sg[tile];
                        }
                        for (uint32_t pi = tid; pi < fn; pi += BM25_THREADS) {
                            const uint32_t l = fp[pi].x - row0;
                            const float S = __uint_as_float(atomicExch(reinterpret_cast<unsigned int *>(&aux[l]), 0u));
                            if (f32_is_normal(S)) {
                                const float c = bm25_sat(S, p.k, kp1, idf);
                                if (c == c) {
                                    score[l] = __fadd_rn(score[l], c);
                                    if (THRESH) mask[l] |= bit;
                                }
                            }
                        }
                        __syncthreads();
                    }
                }
                j = jn;
                if (pre) {
#pragma unroll
                    for (int u = 0; u < 4; u++) rec[u] = nrec[u];
                }
            }
        }
        __syncthreads();
    }

    // ------------------------------------------------ OMC multipliers for this tile
    uint32_t omc_lo = 0, omc_hi = 0;
    if (OMC) {
        for (uint32_t i = tid; i < BM25_TILE; i += BM25_THREADS) aux[i] = 1.0f;
        // binary search [row0, row0+TILE) in omc_row (uniform across the block)
        uint32_t lo = 0, hi = p.n_omc;
        while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (p.omc_row[m] < row0) lo = m + 1; else hi = m; }
        omc_lo = lo; hi = p.n_omc;
        const uint64_t rend = uint64_t(row0) + BM25_TILE;
        while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (uint64_t(p.omc_row[m]) < rend) lo = m + 1; else hi = m; }
        omc_hi = lo;
        __syncthreads();
        for (uint32_t i = omc_lo + tid; i < omc_hi; i += BM25_THREADS) aux[p.omc_row[i] - row0] = p.omc_mult[i];
        __syncthreads();
    }

    // ------------------------------------------------ scan: count, extrema, gated top-n
    const float mh = p.min_hint ? p.min_hint[q] : 0.f;
    unsigned long long tau = s_tau;
    uint32_t matched = 0;
    float lmax = 0.f, lmin = 0.f;
    const uint64_t rows_here = min(uint64_t(BM25_TILE), p.n_rows - row0);
    float tau_f = tau ? key_score(tau) : -INFINITY;   // cheap float pre-filter for the rank key compare
    __shared__ uint32_t s_ovf;
    // One pass over the tile.  chunked=false: no barriers, pushes are overflow-checked (the common
    // case once the query's threshold has warmed up: a handful of pushes per tile).  If the buffer
    // overflowed (cold threshold: the first tiles of a query) the pass is redone chunk by chunk with
    // a barrier + compress between chunks.
    auto scan_pass = [&](const bool chunked) {
        matched = 0; lmax = 0.f; lmin = 0.f;
        for (uint32_t base = 0; base < rows_here; base += BM25_CHUNK) {
            const uint32_t l0 = base + tid * 4;                   // 4 consecutive rows per thread: one LDS.128
            bool pushed = false;
            {
                // branch-free bookkeeping: absent rows hold 0.0 (never touched; rows past n_rows too), so
                // fmax/fmin with them are no-ops (folds start at 0.0) and only the rare candidate path branches
                const float4 s4 = *reinterpret_cast<const float4 *>(score + l0);
                float sv[4] = {s4.x, s4.y, s4.z, s4.w};
                if (THRESH) {
                    const uint4 m4 = *reinterpret_cast<const uint4 *>(mask + l0);
                    const uint32_t mv[4] = {m4.x, m4.y, m4.z, m4.w};
#pragma unroll
                    for (int u = 0; u < 4; u++)   // bm25.rs:416-428: keep popcount(mask) >= required
                        sv[u] = (mv[u] != 0u && uint32_t(__popc(mv[u])) >= qd.required) ? sv[u] : 0.f;
                }
                uint32_t cand = 0;
                float pv[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const float s = sv[u];
                    const bool present = s != 0.f;
                    matched += present ? 1u : 0u;
                    if (p.matched_bits && present) atomicOr(&s_mbits[(l0 + u) >> 5], 1u << ((l0 + u) & 31));
                    if (ROWFT && present) p.row_ft[size_t(q) * p.n_tiles * BM25_TILE + row0 + l0 + u] = s;
                    lmax = fmaxf(lmax, s);
                    lmin = fminf(lmin, s);
                    float proxy = __fsub_rn(s, mh);
                    if (OMC) proxy = __fmul_rn(proxy, aux[l0 + u]);
                    pv[u] = proxy;
                    cand |= (present && proxy >= tau_f) ? (1u << u) : 0u;   // NaN fails; ties re-checked on the key
                }
                if (cand) {
#pragma unroll
                    for (int u = 0; u < 4; u++)
                        if ((cand >> u) & 1u) {
                            const unsigned long long key = make_key(pv[u], row0 + l0 + u);
                            if (key > tau) {
                                const uint32_t slot = atomicAdd(&s_cnt, 1u);
                                if (slot < p.cap) tbuf[slot] = key;   // chunked: guaranteed by the compress rule
                                else s_ovf = 1u;
                                pushed = true;
                            }
                        }
                }
            }
            if (!chunked) continue;
            if (!__syncthreads_or(pushed)) continue;               // nothing pushed in this chunk: no overflow risk
            const uint32_t c = s_cnt;   // snapshot, then barrier, so the branch is block-uniform
            __syncthreads();
            if (c + BM25_CHUNK > p.cap && base + BM25_CHUNK < rows_here) {
                // compress: keep the best n_keep (ft travels by re-lookup: key -> row -> score[])
                block_keep_top(tbuf, c, p.cap, p.n_keep, tid);
                const uint32_t kept = min(c, p.n_keep);
                if (tid == 0) s_cnt = kept;
                if (kept == p.n_keep) { tau = max(tau, (unsigned long long)tbuf[p.n_keep - 1]); tau_f = key_score(tau); }
                __syncthreads();
            }
        }
    };
    if (tid == 0) s_ovf = 0u;
    __syncthreads();
    scan_pass(false);
    __syncthreads();
    if (s_ovf) {
        __syncthreads();
        if (tid == 0) { s_cnt = 0u; s_ovf = 0u; }
        __syncthreads();
        scan_pass(true);
    }
    __syncthreads();
    // ---- block reductions of count / extrema
    matched = __reduce_add_sync(0xffffffffu, matched);
    for (int o = 16; o > 0; o >>= 1) {
        lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
    }
    if ((tid & 31) == 0) {
        if (matched) atomicAdd(&s_matched, matched);
        atomicMax(&s_maxo, f32_ordered(lmax));
        atomicMin(&s_mino, f32_ordered(lmin));
    }
    __syncthreads();

    // ---- final emit: best <= n_keep of the buffer
    const size_t slot_base = (size_t(q) * p.n_tiles + tile);
    uint32_t c = s_cnt;
    if (c >= p.n_keep && c > 0) {
        block_keep_top(tbuf, c, p.cap, p.n_keep, tid);
        c = p.n_keep;
        if (tid == 0) atomicMax(p.tau + q, (unsigned long long)tbuf[p.n_keep - 1]);
    }
    for (uint32_t i = tid; i < c; i += BM25_THREADS) {
        p.cand_key[slot_base * p.n_keep + i] = tbuf[i];
        p.cand_ft[slot_base * p.n_keep + i] = score[key_idx(tbuf[i]) - row0];
    }
    if (tid == 0) {
        p.cand_cnt[slot_base] = c;
        p.tile_count[slot_base] = s_matched;
        p.tile_max[slot_base] = f32_unordered(s_maxo);
        p.tile_min[slot_base] = f32_unordered(s_mino);
    }
    if (p.matched_bits && tid < BM25_TILE / 32) p.matched_bits[slot_base * (BM25_TILE / 32) + tid] = s_mbits[tid];
}


// =======================================================================================
// K3b — the scorer for the common query shape: every token resolves to (at most) ONE index term.
//
// Same contract and outputs as bm25_tile_kernel<false, THRESH, OMC> (bit-identical scores: contributions are
// added in token order with explicit round-to-nearest ops), restructured around the POSTINGS instead of the
// row slots:
//   * persistent CTAs pull (tile, query) items from a global counter, tile-major, so the queries that share a
//     tile's hot posting ranges run back to back (L2) and the per-CTA setup is paid once;
//   * the shared-memory accumulators are zeroed once per CTA; every item leaves them clean: a SPARSE item
//     (few postings in the tile) is finished by walking its postings again (L1/L2-hot) and exchanging each
//     slot with 0 — the first visitor owns the document, later visitors see 0 — so neither a zeroing pass nor
//     a scan of the 8192 slots is paid; a DENSE item scans the slots (as K3 did) and zeroes them on the way out;
//   * lanes map to postings one-to-one for short ranges (4-way unrolled only when a range fills the block).
// The hybrid lookup of the vector hits' fulltext scores is not done here (bm25_point_kernel), so this kernel
// does not depend on the vector stage and can overlap the matrix sweep on another stream.
// =======================================================================================
constexpr uint32_t BM25_SPARSE_MAX = BM25_TILE / 4;     // postings of one (query, tile) item up to which the sparse finish is used
constexpr uint32_t BM25_MAX_TOK = 32;          // tokens per query (u32 bitmask, token_score.rs:293)

__host__ __device__ inline size_t bm25_tile2_smem_bytes(bool threshold, bool omc, uint32_t cap) {
    size_t b = size_t(BM25_TILE) * 4;                 // score
    if (omc) b += size_t(BM25_TILE) * 4;              // omc multipliers
    if (threshold) b += size_t(BM25_TILE) * 4;        // token masks
    b += size_t(BM25_TILE) / 8;                       // row_ok bits
    b += size_t(cap) * 8;                             // top buffer keys
    return b + 64;
}

// Per-(tile, query) item descriptors, flattened by bm25_flatten_kernel so that an item needs ONE level of
// global loads (prefetched during the previous item) instead of the chain query -> tokens -> terms -> seg.
struct ItemTok {            // 32 B
    const void *ptr;        // list: first posting of the term inside this tile; dense: the tile's slice of the float array
    uint32_t n;             // list: postings in the tile; dense: BM25_TILE (0 = token absent from this tile)
    uint32_t flags;         // TD_PRE / TD_DENSE
    float w, idf;
    uint32_t bit;
    uint32_t bound;         // dense: float bits of the bound of the tile's contributions (bm25_dense_bound); else unused
};
constexpr uint32_t BM25_FLAT_TOK = 4;   // tokens per query the flat descriptors hold (longer queries: in-kernel table build)
__global__ void __launch_bounds__(256) bm25_flatten_kernel(const Bm25Params p, ItemTok *flat) {
    const TermDesc *terms = p.terms; const TokenDesc *tokens = p.tokens; const QueryDesc *queries = p.queries;
    const uint32_t *seg = p.seg;
    const uint32_t n_tiles = p.n_tiles, n_queries = p.n_queries;
    const uint64_t gid = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    const uint64_t total = uint64_t(n_tiles) * n_queries * BM25_FLAT_TOK;
    if (gid >= total) return;
    const uint32_t j = uint32_t(gid % BM25_FLAT_TOK);
    const uint32_t item = uint32_t(gid / BM25_FLAT_TOK);
    const uint32_t tile = item / n_queries, q = item % n_queries;
    const QueryDesc qd = queries[q];
    ItemTok it{};
    if (j < qd.token_end - qd.token_begin) {
        const TokenDesc tk = tokens[qd.token_begin + j];
        it.idf = tk.idf; it.bit = tk.bit;
        if (tk.term_end > tk.term_begin) {
            const TermDesc td = terms[tk.term_begin];
            it.flags = td.flags; it.w = td.weight;
            if (td.flags & TD_DENSE) {
                it.ptr = reinterpret_cast<const float *>(td.ptr) + size_t(tile) * BM25_TILE;
                it.n = td.len ? BM25_TILE : 0;
                if (td.len) it.bound = __float_as_uint(bm25_dense_bound(reinterpret_cast<const float *>(td.ptr), n_tiles)[tile]);
            } else {
                const uint32_t *sg = seg + size_t(tk.term_begin) * (n_tiles + 1);
                const uint32_t lo = sg[tile], hi = sg[tile + 1];
                it.ptr = reinterpret_cast<const uint2 *>(td.ptr) + lo;
                it.n = hi - lo;
            }
        }
    }
    flat[gid] = it;
}

template <bool THRESH, bool OMC, bool ROWFT = false>
__global__ void __launch_bounds__(BM25_THREADS, 1024 / BM25_THREADS) bm25_tile2_kernel(const Bm25Params p, const ItemTok *flat, unsigned int *work_counter) {
    extern __shared__ __align__(16) uint8_t smem[];
    float *score = reinterpret_cast<float *>(smem);
    float *aux = score + BM25_TILE;                                    // OMC multipliers
    uint32_t *mask = reinterpret_cast<uint32_t *>(score + BM25_TILE * (OMC ? 2 : 1));
    uint32_t *okb = mask + (THRESH ? BM25_TILE : 0);
    uint64_t *tbuf = reinterpret_cast<uint64_t *>(okb + BM25_TILE / 32);
    // per-item counters, double-buffered by item parity: the set of the NEXT item is reset while this one runs, so no
    // thread can still be reading a counter that another thread is already resetting
    __shared__ uint32_t s_cnt2[2], s_matched2[2];
    __shared__ unsigned int s_maxo2[2], s_mino2[2];
    __shared__ const uint2 *t_ptr[BM25_MAX_TOK];
    __shared__ uint32_t t_n[BM25_MAX_TOK], t_bit[BM25_MAX_TOK], t_pre[BM25_MAX_TOK];
    __shared__ float t_w[BM25_MAX_TOK], t_idf[BM25_MAX_TOK];
    __shared__ uint32_t s_ntok, s_item_cur, s_item_next;
    __shared__ uint32_t s_mbits[BM25_TILE / 32];

    const uint32_t tid = threadIdx.x;
    const float kp1 = __fadd_rn(p.k, 1.0f);
    const bool use_ok = p.row_ok_bits != nullptr;
    const bool want_bits = p.matched_bits != nullptr;
    const uint32_t n_items = p.n_tiles * p.n_queries;

    for (uint32_t i = tid; i < BM25_TILE / 4; i += BM25_THREADS) {
        reinterpret_cast<float4 *>(score)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (THRESH) reinterpret_cast<uint4 *>(mask)[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    // items come from a global counter (tile-major: the queries sharing a tile's hot ranges run back to back through
    // L2; dense and sparse items differ 3x in cost, so the deal is dynamic), fetched TWO ahead: while item k runs, the
    // id of item k+1 is already known — its descriptors travel from global memory now — and the id of k+2 is requested
    auto store_tok = [&](const ItemTok &it, uint32_t j) {
        t_ptr[j] = reinterpret_cast<const uint2 *>(it.ptr); t_n[j] = it.n; t_pre[j] = it.flags;
        t_w[j] = it.w; t_idf[j] = it.idf; t_bit[j] = it.bit;
    };
    if (tid == 0) { s_item_cur = atomicAdd(work_counter, 1u); s_item_next = atomicAdd(work_counter, 1u); s_ntok = BM25_FLAT_TOK; }
    if (tid < 2) { s_cnt2[tid] = 0; s_matched2[tid] = 0; s_maxo2[tid] = f32_ordered(0.f); s_mino2[tid] = f32_ordered(0.f); }
    __syncthreads();
    if (flat && s_item_cur < n_items && tid < BM25_FLAT_TOK) store_tok(flat[size_t(s_item_cur) * BM25_FLAT_TOK + tid], tid);
    for (uint32_t par = 0;; par ^= 1u) {
        if (want_bits && tid < BM25_TILE / 32) s_mbits[tid] = 0u;
        __syncthreads();                                   // previous item retired: accumulators clean, table + counters + ids set
        const uint32_t item = s_item_cur;
        if (item >= n_items) break;
        const uint32_t next = s_item_next;
        uint32_t next2 = 0;
        if (tid == 0) next2 = atomicAdd(work_counter, 1u);   // consumed at the end of this item
        const uint32_t tile = item / p.n_queries, q = item % p.n_queries;
        const uint32_t row0 = tile * BM25_TILE;
        uint32_t &s_cnt = s_cnt2[par], &s_matched = s_matched2[par];
        unsigned int &s_maxo = s_maxo2[par], &s_mino = s_mino2[par];
        if (tid == 0) { s_cnt2[par ^ 1u] = 0; s_matched2[par ^ 1u] = 0; s_maxo2[par ^ 1u] = f32_ordered(0.f); s_mino2[par ^ 1u] = f32_ordered(0.f); }
        const QueryDesc qd = p.queries[q];                 // (required / slow-path token range; L2-hot, off the critical path)
        if (!flat) {   // a query of this batch has more than BM25_FLAT_TOK tokens: build the table here
            const uint32_t ntok = min(qd.token_end - qd.token_begin, BM25_MAX_TOK);
            if (tid < ntok) {
                const TokenDesc tk = p.tokens[qd.token_begin + tid];
                ItemTok it{};
                it.idf = tk.idf; it.bit = tk.bit;
                if (tk.term_end > tk.term_begin) {
                    const TermDesc td = p.terms[tk.term_begin];
                    it.flags = td.flags; it.w = td.weight;
                    if (td.flags & TD_DENSE) { it.ptr = reinterpret_cast<const float *>(td.ptr) + row0; it.n = td.len ? BM25_TILE : 0; }
                    else {
                        const uint32_t *sg = p.seg + size_t(tk.term_begin) * (p.n_tiles + 1);
                        it.ptr = reinterpret_cast<const uint2 *>(td.ptr) + sg[tile]; it.n = sg[tile + 1] - sg[tile];
                    }
                }
                store_tok(it, tid);
            }
            if (tid == 0) s_ntok = ntok;
        }
        if (use_ok) {
            const uint32_t *okq = row_ok_of(p.row_ok_bits, p.q_ok_slot, p.ok_words, q);
            for (uint32_t i = tid; i < BM25_TILE / 32; i += BM25_THREADS) okb[i] = okq[row0 / 32 + i];
        }
        if (!flat || use_ok) __syncthreads();
        const uint32_t ntok = s_ntok;
        // in flight during this item: the next item's descriptors and this query's running threshold
        ItemTok nx{};
        if (flat && next < n_items && tid < BM25_FLAT_TOK) nx = flat[size_t(next) * BM25_FLAT_TOK + tid];
        unsigned long long tau = p.tau[q];

        // ---------------------------------------- accumulate, token by token (the reference's summation order)
        uint32_t total = 0;
        bool prev_dense = false;
        // first batch of the next LIST token is requested before the current token is applied
        uint2 pre[4];
        auto preload = [&](uint32_t j, uint2 (&r)[4]) {
            const uint2 *pp = t_ptr[j];
            const uint32_t n = t_n[j];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const uint32_t pi = tid + u * BM25_THREADS;
                r[u] = pi < n ? __ldg(pp + pi) : make_uint2(0xffffffffu, 0u);
            }
        };
        uint32_t list_mask = 0;   // tokens that are non-empty posting ranges (ntok <= 32)
        for (uint32_t j = 0; j < ntok; j++) list_mask |= (t_n[j] != 0 && !(t_pre[j] & TD_DENSE)) ? (1u << j) : 0u;
        auto next_list = [&](uint32_t j) { const uint32_t m = j < 32 ? (list_mask >> j) : 0u; return m ? j + uint32_t(__ffs(m)) - 1u : ntok; };
        uint32_t jl = next_list(0);
        if (jl < ntok) preload(jl, pre);
        for (uint32_t j = 0; j < ntok; j++) {
            const uint32_t n = t_n[j];
            if (n == 0) continue;                          // block-uniform
            total += n;
            const uint2 *pp = t_ptr[j];
            const bool pre_c = (t_pre[j] & TD_PRE) != 0;
            const float w = t_w[j], idf = t_idf[j];
            const uint32_t bit = t_bit[j];
            if (t_pre[j] & TD_DENSE) {
                // hot term: add the tile's slice of its dense contribution array (0.0 where the row has no posting,
                // is filtered out or its contribution was skipped: x + 0.0 == x bit for bit).  Thread t owns the
                // float4 slots t, t+256, ... here AND in the finishing scan, so no barrier is needed between
                // consecutive dense tokens or between the last one and the scan.
                const float4 *dp = reinterpret_cast<const float4 *>(pp);
                constexpr uint32_t F4 = BM25_TILE / 4 / BM25_THREADS;        // float4 slots per thread (8 at 8192 rows)
                static_assert(F4 >= 1 && F4 % (F4 >= 4 ? 4 : F4) == 0, "tile size");
                constexpr uint32_t FB = F4 >= 4 ? 4 : F4;                    // loads in flight per batch
#pragma unroll
                for (uint32_t h = 0; h < F4 / FB; h++) {
                    float4 c4[FB];
#pragma unroll
                    for (uint32_t u = 0; u < FB; u++) c4[u] = __ldg(dp + tid + (h * FB + u) * BM25_THREADS);
#pragma unroll
                    for (uint32_t u = 0; u < FB; u++) {
                        const uint32_t i = tid + (h * FB + u) * BM25_THREADS;
                        float4 s4 = reinterpret_cast<float4 *>(score)[i];
                        s4.x = __fadd_rn(s4.x, c4[u].x); s4.y = __fadd_rn(s4.y, c4[u].y);
                        s4.z = __fadd_rn(s4.z, c4[u].z); s4.w = __fadd_rn(s4.w, c4[u].w);
                        reinterpret_cast<float4 *>(score)[i] = s4;
                        if (THRESH) {
                            uint4 m4 = reinterpret_cast<uint4 *>(mask)[i];
                            m4.x |= c4[u].x != 0.f ? bit : 0u; m4.y |= c4[u].y != 0.f ? bit : 0u;
                            m4.z |= c4[u].z != 0.f ? bit : 0u; m4.w |= c4[u].w != 0.f ? bit : 0u;
                            reinterpret_cast<uint4 *>(mask)[i] = m4;
                        }
                    }
                }
                prev_dense = true;
                continue;
            }
            if (prev_dense) { __syncthreads(); prev_dense = false; }   // a list token scatters across the owners' slots
            auto apply = [&](const uint2 rec) {
                if (rec.x == 0xffffffffu) return;
                const uint32_t l = rec.x - row0;
                if (use_ok && !((okb[l >> 5] >> (l & 31)) & 1u)) return;
                float c;
                if (pre_c) c = __uint_as_float(rec.y);       // contribution precomputed once per batch (NaN = skip)
                else {
                    const float ntf = __fmul_rn(w, __uint_as_float(rec.y));
                    c = f32_is_normal(ntf) ? bm25_sat(ntf, p.k, kp1, idf) : __int_as_float(0x7fc00000);   // bm25.rs:387,501
                }
                if (c == c) {
                    score[l] = __fadd_rn(score[l], c);
                    if (THRESH) mask[l] |= bit;
                }
            };
            // this token's first batch is already here; request the next list token's before applying it
            uint2 cur[4];
#pragma unroll
            for (int u = 0; u < 4; u++) cur[u] = pre[u];
            jl = next_list(j + 1);
            if (jl < ntok) preload(jl, pre);
#pragma unroll
            for (int u = 0; u < 4; u++) apply(cur[u]);
            for (uint32_t base = BM25_THREADS * 4; base < n; base += BM25_THREADS * 4) {   // long ranges: 4 loads in flight per lane
                uint2 r[4];
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const uint32_t pi = base + tid + u * BM25_THREADS;
                    r[u] = pi < n ? __ldg(pp + pi) : make_uint2(0xffffffffu, 0u);
                }
#pragma unroll
                for (int u = 0; u < 4; u++) apply(r[u]);
            }
            __syncthreads();                               // the next token may touch the same rows
        }

        if (OMC) {   // multipliers of this tile's rows (search.rs:39-48), rare
            for (uint32_t i = tid; i < BM25_TILE; i += BM25_THREADS) aux[i] = 1.0f;
            uint32_t lo = 0, hi = p.n_omc;
            while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (p.omc_row[m] < row0) lo = m + 1; else hi = m; }
            const uint32_t omc_lo = lo;
            hi = p.n_omc;
            const uint64_t rend = uint64_t(row0) + BM25_TILE;
            while (lo < hi) { uint32_t m = (lo + hi) >> 1; if (uint64_t(p.omc_row[m]) < rend) lo = m + 1; else hi = m; }
            __syncthreads();
            for (uint32_t i = omc_lo + tid; i < lo; i += BM25_THREADS) aux[p.omc_row[i] - row0] = p.omc_mult[i];
            __syncthreads();
        }

        // ---------------------------------------- finish: count, extrema, gated top-n; leave the accumulators clean
        const float mh = p.min_hint ? p.min_hint[q] : 0.f;
        float tau_f = tau ? key_score(tau) : -INFINITY;
        uint32_t matched = 0;
        float lmax = 0.f, lmin = 0.f;
        const uint64_t rows_here = min(uint64_t(BM25_TILE), p.n_rows - row0);
        auto consider = [&](float s, uint32_t l) -> bool {   // candidate test of one matched row; true when it pushed
            float proxy = __fsub_rn(s, mh);
            if (OMC) proxy = __fmul_rn(proxy, aux[l]);
            if (!(proxy >= tau_f)) return false;                            // NaN fails; ties re-checked on the key
            const unsigned long long key = make_key(proxy, row0 + l);
            if (key <= tau) return false;
            const uint32_t slot = atomicAdd(&s_cnt, 1u);
            if (slot < p.cap) tbuf[slot] = key;                             // s_cnt > cap afterwards == overflow
            return true;
        };
        auto visit = [&](float s, uint32_t l) -> bool {   // one matched row
            matched++;
            if (want_bits) atomicOr(&s_mbits[l >> 5], 1u << (l & 31));
            if (ROWFT) p.row_ft[size_t(q) * p.n_tiles * BM25_TILE + row0 + l] = s;
            lmax = fmaxf(lmax, s);
            lmin = fminf(lmin, s);
            return consider(s, l);
        };
        // without OMC / a min hint a candidate's raw score is its key's score (proxy == score): nothing is re-read at emit
        const bool ft_from_key = !OMC && mh == 0.f;
        const bool sparse = total != 0 && total <= BM25_SPARSE_MAX && p.cap >= BM25_SPARSE_MAX && ft_from_key;
        auto scan_pass = [&](const bool chunked) {
            matched = 0; lmax = 0.f; lmin = 0.f;
            for (uint32_t base = 0; base < rows_here; base += BM25_CHUNK) {
                const uint32_t l0 = base + tid * 4;
                bool pushed = false;
                const float4 s4 = *reinterpret_cast<const float4 *>(score + l0);
                float sv[4] = {s4.x, s4.y, s4.z, s4.w};
                if (THRESH) {
                    const uint4 m4 = *reinterpret_cast<const uint4 *>(mask + l0);
                    const uint32_t mv[4] = {m4.x, m4.y, m4.z, m4.w};
#pragma unroll
                    for (int u = 0; u < 4; u++)   // bm25.rs:416-428: keep popcount(mask) >= required
                        sv[u] = (mv[u] != 0u && uint32_t(__popc(mv[u])) >= qd.required) ? sv[u] : 0.f;
                }
                if (!OMC && !want_bits) {
                    // common case: branch-free bookkeeping of the 4 slots, one candidate test on their maximum
                    // (absent rows hold 0.0: no-ops for the folds, which start at 0.0, token_score.rs:398-401)
                    matched += (sv[0] != 0.f ? 1u : 0u) + (sv[1] != 0.f ? 1u : 0u) + (sv[2] != 0.f ? 1u : 0u) + (sv[3] != 0.f ? 1u : 0u);
                    const float m4 = fmaxf(fmaxf(sv[0], sv[1]), fmaxf(sv[2], sv[3]));
                    lmax = fmaxf(lmax, m4);
                    lmin = fminf(lmin, fminf(fminf(sv[0], sv[1]), fminf(sv[2], sv[3])));
                    if (__fsub_rn(m4, mh) >= tau_f) {
#pragma unroll
                        for (int u = 0; u < 4; u++)
                            if (sv[u] != 0.f) pushed |= consider(sv[u], l0 + u);
                    }
                } else {
#pragma unroll
                    for (int u = 0; u < 4; u++)
                        if (sv[u] != 0.f) pushed |= visit(sv[u], l0 + u);
                }
                if (!chunked) continue;
                if (!__syncthreads_or(pushed)) continue;
                const uint32_t c = s_cnt;
                __syncthreads();
                if (c + BM25_CHUNK > p.cap && base + BM25_CHUNK < rows_here) {
                    block_keep_top(tbuf, c, p.cap, p.n_keep, tid);
                    const uint32_t kept = min(c, p.n_keep);
                    if (tid == 0) s_cnt = kept;
                    if (kept == p.n_keep) { tau = max(tau, (unsigned long long)tbuf[p.n_keep - 1]); tau_f = key_score(tau); }
                    __syncthreads();
                }
            }
        };
        auto reduce = [&]() {   // block reductions of count / extrema
            matched = __reduce_add_sync(0xffffffffu, matched);
            for (int o = 16; o > 0; o >>= 1) {
                lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
                lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
            }
            if ((tid & 31) == 0 && matched) {
                atomicAdd(&s_matched, matched);
                atomicMax(&s_maxo, f32_ordered(lmax));
                atomicMin(&s_mino, f32_ordered(lmin));
            }
        };
        if (sparse) {
            // walk the postings again; the first visitor of a row takes its sum and clears the slot
            for (uint32_t j = 0; j < ntok; j++) {
                const uint32_t n = t_n[j];
                const uint2 *pp = t_ptr[j];
                for (uint32_t pi = tid; pi < n; pi += BM25_THREADS) {
                    const uint32_t l = __ldg(&pp[pi].x) - row0;
                    float s = __uint_as_float(atomicExch(reinterpret_cast<unsigned int *>(&score[l]), 0u));
                    if (s != 0.f) {
                        if (THRESH) {   // the masks are stable during this walk (cleared below)
                            const uint32_t m = mask[l];
                            if (!(m != 0u && uint32_t(__popc(m)) >= qd.required)) continue;   // bm25.rs:416-428
                        }
                        visit(s, l);
                    }
                }
            }
            if (THRESH) {
                __syncthreads();
                for (uint32_t j = 0; j < ntok; j++) {
                    const uint32_t n = t_n[j];
                    const uint2 *pp = t_ptr[j];
                    for (uint32_t pi = tid; pi < n; pi += BM25_THREADS) mask[__ldg(&pp[pi].x) - row0] = 0u;
                }
            }
            reduce();
            __syncthreads();
        } else if (total != 0) {
            // DENSE: scan the slots (4 per thread per step: one LDS.128, owner-aligned with the dense adds)
            scan_pass(false);
            reduce();
            __syncthreads();
            if (s_cnt > p.cap) {   // cold threshold overflowed the candidate buffer: redo chunk by chunk with a compress between chunks
                __syncthreads();
                if (tid == 0) { s_cnt = 0u; s_matched = 0u; s_maxo = f32_ordered(0.f); s_mino = f32_ordered(0.f); }
                __syncthreads();
                scan_pass(true);
                reduce();
                __syncthreads();
            }
        } else {
            __syncthreads();
        }
        // ---- emit: best <= n_keep of the buffer
        const size_t slot_base = (size_t(q) * p.n_tiles + tile);
        uint32_t c = min(s_cnt, p.cap);
        if (c >= p.n_keep && c > 0) {
            block_keep_top(tbuf, c, p.cap, p.n_keep, tid);
            c = p.n_keep;
            if (tid == 0) atomicMax(p.tau + q, (unsigned long long)tbuf[p.n_keep - 1]);
        }
        for (uint32_t i = tid; i < c; i += BM25_THREADS) {
            const uint64_t key = tbuf[i];
            p.cand_key[slot_base * p.n_keep + i] = key;
            p.cand_ft[slot_base * p.n_keep + i] = ft_from_key ? key_score(key) : score[key_idx(key) - row0];
        }
        if (want_bits && tid < BM25_TILE / 32) p.matched_bits[slot_base * (BM25_TILE / 32) + tid] = s_mbits[tid];
        if (!sparse && total != 0) {
            if (!ft_from_key) __syncthreads();             // emit read the scores of other owners' slots
            for (uint32_t i = tid; i < BM25_TILE / 4; i += BM25_THREADS) {   // owner-aligned with the scan: no barrier needed before it
                reinterpret_cast<float4 *>(score)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (THRESH) reinterpret_cast<uint4 *>(mask)[i] = make_uint4(0u, 0u, 0u, 0u);
            }
        }
        if (tid == 0) {
            p.cand_cnt[slot_base] = c;
            p.tile_count[slot_base] = s_matched;
            p.tile_max[slot_base] = f32_unordered(s_maxo);
            p.tile_min[slot_base] = f32_unordered(s_mino);
        }
        if (flat && tid < BM25_FLAT_TOK) store_tok(nx, tid);   // the next item's table (this item no longer reads it)
        if (tid == 0) { s_item_cur = next; s_item_next = next2; }
    }
}

// =======================================================================================
// K3c — the scorer without accumulator arrays (plain queries: no threshold, no OMC, <= BM25_FLAT_TOK tokens,
// every token <= 1 term).  Same contract, outputs and bits as bm25_tile2_kernel<false, false>.
//
// A row's score is the fold of its tokens' contributions in token order.  K3b materialises that fold in a
// float[TILE] array per item: every dense token costs a shared-memory read-modify-write of the whole tile, then a
// scan re-reads it and a zeroing pass clears it.  Here the fold lives in REGISTERS:
//   * rows that appear in some LIST token (few: list tokens are the non-hot terms) are marked in 1 KB bitmaps (one per
//     list token + their union) by a first walk over the postings; after the scan below, a second walk scores them: the
//     posting of the FIRST list token that holds the row folds all tokens in order — a scalar load from each dense
//     token's contribution array (L1-hot: the scan just streamed those slices), and a binary search in another list
//     token's tile slice only where that token's bitmap has the row;
//   * every other row can only receive dense contributions: the scan folds the dense tokens' float4 slices
//     straight from L2 into registers (adding the 0.0 of an absent row changes no bit), masks the rows the union
//     bitmap marks, and does the bookkeeping (count, extrema, gated candidates) on the spot.
// An item without dense tokens costs its postings only; an item without list tokens needs no bitmap and one
// barrier.  No float accumulators, no zeroing passes: ~21 KB of shared memory per CTA (bitmaps + candidate buffer).  When a cold threshold lets more
// than `cap` candidates through, the best n_keep of the first `cap` arrivals give a valid tighter threshold and the
// item is redone with it (first tiles of a query only).
// =======================================================================================
__host__ __device__ inline size_t bm25_tile3_smem_bytes(uint32_t cap) { return size_t(BM25_TILE) / 8 * (BM25_FLAT_TOK + 1) + size_t(cap) * 8 + 64; }

__device__ __forceinline__ void t3_consider(float s, uint32_t row, unsigned long long tau, float tau_f, uint32_t *s_cnt,
                                            uint64_t *tbuf, uint32_t cap) {
    if (!(s >= tau_f)) return;                                          // NaN fails; ties re-checked on the key
    const unsigned long long key = make_key(s, row);
    if (key <= tau) return;
    const uint32_t slot = atomicAdd(s_cnt, 1u);
    if (slot < cap) tbuf[slot] = key;                                   // *s_cnt > cap afterwards == overflow
}
__device__ __forceinline__ bool t3_find(const uint2 *pp, uint32_t n, uint32_t row, uint32_t *payload) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (__ldg(&pp[m].x) < row) lo = m + 1; else hi = m; }
    if (lo < n) { const uint2 r = __ldg(pp + lo); if (r.x == row) { *payload = r.y; return true; } }
    return false;
}
// score of a row that list token j holds (posting `rec`): the item's tokens folded in token order (the reference's
// summation order) — dense tokens by row, other list tokens by binary search where their bitmap has the row
__device__ __noinline__ float t3_fold(const ItemTok *tab, const uint32_t *bm, const uint32_t j, const uint2 rec, const uint32_t l,
                                         const float k, const float kp1) {
    constexpr uint32_t W = BM25_TILE / 32;
    const uint32_t w = l >> 5, bit = 1u << (l & 31u);
    // the dense tokens' contributions, loaded together: one memory latency per row, not one per token (when the scan
    // of the item was skipped, these rows are not in L1)
    // (registers, picked by selects below: the token loop stays rolled, one copy of t3_find)
    static_assert(BM25_FLAT_TOK == 4, "t3_fold holds one dense contribution per flat token");
    auto dense_at = [&](const uint32_t i) {
        return (tab[i].n && (tab[i].flags & TD_DENSE)) ? __ldg(reinterpret_cast<const float *>(tab[i].ptr) + l) : 0.f;
    };
    const float cd0 = dense_at(0), cd1 = dense_at(1), cd2 = dense_at(2), cd3 = dense_at(3);
    float s = 0.f;
#pragma unroll 1
    for (uint32_t i = 0; i < BM25_FLAT_TOK; i++) {
        const uint32_t ni = tab[i].n;
        if (ni == 0) continue;
        const uint32_t fi = tab[i].flags;
        float ci;
        if (fi & TD_DENSE) ci = i == 0 ? cd0 : i == 1 ? cd1 : i == 2 ? cd2 : cd3;   // 0.0 = absent
        else {
            uint32_t pay = rec.y;
            if (i != j) {                              // (another non-empty list token: the per-token bitmaps are in use)
                if (!(bm[i * W + w] & bit)) continue;
                if (!t3_find(reinterpret_cast<const uint2 *>(tab[i].ptr), ni, rec.x, &pay)) continue;
            }
            if (fi & TD_PRE) ci = __uint_as_float(pay);                    // NaN = skipped contribution
            else {
                const float ntf = __fmul_rn(tab[i].w, __uint_as_float(pay));
                ci = f32_is_normal(ntf) ? bm25_sat(ntf, k, kp1, tab[i].idf) : __int_as_float(0x7fc00000);   // bm25.rs:387,501
            }
        }
        if (ci == ci) s = __fadd_rn(s, ci);
    }
    return s;
}
// candidate test of the 4 rows of one float4 slot (rare once the threshold is warm: kept out of line so the scan loop
// stays small — the scorers' code footprint is what the instruction cache sees from 30 unsynchronised warps)
__device__ __noinline__ void t3_consider4(const float s0, const float s1, const float s2, const float s3, const uint32_t row,
                                          const unsigned long long tau, const float tau_f, uint32_t *s_cnt, uint64_t *tbuf, const uint32_t cap) {
    if (s0 != 0.f) t3_consider(s0, row, tau, tau_f, s_cnt, tbuf, cap);
    if (s1 != 0.f) t3_consider(s1, row + 1u, tau, tau_f, s_cnt, tbuf, cap);
    if (s2 != 0.f) t3_consider(s2, row + 2u, tau, tau_f, s_cnt, tbuf, cap);
    if (s3 != 0.f) t3_consider(s3, row + 3u, tau, tau_f, s_cnt, tbuf, cap);
}
__device__ __forceinline__ uint32_t f32_ne0_mask(const float x) {   // 0xffffffff when x != 0 (or NaN), else 0: one FSET
    uint32_t r;
    asm("set.neu.u32.f32 %0, %1, 0f00000000;" : "=r"(r) : "f"(x));
    return r;
}
// the dense part of an item: ND dense tokens (token order); thread t owns the float4 slots t, t + STRIDE, ...
// Software-pipelined: the loads of batch h+1 are in flight while batch h is folded.  `pos`: every contribution of the
// item is >= 0 (weights, idf, k non-negative), so no score is below the fold's start and the minimum stays 0.
template <uint32_t ND, uint32_t STRIDE>
__device__ __forceinline__ void t3_scan(const float4 *d0, const float4 *d1, const float4 *d2, const float4 *d3,
                                        const uint32_t *touched, const bool any_list, const bool pos, const uint32_t row0, const uint32_t tid,
                                        const unsigned long long tau, const float tau_f, uint32_t *s_cnt, uint64_t *tbuf,
                                        const uint32_t cap, uint32_t &matched, float &lmax, float &lmin) {
    constexpr uint32_t F4 = BM25_TILE / 4 / STRIDE;         // float4 slots per thread (8 at 8192 rows x 256 threads, 64 per lane of a warp)
    constexpr uint32_t FB = (ND <= 2 && F4 >= 4) ? 2 : 1;   // slots per batch
    constexpr uint32_t NB = F4 / FB;                        // batches
    static_assert(F4 >= 2 && NB % 2 == 0, "tile size");
    const float4 *dp[4] = {d0, d1, d2, d3};
    const uint32_t *tw = touched + (tid >> 3);              // slot i = tid + j * STRIDE: word (tid >> 3) + j * STRIDE / 8, shift (tid & 7) * 4
    const uint32_t tsh = (tid & 7u) * 4u;
    float4 ca[ND][FB], cb[ND][FB];
    auto load = [&](float4 (&c)[ND][FB], const uint32_t h) {
#pragma unroll
        for (uint32_t u = 0; u < FB; u++)
#pragma unroll
            for (uint32_t d = 0; d < ND; d++) c[d][u] = __ldg(dp[d] + tid + (h * FB + u) * STRIDE);
    };
    auto fold = [&](const float4 (&c)[ND][FB], const uint32_t h) {
#pragma unroll
        for (uint32_t u = 0; u < FB; u++) {
            const uint32_t i = tid + (h * FB + u) * STRIDE;
            float sv[4] = {c[0][u].x, c[0][u].y, c[0][u].z, c[0][u].w};   // 0.0 + c == c for the values stored (never -0.0)
#pragma unroll
            for (uint32_t d = 1; d < ND; d++) {
                sv[0] = __fadd_rn(sv[0], c[d][u].x); sv[1] = __fadd_rn(sv[1], c[d][u].y);
                sv[2] = __fadd_rn(sv[2], c[d][u].z); sv[3] = __fadd_rn(sv[3], c[d][u].w);
            }
            if (any_list) {   // rows scored by a posting walker (4 rows = 4 bits of one bitmap word)
                const uint32_t bits = (tw[(h * FB + u) * (STRIDE / 8)] >> tsh) & 0xfu;
                if (bits) {
#pragma unroll
                    for (int k = 0; k < 4; k++) sv[k] = ((bits >> k) & 1u) ? 0.f : sv[k];
                }
            }
            matched -= f32_ne0_mask(sv[0]) + f32_ne0_mask(sv[1]) + f32_ne0_mask(sv[2]) + f32_ne0_mask(sv[3]);   // -(-1) per non-zero
            const float m4 = fmaxf(fmaxf(sv[0], sv[1]), fmaxf(sv[2], sv[3]));
            lmax = fmaxf(lmax, m4);
            if (!pos) lmin = fminf(lmin, fminf(fminf(sv[0], sv[1]), fminf(sv[2], sv[3])));
            if (m4 >= tau_f) t3_consider4(sv[0], sv[1], sv[2], sv[3], row0 + i * 4u, tau, tau_f, s_cnt, tbuf, cap);
        }
    };
    load(ca, 0);
#pragma unroll 1
    for (uint32_t h = 0; h < NB; h += 2) {
        // the candidate buffer overflowed: the item is redone with a tighter threshold, which recomputes the count and
        // the extrema, and takes its threshold from keys already in the buffer — the rest of this pass changes nothing
        // (a cold threshold overflows after a few hundred rows of an 8192-row scan)
        if (h && *reinterpret_cast<volatile const uint32_t *>(s_cnt) > cap) break;
        load(cb, h + 1);
        fold(ca, h);
        if (h + 2 < NB) load(ca, h + 2);
        fold(cb, h + 1);
    }
}

// Skipping the dense part of an item.  A row that no list token holds scores the fold of its dense tokens'
// contributions in token order, and each contribution is at most its token's tile_bound.  `ub` folds those bounds in
// the same order with the same rounded adds; round-to-nearest addition is monotone, so ub >= the score of every
// dense-only row of the item.  When `pos` holds and ub < tau_f, t3_scan would change nothing but the count:
//   * candidates: every dense-only row fails t3_consider's s >= tau_f, so none is pushed;
//   * count: under `pos` every stored contribution is > 0 (or a zero, which the bitmap leaves clear) and never NaN,
//     so a row's fold is != 0 exactly when one of its bits is set — t3_count counts the same rows the scan would;
//   * maximum: tau only rises, and its final value is attained by n_keep real rows of the query (the seed's rows or
//     a tile's emitted keys; a key's score is exact).  A skipped row is < the tau_f of its item <= the final tau_f, so
//     those rows are never skipped, their tiles' tile_max hold them, and the query's maximum over its tiles' tile_max
//     — all any reader takes from tile_max — is >= the final tau_f > every skipped row;
//   * minimum: lmin stays 0 under `pos`.
// The decision must be the same in every thread of the item: t3_count gives thread t whole bitmap words, t3_scan gives
// it float4 slots, so a mixed decision would count some rows twice and others never.  Hence one threshold per item:
// K3c shares thread 0's load through shared memory, K3d broadcasts lane 0's (other CTAs raise tau[q] meanwhile, so
// separate loads could differ).  With a negative weight, idf or k (`pos` false) the item is always scanned.  K3c / K3d never run with matched_bits or
// row_ft (facets, groups, sortBy), the outputs that would need each row.
__device__ __forceinline__ float t3_dense_ub(const ItemTok *tab) {
    float ub = 0.f;
#pragma unroll
    for (uint32_t j = 0; j < BM25_FLAT_TOK; j++)
        if (tab[j].n && (tab[j].flags & TD_DENSE)) ub = __fadd_rn(ub, __uint_as_float(tab[j].bound));
    return ub;
}
// the count pass that replaces t3_scan: rows outside every list token with some dense contribution, from the dense
// tokens' presence bitmaps (thread t owns the words t, t + STRIDE, ...)
template <uint32_t STRIDE>
__device__ __noinline__ uint32_t t3_count(const ItemTok *tab, const uint32_t *touched, const bool any_list, const uint32_t n_tiles,
                                          const uint32_t tile, const uint32_t tid) {
    constexpr uint32_t W = BM25_TILE / 32;
    const uint32_t *bp[BM25_FLAT_TOK];
#pragma unroll
    for (uint32_t j = 0; j < BM25_FLAT_TOK; j++)
        bp[j] = (tab[j].n && (tab[j].flags & TD_DENSE))
                    ? bm25_dense_bits(reinterpret_cast<const float *>(tab[j].ptr) - size_t(tile) * BM25_TILE, n_tiles) + size_t(tile) * W
                    : nullptr;
    uint32_t m = 0;
#pragma unroll 2
    for (uint32_t w = tid; w < W; w += STRIDE) {
        uint32_t u = 0;
#pragma unroll
        for (uint32_t j = 0; j < BM25_FLAT_TOK; j++) if (bp[j]) u |= __ldg(bp[j] + w);
        if (any_list) u &= ~touched[w];
        m += __popc(u);
    }
    return m;
}

__global__ void __launch_bounds__(BM25_THREADS, 1024 / BM25_THREADS) bm25_tile3_kernel(const Bm25Params p, const ItemTok *flat, unsigned int *work_counter) {
    constexpr uint32_t W = BM25_TILE / 32;                                  // bitmap words per tile
    extern __shared__ __align__(16) uint8_t smem[];
    uint32_t *touched = reinterpret_cast<uint32_t *>(smem);                 // rows that appear in some list token
    uint32_t *bm = touched + W;                                             // [BM25_FLAT_TOK][W]: rows of each list token
    uint64_t *tbuf = reinterpret_cast<uint64_t *>(bm + BM25_FLAT_TOK * W);
    // per-item counters and the token table, double-buffered by item parity (the next item's set is prepared while
    // this one still reads its own)
    __shared__ uint32_t s_cnt2[2], s_matched2[2];
    __shared__ unsigned int s_maxo2[2], s_mino2[2];
    __shared__ ItemTok s_tab[2][BM25_FLAT_TOK];
    __shared__ uint32_t s_item_cur, s_item_next;
    __shared__ uint32_t s_dense[2];                        // dense passes, of which skipped (thread 0 only)
    // the item's running threshold, loaded by thread 0 and double-buffered by item parity: every thread of the CTA
    // gates by the same value, so the dense-skip decision is block-uniform (t3_count and t3_scan split rows differently)
    __shared__ unsigned long long s_tau2[2];

    const uint32_t tid = threadIdx.x;
    const float kp1 = __fadd_rn(p.k, 1.0f);
    const uint32_t n_items = p.n_tiles * p.n_queries;
    const uint32_t *okbits = p.row_ok_bits;

    for (uint32_t i = tid; i < (BM25_FLAT_TOK + 1) * W; i += BM25_THREADS) touched[i] = 0u;
    if (tid == 0) { s_item_cur = atomicAdd(work_counter, 1u); s_item_next = atomicAdd(work_counter, 1u); s_dense[0] = s_dense[1] = 0u; }
    if (tid < 2) { s_cnt2[tid] = 0; s_matched2[tid] = 0; s_maxo2[tid] = f32_ordered(0.f); s_mino2[tid] = f32_ordered(0.f); }
    __syncthreads();
    if (s_item_cur < n_items && tid < BM25_FLAT_TOK) s_tab[0][tid] = flat[size_t(s_item_cur) * BM25_FLAT_TOK + tid];
    unsigned long long tau_next = 0ull;                    // (thread 0)
    if (tid == 0) {
        s_tau2[0] = 0ull;
        if (s_item_cur < n_items) s_tau2[0] = __ldcg(p.tau + s_item_cur % p.n_queries);   // (L2: other CTAs raise it)
    }

    for (uint32_t par = 0;; par ^= 1u) {
        __syncthreads();                                   // previous item retired: bitmaps clean, table + counters + ids set
        const uint32_t item = s_item_cur;
        if (item >= n_items) break;
        const uint32_t next = s_item_next;
        uint32_t next2 = 0;
        if (tid == 0) next2 = atomicAdd(work_counter, 1u);   // consumed at the end of this item
        const uint32_t tile = item / p.n_queries, q = item % p.n_queries;
        const uint32_t row0 = tile * BM25_TILE;
        uint32_t *s_cnt = &s_cnt2[par];
        if (tid == 0) { s_cnt2[par ^ 1u] = 0; s_matched2[par ^ 1u] = 0; s_maxo2[par ^ 1u] = f32_ordered(0.f); s_mino2[par ^ 1u] = f32_ordered(0.f); }
        // in flight during this item: the next item's descriptors and its query's running threshold
        ItemTok nx{};
        if (next < n_items && tid < BM25_FLAT_TOK) nx = flat[size_t(next) * BM25_FLAT_TOK + tid];
        unsigned long long tau = s_tau2[par];
        if (tid == 0 && next < n_items) tau_next = __ldcg(p.tau + next % p.n_queries);

        // the item's tokens: dense slices in token order; list tokens counted
        const ItemTok *tab = s_tab[par];
        const float4 *d0 = nullptr, *d1 = nullptr, *d2 = nullptr, *d3 = nullptr;
        uint32_t nd = 0, n_list = 0;
        bool pos = p.k >= 0.f;
#pragma unroll
        for (uint32_t j = 0; j < BM25_FLAT_TOK; j++) {
            const uint32_t n = tab[j].n;
            if (n == 0) continue;
            pos = pos && tab[j].w >= 0.f && tab[j].idf >= 0.f;
            if (tab[j].flags & TD_DENSE) {
                const float4 *dp = reinterpret_cast<const float4 *>(tab[j].ptr);
                if (nd == 0) d0 = dp; else if (nd == 1) d1 = dp; else if (nd == 2) d2 = dp; else d3 = dp;
                nd++;
            } else n_list++;
        }
        const bool any_list = n_list != 0;
        // per-token bitmaps are needed to find the owner of a row that sits in several list tokens, and they carry the
        // outcome of the filter / tombstone check; one unfiltered list token needs neither
        const bool use_bm = n_list > 1 || okbits != nullptr;

        for (;;) {   // (repeats only when a cold threshold overflowed the candidate buffer)
            const float tau_f = tau ? key_score(tau) : -INFINITY;
            uint32_t matched = 0;
            float lmax = 0.f, lmin = 0.f;
            // ---------------------------------------- mark the rows of the list tokens
            if (any_list && (nd || use_bm)) {
#pragma unroll 1
                for (uint32_t j = 0; j < BM25_FLAT_TOK; j++) {
                    const uint32_t n = tab[j].n;
                    if (n == 0 || (tab[j].flags & TD_DENSE)) continue;     // block-uniform
                    const uint2 *pp = reinterpret_cast<const uint2 *>(tab[j].ptr);
                    for (uint32_t pi = tid; pi < n; pi += BM25_THREADS) {
                        const uint32_t row = __ldg(&pp[pi].x);
                        if (okbits && !((__ldg(okbits + (row >> 5)) >> (row & 31u)) & 1u)) continue;
                        const uint32_t l = row - row0, bit = 1u << (l & 31u);
                        if (nd) atomicOr(&touched[l >> 5], bit);
                        if (use_bm) atomicOr(&bm[j * W + (l >> 5)], bit);
                    }
                }
                __syncthreads();
            }
            // ---------------------------------------- rows outside every list: dense tokens only, folded in registers
            // (or only counted, when no such row can reach the threshold)
            const bool skip = nd && pos && t3_dense_ub(tab) < tau_f;
            if (nd && tid == 0) { s_dense[0]++; s_dense[1] += skip; }
            if (skip) matched += t3_count<BM25_THREADS>(tab, touched, any_list, p.n_tiles, tile, tid);
            else switch (nd) {
                case 0: break;
                case 1: t3_scan<1, BM25_THREADS>(d0, d1, d2, d3, touched, any_list, pos, row0, tid, tau, tau_f, s_cnt, tbuf, p.cap, matched, lmax, lmin); break;
                case 2: t3_scan<2, BM25_THREADS>(d0, d1, d2, d3, touched, any_list, pos, row0, tid, tau, tau_f, s_cnt, tbuf, p.cap, matched, lmax, lmin); break;
                case 3: t3_scan<3, BM25_THREADS>(d0, d1, d2, d3, touched, any_list, pos, row0, tid, tau, tau_f, s_cnt, tbuf, p.cap, matched, lmax, lmin); break;
                default: t3_scan<4, BM25_THREADS>(d0, d1, d2, d3, touched, any_list, pos, row0, tid, tau, tau_f, s_cnt, tbuf, p.cap, matched, lmax, lmin); break;
            }
            // ---------------------------------------- rows of the list tokens: the FIRST list token holding the row folds
            // it (the scan just pulled the dense slices through L1; other lists are consulted only where their bit is set)
            if (any_list) {
#pragma unroll 1
                for (uint32_t j = 0; j < BM25_FLAT_TOK; j++) {
                    const uint32_t n = tab[j].n;
                    if (n == 0 || (tab[j].flags & TD_DENSE)) continue;
                    const uint2 *pp = reinterpret_cast<const uint2 *>(tab[j].ptr);
                    for (uint32_t pi = tid; pi < n; pi += BM25_THREADS) {
                        const uint2 rec = __ldg(pp + pi);
                        const uint32_t l = rec.x - row0, w = l >> 5, bit = 1u << (l & 31u);
                        if (use_bm) {
                            if (!(bm[j * W + w] & bit)) continue;          // failed the row check
                            uint32_t earlier = 0;
                            for (uint32_t jj = 0; jj < j; jj++) earlier |= bm[jj * W + w];   // (all-zero for dense / empty tokens)
                            if (earlier & bit) continue;                   // an earlier list token owns the row
                        }
                        const float s = t3_fold(tab, bm, j, rec, l, p.k, kp1);
                        if (s != 0.f) {
                            matched++;
                            lmax = fmaxf(lmax, s);
                            lmin = fminf(lmin, s);
                            t3_consider(s, rec.x, tau, tau_f, s_cnt, tbuf, p.cap);
                        }
                    }
                }
            }
            // block reductions of count / extrema
            matched = __reduce_add_sync(0xffffffffu, matched);
            if (matched) {   // (warp-uniform)
                for (int o = 16; o > 0; o >>= 1) {
                    lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
                    lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
                }
                if ((tid & 31) == 0) {
                    atomicAdd(&s_matched2[par], matched);
                    atomicMax(&s_maxo2[par], f32_ordered(lmax));
                    atomicMin(&s_mino2[par], f32_ordered(lmin));
                }
            }
            __syncthreads();                                   // counters final; nobody reads the bitmaps any more
            if (any_list) {
                if (nd) for (uint32_t i = tid; i < W; i += BM25_THREADS) touched[i] = 0u;
                if (use_bm) for (uint32_t i = tid; i < BM25_FLAT_TOK * W; i += BM25_THREADS) bm[i] = 0u;
            }
            if (*s_cnt <= p.cap) break;
            // overflow: the n_keep-th best of the first `cap` arrivals bounds the tile's n_keep-th best from below
            block_keep_top(tbuf, p.cap, p.cap, p.n_keep, tid);
            const unsigned long long kth = tbuf[p.n_keep - 1] - 1ull;   // keys are unique: "> kth" keeps that row itself
            tau = kth > tau ? kth : tau;
            __syncthreads();                                   // everybody has read tbuf / the counters
            if (tid == 0) { s_cnt2[par] = 0; s_matched2[par] = 0; s_maxo2[par] = f32_ordered(0.f); s_mino2[par] = f32_ordered(0.f); }
            __syncthreads();
        }
        // ---- emit: best <= n_keep of the buffer
        const size_t slot_base = (size_t(q) * p.n_tiles + tile);
        uint32_t c = *s_cnt;
        if (c >= p.n_keep && c > 0) {
            block_keep_top(tbuf, c, p.cap, p.n_keep, tid);
            c = p.n_keep;
            if (tid == 0) atomicMax(p.tau + q, (unsigned long long)tbuf[p.n_keep - 1]);
        }
        for (uint32_t i = tid; i < c; i += BM25_THREADS) {
            const uint64_t key = tbuf[i];
            p.cand_key[slot_base * p.n_keep + i] = key;
            p.cand_ft[slot_base * p.n_keep + i] = key_score(key);   // no OMC, no min hint: the key's score IS the raw score
        }
        if (tid == 0) {
            p.cand_cnt[slot_base] = c;
            p.tile_count[slot_base] = s_matched2[par];
            p.tile_max[slot_base] = f32_unordered(s_maxo2[par]);
            p.tile_min[slot_base] = f32_unordered(s_mino2[par]);
        }
        if (tid < BM25_FLAT_TOK) s_tab[par ^ 1u][tid] = nx;   // the next item's table
        if (tid == 0) { s_item_cur = next; s_item_next = next2; s_tau2[par ^ 1u] = tau_next; }
    }
    if (tid == 0 && p.dense_stat && s_dense[0]) { atomicAdd(p.dense_stat, s_dense[0]); atomicAdd(p.dense_stat + 1, s_dense[1]); }
}

// =======================================================================================
// K3d — the same scorer with a WARP per (tile, query) item instead of a CTA: no block barrier anywhere, the per-item
// fixed work (descriptors, reductions, selection, emit) is executed by one warp instead of eight, and 30 warps per
// SM progress independently (an item's latency chain stalls only its own warp).  Plain queries with n_keep <= 32.
// Per warp: the ownership bitmaps (5 KB), 256 candidate keys, the token table.
// =======================================================================================
constexpr uint32_t BW_WARPS = 6, BW_CAP = 256;
struct __align__(16) WarpScratch {
    uint32_t touched[BM25_TILE / 32];
    uint32_t bm[BM25_FLAT_TOK * (BM25_TILE / 32)];
    uint64_t tbuf[BW_CAP];
    ItemTok tab[BM25_FLAT_TOK];
    uint32_t cnt, dense_items, dense_skipped, pad;   // (lane 0: dense passes, of which skipped)
};
// the n largest of buf[0, count) (count <= BW_CAP, n <= 32), descending, into buf[0, n); returns the n-th (0 if count < n)
__device__ __noinline__ unsigned long long warp_keep_top(uint64_t *buf, const uint32_t count, const uint32_t n, const uint32_t lane) {
    constexpr uint32_t PER = BW_CAP / 32;
    unsigned long long k[PER];
#pragma unroll
    for (uint32_t u = 0; u < PER; u++) k[u] = lane + 32u * u < count ? buf[lane + 32u * u] : 0ull;
    __syncwarp();
    unsigned long long mine = 0ull, last = 0ull;
    for (uint32_t r = 0; r < n; r++) {
        unsigned long long m = k[0];
#pragma unroll
        for (uint32_t u = 1; u < PER; u++) m = k[u] > m ? k[u] : m;
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long om = __shfl_xor_sync(0xffffffffu, m, o);
            m = om > m ? om : m;
        }
        last = m;
        if (m == 0ull) break;
        if (lane == r) mine = m;
#pragma unroll
        for (uint32_t u = 0; u < PER; u++) if (k[u] == m) k[u] = 0ull;   // keys are unique
    }
    if (lane < n) buf[lane] = mine;
    __syncwarp();
    return last;
}
// Phase profile of K3d (OC_BM25_PHASE_PROFILE, defined only by `make phaseprof`, which builds a separate library for
// tools/profile_k3d.py): lane 0 of each warp appends one BwProfItem per item and one BwProfWarp per warp.  The spans
// are clock64 deltas (per SM clock), the warp times %globaltimer (ns, comparable across SMs).
enum { BWP_DESC, BWP_MARK, BWP_DENSE, BWP_FOLD, BWP_CLEAR, BWP_KEEP, BWP_EMIT, BWP_N };
struct BwProfItem {
    uint32_t item, cls;      // cls: nd | n_list << 4 | skip << 8 | passes << 12 (1 + threshold redos)
    uint32_t postings, cand; // list postings in the tile (all list tokens), candidates pushed (last pass)
    uint32_t span[BWP_N];    // cycles per phase
    uint32_t smid;
};
struct BwProfWarp { unsigned long long t0, t1, c0, c1; uint32_t smid, items, pad[2]; };
struct BwProf { BwProfItem *items; BwProfWarp *warps; unsigned int *n_items, *n_warps; uint32_t cap_items, cap_warps; };
#ifdef OC_BM25_PHASE_PROFILE
__device__ BwProf g_bw_prof;
__device__ __forceinline__ unsigned long long bw_gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ uint32_t bw_smid() { uint32_t s; asm volatile("mov.u32 %0, %%smid;" : "=r"(s)); return s; }
#define BW_PROF(...) __VA_ARGS__
#define BW_LAP(ph) do { const long long t_ = clock64(); pspan[ph] += uint32_t(t_ - pclk); pclk = t_; } while (0)
#else
#define BW_PROF(...)
#define BW_LAP(ph) do { } while (0)
#endif
__global__ void __launch_bounds__(BW_WARPS * 32, 5) bm25_warp_kernel(const Bm25Params p, const ItemTok *flat, unsigned int *work_counter) {
    constexpr uint32_t W = BM25_TILE / 32;
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t lane = threadIdx.x & 31u;
    WarpScratch &ws = reinterpret_cast<WarpScratch *>(smem)[threadIdx.x >> 5];
    uint32_t *touched = ws.touched, *bm = ws.bm;
    const ItemTok *tab = ws.tab;
    const float kp1 = __fadd_rn(p.k, 1.0f);
    const uint32_t n_items = p.n_tiles * p.n_queries;
    const uint32_t *okbits = p.row_ok_bits;

    for (uint32_t i = lane; i < W; i += 32) touched[i] = 0u;
    for (uint32_t i = lane; i < BM25_FLAT_TOK * W; i += 32) bm[i] = 0u;
    if (lane == 0) { ws.cnt = 0u; ws.dense_items = 0u; ws.dense_skipped = 0u; }
    uint32_t item = 0, next = 0;
    if (lane == 0) { item = atomicAdd(work_counter, 1u); next = atomicAdd(work_counter, 1u); }
    item = __shfl_sync(0xffffffffu, item, 0); next = __shfl_sync(0xffffffffu, next, 0);
    ItemTok cur{};
    if (item < n_items && lane < BM25_FLAT_TOK) cur = flat[size_t(item) * BM25_FLAT_TOK + lane];
    unsigned long long tau_next = 0ull;
    if (item < n_items) tau_next = __ldcg(p.tau + item % p.n_queries);
    BW_PROF(const unsigned long long prof_t0 = bw_gtime(), prof_c0 = clock64(); uint32_t prof_items = 0;)

    while (item < n_items) {
        BW_PROF(uint32_t pspan[BWP_N] = {}; long long pclk = clock64(); uint32_t prof_passes = 0, prof_skip = 0, prof_post = 0;)
        uint32_t next2 = 0;
        if (lane == 0) next2 = atomicAdd(work_counter, 1u);   // consumed at the end of this item
        const uint32_t tile = item / p.n_queries, q = item % p.n_queries;
        const uint32_t row0 = tile * BM25_TILE;
        if (lane < BM25_FLAT_TOK) ws.tab[lane] = cur;
        ItemTok nx{};
        if (next < n_items && lane < BM25_FLAT_TOK) nx = flat[size_t(next) * BM25_FLAT_TOK + lane];
        // lane 0's value for every lane: the dense-skip decision must be warp-uniform (t3_count and t3_scan split rows
        // differently), whatever each lane's load returned
        unsigned long long tau = __shfl_sync(0xffffffffu, tau_next, 0);
        if (next < n_items) tau_next = __ldcg(p.tau + next % p.n_queries);
        __syncwarp();

        const float4 *d0 = nullptr, *d1 = nullptr, *d2 = nullptr, *d3 = nullptr;
        uint32_t nd = 0, n_list = 0;
        bool pos = p.k >= 0.f;
#pragma unroll
        for (uint32_t j = 0; j < BM25_FLAT_TOK; j++) {
            const uint32_t n = tab[j].n;
            if (n == 0) continue;
            pos = pos && tab[j].w >= 0.f && tab[j].idf >= 0.f;
            if (tab[j].flags & TD_DENSE) {
                const float4 *dp = reinterpret_cast<const float4 *>(tab[j].ptr);
                if (nd == 0) d0 = dp; else if (nd == 1) d1 = dp; else if (nd == 2) d2 = dp; else d3 = dp;
                nd++;
            } else { n_list++; BW_PROF(prof_post += n;) }
        }
        const bool any_list = n_list != 0;
        const bool use_bm = n_list > 1 || okbits != nullptr;
        uint32_t matched;
        float lmax, lmin;
        BW_LAP(BWP_DESC);
        for (;;) {   // (repeats only when a cold threshold overflowed the candidate buffer)
            const float tau_f = tau ? key_score(tau) : -INFINITY;
            matched = 0; lmax = 0.f; lmin = 0.f;
            BW_PROF(prof_passes++;)
            if (any_list && (nd || use_bm)) {   // mark the rows of the list tokens
#pragma unroll 1
                for (uint32_t j = 0; j < BM25_FLAT_TOK; j++) {
                    const uint32_t n = tab[j].n;
                    if (n == 0 || (tab[j].flags & TD_DENSE)) continue;
                    const uint2 *pp = reinterpret_cast<const uint2 *>(tab[j].ptr);
                    for (uint32_t pi = lane; pi < n; pi += 32) {
                        const uint32_t row = __ldg(&pp[pi].x);
                        if (okbits && !((__ldg(okbits + (row >> 5)) >> (row & 31u)) & 1u)) continue;
                        const uint32_t l = row - row0, bit = 1u << (l & 31u);
                        if (nd) atomicOr(&touched[l >> 5], bit);
                        if (use_bm) atomicOr(&bm[j * W + (l >> 5)], bit);
                    }
                }
                __syncwarp();
            }
            BW_LAP(BWP_MARK);
            // rows outside every list: dense tokens only, folded in registers (or only counted: see t3_count)
            const bool skip = nd && pos && t3_dense_ub(tab) < tau_f;
            if (nd && lane == 0) { ws.dense_items++; ws.dense_skipped += skip; }
            BW_PROF(prof_skip = skip;)
            if (skip) matched += t3_count<32>(tab, touched, any_list, p.n_tiles, tile, lane);
            else switch (nd) {
                case 0: break;
                case 1: t3_scan<1, 32>(d0, d1, d2, d3, touched, any_list, pos, row0, lane, tau, tau_f, &ws.cnt, ws.tbuf, BW_CAP, matched, lmax, lmin); break;
                case 2: t3_scan<2, 32>(d0, d1, d2, d3, touched, any_list, pos, row0, lane, tau, tau_f, &ws.cnt, ws.tbuf, BW_CAP, matched, lmax, lmin); break;
                case 3: t3_scan<3, 32>(d0, d1, d2, d3, touched, any_list, pos, row0, lane, tau, tau_f, &ws.cnt, ws.tbuf, BW_CAP, matched, lmax, lmin); break;
                default: t3_scan<4, 32>(d0, d1, d2, d3, touched, any_list, pos, row0, lane, tau, tau_f, &ws.cnt, ws.tbuf, BW_CAP, matched, lmax, lmin); break;
            }
            BW_LAP(BWP_DENSE);
            if (any_list) {   // rows of the list tokens: the first list token holding the row folds it
#pragma unroll 1
                for (uint32_t j = 0; j < BM25_FLAT_TOK; j++) {
                    const uint32_t n = tab[j].n;
                    if (n == 0 || (tab[j].flags & TD_DENSE)) continue;
                    const uint2 *pp = reinterpret_cast<const uint2 *>(tab[j].ptr);
                    for (uint32_t pi = lane; pi < n; pi += 32) {
                        const uint2 rec = __ldg(pp + pi);
                        const uint32_t l = rec.x - row0, w = l >> 5, bit = 1u << (l & 31u);
                        if (use_bm) {
                            if (!(bm[j * W + w] & bit)) continue;          // failed the row check
                            uint32_t earlier = 0;
                            for (uint32_t jj = 0; jj < j; jj++) earlier |= bm[jj * W + w];
                            if (earlier & bit) continue;                   // an earlier list token owns the row
                        }
                        const float s = t3_fold(tab, bm, j, rec, l, p.k, kp1);
                        if (s != 0.f) {
                            matched++;
                            lmax = fmaxf(lmax, s);
                            lmin = fminf(lmin, s);
                            t3_consider(s, rec.x, tau, tau_f, &ws.cnt, ws.tbuf, BW_CAP);
                        }
                    }
                }
            }
            __syncwarp();                                      // candidate pushes and bitmap reads of all lanes are done
            BW_LAP(BWP_FOLD);
            if (any_list) {
                if (nd) for (uint32_t i = lane; i < W; i += 32) touched[i] = 0u;
                if (use_bm) for (uint32_t i = lane; i < BM25_FLAT_TOK * W; i += 32) bm[i] = 0u;
            }
            BW_LAP(BWP_CLEAR);
            if (ws.cnt <= BW_CAP) break;
            // overflow: the n_keep-th best of the first BW_CAP arrivals bounds the tile's n_keep-th best from below
            const unsigned long long kth = warp_keep_top(ws.tbuf, BW_CAP, p.n_keep, lane) - 1ull;   // "> kth" keeps that row itself
            tau = kth > tau ? kth : tau;
            if (lane == 0) ws.cnt = 0u;
            __syncwarp();
            BW_LAP(BWP_KEEP);
        }
        matched = __reduce_add_sync(0xffffffffu, matched);
        for (int o = 16; o > 0; o >>= 1) {
            lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
            lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
        }
        // ---- emit: best <= n_keep of the buffer
        const size_t slot_base = (size_t(q) * p.n_tiles + tile);
        uint32_t c = ws.cnt;
        BW_PROF(const uint32_t prof_cand = c;)
        BW_LAP(BWP_EMIT);
        if (c >= p.n_keep && c > 0) {
            const unsigned long long kth = warp_keep_top(ws.tbuf, c, p.n_keep, lane);
            c = p.n_keep;
            if (lane == 0) atomicMax(p.tau + q, kth);
        }
        BW_LAP(BWP_KEEP);
        for (uint32_t i = lane; i < c; i += 32) {
            const uint64_t key = ws.tbuf[i];
            p.cand_key[slot_base * p.n_keep + i] = key;
            p.cand_ft[slot_base * p.n_keep + i] = key_score(key);
        }
        __syncwarp();
        if (lane == 0) {
            p.cand_cnt[slot_base] = c;
            p.tile_count[slot_base] = matched;
            p.tile_max[slot_base] = lmax;
            p.tile_min[slot_base] = lmin;
            ws.cnt = 0u;
        }
        // the next item's descriptors arrived during this one: pull the head of each of its posting ranges / dense slices
        // towards L1 so its first dependent loads do not pay the L2 round trip
        if (lane < BM25_FLAT_TOK && nx.n) {
            const char *pf = reinterpret_cast<const char *>(nx.ptr);
            const uint32_t bytes = (nx.flags & TD_DENSE) ? 1024u : min(nx.n * 8u, 1024u);
            for (uint32_t o = 0; o < bytes; o += 128u) asm volatile("prefetch.global.L1 [%0];" ::"l"(pf + o));
        }
        BW_LAP(BWP_EMIT);
        BW_PROF(if (lane == 0 && g_bw_prof.n_items) {   // (no buffers set: nothing recorded)
            const BwProf &g = g_bw_prof;
            const uint32_t s = atomicAdd(g.n_items, 1u);
            if (s < g.cap_items) {
                BwProfItem &r = g.items[s];
                r.item = item; r.cls = nd | n_list << 4 | prof_skip << 8 | prof_passes << 12;
                r.postings = prof_post; r.cand = prof_cand; r.smid = bw_smid();
                for (int ph = 0; ph < BWP_N; ph++) r.span[ph] = pspan[ph];
            }
            prof_items++;
        })
        cur = nx;
        item = next;
        next = __shfl_sync(0xffffffffu, next2, 0);
        __syncwarp();
    }
    if (lane == 0 && p.dense_stat && ws.dense_items) { atomicAdd(p.dense_stat, ws.dense_items); atomicAdd(p.dense_stat + 1, ws.dense_skipped); }
    BW_PROF(if (lane == 0 && g_bw_prof.n_warps) {
        const BwProf &g = g_bw_prof;
        const uint32_t s = atomicAdd(g.n_warps, 1u);
        if (s < g.cap_warps) {
            BwProfWarp &r = g.warps[s];
            r.t0 = prof_t0; r.t1 = bw_gtime(); r.c0 = prof_c0; r.c1 = clock64(); r.smid = bw_smid(); r.items = prof_items;
        }
    })
}

// ---------------------------------------------------------------------------------------
// Hybrid: the fulltext score of each vector hit's document (token_score.rs:416-419 needs it for the <= limit
// documents of the vector map), by POINT lookups instead of a pass inside the tile scorer: one warp per
// (query, hit), lane i evaluates token i — binary search of the row in each of the token's posting lists, the
// same rounded ops and the same term / token order as the tile kernels — and lane 0 adds the token
// contributions in order, so the value is bit-identical to what the tile accumulators held.
// ---------------------------------------------------------------------------------------
struct PointParams {
    const TermDesc *terms; const TokenDesc *tokens; const QueryDesc *queries;
    uint32_t n_queries, v_stride;
    const uint32_t *v_row;        // [q][v_stride] string row of each vector hit, 0xffffffff = none
    const uint32_t *row_ok_bits;  // NULL or bitmap over rows
    float k;
    int threshold;
    float *v_ft; uint8_t *v_present;
    const uint32_t *q_ok_slot;    // NULL, or [n_queries] slot of each query in row_ok_bits (per-query where-filters)
    uint64_t ok_words;
};
__device__ __forceinline__ bool posting_find(const TermDesc &td, uint32_t row, uint32_t *payload) {
    const uint2 *pp = reinterpret_cast<const uint2 *>(td.ptr);
    uint32_t lo = 0, hi = td.len;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (__ldg(&pp[m].x) < row) lo = m + 1; else hi = m; }
    if (lo < td.len) { const uint2 r = __ldg(pp + lo); if (r.x == row) { *payload = r.y; return true; } }
    return false;
}
__global__ void __launch_bounds__(256) bm25_point_kernel(const PointParams p) {
    const uint32_t wid = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
    if (wid >= p.n_queries * p.v_stride) return;
    const uint32_t q = wid / p.v_stride;
    const uint32_t r = p.v_row[wid];
    const QueryDesc qd = p.queries[q];
    const float kp1 = __fadd_rn(p.k, 1.0f);
    float score = 0.f;
    uint32_t mask = 0;
    bool ok = r != 0xffffffffu;
    if (ok && p.row_ok_bits) ok = (row_ok_of(p.row_ok_bits, p.q_ok_slot, p.ok_words, q)[r >> 5] >> (r & 31)) & 1u;
    if (ok) {
        for (uint32_t t0 = qd.token_begin; t0 < qd.token_end; t0 += 32) {
            const uint32_t ti = t0 + lane;
            float c = __int_as_float(0x7fc00000);
            uint32_t bit = 0;
            if (ti < qd.token_end) {
                const TokenDesc tk = p.tokens[ti];
                bit = tk.bit;
                const uint32_t nt = tk.term_end - tk.term_begin;
                if (nt == 1) {
                    const TermDesc td = p.terms[tk.term_begin];
                    uint32_t pay;
                    if (td.flags & TD_DENSE) {
                        const float cd = reinterpret_cast<const float *>(td.ptr)[r];
                        if (cd != 0.f) c = cd;
                    } else if (posting_find(td, r, &pay)) {
                        if (td.flags & 1u) c = __uint_as_float(pay);
                        else {
                            const float ntf = __fmul_rn(td.weight, __uint_as_float(pay));
                            if (f32_is_normal(ntf)) c = bm25_sat(ntf, p.k, kp1, tk.idf);
                        }
                    }
                } else if (nt > 1) {
                    float S = 0.f;   // S += weight(1.0) * ntf in term order (token_score.rs:266-271)
                    for (uint32_t e = tk.term_begin; e < tk.term_end; e++) {
                        const TermDesc td = p.terms[e];
                        uint32_t pay;
                        if (posting_find(td, r, &pay)) S = __fadd_rn(S, __fmul_rn(td.weight, __uint_as_float(pay)));
                    }
                    if (f32_is_normal(S)) c = bm25_sat(S, p.k, kp1, tk.idf);
                }
            }
            const uint32_t nhere = min(32u, qd.token_end - t0);
            for (uint32_t i = 0; i < nhere; i++) {      // token order
                const float ci = __shfl_sync(0xffffffffu, c, i);
                const uint32_t bi = __shfl_sync(0xffffffffu, bit, i);
                if (ci == ci) { score = __fadd_rn(score, ci); mask |= bi; }
            }
        }
    }
    if (lane == 0) {
        // the query's own threshold mode (a batch with per-query parameters mixes queries with and without one)
        const bool thr = p.threshold && (qd.flags & QF_THRESHOLD);
        const bool present = ok && (thr ? (mask != 0u && uint32_t(__popc(mask)) >= qd.required) : score != 0.f);
        p.v_ft[wid] = present ? score : 0.f;
        p.v_present[wid] = present ? 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------
// Warm start of the per-query candidate threshold (plain queries, n_keep <= 32): the tile scorers gate candidates by
// tau[q], which the first tiles of a query would otherwise have to discover themselves (every matched row of those
// tiles passes a cold threshold).  One warp per query scores the first 64 documents of the query's RAREST list
// token exactly (the fold of bm25_tile3_kernel: dense arrays by row, other lists by binary search) — documents that
// hold the rarest term are where the top of the ranking lives — and publishes (n_keep-th best key) - 1: n_keep real
// rows reach it, so it is a valid lower bound of the final n_keep-th best and pruning by it cannot change a result.
// ---------------------------------------------------------------------------------------
constexpr uint32_t SEED_PER_LANE = 2, SEED_MAX_PER_LANE = 8;
__global__ void __launch_bounds__(256) bm25_seed_kernel(const Bm25Params p) {
    const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (q >= p.n_queries) return;
    const QueryDesc qd = p.queries[q];
    const uint32_t ntok = qd.token_end - qd.token_begin;
    if (ntok == 0 || ntok > BM25_FLAT_TOK || p.n_keep > 32) return;
    const float kp1 = __fadd_rn(p.k, 1.0f);
    uint32_t best = 0xffffffffu, best_len = 0xffffffffu;
    for (uint32_t j = 0; j < ntok; j++) {
        const TokenDesc tk = p.tokens[qd.token_begin + j];
        if (tk.term_end - tk.term_begin != 1) continue;
        const TermDesc td = p.terms[tk.term_begin];
        if (!(td.flags & TD_DENSE) && td.len >= p.n_keep && td.len < best_len) { best = j; best_len = td.len; }
    }
    // no list token with n_keep postings (every token hot or very rare): score the first 256 rows of the store instead — a
    // weaker bound, but enough to stop the first tiles from pushing every matched row
    const bool fallback = best == 0xffffffffu;                             // (warp-uniform)
    if (fallback && p.n_rows < 32u * SEED_MAX_PER_LANE) return;
    const uint32_t per = fallback ? SEED_MAX_PER_LANE : SEED_PER_LANE;
    const uint2 *pb = fallback ? nullptr : reinterpret_cast<const uint2 *>(p.terms[p.tokens[qd.token_begin + best].term_begin].ptr);
    unsigned long long keys[SEED_MAX_PER_LANE];
#pragma unroll
    for (uint32_t u = 0; u < SEED_MAX_PER_LANE; u++) {
        keys[u] = 0ull;
        if (u >= per) continue;
        const uint32_t pi = lane + 32u * u;
        uint2 rec = make_uint2(pi, 0u);                                    // fallback: row pi
        if (!fallback) {
            if (pi >= best_len) continue;
            rec = __ldg(pb + pi);
        }
        if (p.row_ok_bits && !((__ldg(p.row_ok_bits + (rec.x >> 5)) >> (rec.x & 31u)) & 1u)) continue;
        float s = 0.f;
        for (uint32_t i = 0; i < ntok; i++) {                              // token order
            const TokenDesc tk = p.tokens[qd.token_begin + i];
            if (tk.term_end - tk.term_begin != 1) continue;
            const TermDesc td = p.terms[tk.term_begin];
            float ci;
            if (td.flags & TD_DENSE) ci = __ldg(reinterpret_cast<const float *>(td.ptr) + rec.x);
            else {
                uint32_t pay = rec.y;
                if (i != best && !posting_find(td, rec.x, &pay)) continue;
                if (td.flags & TD_PRE) ci = __uint_as_float(pay);
                else {
                    const float ntf = __fmul_rn(td.weight, __uint_as_float(pay));
                    ci = f32_is_normal(ntf) ? bm25_sat(ntf, p.k, kp1, tk.idf) : __int_as_float(0x7fc00000);
                }
            }
            if (ci == ci) s = __fadd_rn(s, ci);
        }
        if (s != 0.f && s == s) keys[u] = make_key(s, rec.x);
    }
    unsigned long long kth = 0ull;
    for (uint32_t r = 0; r < p.n_keep; r++) {
        unsigned long long m = keys[0];
#pragma unroll
        for (uint32_t u = 1; u < SEED_MAX_PER_LANE; u++) m = keys[u] > m ? keys[u] : m;
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long om = __shfl_xor_sync(0xffffffffu, m, o);
            m = om > m ? om : m;
        }
        kth = m;
        if (m == 0ull) break;                                              // fewer than n_keep scored rows: no seed
#pragma unroll
        for (uint32_t u = 0; u < SEED_MAX_PER_LANE; u++) if (keys[u] == m) keys[u] = 0ull;   // keys are unique (row index)
    }
    if (lane == 0 && kth > 1ull) p.tau[q] = kth - 1ull;                    // "> tau" keeps the kth row itself
}

}  // namespace oc
