// emb_scan.cuh — K1: exact cosine top-k sweep over the device-resident embedding matrix.
//
// Replaces the external oramacore_fields::embedding::EmbeddingStorage::search call made by
// EmbeddingFieldStorage::search (read/index/embedding_field.rs:250-266) and fuses the
// post-processing of :268-276 (1 - d, rescale_score, >= similarity) into the merge.
//
// Roofline: HBM.  Algorithmic bytes per sweep = n_rows * stride * 4 (+ n_rows * 4 for the
// inverse norms); one sweep serves QB (<= 4) queries.  Layout: row-major [n_rows][stride]
// fp32, stride = dim rounded up to 128 floats (zero padded) so every lane owns whole
// 16-byte vectors; inv_norm[n_rows] fp32 (NaN = tombstoned / filtered-out row).
//
// Structure (persistent, one CTA per SM): a dedicated producer warp streams R-row tiles
// into an S-stage shared-memory ring with 1-D bulk async copies (TMA engine, mbarrier
// complete_tx); 8 consumer warps each take whole rows from the ring: lane l reads
// float4 #(l + 32 j) (conflict-free LDS.128), FMAs against the query held in registers,
// warp-shuffle reduction, then a threshold-gated insert into a warp-private top-k buffer
// (bitonic compress when full).  The 8 warp lists are merged per CTA at the end; a second
// tiny kernel merges the per-CTA lists and applies rescale / similarity.
#pragma once
#include "oc_common.cuh"

namespace oc {

constexpr int SCAN_CONSUMER_WARPS = 8;
constexpr int SCAN_THREADS = (SCAN_CONSUMER_WARPS + 1) * 32;  // + producer warp

struct ScanParams {
    const void *rows;         // [n_rows][stride] fp32 or bf16 (OC_DTYPE_*)
    const float *inv_norm;    // [n_rows] (NaN => skip row)
    uint64_t n_rows;
    uint32_t stride;          // floats, multiple of 128
    const float *queries;     // [nq][stride] zero padded
    const float *inv_qnorm;   // [nq]
    uint32_t n_keep;          // candidates kept per CTA per query (= limit)
    uint32_t wcap;            // warp buffer capacity, pow2 >= 2*n_keep, >= 32
    uint32_t rows_per_stage;  // multiple of 8
    uint32_t n_stages;
    uint32_t n_ctas_total;    // candidate slots per query (>= gridDim.x)
    uint64_t *cand;           // [nq][n_ctas_total][n_keep] keys, KEY_NONE padded
    // per-query where-filters (oc_search_params.q_filters): NULL, or [n_slots][row_words] row bitmaps; query q passes
    // row r when q_slot[q] == SLOT_NONE or bit r of slot q_slot[q] is set
    const uint32_t *row_bits;
    uint64_t row_words;
    const uint32_t *q_slot;   // [nq]
};
constexpr uint32_t SLOT_NONE = 0xffffffffu;
__device__ __forceinline__ bool slot_row_ok(const uint32_t *row_bits, uint64_t row_words, uint32_t slot, uint64_t row) {
    return slot == SLOT_NONE || ((__ldg(row_bits + size_t(slot) * row_words + (row >> 5)) >> (row & 31)) & 1u);
}

__host__ __device__ inline size_t scan_smem_bytes(uint32_t stride, uint32_t rows_per_stage,
                                                  uint32_t n_stages, uint32_t wcap, uint32_t qb, uint32_t esz = 4) {
    size_t b = size_t(n_stages) * rows_per_stage * stride * esz;    // row ring
    b += size_t(n_stages) * rows_per_stage * 4;                     // inverse-norm ring
    b += size_t(n_stages) * 2 * 8;                                  // full/empty mbarriers
    b += size_t(SCAN_CONSUMER_WARPS) * qb * wcap * 8;               // warp top-k buffers
    return b + 128;
}

// 4 consecutive elements of a row as fp32: fp32 rows -> one LDS/LDG.128; bf16 rows -> one 8-byte load,
// widened exactly (bf16 -> fp32 is a 16-bit shift).
template <typename T> struct RowLoad;
template <> struct RowLoad<float> {
    static constexpr uint32_t ESZ = 4;
    __device__ static __forceinline__ float4 ld(const void *row, uint32_t chunk) {
        return reinterpret_cast<const float4 *>(row)[chunk];
    }
};
struct bf16_t { uint16_t v; };
template <> struct RowLoad<bf16_t> {
    static constexpr uint32_t ESZ = 2;
    __device__ static __forceinline__ float4 ld(const void *row, uint32_t chunk) {
        const uint2 r = reinterpret_cast<const uint2 *>(row)[chunk];
        return make_float4(__uint_as_float(r.x << 16), __uint_as_float(r.x & 0xffff0000u),
                           __uint_as_float(r.y << 16), __uint_as_float(r.y & 0xffff0000u));
    }
};

// Rank key of a row: -(cosine distance), distance = 1 - cos (embedding_field.rs:246-249), cos = dot * inv|x| * inv|q|.
// The multiply by inv|q| is fused with the subtraction.  Spelled out so that every kernel that scores a row (K1 at
// every QB, the K2 re-score) rounds identically: left to the compiler, the contraction depended on the surrounding
// code, and K1 with QB = 1 scored the same row a few ulp apart from QB = 2 / 4 and from K2.
__device__ __forceinline__ float cos_rank_key(float dot, float inr, float iqn) {
    return -fmaf(-__fmul_rn(dot, inr), iqn, 1.0f);
}

template <int NCH, int QB, typename T>
__global__ void __launch_bounds__(SCAN_THREADS, 1) emb_scan_kernel(const ScanParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const uint32_t stride = p.stride;
    const uint32_t R = p.rows_per_stage, S = p.n_stages;
    constexpr uint32_t ESZ = RowLoad<T>::ESZ;
    uint8_t *ring = smem;
    float *nring = reinterpret_cast<float *>(ring + size_t(S) * R * stride * ESZ);
    uint64_t *full = reinterpret_cast<uint64_t *>(nring + size_t(S) * R);
    uint64_t *empty = full + S;
    uint64_t *wbuf = empty + S;  // [QB][8 warps][wcap]

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t n_tiles = (p.n_rows + R - 1) / R;
    // tiles owned by this CTA: blockIdx.x, blockIdx.x + grid, ...
    const uint64_t my_tiles = (n_tiles > blockIdx.x) ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < S; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], SCAN_CONSUMER_WARPS);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == SCAN_CONSUMER_WARPS) {
        // ===================== producer warp (one elected lane) =====================
        if (lane == 0) {
            const uint64_t pol = l2_policy_evict_first();
            for (uint64_t it = 0; it < my_tiles; it++) {
                const uint32_t s = uint32_t(it % S);
                const uint32_t ph = uint32_t((it / S) & 1);
                mbar_wait(&empty[s], ph ^ 1);
                const uint64_t tile = blockIdx.x + it * gridDim.x;
                const uint64_t row0 = tile * R;
                const uint32_t nr = uint32_t(min(uint64_t(R), p.n_rows - row0));
                const uint32_t bytes_rows = nr * stride * ESZ;
                const uint32_t bytes_norm = ((nr * 4 + 15) / 16) * 16;  // n_rows padded alloc
                mbar_expect_tx(&full[s], bytes_rows + bytes_norm);
                bulk_g2s_hint(ring + size_t(s) * R * stride * ESZ, static_cast<const uint8_t *>(p.rows) + row0 * stride * ESZ,
                              bytes_rows, &full[s], pol);
                bulk_g2s(nring + size_t(s) * R, p.inv_norm + row0, bytes_norm, &full[s]);
            }
        }
        return;
    }

    // ===================== consumer warps =====================
    float4 qv[QB][NCH];
    float iqn[QB];
#pragma unroll
    for (int q = 0; q < QB; q++) {
        const float4 *qp = reinterpret_cast<const float4 *>(p.queries + size_t(q) * stride);
#pragma unroll
        for (int j = 0; j < NCH; j++) qv[q][j] = qp[lane + 32 * j];
        iqn[q] = p.inv_qnorm[q];
    }
    float tau[QB];
    uint32_t cnt[QB];
    uint64_t *mybuf[QB];
#pragma unroll
    for (int q = 0; q < QB; q++) {
        tau[q] = -INFINITY;
        cnt[q] = 0;
        mybuf[q] = wbuf + (size_t(q) * SCAN_CONSUMER_WARPS + warp) * p.wcap;
    }
    // -inf never passes `kf > tau`, so rows scoring -inf (cos = -inf cannot happen) are moot;
    // NaN (tombstone / filtered) fails the comparison as well.

    for (uint64_t it = 0; it < my_tiles; it++) {
        const uint32_t s = uint32_t(it % S);
        const uint32_t ph = uint32_t((it / S) & 1);
        const uint64_t tile = blockIdx.x + it * gridDim.x;
        const uint64_t row0 = tile * R;
        const uint32_t nr = uint32_t(min(uint64_t(R), p.n_rows - row0));
        mbar_wait(&full[s], ph);
        const uint8_t *st = ring + size_t(s) * R * stride * ESZ;
        const float *sn = nring + size_t(s) * R;
        for (uint32_t r = warp; r < nr; r += SCAN_CONSUMER_WARPS) {
            const void *rp = st + size_t(r) * stride * ESZ;
            float acc[QB];
#pragma unroll
            for (int q = 0; q < QB; q++) acc[q] = 0.f;
#pragma unroll
            for (int j = 0; j < NCH; j++) {
                const float4 x = RowLoad<T>::ld(rp, lane + 32 * j);
#pragma unroll
                for (int q = 0; q < QB; q++) {
                    acc[q] = fmaf(x.x, qv[q][j].x, acc[q]);
                    acc[q] = fmaf(x.y, qv[q][j].y, acc[q]);
                    acc[q] = fmaf(x.z, qv[q][j].z, acc[q]);
                    acc[q] = fmaf(x.w, qv[q][j].w, acc[q]);
                }
            }
            const float inr = sn[r];
#pragma unroll
            for (int q = 0; q < QB; q++) {
                const float kf = cos_rank_key(warp_sum(acc[q]), inr, iqn[q]);
                // warp-uniform; a row the query's own filter rejects is skipped here, where a NaN inverse norm would
                // skip it in a single-filter sweep (slot and bit are only read for rows that clear the threshold)
                if (kf > tau[q] && (!p.row_bits || slot_row_ok(p.row_bits, p.row_words, __ldg(p.q_slot + q), row0 + r))) {
                    if (cnt[q] == p.wcap) {
                        warp_bitonic_desc(mybuf[q], p.wcap, lane);
                        cnt[q] = p.n_keep;
                        tau[q] = key_score(mybuf[q][p.n_keep - 1]);
                        __syncwarp();
                    }
                    if (kf > tau[q]) {
                        if (lane == 0) mybuf[q][cnt[q]] = make_key(kf, uint32_t(row0 + r));
                        cnt[q]++;
                    }
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }

    // ---- per-warp final compress, then CTA-level merge of the 8 warp lists per query ----
#pragma unroll
    for (int q = 0; q < QB; q++) {
        __syncwarp();
        for (uint32_t i = cnt[q] + lane; i < p.wcap; i += 32) mybuf[q][i] = KEY_NONE;
    }
    const uint32_t ctid = threadIdx.x;  // < 256
    const uint32_t region = SCAN_CONSUMER_WARPS * p.wcap;
#pragma unroll
    for (int q = 0; q < QB; q++) {
        uint64_t *reg = wbuf + size_t(q) * region;
        group_bitonic_desc(reg, region, ctid, SCAN_CONSUMER_WARPS * 32, 1);
        uint64_t *out = p.cand + (size_t(q) * p.n_ctas_total + blockIdx.x) * p.n_keep;
        for (uint32_t i = ctid; i < p.n_keep; i += SCAN_CONSUMER_WARPS * 32) out[i] = reg[i];
    }
}

// ---------------------------------------------------------------------------------------
// Row preparation: inverse L2 norms of newly inserted rows (one warp per row).
// ---------------------------------------------------------------------------------------
// round-to-nearest-even bf16 of an fp32 value, as the fp32 it denotes (what cvt.rn.bf16x2.f32 produces)
__device__ __forceinline__ float bf16_round_f32(float x) {
    const uint32_t u = __float_as_uint(x);
    const uint32_t r = ((u & 0x7fffffffu) > 0x7f800000u) ? (u | 0x00400000u) : (u + 0x7fffu + ((u >> 16) & 1u));
    return __uint_as_float(r & 0xffff0000u);
}
template <typename T>
__global__ void emb_inv_norm_kernel(const void *rows, uint32_t stride, uint64_t row_begin, uint64_t row_end, float *inv_norm) {
    const uint64_t r = row_begin + (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
    const uint32_t lane = threadIdx.x & 31;
    if (r >= row_end) return;
    const void *rp = static_cast<const uint8_t *>(rows) + r * stride * RowLoad<T>::ESZ;
    float s = 0.f;
    for (uint32_t j = lane; j < stride / 4; j += 32) {
        const float4 x = RowLoad<T>::ld(rp, j);
        s = fmaf(x.x, x.x, s); s = fmaf(x.y, x.y, s); s = fmaf(x.z, x.z, s); s = fmaf(x.w, x.w, s);
    }
    s = warp_sum(s);
    if (lane == 0) inv_norm[r] = s > 0.f ? 1.0f / sqrtf(s) : 0.f;
}

// Query preparation: zero-pad to stride, 1/|q| and (optional) rho_q = |q - bf16(q)| / |q| (one warp per query).
__global__ void emb_prep_queries_kernel(const float *q_in, uint32_t dim, uint32_t stride, uint32_t nq,
                                        float *q_out, float *inv_qnorm, float *rho_q) {
    const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
    if (q >= nq) return;
    float s = 0.f, sd = 0.f;
#pragma unroll 8
    for (uint32_t j = lane; j < stride; j += 32) {
        const float v = j < dim ? __ldg(q_in + size_t(q) * dim + j) : 0.f;
        q_out[size_t(q) * stride + j] = v;
        s = fmaf(v, v, s);
        const float d = v - bf16_round_f32(v);
        sd = fmaf(d, d, sd);
    }
    s = warp_sum(s);
    sd = warp_sum(sd);
    if (lane == 0) {
        inv_qnorm[q] = s > 0.f ? 1.0f / sqrtf(s) : 0.f;
        if (rho_q) rho_q[q] = s > 0.f ? sqrtf(sd / s) * 1.001f : 0.f;
    }
}

// Effective inverse norms under a DocumentId filter bitmap (FilterResult::contains,
// embedding_field.rs:54-61): filtered-out rows become NaN and never enter a top-k.
__global__ void emb_apply_filter_kernel(const float *inv_norm, const uint64_t *row_doc_ids, uint64_t n_rows,
                                        const uint64_t *filter_bits, uint64_t filter_nbits, float *out) {
    const uint64_t r = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    const uint64_t doc = row_doc_ids[r];
    const bool ok = doc < filter_nbits && ((filter_bits[doc >> 6] >> (doc & 63)) & 1ull);
    out[r] = ok ? inv_norm[r] : __int_as_float(0x7fc00000);
}

// ---------------------------------------------------------------------------------------
// Block-level streaming top-n over a list of keys in global memory (shared by the scan
// merge and the fusion kernels).  buf: CAPB u64 in shared memory, CAPB pow2 >= 2*n.
// Returns (uniformly) the number of keys kept, sorted descending in buf[0..kept).
// ---------------------------------------------------------------------------------------
template <typename LoadKey>
__device__ inline uint32_t block_topn_stream(uint64_t *buf, uint32_t capb, uint32_t n, uint64_t total,
                                             LoadKey load) {
    uint32_t kept = 0;
    uint64_t pos = 0;
    if (total == 0) return 0;
    while (pos < total) {
        const uint32_t take = uint32_t(min(uint64_t(capb - kept), total - pos));
        for (uint32_t i = threadIdx.x; i < capb - kept; i += blockDim.x)
            buf[kept + i] = i < take ? load(pos + i) : KEY_NONE;
        group_bitonic_desc(buf, capb, threadIdx.x, blockDim.x, 0);
        kept = min(n, kept + take);
        pos += take;
    }
    // trim KEY_NONE padding from the count
    __shared__ uint32_t s_real;
    if (threadIdx.x == 0) {
        uint32_t c = kept;
        while (c > 0 && buf[c - 1] == KEY_NONE) c--;
        s_real = c;
    }
    __syncthreads();
    return s_real;
}

struct ScanMergeParams {
    const uint64_t *cand;       // [nq][n_lists][n_keep]
    uint32_t n_lists, n_keep;
    uint32_t limit;
    uint32_t capb;
    const uint64_t *row_doc_ids;  // NULL => identity
    int rescale_e5;
    float similarity;
    uint64_t *out_doc;   // [nq][limit]
    float *out_score;    // [nq][limit]
    uint32_t *out_row;   // [nq][limit] (row index, for hybrid fusion); may be NULL
    uint32_t *out_count; // [nq]
    float *out_raw;      // [nq][limit] rank key (-distance) of each kept hit; may be NULL
    // per-query parameters: NULL, or [nq] each query's own depth (<= limit) and similarity.  A query's top-L is the
    // first L entries of its top-limit list (keys are unique), so the list is cut before the similarity test.
    const uint32_t *q_limit;
    const float *q_sim;
};

// Model::rescale_score (python/embeddings.rs:71-92)
__device__ __forceinline__ float rescale_score(float s, int is_e5) {
    if (!is_e5) return s;
    const float MIN = 0.7f, MAX = 1.0f, DELTA = MAX - MIN;
    float c = s;
    if (c < MIN) c = MIN;
    if (c > MAX) c = MAX;
    return (c - MIN) / DELTA;
}

__global__ void __launch_bounds__(256) emb_scan_merge_kernel(const ScanMergeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *buf = reinterpret_cast<uint64_t *>(smem);
    const uint32_t q = blockIdx.x;
    const uint64_t total = uint64_t(p.n_lists) * p.n_keep;
    const uint64_t *src = p.cand + size_t(q) * total;
    uint32_t got;
    if (p.limit <= 32 && p.n_lists <= blockDim.x) {
        // the per-CTA lists are already sorted: `limit` rounds of a block arg-max over the list heads
        __shared__ uint64_t s_wk[8];
        __shared__ uint32_t s_wt[8];
        uint32_t head = 0;
        const uint64_t *mine = src + size_t(threadIdx.x) * p.n_keep;
        uint32_t n_real = 0;
        for (uint32_t r = 0; r < p.limit; r++) {
            uint64_t best = (threadIdx.x < p.n_lists && head < p.n_keep) ? mine[head] : KEY_NONE;
            uint32_t who = threadIdx.x;
            for (int o = 16; o > 0; o >>= 1) {
                const uint64_t ob = __shfl_xor_sync(0xffffffffu, best, o);
                const uint32_t ow = __shfl_xor_sync(0xffffffffu, who, o);
                if (ob > best) { best = ob; who = ow; }
            }
            if ((threadIdx.x & 31) == 0) { s_wk[threadIdx.x >> 5] = best; s_wt[threadIdx.x >> 5] = who; }
            __syncthreads();
            uint64_t b = s_wk[0]; uint32_t bw = s_wt[0];
            for (uint32_t w = 1; w < blockDim.x / 32; w++) if (s_wk[w] > b) { b = s_wk[w]; bw = s_wt[w]; }
            if (threadIdx.x == bw && b != KEY_NONE) head++;
            if (threadIdx.x == 0) buf[r] = b;
            if (b != KEY_NONE) n_real++;
            __syncthreads();
        }
        got = n_real;
    } else {
        got = block_topn_stream(buf, p.capb, p.limit, total, [&](uint64_t i) { return src[i]; });
    }
    __shared__ uint32_t s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    if (p.q_limit) got = min(got, p.q_limit[q]);
    const float similarity = p.q_sim ? p.q_sim[q] : p.similarity;
    for (uint32_t i = threadIdx.x; i < p.limit; i += blockDim.x) {
        uint64_t doc = 0; float score = 0.f; uint32_t row = 0xffffffffu;
        if (i < got) {
            const uint64_t k = buf[i];
            row = key_idx(k);
            const float distance = -key_score(k);
            const float sim = 1.0f - distance;                 // embedding_field.rs:270
            score = rescale_score(sim, p.rescale_e5);          // :271
            if (score >= similarity) {                         // :272 (kept hits form a prefix)
                doc = p.row_doc_ids ? p.row_doc_ids[row] : uint64_t(row);
                atomicAdd(&s_cnt, 1u);
            } else {
                score = 0.f; row = 0xffffffffu;
            }
        }
        p.out_doc[size_t(q) * p.limit + i] = doc;
        p.out_score[size_t(q) * p.limit + i] = score;
        if (p.out_row) p.out_row[size_t(q) * p.limit + i] = row;
        if (p.out_raw) p.out_raw[size_t(q) * p.limit + i] = (i < got && row != 0xffffffffu) ? key_score(buf[i]) : 0.f;
    }
    __syncthreads();
    if (threadIdx.x == 0) p.out_count[q] = s_cnt;
}

}  // namespace oc
