// emb_gemm.cuh — K2: batched-query embedding scan on the Hopper tensor cores (wgmma).
//
// Same contract as K1 (EmbeddingFieldStorage::search, read/index/embedding_field.rs:250-278)
// but for a BATCH of queries, where the distance computation is a true dense GEMM
// S[q][r] = sum_k Q[q][k] * X[r][k] (north_star: "tensor cores used only when batched
// queries make the distance a true dense GEMM").  One matrix sweep serves the whole batch.
//
//   * operands (GemmOp): an fp32 store is swept through its fp16 copy (oc_emb.rows_f16: every row scaled by a power of
//     two that puts its largest |x_i| in [2^14, 2^15), then rounded to nearest; the scale comes back exactly with the
//     row's inverse norm) with wgmma .f16, algorithmic bytes = n_rows * (stride * 2 + 8) per batch; without the copy
//     (OC_EMB_F16=0) the fp32 rows are read straight from HBM by wgmma .tf32 (the tensor core drops the low 13
//     mantissa bits), n_rows * (stride * 4 + 4); bf16 stores use wgmma .bf16;
//   * CTA tile: M = 128 queries (A operand, two consumer warpgroups of 64) x N = 256 rows (B operand),
//     K-blocks of 128 bytes = one swizzle row; one producer warp fills a 4-stage shared-memory ring
//     with TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B) under full / empty mbarriers, each consumer
//     warpgroup issues wgmma.mma_async m64n256 into 128 fp32 accumulator registers per thread;
//   * CTA pairs: with an even number of query groups the sweep is launched in clusters of 2 CTAs, query
//     groups 2i and 2i + 1 of the same row partition.  Each CTA loads one 128-row half of every row tile
//     with TMA multicast into both CTAs' rings, so each row leaves L2 once per batch instead of once per
//     query group; a stage is refilled only when the consumers of BOTH CTAs have released it.  Launched
//     without a cluster (odd group counts, the kernel test harness) a CTA loads the whole tile itself;
//     tm_x's box is GEMM_N / (cluster size) rows;
//   * epilogue, straight from the accumulator registers: a thread holds 2 queries x 64 rows of the
//     tile (wgmma's D fragment), taken in two halves of 32 rows (one per 128-row half of the tile),
//     scales them by the rows' inverse norms and pushes every row whose
//     approximate score clears the query's threshold into a private candidate list — one list per
//     (query, CTA, lane % 4); the threshold is the query's running K'-th best, seeded by a one-tile
//     threshold pass of the same kernel and shared across CTAs through an atomicMax'd global array
//     (any subset's K'-th best bounds the global one);
//   * the sweep's scores are only used to SELECT candidates.  The merge kernel re-scores the
//     best K' candidates per query in exact fp32 with K1's arithmetic (bit-identical scores) and
//     PROVES the answer: every non-candidate row has approx <= max(final threshold, K'-th
//     selected), and |approx - exact| <= eps for the sweep's arithmetic (GEMM_EPS_* below), so
//     when the limit-th exact score clears bound + eps the exact top-`limit` is inside the
//     candidate set.  Queries that fail the proof are re-run through the exact K1 sweep by the
//     host (rare).
//   * kernels in this file: emb_gemm_kernel<OP>, gemm_thr_kernel, emb_gemm_merge_kernel.  emb_gemm_kernel<OP, true>
//     (score dump) is instantiated only by the kernel test harness (tests/kernels).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "emb_scan.cuh"

namespace oc {

constexpr uint32_t GEMM_CONSUMER_WG = 2;                          // warpgroups issuing wgmma, 64 queries each
// warps 0-7: consumers, warps 8-11: the producer warpgroup (warp 8 issues the TMA loads).  A whole producer warpgroup
// lets setmaxnreg move registers to the consumers: 168 per thread at launch (64K / 384), then 40 for the producers
// and 232 for the consumers (128 accumulators + the epilogue)
constexpr int GEMM_THREADS = (GEMM_CONSUMER_WG + 1) * 128;
constexpr uint32_t GEMM_PRODUCER_REGS = 40, GEMM_CONSUMER_REGS = 232;
constexpr uint32_t GEMM_M = 128;       // queries per CTA
constexpr uint32_t GEMM_N = 256;       // rows per tile
constexpr uint32_t GEMM_KB = 32;       // fp32 elements per K-block (one 128 B swizzle row); bf16 / fp16 rows: 64
constexpr uint32_t GEMM_STAGES = 4;
constexpr uint32_t GEMM_CLUSTER = 2;   // CTAs of a paired launch (two query groups sharing each row tile)
constexpr uint32_t GEMM_A_BYTES = GEMM_M * 128;   // 16 KB
constexpr uint32_t GEMM_B_BYTES = GEMM_N * 128;   // 32 KB
constexpr uint32_t GEMM_STAGE_BYTES = GEMM_A_BYTES + GEMM_B_BYTES;
constexpr uint32_t GEMM_LISTS_PER_CTA = 4;        // candidate lists per (query, CTA): one per lane % 4 of the D fragment
constexpr uint32_t GEMM_LIST_CAP = 128;           // entries of one (query, list) candidate buffer
constexpr uint32_t GEMM_OVF_CAP = 2048;           // per-query spill area shared by its lists (global atomics; rare)
constexpr uint32_t GEMM_MERGE_BUF = 4096;         // keys the merge kernel holds in shared memory
constexpr uint32_t GEMM_MAX_RESCORE = 2048;       // candidates re-scored exactly per query; more => exact sweep
constexpr uint32_t GEMM_MAX_LIMIT = 128;          // largest `limit` the tensor-core scan serves (seeds need >= limit row groups)
// Rigorous bounds on |approx - exact| of the COSINE for each sweep arithmetic (tests/test_proof_bounds.py).
// With x~ = x + dx, q~ = q + dq the tensor core accumulates sum x~_i q~_i, so
//   |approx - exact| <= (rho_x + rho_q + rho_x rho_q) |x||q| + acc,   rho = |d| / |.|   (Cauchy-Schwarz),
// acc = the fp32 accumulation of the tensor core (<= 1024 adds x 2^-23, truncating: 1.3e-4 |x||q|) plus the
// rounding of the exact fp32 re-score it is compared with (<= 1024 x 2^-24, twice): GEMM_EPS_ACC.
//   tf32: the tensor core drops the low 13 mantissa bits of both operands: rho <= 2^-10 each, worst case taken
//         -> GEMM_EPS_TF32 (constant);
//   bf16 store: the rows are exact bf16 values (rho_x = 0); the query is rounded to bf16 (unit roundoff 2^-8):
//         the worst case 2^-8 is ~2.4x the actual residual norm of a rounded vector, so the MEASURED residual
//         rho_q per query (emb_prep_queries_kernel) is used, capped at the worst case.
//   fp16 copy of an fp32 store: row and query are each scaled by a power of two (exact) that puts the largest |v_i| in
//         [2^14, 2^15), then rounded to nearest fp16 (11 significant bits): rho <= 2^-11 for the normal components,
//         and a component that lands in fp16's subnormal range is off by <= 2^-25 absolute, <= 2^-34 |v| over 1024
//         of them: rho <= 2^-11 + 2^-34 per operand -> GEMM_EPS_F16 (constant).  The sweep's scores are then in
//         units of cos * |q| * 2^e_q (the query's scale), and gemm_thr_kernel scales eps_v alike.
constexpr float GEMM_EPS_ACC = 2.5e-4f;
constexpr float GEMM_EPS_TF32 = 2.25e-3f;
constexpr float GEMM_EPS_F16 = 1.25e-3f;
constexpr float GEMM_RHO_BF16_WORST = 3.90625e-3f;   // 2^-8: cap of a measured rho (a sound upper bound by itself)

// operand kind of the sweep (the template argument of emb_gemm_kernel)
enum GemmOp : int {
    GEMM_TF32 = 0,   // fp32 rows and query, wgmma .tf32, 32 elements per K-block
    GEMM_BF16 = 1,   // bf16 store and bf16-rounded query, wgmma .bf16, 64 elements per K-block
    GEMM_F16 = 2,    // power-of-two scaled fp16 copies of an fp32 store and of the query, wgmma .f16, 64 per K-block
};

struct GemmParams {
    uint64_t n_rows;
    uint32_t n_kblocks;        // stride / 32 (tf32) or stride / 64 (bf16, fp16)
    const float *inv_norm;     // [n_rows] (NaN => skipped)
    uint32_t n_queries;        // B (real queries)
    uint32_t n_qgroups;        // ceil(B / 128)
    uint32_t ctas_per_group;   // gridDim.x / n_qgroups
    uint32_t cap;              // GEMM_LIST_CAP
    unsigned int *thr;         // [n_queries] per-query gather thresholds (cos*|q| units, order-preserving uint): seeded by
                               // gemm_thr_kernel, raised with atomicMax whenever a list proves a better bound (see gemm_compact)
    const float *eps_v;        // [n_queries] error bound of the sweep's scores in the same units
    uint32_t limit;            // top-`limit` wanted
    uint32_t lists_per_query;  // candidate lists per query: ctas_per_group * GEMM_LISTS_PER_CTA
    int max_mode;              // 1 => threshold pass: record each list's best approximate score, push nothing
    uint32_t tile_limit;       // max row tiles per CTA (0 = all); the threshold pass looks at one
    float *gmax;               // [n_qgroups*128][lists_per_query] best score per list (max_mode)
    uint64_t *cand;            // [n_qgroups*128][lists_per_query][cap]
    uint32_t *cand_cnt;        // [n_qgroups*128][lists_per_query]
    uint64_t *ovf;             // [n_queries][ovf_cap] spill area: a full private list is appended here
    uint32_t *ovf_cnt;         // [n_queries] (may exceed ovf_cap: the merge then sends the query to the exact sweep)
    uint32_t ovf_cap;
    // per-query where-filters (as ScanParams): NULL, or [n_slots][row_words] row bitmaps, row_words a multiple of 4
    // covering every tile; query q keeps row r when q_slot[q] == SLOT_NONE or bit r of its slot is set
    const uint32_t *row_bits;
    uint64_t row_words;
    const uint32_t *q_slot;    // [n_queries]
};
// emb_gemm_kernel<GEMM_F16>: row_scale [n_rows] = the power of two that turns a row of the fp16 copy back into the stored
// row (NaN for a row with a non-finite element), staged multiplied into the inverse norms.  (A field of its own type, so
// that the tf32 and bf16 kernels keep their parameter block.)
struct GemmF16Params : GemmParams {
    const float *row_scale;
};
// The 32 rows a thread holds of a 128-row half tile (rows row0 + 2 (lane & 3) + 8 (j >> 1) + (j & 1), j < 32) as bit j
// of a mask, from the half's 4 words of a row bitmap: word w gives bits 8w .. 8w + 7 (its bits 8m + 2 (lane & 3) + {0, 1}).
__device__ __forceinline__ uint32_t gemm_tile_row_mask(const uint32_t *bits, uint32_t lane) {
    const uint4 w = __ldg(reinterpret_cast<const uint4 *>(bits));
    const uint32_t s = 2 * (lane & 3);
    auto pick = [s](uint32_t x) {
        x = (x >> s) & 0x03030303u;
        x = (x | (x >> 6)) & 0x000f000fu;
        return (x | (x >> 12)) & 0xffu;
    };
    return pick(w.x) | (pick(w.y) << 8) | (pick(w.z) << 16) | (pick(w.w) << 24);
}
// emb_gemm_kernel<OP, DUMP = true> (test harness only): the epilogue writes every approximate score v of a live
// (query, row) pair to dump[q * n_rows + row] instead of gathering candidates
struct GemmDumpParams : GemmF16Params {
    float *dump;               // [n_queries][n_rows]
};
template <int OP, bool DUMP> struct GemmKernelParams { using type = GemmParams; };
template <> struct GemmKernelParams<GEMM_F16, false> { using type = GemmF16Params; };
template <int OP> struct GemmKernelParams<OP, true> { using type = GemmDumpParams; };

__host__ __device__ inline size_t gemm_smem_bytes() {
    return 1024 /*align slack*/ + size_t(GEMM_STAGES) * GEMM_STAGE_BYTES + GEMM_CONSUMER_WG * 2 * GEMM_N * 4 /*inv norms*/
           + 256 /*barriers*/;
}

// ---- TMA / wgmma PTX wrappers ------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, uint64_t *bar, int32_t c0, int32_t c1,
                                            uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(hint)
        : "memory");
}
// the same box written to the same shared-memory offset of every CTA in cta_mask, each CTA's mbarrier at `bar`'s
// offset receiving complete_tx of the box's bytes
__device__ __forceinline__ void tma_load_2d_multicast(void *dst, const CUtensorMap *map, uint64_t *bar, int32_t c0, int32_t c1,
                                                      uint16_t cta_mask, uint64_t hint) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
        " [%0], [%1, {%3, %4}], [%2], %5, %6;" ::"r"(smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask), "l"(hint)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// ---- thread-block clusters (1 CTA when launched without a cluster) ----
__device__ __forceinline__ uint32_t cluster_nctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// per-thread register budget of the calling warpgroup (all its warps execute the same one)
template <uint32_t R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
// every thread of every CTA of the cluster (need not be warp-converged)
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at `bar`'s shared-memory offset in CTA `cta` of the cluster.  Default (.cta) release scope:
// what it orders is the arriving warp's wgmma reads of a stage, already complete (wgmma.wait_group), before the
// partner's TMA overwrites it; .release.cluster would put a MEMBAR.GPU in front of every arrival of the K loop.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t *bar, uint32_t cta) {
    asm volatile(
        "{\n\t.reg .b32 ra;\n\t"
        "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
        "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}" ::"r"(smem_u32(bar)), "r"(cta)
        : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma:
// start>>4 [0,14) | LBO>>4 [16,30) = 1 (unused when swizzled) | SBO>>4 [32,46) = 1024/16 (8-row groups) | layout [62,64) = 1
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
    return uint64_t((smem_addr >> 4) & 0x3fffu) | (uint64_t(1) << 16) | (uint64_t(64) << 32) | (uint64_t(1) << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 256] (+)= A[64 x K] * B[256 x K]^T, both K-major in shared memory; K = 8 (tf32) or 16 (bf16, fp16) = 32 bytes
template <int OP>
__device__ __forceinline__ void wgmma_m64n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
#define OC_WGMMA_D                                                                                                             \
    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "         \
    "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "          \
    "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, "          \
    "%68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, "          \
    "%90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, "          \
    "%110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define OC_WGMMA_OPS                                                                                                           \
    "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),               \
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),                 \
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),                \
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),                \
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),                \
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),                \
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),                \
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]),                \
        "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),                \
        "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]),                \
        "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]),                \
        "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]),                \
        "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]),           \
        "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]),        \
        "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]),        \
        "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
    if constexpr (OP == GEMM_BF16)
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 " OC_WGMMA_D ", %128, %129, p, 1, 1, 0, 0;\n\t}"
            : OC_WGMMA_OPS
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
    else if constexpr (OP == GEMM_F16)
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " OC_WGMMA_D ", %128, %129, p, 1, 1, 0, 0;\n\t}"
            : OC_WGMMA_OPS
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "setp.ne.b32 p, %130, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 " OC_WGMMA_D ", %128, %129, p, 1, 1;\n\t}"
            : OC_WGMMA_OPS
            : "l"(adesc), "l"(bdesc), "r"(accumulate));
#undef OC_WGMMA_D
#undef OC_WGMMA_OPS
}

constexpr uint64_t TMA_EVICT_FIRST = 0x12F0000000000000ull;
constexpr uint64_t TMA_EVICT_LAST = 0x14F0000000000000ull;

// ---- the epilogue: one thread = 2 queries x 32 rows of the tile, one private list per query --------------------
// The threshold only has to stay <= a_lim - 2 eps (a_lim = the limit-th best approximate score of the whole
// store): the seed is a coarse sample bound, so when a list fills up the warp tightens it — the limit-th largest
// score of ANY `limit` distinct rows bounds a_lim from below — drops what fell under the new threshold and shares
// it with the other CTAs through an atomicMax'd global (gemm_compact).  Only a list that is still full after
// that is appended to the query's spill area.
struct GemmEpi {
    uint32_t cnt = 0;
    float thr = 0.f;
    float best = 0.f;
};
__device__ __noinline__ void gemm_spill(const GemmParams &p, uint32_t q, const uint64_t *mybuf, uint32_t cnt) {
    const uint32_t base = atomicAdd(p.ovf_cnt + q, cnt);
    if (base + cnt <= p.ovf_cap)
        for (uint32_t i = 0; i < cnt; i++) p.ovf[size_t(q) * p.ovf_cap + base + i] = mybuf[i];
}
// Warp-cooperative tightening of the lists of the lanes in `need` (register-only: 4 keys per lane, cap <= 128).
// Lane l owns list my_list of query my_q (both passed per lane).  For lane l: kth = limit-th largest score of its
// list (bitwise search on the order-preserving key, one __reduce_add_sync per bit); thr_l = max(thr_l, kth - 2 eps_l);
// entries <= thr_l are dropped, the rest compacted in place.  Returns, for the calling lane, its new (cnt, thr).
__device__ __noinline__ void gemm_compact(const GemmParams &p, uint32_t need, uint32_t my_q, uint32_t my_list, uint32_t lane,
                                          GemmEpi &e) {
    while (need) {
        const uint32_t l = __ffs(need) - 1;
        need &= need - 1;
        const uint32_t lq = __shfl_sync(0xffffffffu, my_q, l);
        const uint32_t llist = __shfl_sync(0xffffffffu, my_list, l);
        uint64_t *lbuf = p.cand + (size_t(lq) * p.lists_per_query + llist) * p.cap;
        const uint32_t lcnt = __shfl_sync(0xffffffffu, e.cnt, l);
        float lthr = __shfl_sync(0xffffffffu, e.thr, l);
        __syncwarp();                                         // lane l's pushes are visible to the whole warp
        uint64_t k[4];
        uint32_t o[4];
#pragma unroll
        for (uint32_t u = 0; u < 4; u++) {
            const uint32_t i = lane + 32 * u;
            k[u] = i < lcnt ? lbuf[i] : KEY_NONE;
            o[u] = uint32_t(k[u] >> 32);                      // order-preserving score bits (0 for KEY_NONE)
        }
        if (lcnt >= p.limit) {
            uint32_t prefix = 0;
            for (int bit = 31; bit >= 0; bit--) {             // largest value v with |{keys >= v}| >= limit
                const uint32_t cand = prefix | (1u << bit);
                uint32_t c = 0;
#pragma unroll
                for (uint32_t u = 0; u < 4; u++) c += o[u] >= cand ? 1u : 0u;
                c = __reduce_add_sync(0xffffffffu, c);
                if (c >= p.limit) prefix = cand;
            }
            const float kth = f32_unordered(prefix);
            const float ev = p.eps_v[lq];
            const float nthr = kth - 2.0f * ev;               // eps = inf (zero query) -> -inf: no change
            if (nthr > lthr) lthr = nthr;
        }
        // compact: keep the entries above the (possibly raised) threshold
        uint32_t base = 0;
        __syncwarp();
#pragma unroll
        for (uint32_t u = 0; u < 4; u++) {
            const bool keep = k[u] != KEY_NONE && key_score(k[u]) > lthr;
            const uint32_t m = __ballot_sync(0xffffffffu, keep);
            if (keep) lbuf[base + __popc(m & ((1u << lane) - 1u))] = k[u];
            base += __popc(m);
        }
        __syncwarp();
        if (lane == l) {
            e.cnt = base;
            if (lthr > e.thr) { e.thr = lthr; atomicMax(p.thr + lq, f32_ordered(lthr)); }
            if (e.cnt + 32 > p.cap) { gemm_spill(p, lq, lbuf, e.cnt); e.cnt = 0; }   // still full: a dense cluster
        }
        __syncwarp();
    }
}

// Accumulator of the j-th of the 32 rows (rows 2 (lane & 3) + 8 (j >> 1) + (j & 1) of the 128-row half u of the tile)
// a thread holds for its query h.
__host__ __device__ constexpr uint32_t gemm_frag(uint32_t u, uint32_t h, uint32_t j) {
    return 64 * u + 4 * (j >> 1) + 2 * h + (j & 1);
}
// A stage is free again once the consumer warps of every CTA it is loaded into have arrived on its `empty` barrier.
__device__ __forceinline__ void gemm_release(uint64_t *empty, uint32_t csize) {
    if (csize == 1) mbar_arrive(empty);
    else
        for (uint32_t r = 0; r < csize; r++) mbar_arrive_cluster(empty, r);
}

// One CTA = one query group (128 queries) x one row partition c of the store (tiles c, c + ctas_per_group, ...).
// The CTAs of a cluster (blockIdx.x 2i, 2i + 1; n_qgroups even) share c, hence the tiles and the stage sequence.
// wgmma D fragment of m64n256 (per warpgroup): warp w holds rows [16w, 16w + 16); lane holds rows lane/4 and
// lane/4 + 8, columns 8j + 2 (lane % 4) + {0, 1} for j = 0..31, in d[4j + 2h + {0, 1}] (h = row half); the
// tile's 128-row half u is j = 16u .. 16u + 15.
template <int OP, bool DUMP = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
emb_gemm_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_x,
                const typename GemmKernelParams<OP, DUMP>::type p) {
    extern __shared__ __align__(1024) uint8_t smem_gemm[];
    // SWIZZLE_128B tiles need 1024-byte alignment of the shared-memory address (the same offset in every CTA: the
    // multicast writes both CTAs of a pair at one offset)
    uint8_t *ring = smem_gemm + ((1024u - (smem_u32(smem_gemm) & 1023u)) & 1023u);
    float *inr_s = reinterpret_cast<float *>(ring + GEMM_STAGES * GEMM_STAGE_BYTES);   // [wg][2][GEMM_N]
    uint64_t *bars = reinterpret_cast<uint64_t *>(inr_s + GEMM_CONSUMER_WG * 2 * GEMM_N);
    uint64_t *full = bars, *empty = bars + GEMM_STAGES;

    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t grp = blockIdx.x % p.n_qgroups;     // query group
    const uint32_t c = blockIdx.x / p.n_qgroups;       // row partition
    const uint32_t csize = cluster_nctarank();         // 1, or GEMM_CLUSTER for a paired launch
    const uint64_t n_tiles = (p.n_rows + GEMM_N - 1) / GEMM_N;
    uint64_t my_tiles = (n_tiles > c) ? (n_tiles - c + p.ctas_per_group - 1) / p.ctas_per_group : 0;
    if (p.tile_limit && my_tiles > p.tile_limit) my_tiles = p.tile_limit;
    const uint32_t nkb = p.n_kblocks;
    constexpr int32_t KSTEP = OP == GEMM_TF32 ? GEMM_KB : 2 * GEMM_KB;

    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < GEMM_STAGES; s++) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], GEMM_CONSUMER_WG * 4 * csize);
        }
        fence_mbar_init();
        tma_prefetch_desc(&tm_q);
        tma_prefetch_desc(&tm_x);
    }
    // the partner CTA multicasts into this CTA's ring and arrives on its barriers: both must be initialised first
    if (csize > 1) cluster_sync();
    else __syncthreads();

    if (warp >= GEMM_CONSUMER_WG * 4) {
        // ===================== TMA producer =====================
        setmaxnreg_dec<GEMM_PRODUCER_REGS>();
        if (warp == GEMM_CONSUMER_WG * 4 && lane == 0) {
            // this CTA's share of the row tile: all of it, or one half multicast into both CTAs of the pair
            const uint32_t crank = cluster_ctarank(), b_rows = GEMM_N / csize;
            const uint16_t cta_mask = uint16_t((1u << csize) - 1u);
            uint64_t n = 0;
            for (uint64_t it = 0; it < my_tiles; it++) {
                const uint64_t row0 = (c + it * p.ctas_per_group) * GEMM_N + crank * b_rows;
                for (uint32_t kb = 0; kb < nkb; kb++, n++) {
                    const uint32_t s = uint32_t(n % GEMM_STAGES), ph = uint32_t((n / GEMM_STAGES) & 1);
                    mbar_wait(&empty[s], ph ^ 1);
                    uint8_t *a_dst = ring + s * GEMM_STAGE_BYTES;
                    uint8_t *b_dst = a_dst + GEMM_A_BYTES + crank * b_rows * 128;
                    mbar_expect_tx(&full[s], GEMM_STAGE_BYTES);   // the whole stage lands in every CTA
                    // rows past the padded query matrix / the store are zero-filled by TMA
                    tma_load_2d(a_dst, &tm_q, &full[s], int32_t(kb) * KSTEP, int32_t(grp * GEMM_M), TMA_EVICT_LAST);
                    if (csize == 1) tma_load_2d(b_dst, &tm_x, &full[s], int32_t(kb) * KSTEP, int32_t(row0), TMA_EVICT_FIRST);
                    else tma_load_2d_multicast(b_dst, &tm_x, &full[s], int32_t(kb) * KSTEP, int32_t(row0), cta_mask, TMA_EVICT_FIRST);
                }
            }
        }
        // no CTA leaves while its partner may still write into its ring or arrive on its barriers
        if (csize > 1) cluster_sync();
        return;
    }

    // ===================== consumers: wgmma + epilogue =====================
    setmaxnreg_inc<GEMM_CONSUMER_REGS>();
    const uint32_t wg = warp >> 2, t = threadIdx.x & 127;
    const uint32_t lists = p.lists_per_query;
    const uint32_t my_list = c * GEMM_LISTS_PER_CTA + (lane & 3);
    uint32_t q[2];
    bool live[2];
    GemmEpi e[2];
    uint32_t slot[2];
#pragma unroll
    for (uint32_t h = 0; h < 2; h++) {
        q[h] = grp * GEMM_M + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        live[h] = q[h] < p.n_queries;
        slot[h] = (!DUMP && p.row_bits && live[h]) ? p.q_slot[q[h]] : SLOT_NONE;
        e[h].thr = live[h] ? -INFINITY : INFINITY;     // refreshed from the query's global threshold before every tile
        e[h].best = -INFINITY;                         // max_mode: best approximate score seen by this list
    }
    float d[128];
#pragma unroll
    for (uint32_t i = 0; i < 128; i++) d[i] = 0.f;
    uint64_t n = 0;
    for (uint64_t it = 0; it < my_tiles; it++) {
        const uint64_t row0 = (c + it * p.ctas_per_group) * GEMM_N;
        float *inr = inr_s + (wg * 2 + uint32_t(it & 1)) * GEMM_N;
#pragma unroll
        for (uint32_t i = t; i < GEMM_N; i += 128) {
            const uint64_t r = row0 + i;
            if constexpr (OP == GEMM_F16)   // row_scale is a power of two: the product is exact
                inr[i] = r < p.n_rows ? __ldg(p.inv_norm + r) * __ldg(p.row_scale + r) : __int_as_float(0x7fc00000);
            else
                inr[i] = r < p.n_rows ? __ldg(p.inv_norm + r) : __int_as_float(0x7fc00000);
        }
        // requested before the main loop, consumed after it: the L2 round trip hides behind the MMAs of this tile
        unsigned int tg[2];
#pragma unroll
        for (uint32_t h = 0; h < 2; h++)
            tg[h] = (!DUMP && live[h] && !p.max_mode) ? *reinterpret_cast<volatile unsigned int *>(p.thr + q[h]) : 0u;
        uint32_t prev_s = 0;
        for (uint32_t kb = 0; kb < nkb; kb++, n++) {
            const uint32_t s = uint32_t(n % GEMM_STAGES), ph = uint32_t((n / GEMM_STAGES) & 1);
            mbar_wait(&full[s], ph);
            const uint32_t a_addr = smem_u32(ring + s * GEMM_STAGE_BYTES);
            const uint64_t adesc = wgmma_desc_sw128(a_addr + wg * (GEMM_A_BYTES / 2));
            const uint64_t bdesc = wgmma_desc_sw128(a_addr + GEMM_A_BYTES);
            wgmma_fence();
#pragma unroll
            for (uint32_t k = 0; k < 4; k++)   // 32 B of K per instruction: advance the start address by 32 B (>> 4 = 2)
                wgmma_m64n256<OP>(d, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0);
            wgmma_commit();
            if (kb > 0) {                      // the previous K-block's MMAs have retired: free its stage
                wgmma_wait<1>();
                if (lane == 0) gemm_release(&empty[prev_s], csize);
            }
            prev_s = s;
        }
        wgmma_wait<0>();
        if (lane == 0) gemm_release(&empty[prev_s], csize);
        named_bar_sync(1 + wg, 128);           // this warpgroup's inverse norms are in shared memory

        // in 128-row halves of the tile: 32 rows per (thread, query) at a time keep v[] at 32 registers, and each
        // half pushes at most 32 entries into a list between two list-full tests
#pragma unroll
        for (uint32_t u = 0; u < 2; u++) {
            const uint64_t rowu = row0 + 128 * u;
            const float2 *inr2 = reinterpret_cast<const float2 *>(inr + 128 * u);
#pragma unroll
            for (uint32_t h = 0; h < 2; h++) {
                GemmEpi &E = e[h];
                if (u == 0 && tg[h]) E.thr = fmaxf(E.thr, f32_unordered(tg[h]));   // the query's threshold as raised by every CTA so far
                // scaled in place (the next tile's first wgmma overwrites the accumulators): no extra registers
#pragma unroll
                for (uint32_t j = 0; j < 16; j++) {
                    const float2 w = inr2[4 * j + (lane & 3)];
                    d[gemm_frag(u, h, 2 * j + 0)] *= w.x;   // cos * |q|
                    d[gemm_frag(u, h, 2 * j + 1)] *= w.y;
                }
                if constexpr (DUMP) {
                    const uint64_t rb = rowu + 2 * (lane & 3);
#pragma unroll
                    for (uint32_t j = 0; j < 32; j++) {
                        const uint64_t r = rb + 8 * (j >> 1) + (j & 1);
                        if (live[h] && r < p.n_rows) p.dump[size_t(q[h]) * p.n_rows + r] = d[gemm_frag(u, h, j)];
                    }
                    continue;
                }
                if (p.max_mode) {
                    // a row the query's own filter rejects must not raise its bound (it is NaN in a single-filter sweep)
                    const uint32_t ok = slot[h] == SLOT_NONE ? 0xffffffffu
                                                             : gemm_tile_row_mask(p.row_bits + size_t(slot[h]) * p.row_words + rowu / 32, lane);
#pragma unroll
                    for (uint32_t j = 0; j < 32; j++)
                        if ((ok >> j) & 1u) E.best = fmaxf(E.best, d[gemm_frag(u, h, j)]);   // NaN (dead rows) ignored
                    continue;
                }
                uint32_t mask = 0;
#pragma unroll
                for (uint32_t j = 0; j < 32; j++) mask |= (d[gemm_frag(u, h, j)] > E.thr ? 1u : 0u) << j;   // NaN fails
                // per-query filter: only rows that already clear the threshold look at the bitmap (the common path of
                // the sweep loads nothing more)
                if (mask && slot[h] != SLOT_NONE)
                    mask &= gemm_tile_row_mask(p.row_bits + size_t(slot[h]) * p.row_words + rowu / 32, lane);
                if (mask) {   // rare once the threshold has tightened
                    uint64_t *mybuf = p.cand + (size_t(q[h]) * lists + my_list) * p.cap;
                    const uint32_t rb = uint32_t(rowu) + 2 * (lane & 3);
#pragma unroll
                    for (uint32_t j = 0; j < 32; j++)
                        if ((mask >> j) & 1u) { mybuf[E.cnt] = make_key(d[gemm_frag(u, h, j)], rb + 8 * (j >> 1) + (j & 1)); E.cnt++; }
                }
                const uint32_t need = __ballot_sync(0xffffffffu, E.cnt + 32 > p.cap);
                if (need) gemm_compact(p, need, q[h], my_list, lane, E);
            }
        }
    }
    if constexpr (!DUMP) {
#pragma unroll
        for (uint32_t h = 0; h < 2; h++) {
            if (p.max_mode) p.gmax[size_t(q[h]) * lists + my_list] = live[h] ? e[h].best : -INFINITY;
            else p.cand_cnt[size_t(q[h]) * lists + my_list] = live[h] ? e[h].cnt : 0;
        }
    }
    if (csize > 1) cluster_sync();
}

// ---------------------------------------------------------------------------------------
// Merge: gathered candidates -> the ones that can still be in the exact top-`limit` -> exact fp32
// re-score (K1 arithmetic) -> top-`limit`.
//
// Exactness argument (eps = bound on |approx - exact| of this query, in cos*|q| units):
//   * the sweep gathered EVERY row with approx > thr, thr = LB - 2 eps, LB <= a_lim := the limit-th best
//     approximate score of the whole store (LB is attained by `limit` distinct rows: gemm_thr_kernel), so the
//     gathered set holds the global top-`limit` by approximate score and a_lim is known exactly;
//   * the `limit` rows with the best approximate scores have exact >= a_lim - eps, hence the limit-th best
//     EXACT score s* >= a_lim - eps, and a row can only belong to the exact top-`limit` if
//     approx >= s* - eps >= a_lim - 2 eps: those rows (all gathered, since a_lim - 2 eps >= thr) are re-scored
//     exactly and ranked.  Nothing is assumed about the distribution of the scores: near-duplicate clusters
//     only make the re-scored set larger (the whole cluster instead of a few dozen rows).
// The host re-runs a query through the exact sweep only if a buffer overflowed (out_unproven): more than
// GEMM_OVF_CAP spilled candidates or more than GEMM_MAX_RESCORE rows within 2 eps of the limit-th best.
// ---------------------------------------------------------------------------------------
struct GemmMergeParams {
    const uint64_t *cand; const uint32_t *cand_cnt;
    uint32_t n_lists, cap;
    const uint64_t *ovf; const uint32_t *ovf_cnt; uint32_t ovf_cap;
    const float *eps_v;          // [B] per-query eps in cos*|q| units (gemm_thr_kernel)
    uint32_t limit;
    const void *rows; int rows_bf16; uint32_t stride; const float *inv_norm;
    const float *queries;        // [B][stride] padded fp32 (exact re-score always uses the fp32 query)
    const float *inv_qnorm;      // [B]
    const uint64_t *row_doc_ids;
    int rescale_e5; float similarity;
    uint64_t *out_doc; float *out_score; uint32_t *out_row; uint32_t *out_count; float *out_raw;
    uint8_t *out_unproven;       // [B] 1 => host must re-run this query through the exact sweep
    uint32_t *out_rescored;      // [B] rows re-scored exactly (diagnostics), may be NULL
    const uint32_t *q_limit;     // NULL, or [B] each query's own depth (<= limit): its list is cut there ...
    const float *q_sim;          // ... before its own similarity test (NULL: similarity)
};
__host__ __device__ inline size_t gemm_merge_smem_bytes() { return size_t(GEMM_MERGE_BUF + GEMM_MAX_RESCORE + GEMM_MAX_LIMIT) * 8; }

__global__ void __launch_bounds__(512, 2) emb_gemm_merge_kernel(const GemmMergeParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *buf = reinterpret_cast<uint64_t *>(smem);          // [GEMM_MERGE_BUF] gathered approximate keys
    uint64_t *exact = buf + GEMM_MERGE_BUF;                       // [GEMM_MAX_RESCORE] filtered keys, then exact keys
    uint64_t *sel = exact + GEMM_MAX_RESCORE;                     // [GEMM_MAX_LIMIT]
    __shared__ uint32_t s_cnt, s_m, s_off[512];
    __shared__ unsigned int s_alim;
    const uint32_t q = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint64_t *src = p.cand + size_t(q) * p.n_lists * p.cap;
    const uint32_t *cnts = p.cand_cnt + size_t(q) * p.n_lists;
    const uint64_t *osrc = p.ovf + size_t(q) * p.ovf_cap;
    const uint32_t n_ovf_raw = p.ovf_cnt[q];
    bool lost = n_ovf_raw > p.ovf_cap;                            // a spill did not fit: candidates are missing
    const uint32_t n_ovf = min(n_ovf_raw, p.ovf_cap);
    // ---- gather: exclusive scan of the list lengths (host guarantees n_lists <= 512), then the spill area
    uint32_t nv;
    {
        const uint32_t mine = (tid < p.n_lists) ? min(cnts[tid], p.cap) : 0u;
        uint32_t tot;
        const uint32_t off = block_exclusive_scan(mine, &tot);
        s_off[tid] = off;
        nv = tot + n_ovf;
    }
    if (tid == 0) { s_cnt = 0; s_m = 0; s_alim = 0; }
    __syncthreads();
    const bool in_smem = nv <= GEMM_MERGE_BUF;
    const float eps_v = p.eps_v[q];
    float a_lim = -INFINITY;                                      // limit-th best approximate score (if there are that many)
    if (in_smem) {
        for (uint32_t l = tid; l < p.n_lists; l += blockDim.x) {
            const uint32_t c = min(cnts[l], p.cap), o = s_off[l];
            for (uint32_t k = 0; k < c; k++) buf[o + k] = src[size_t(l) * p.cap + k];
        }
        for (uint32_t i = tid; i < n_ovf; i += blockDim.x) buf[nv - n_ovf + i] = osrc[i];
        __syncthreads();
        if (nv >= p.limit) {
            const uint32_t got = block_select_largest(buf, nv, p.limit, sel);   // unsorted
            uint64_t mn = ~0ull;
            for (uint32_t i = tid; i < got; i += blockDim.x) mn = min(mn, sel[i]);
            for (int o = 16; o > 0; o >>= 1) mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            if (lane == 0 && mn != ~0ull) atomicMax(&s_alim, ~uint32_t(mn >> 32));   // min of keys == max of complemented score bits
            __syncthreads();
            a_lim = f32_unordered(~s_alim);
        }
    } else {
        // too many candidates for shared memory (degenerate thresholds): stream them
        const uint64_t total = uint64_t(p.n_lists) * p.cap + n_ovf;
        const uint32_t got = block_topn_stream(buf, GEMM_MERGE_BUF, p.limit, total, [&](uint64_t i) -> uint64_t {
            if (i >= uint64_t(p.n_lists) * p.cap) return osrc[i - uint64_t(p.n_lists) * p.cap];
            const uint32_t l = uint32_t(i / p.cap), k = uint32_t(i % p.cap);
            return k < min(cnts[l], p.cap) ? src[i] : KEY_NONE;
        });
        if (got == p.limit) a_lim = key_score(buf[p.limit - 1]);
        __syncthreads();
    }
    // ---- filter: only rows with approx >= a_lim - 2 eps can reach the exact top-`limit`
    const float cut = (a_lim == -INFINITY) ? -INFINITY : a_lim - 2.0f * eps_v;   // eps_v = inf (zero query) -> -inf
    auto stage = [&](uint64_t k) {
        if (k != KEY_NONE && key_score(k) >= cut) {
            const uint32_t s = atomicAdd(&s_m, 1u);
            if (s < GEMM_MAX_RESCORE) exact[s] = k;
        }
    };
    if (in_smem) {
        for (uint32_t i = tid; i < nv; i += blockDim.x) stage(buf[i]);
    } else {
        for (uint32_t l = warp; l < p.n_lists; l += blockDim.x / 32) {
            const uint32_t c = min(cnts[l], p.cap);
            for (uint32_t k = lane; k < c; k += 32) stage(src[size_t(l) * p.cap + k]);
        }
        for (uint32_t i = tid; i < n_ovf; i += blockDim.x) stage(osrc[i]);
    }
    __syncthreads();
    const uint32_t m_raw = s_m;
    if (m_raw > GEMM_MAX_RESCORE) lost = true;
    const uint32_t M = min(m_raw, GEMM_MAX_RESCORE);
    // ---- exact fp32 re-score, one warp per candidate, K1's lane layout and FMA order
    const float iqn = p.inv_qnorm[q];
    const float4 *qp = reinterpret_cast<const float4 *>(p.queries + size_t(q) * p.stride);
    for (uint32_t i = warp; i < M; i += blockDim.x / 32) {
        const uint32_t row = key_idx(exact[i]);
        const void *rp = static_cast<const uint8_t *>(p.rows) + size_t(row) * p.stride * (p.rows_bf16 ? 2 : 4);
        // all row loads are issued before the first use (the rows were streamed evict-first: DRAM latency)
        float4 xr[8];
        const uint32_t nch = p.stride / 128;   // <= 8
#pragma unroll
        for (uint32_t j = 0; j < 8; j++)
            if (j < nch) xr[j] = p.rows_bf16 ? RowLoad<bf16_t>::ld(rp, lane + 32 * j) : RowLoad<float>::ld(rp, lane + 32 * j);
        float acc = 0.f;
#pragma unroll
        for (uint32_t j = 0; j < 8; j++)
            if (j < nch) {
                const float4 x = xr[j], y = qp[lane + 32 * j];
                acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
            }
        const float kf = cos_rank_key(warp_sum(acc), p.inv_norm[row], iqn);
        __syncwarp();
        if (lane == 0) exact[i] = make_key(kf, row);
    }
    __syncthreads();
    // ---- rank the exact keys: sort all when few, else select the best `limit` and sort those
    const uint32_t n_top = min(M, p.limit);
    if (M <= 256) {
        const uint32_t np2 = max(32u, next_pow2(M));
        for (uint32_t i = M + tid; i < np2; i += blockDim.x) exact[i] = KEY_NONE;
        group_bitonic_desc(exact, np2, tid, blockDim.x, 0);
    } else {
        for (uint32_t i = tid; i < GEMM_MAX_LIMIT; i += blockDim.x) sel[i] = KEY_NONE;
        __syncthreads();
        block_select_largest(exact, M, p.limit, sel);
        group_bitonic_desc(sel, GEMM_MAX_LIMIT, tid, blockDim.x, 0);
        for (uint32_t i = tid; i < GEMM_MAX_LIMIT; i += blockDim.x) exact[i] = sel[i];
        __syncthreads();
    }
    const uint32_t n_mine = p.q_limit ? min(n_top, p.q_limit[q]) : n_top;
    const float similarity = p.q_sim ? p.q_sim[q] : p.similarity;
    for (uint32_t i = tid; i < p.limit; i += blockDim.x) {
        uint64_t doc = 0; float score = 0.f, raw = 0.f; uint32_t row = 0xffffffffu;
        if (i < n_mine) {
            const uint64_t k = exact[i];
            const uint32_t r = key_idx(k);
            const float distance = -key_score(k);
            const float sim = 1.0f - distance;
            const float sc = rescale_score(sim, p.rescale_e5);
            if (sc >= similarity) {
                doc = p.row_doc_ids ? p.row_doc_ids[r] : uint64_t(r);
                score = sc; row = r; raw = key_score(k);
                atomicAdd(&s_cnt, 1u);
            }
        }
        p.out_doc[size_t(q) * p.limit + i] = doc;
        p.out_score[size_t(q) * p.limit + i] = score;
        if (p.out_row) p.out_row[size_t(q) * p.limit + i] = row;
        if (p.out_raw) p.out_raw[size_t(q) * p.limit + i] = raw;
    }
    __syncthreads();
    if (tid == 0) {
        p.out_count[q] = s_cnt;
        p.out_unproven[q] = lost ? 1 : 0;
        if (p.out_rescored) p.out_rescored[q] = M;
    }
}

// Threshold pass, step 2.  Every list of the threshold pass reported the best approximate score of a
// disjoint group of rows; the limit-th largest of those group maxima is attained by `limit` distinct rows,
// hence a valid lower bound LB of the query's global limit-th best approximate score — in the same
// arithmetic the sweep compares with.  The sweep gathers every row above thr = LB - 2 eps (see the merge).
// eps (cosine) = eps_const + rho_q (bf16: the rows enter the sweep exactly, rho_x = 0), scaled to the sweep's cos*|q|
// units (times 2^e_q for the fp16 sweep).
struct GemmThrParams {
    const float *gmax; uint32_t lists, limit;
    const float *inv_qnorm;
    float eps_const;
    const float *rho_q;       // [B] relative bf16 residual norm of each query, or NULL
    unsigned int *thr;        // [B] out: seed threshold, order-preserving uint (atomicMax'ed by the sweep)
    float *eps_v;             // [B] out
    uint32_t *ovf_cnt;        // [B] reset here: the spill cursors of the sweep that follows
    const float *q_scale;     // [B] GEMM_F16: the power of two 2^e_q the fp16 query was scaled by (the sweep's scores, hence
                              // gmax and thr, are in cos*|q|*2^e_q units: eps_v is scaled alike), or NULL
};
__global__ void __launch_bounds__(256) gemm_thr_kernel(const GemmThrParams p) {
    __shared__ uint64_t keys[512];
    const uint32_t q = blockIdx.x, tid = threadIdx.x;
    const uint32_t n = min(p.lists, 512u), np2 = max(64u, next_pow2(n));
    for (uint32_t i = tid; i < np2; i += blockDim.x) {
        const float v = i < n ? p.gmax[size_t(q) * p.lists + i] : -INFINITY;
        keys[i] = (v == v && v > -INFINITY) ? make_key(v, i) : KEY_NONE;
    }
    group_bitonic_desc(keys, np2, tid, blockDim.x, 0);
    if (tid == 0) {
        const float rq = p.rho_q ? fminf(p.rho_q[q], GEMM_RHO_BF16_WORST) : 0.f;
        const float eps_cos = p.eps_const + rq;
        const float iqn = p.inv_qnorm[q];
        float ev = iqn > 0.f ? __fdiv_ru(eps_cos, iqn) : INFINITY;
        if (p.q_scale) ev *= p.q_scale[q];                     // a power of two: exact
        float thr = -INFINITY;
        if (n >= p.limit && keys[p.limit - 1] != KEY_NONE && ev < INFINITY) thr = key_score(keys[p.limit - 1]) - 2.0f * ev;
        p.thr[q] = f32_ordered(thr);
        p.eps_v[q] = ev;
        p.ovf_cnt[q] = 0u;
    }
}

// fp32 -> bf16 (round to nearest even) of the padded queries: the B operand of the bf16 sweep
__global__ void f32_to_bf16_kernel(const float *in, uint16_t *out, size_t n) {
    const size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t u = __float_as_uint(in[i]);
    const uint32_t r = ((u & 0x7fffffffu) > 0x7f800000u) ? (u | 0x00400000u) : (u + 0x7fffu + ((u >> 16) & 1u));
    out[i] = uint16_t(r >> 16);
}

// ---- fp16 operands of the GEMM_F16 sweep ----
// One warp: out[i] = fp16_rn(v[i] * 2^s) for i < n, s chosen so that the largest |v_i| * 2^s lies in [2^14, 2^15)
// (the scaling is exact; nothing overflows, and rounding to nearest loses at most 2^-11 relative per component).
// Returns s; 0 for an all-zero vector; F16_NONFINITE (and NaN in every element) when some v_i is inf or NaN.
constexpr int F16_NONFINITE = -0x10000;
__device__ __forceinline__ int f16_scaled_copy_warp(const float *v, uint32_t n, uint16_t *out, uint32_t lane) {
    uint32_t mx = 0;   // largest |v_i| as bits: inf and NaN compare above every finite value
    for (uint32_t j = lane; j < n; j += 32) mx = max(mx, __float_as_uint(v[j]) & 0x7fffffffu);
    mx = __reduce_max_sync(0xffffffffu, mx);
    if (mx >= 0x7f800000u) {
        for (uint32_t j = lane; j < n; j += 32) out[j] = 0x7e00u;
        return F16_NONFINITE;
    }
    int s = 0;
    if (mx) {   // floor(log2 max|v_i|), subnormal maxima included
        const int k = mx >= 0x00800000u ? int(mx >> 23) - 127 : (31 - __clz(int(mx))) - 149;
        s = 14 - k;
    }
    for (uint32_t j = lane; j < n; j += 32) out[j] = __half_as_ushort(__float2half_rn(scalbnf(v[j], s)));
    return s;
}
// Rows [row_begin, row_end) of an fp32 store -> their fp16 copy and row_scale = 2^-s (one warp per row).  A row with a
// non-finite element gets a NaN scale, so its inverse norm in the sweep is NaN and the row is never gathered.
__global__ void emb_f16_rows_kernel(const float *rows, uint32_t stride, uint64_t row_begin, uint64_t row_end,
                                    uint16_t *rows_f16, float *row_scale) {
    const uint64_t r = row_begin + (uint64_t(blockIdx.x) * blockDim.x + threadIdx.x) / 32;
    if (r >= row_end) return;
    const uint32_t lane = threadIdx.x & 31;
    const int s = f16_scaled_copy_warp(rows + r * stride, stride, rows_f16 + r * stride, lane);
    if (lane == 0) row_scale[r] = s == F16_NONFINITE ? __int_as_float(0x7fc00000) : scalbnf(1.0f, -s);
}
// Padded fp32 queries [nq][stride] -> the fp16 query operand and q_scale = 2^s (one warp per query).  A query with a
// non-finite element keeps scale 1 and NaN operands: all its scores are NaN and nothing is gathered, as in the tf32 sweep.
__global__ void emb_f16_queries_kernel(const float *q_pad, uint32_t stride, uint32_t nq, uint16_t *q_f16, float *q_scale) {
    const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
    if (q >= nq) return;
    const int s = f16_scaled_copy_warp(q_pad + size_t(q) * stride, stride, q_f16 + size_t(q) * stride, lane);
    if (lane == 0) q_scale[q] = s == F16_NONFINITE ? 1.0f : scalbnf(1.0f, s);
}

// copies the exact-path results of re-run queries into their slots of the batch outputs
__global__ void scatter_rows_kernel(const uint32_t *qmap, uint32_t n, uint32_t limit, const uint64_t *sdoc,
                                    const float *sscore, const uint32_t *srow, const uint32_t *scnt, const float *sraw,
                                    uint64_t *ddoc, float *dscore, uint32_t *drow, uint32_t *dcnt, float *draw) {
    const uint32_t i = blockIdx.x, t = threadIdx.x;
    if (i >= n) return;
    const uint32_t q = qmap[i];
    for (uint32_t k = t; k < limit; k += blockDim.x) {
        ddoc[size_t(q) * limit + k] = sdoc[size_t(i) * limit + k];
        dscore[size_t(q) * limit + k] = sscore[size_t(i) * limit + k];
        drow[size_t(q) * limit + k] = srow[size_t(i) * limit + k];
        draw[size_t(q) * limit + k] = sraw[size_t(i) * limit + k];
    }
    if (t == 0) dcnt[q] = scnt[i];
}

}  // namespace oc
