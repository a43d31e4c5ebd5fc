// Test-only entry points into the K2 kernels of emb_gemm.cuh (the batched tensor-core embedding scan).
// Not part of the library's ABI: the tests load this through ctypes to run one kernel at a time on inputs
// they build themselves — the sweep with its approximate scores dumped (emb_gemm_kernel<BF16, true>), the
// threshold kernel and the merge kernel — and compare the results with numpy restatements.
// Every function takes and returns host arrays, runs synchronously and returns 0 or -1 (h_last_error()).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <vector>

#include "emb_gemm.cuh"
#include "emb_scan.cuh"
#include "tmap.cuh"

using namespace oc;

static char g_err[512] = "";
#define HC(x)                                                                                             \
    do {                                                                                                  \
        cudaError_t _e = (x);                                                                             \
        if (_e != cudaSuccess) {                                                                          \
            snprintf(g_err, sizeof(g_err), "%s: %s (line %d)", #x, cudaGetErrorString(_e), __LINE__);   \
            return -1;                                                                                    \
        }                                                                                                 \
    } while (0)

// device copies freed on scope exit
struct Dev {
    std::vector<void *> ptrs;
    ~Dev() { for (void *p : ptrs) cudaFree(p); }
    template <typename T> T *alloc(size_t n) {
        void *p = nullptr;
        if (cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)) != cudaSuccess) return nullptr;
        ptrs.push_back(p);
        return static_cast<T *>(p);
    }
};
#define HALLOC(var, T, n, dev)                                                          \
    T *var = (dev).alloc<T>(n);                                                         \
    if (!var) { snprintf(g_err, sizeof(g_err), "cudaMalloc %s failed", #var); return -1; }
#define HUP(var, T, n, dev, src)                                                        \
    HALLOC(var, T, n, dev);                                                             \
    HC(cudaMemcpy(var, src, (n) * sizeof(T), cudaMemcpyHostToDevice))

extern "C" const char *h_last_error(void) { return g_err; }

extern "C" void h_constants(uint32_t *out) {
    out[0] = GEMM_M; out[1] = GEMM_N; out[2] = GEMM_KB; out[3] = GEMM_STAGES; out[4] = GEMM_LIST_CAP;
    out[5] = GEMM_OVF_CAP; out[6] = GEMM_MERGE_BUF; out[7] = GEMM_MAX_RESCORE; out[8] = GEMM_MAX_LIMIT;
    out[9] = GEMM_LISTS_PER_CTA;
}

// Library query preparation (emb_prep_queries_kernel): zero padding, 1 / |q| and the bf16 residual rho_q.
extern "C" int h_prep_queries(const float *q, uint32_t dim, uint32_t stride, uint32_t nq, float *q_pad, float *inv_qnorm,
                              float *rho_q) {
    Dev dv;
    HUP(d_q, float, size_t(nq) * dim, dv, q);
    HALLOC(d_pad, float, size_t(nq) * stride, dv);
    HALLOC(d_inv, float, nq, dv);
    HALLOC(d_rho, float, nq, dv);
    emb_prep_queries_kernel<<<(nq + 7) / 8, 256>>>(d_q, dim, stride, nq, d_pad, d_inv, d_rho);
    HC(cudaGetLastError());
    HC(cudaMemcpy(q_pad, d_pad, size_t(nq) * stride * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(inv_qnorm, d_inv, nq * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(rho_q, d_rho, nq * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// The sweep with DUMP = true.  rows: [n_rows][stride] (fp32, or bf16 bits when bf16); queries: [Bpad][stride] in the
// same element type, Bpad = ceil(B / 128) * 128 (the library pads with zero rows); inv_norm: [n_rows] (NaN = dead row).
// cpg: CTAs per query group (0 = the library's choice, one CTA per SM).  dump: [dump_len] floats, copied to the
// device first (the caller pre-fills a sentinel) and back after the sweep.
extern "C" int h_gemm_dump(const void *rows, const float *inv_norm, uint64_t n_rows, uint32_t stride, int bf16,
                           const void *queries, uint32_t B, uint32_t cpg, float *dump, size_t dump_len) {
    const size_t esz = bf16 ? 2 : 4;
    const uint32_t n_qgroups = (B + GEMM_M - 1) / GEMM_M, Bpad = n_qgroups * GEMM_M;
    if (dump_len < size_t(B) * n_rows) { snprintf(g_err, sizeof(g_err), "dump too small"); return -1; }
    int dev = 0, sms = 0;
    HC(cudaGetDevice(&dev));
    HC(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (cpg == 0) cpg = std::min<uint32_t>(512 / GEMM_LISTS_PER_CTA, std::max<uint32_t>(1, uint32_t(sms) / n_qgroups));
    Dev dv;
    HUP(d_rows, uint8_t, n_rows * stride * esz, dv, rows);
    HUP(d_inv, float, n_rows, dv, inv_norm);
    HUP(d_q, uint8_t, size_t(Bpad) * stride * esz, dv, queries);
    HUP(d_dump, float, dump_len, dv, dump);
    CUtensorMap tm_q, tm_x;
    for (auto s : {make_tmap_2d(&tm_q, d_q, Bpad, stride, GEMM_M, bf16), make_tmap_2d(&tm_x, d_rows, n_rows, stride, GEMM_N, bf16)})
        if (s.what) { snprintf(g_err, sizeof(g_err), "%s failed: %d", s.what, s.code); return -1; }
    GemmDumpParams gp{};
    gp.n_rows = n_rows; gp.n_kblocks = stride / (bf16 ? 2 * GEMM_KB : GEMM_KB); gp.inv_norm = d_inv; gp.n_queries = B;
    gp.n_qgroups = n_qgroups; gp.ctas_per_group = cpg; gp.cap = GEMM_LIST_CAP; gp.lists_per_query = cpg * GEMM_LISTS_PER_CTA;
    gp.limit = 1; gp.dump = d_dump;
    const size_t smem = gemm_smem_bytes();
    if (bf16) {
        HC(cudaFuncSetAttribute(emb_gemm_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
        emb_gemm_kernel<true, true><<<cpg * n_qgroups, GEMM_THREADS, smem>>>(tm_q, tm_x, gp);
    } else {
        HC(cudaFuncSetAttribute(emb_gemm_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
        emb_gemm_kernel<false, true><<<cpg * n_qgroups, GEMM_THREADS, smem>>>(tm_q, tm_x, gp);
    }
    HC(cudaGetLastError());
    HC(cudaDeviceSynchronize());
    HC(cudaMemcpy(dump, d_dump, dump_len * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// gemm_thr_kernel on group maxima gmax [B][lists]; rho_q may be NULL.  ovf_cnt_out receives the reset spill cursors
// (pre-filled on the device with 0xffffffff).
extern "C" int h_gemm_thr(const float *gmax, uint32_t B, uint32_t lists, uint32_t limit, const float *inv_qnorm,
                          float eps_const, const float *rho_q, uint32_t *thr_out, float *eps_out, uint32_t *ovf_cnt_out) {
    Dev dv;
    HUP(d_gmax, float, size_t(B) * lists, dv, gmax);
    HUP(d_iqn, float, B, dv, inv_qnorm);
    float *d_rho = nullptr;
    if (rho_q) { HUP(r, float, B, dv, rho_q); d_rho = r; }
    HALLOC(d_thr, uint32_t, B, dv);
    HALLOC(d_eps, float, B, dv);
    HALLOC(d_ovf, uint32_t, B, dv);
    HC(cudaMemset(d_ovf, 0xff, size_t(B) * 4));
    GemmThrParams tp{};
    tp.gmax = d_gmax; tp.lists = lists; tp.limit = limit; tp.inv_qnorm = d_iqn; tp.eps_const = eps_const; tp.rho_q = d_rho;
    tp.thr = d_thr; tp.eps_v = d_eps; tp.ovf_cnt = d_ovf;
    gemm_thr_kernel<<<B, 256>>>(tp);
    HC(cudaGetLastError());
    HC(cudaMemcpy(thr_out, d_thr, size_t(B) * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(eps_out, d_eps, size_t(B) * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(ovf_cnt_out, d_ovf, size_t(B) * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// emb_gemm_merge_kernel on candidate lists cand [B][n_lists][cap] (cand_cnt [B][n_lists]) and spill areas
// ovf [B][ovf_cap] (ovf_cnt [B], may exceed ovf_cap).  rows: the store [n_rows][stride] (fp32 or bf16 bits),
// queries: padded fp32 [B][stride].  Documents are row indices.  Outputs: [B][limit] doc / score / row / raw,
// [B] count / unproven / rescored.
extern "C" int h_gemm_merge(const uint64_t *cand, const uint32_t *cand_cnt, uint32_t B, uint32_t n_lists, uint32_t cap,
                            const uint64_t *ovf, const uint32_t *ovf_cnt, uint32_t ovf_cap, const float *eps_v,
                            uint32_t limit, const void *rows, int rows_bf16, uint64_t n_rows, uint32_t stride,
                            const float *inv_norm, const float *queries, const float *inv_qnorm, int rescale_e5,
                            float similarity, uint64_t *out_doc, float *out_score, uint32_t *out_row, float *out_raw,
                            uint32_t *out_count, uint8_t *out_unproven, uint32_t *out_rescored) {
    if (n_lists > 512 || limit > GEMM_MAX_LIMIT) { snprintf(g_err, sizeof(g_err), "n_lists > 512 or limit > %u", GEMM_MAX_LIMIT); return -1; }
    const size_t esz = rows_bf16 ? 2 : 4;
    Dev dv;
    HUP(d_cand, uint64_t, size_t(B) * n_lists * cap, dv, cand);
    HUP(d_cnt, uint32_t, size_t(B) * n_lists, dv, cand_cnt);
    HUP(d_ovf, uint64_t, size_t(B) * ovf_cap, dv, ovf);
    HUP(d_ovfcnt, uint32_t, B, dv, ovf_cnt);
    HUP(d_eps, float, B, dv, eps_v);
    HUP(d_rows, uint8_t, n_rows * stride * esz, dv, rows);
    HUP(d_inv, float, n_rows, dv, inv_norm);
    HUP(d_q, float, size_t(B) * stride, dv, queries);
    HUP(d_iqn, float, B, dv, inv_qnorm);
    HALLOC(d_doc, uint64_t, size_t(B) * limit, dv);
    HALLOC(d_score, float, size_t(B) * limit, dv);
    HALLOC(d_row, uint32_t, size_t(B) * limit, dv);
    HALLOC(d_raw, float, size_t(B) * limit, dv);
    HALLOC(d_count, uint32_t, B, dv);
    HALLOC(d_unp, uint8_t, B, dv);
    HALLOC(d_resc, uint32_t, B, dv);
    GemmMergeParams mp{};
    mp.cand = d_cand; mp.cand_cnt = d_cnt; mp.n_lists = n_lists; mp.cap = cap;
    mp.ovf = d_ovf; mp.ovf_cnt = d_ovfcnt; mp.ovf_cap = ovf_cap; mp.eps_v = d_eps; mp.limit = limit;
    mp.rows = d_rows; mp.rows_bf16 = rows_bf16; mp.stride = stride; mp.inv_norm = d_inv; mp.queries = d_q;
    mp.inv_qnorm = d_iqn; mp.row_doc_ids = nullptr; mp.rescale_e5 = rescale_e5; mp.similarity = similarity;
    mp.out_doc = d_doc; mp.out_score = d_score; mp.out_row = d_row; mp.out_count = d_count; mp.out_raw = d_raw;
    mp.out_unproven = d_unp; mp.out_rescored = d_resc;
    HC(cudaFuncSetAttribute(emb_gemm_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(gemm_merge_smem_bytes())));
    emb_gemm_merge_kernel<<<B, 512, gemm_merge_smem_bytes()>>>(mp);
    HC(cudaGetLastError());
    HC(cudaMemcpy(out_doc, d_doc, size_t(B) * limit * 8, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(out_score, d_score, size_t(B) * limit * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(out_row, d_row, size_t(B) * limit * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(out_raw, d_raw, size_t(B) * limit * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(out_count, d_count, size_t(B) * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(out_unproven, d_unp, B, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(out_rescored, d_resc, size_t(B) * 4, cudaMemcpyDeviceToHost));
    return 0;
}
