// Test-only entry points into the fp16 sweep of an fp32 store (emb_gemm.cuh, GEMM_F16): the library's fp16 operands
// (emb_f16_rows_kernel, emb_f16_queries_kernel), the sweep with its approximate scores dumped
// (emb_gemm_kernel<GEMM_F16, true>) and the threshold kernel with the queries' scales.  Not part of the library's ABI:
// tests/test_gpu_gemm_f16_numerics.py loads this through ctypes next to libgemm_harness.so.
// Every function takes and returns host arrays, runs synchronously and returns 0 or -1 (h16_last_error()).
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

extern "C" const char *h16_last_error(void) { return g_err; }

// The library's fp16 operands of fp32 vectors [n][stride]: the store's copy (emb_f16_rows_kernel, scale = 2^-s) when
// is_query == 0, the query operand (emb_f16_queries_kernel, scale = 2^s) otherwise.  out: [n][stride] fp16 bits.
extern "C" int h16_operands(const float *v, uint64_t n, uint32_t stride, int is_query, uint16_t *out, float *scale) {
    Dev dv;
    HUP(d_v, float, n * stride, dv, v);
    HALLOC(d_out, uint16_t, n * stride, dv);
    HALLOC(d_scale, float, n, dv);
    const unsigned blocks = unsigned((n + 7) / 8);
    if (is_query) emb_f16_queries_kernel<<<blocks, 256>>>(d_v, stride, uint32_t(n), d_out, d_scale);
    else emb_f16_rows_kernel<<<blocks, 256>>>(d_v, stride, 0, n, d_out, d_scale);
    HC(cudaGetLastError());
    HC(cudaMemcpy(out, d_out, n * stride * 2, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(scale, d_scale, n * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// The fp16 sweep with DUMP = true.  rows_f16: [n_rows][stride] fp16 bits, row_scale / inv_norm: [n_rows] (NaN inverse
// norm = dead row); q_f16: [Bpad][stride] fp16 bits, Bpad = ceil(B / 128) * 128.  cpg: CTAs per query group (0 = the
// library's choice, one CTA per SM).  dump: [dump_len] floats, copied to the device first (the caller pre-fills a
// sentinel) and back after the sweep.
extern "C" int h16_gemm_dump(const uint16_t *rows_f16, const float *inv_norm, const float *row_scale, uint64_t n_rows,
                             uint32_t stride, const uint16_t *q_f16, uint32_t B, uint32_t cpg, float *dump, size_t dump_len) {
    const uint32_t n_qgroups = (B + GEMM_M - 1) / GEMM_M, Bpad = n_qgroups * GEMM_M;
    if (dump_len < size_t(B) * n_rows) { snprintf(g_err, sizeof(g_err), "dump too small"); return -1; }
    int dev = 0, sms = 0;
    HC(cudaGetDevice(&dev));
    HC(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (cpg == 0) cpg = std::min<uint32_t>(512 / GEMM_LISTS_PER_CTA, std::max<uint32_t>(1, uint32_t(sms) / n_qgroups));
    Dev dv;
    HUP(d_rows, uint16_t, n_rows * stride, dv, rows_f16);
    HUP(d_inv, float, n_rows, dv, inv_norm);
    HUP(d_scale, float, n_rows, dv, row_scale);
    HUP(d_q, uint16_t, size_t(Bpad) * stride, dv, q_f16);
    HUP(d_dump, float, dump_len, dv, dump);
    CUtensorMap tm_q, tm_x;
    for (auto s : {make_tmap_2d(&tm_q, d_q, Bpad, stride, GEMM_M, GEMM_F16),
                   make_tmap_2d(&tm_x, d_rows, n_rows, stride, GEMM_N, GEMM_F16)})
        if (s.what) { snprintf(g_err, sizeof(g_err), "%s failed: %d", s.what, s.code); return -1; }
    GemmDumpParams gp{};
    gp.n_rows = n_rows; gp.n_kblocks = stride / (2 * GEMM_KB); gp.inv_norm = d_inv; gp.n_queries = B;
    gp.n_qgroups = n_qgroups; gp.ctas_per_group = cpg; gp.cap = GEMM_LIST_CAP; gp.lists_per_query = cpg * GEMM_LISTS_PER_CTA;
    gp.limit = 1; gp.dump = d_dump; gp.row_scale = d_scale;
    const size_t smem = gemm_smem_bytes();
    HC(cudaFuncSetAttribute(emb_gemm_kernel<GEMM_F16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    emb_gemm_kernel<GEMM_F16, true><<<cpg * n_qgroups, GEMM_THREADS, smem>>>(tm_q, tm_x, gp);
    HC(cudaGetLastError());
    HC(cudaDeviceSynchronize());
    HC(cudaMemcpy(dump, d_dump, dump_len * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// gemm_thr_kernel for the fp16 sweep on group maxima gmax [B][lists]: q_scale [B] = the queries' 2^e_q (h16_operands
// with is_query = 1).  ovf_cnt_out receives the reset spill cursors (pre-filled on the device with 0xffffffff).
extern "C" int h16_gemm_thr(const float *gmax, uint32_t B, uint32_t lists, uint32_t limit, const float *inv_qnorm,
                            float eps_const, const float *q_scale, uint32_t *thr_out, float *eps_out, uint32_t *ovf_cnt_out) {
    Dev dv;
    HUP(d_gmax, float, size_t(B) * lists, dv, gmax);
    HUP(d_iqn, float, B, dv, inv_qnorm);
    HUP(d_qs, float, B, dv, q_scale);
    HALLOC(d_thr, uint32_t, B, dv);
    HALLOC(d_eps, float, B, dv);
    HALLOC(d_ovf, uint32_t, B, dv);
    HC(cudaMemset(d_ovf, 0xff, size_t(B) * 4));
    GemmThrParams tp{};
    tp.gmax = d_gmax; tp.lists = lists; tp.limit = limit; tp.inv_qnorm = d_iqn; tp.eps_const = eps_const; tp.rho_q = nullptr;
    tp.q_scale = d_qs; tp.thr = d_thr; tp.eps_v = d_eps; tp.ovf_cnt = d_ovf;
    gemm_thr_kernel<<<B, 256>>>(tp);
    HC(cudaGetLastError());
    HC(cudaMemcpy(thr_out, d_thr, size_t(B) * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(eps_out, d_eps, size_t(B) * 4, cudaMemcpyDeviceToHost));
    HC(cudaMemcpy(ovf_cnt_out, d_ovf, size_t(B) * 4, cudaMemcpyDeviceToHost));
    return 0;
}
