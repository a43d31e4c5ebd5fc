// tmap.cuh — TMA tensor maps of the K2 sweep's operands (emb_gemm.cuh), shared by the library and the
// kernel test harness so that both hand the sweep byte-identical descriptors.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "emb_gemm.cuh"

namespace oc {

// The driver entry point is fetched through the runtime: no -lcuda link.
typedef CUresult (*EncodeTiled_t)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct TmapStatus {
    const char *what;   // nullptr on success, else the step that failed
    int code;           // its cudaError_t / CUresult
};

// [n_rows][stride] row-major matrix of the sweep's operand kind `op` (GemmOp: fp32, bf16 or fp16 elements), boxes of
// 128 bytes of K x box_rows rows, SWIZZLE_128B (the layout wgmma_desc_sw128 describes); rows past n_rows read as zeros.
inline TmapStatus make_tmap_2d(CUtensorMap *m, const void *base, uint64_t n_rows, uint32_t stride, uint32_t box_rows,
                               int op) {
    static EncodeTiled_t fn = nullptr;
    if (!fn) {
        void *f = nullptr;
        cudaDriverEntryPointQueryResult qr;
        const cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qr);
        if (e != cudaSuccess) return {"cudaGetDriverEntryPoint(cuTensorMapEncodeTiled)", int(e)};
        if (!f || qr != cudaDriverEntryPointSuccess) return {"cuTensorMapEncodeTiled unavailable", int(qr)};
        fn = (EncodeTiled_t)f;
    }
    const bool half = op != GEMM_TF32;   // 16-bit elements
    const CUtensorMapDataType dt = op == GEMM_BF16  ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                   : op == GEMM_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                                    : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    cuuint64_t dims[2] = {stride, n_rows};
    cuuint64_t strides[1] = {cuuint64_t(stride) * (half ? 2 : 4)};
    cuuint32_t box[2] = {half ? 2 * GEMM_KB : GEMM_KB, box_rows};   // 128 bytes of K
    cuuint32_t estr[2] = {1, 1};
    // L2 promotion granule = the 128-byte box row: a larger granule would also pull the neighbouring K-block
    // of the row into L2, which another CTA's load may evict before it is used (extra DRAM reads)
    const CUtensorMapL2promotion promo = CU_TENSOR_MAP_L2_PROMOTION_L2_128B;
    CUresult r = fn(m, dt, 2, const_cast<void *>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return {"cuTensorMapEncodeTiled", int(r)};
    return {nullptr, 0};
}

}  // namespace oc
