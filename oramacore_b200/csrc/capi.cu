// capi.cu — host side of liboramacore_b200.so: the C ABI declared in
// include/oramacore_b200.h over the sm_90a kernels (emb_scan.cuh, bm25.cuh, fuse.cuh).
// No torch, no CPU fallback: every entry point needs a live CUDA device.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <limits>
#include <map>
#include <memory>
#include <mutex>
#include <utility>
#include <string>
#include <unordered_map>
#include <vector>

#include "bm25.cuh"
#include "comm.h"
#include "dict.h"
#include "stem_en.h"
#include "emb_gemm.cuh"
#include "emb_scan.cuh"
#include "fuse.cuh"
#include "geo.cuh"
#include "group.cuh"
#include "pins.cuh"
#include "sort.cuh"
#include "tmap.cuh"
#include "oramacore_b200.h"

using namespace oc;

// ------------------------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";
static int fail(int code, const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
#define CU(x)                                                                                   \
    do {                                                                                        \
        cudaError_t _e = (x);                                                                   \
        if (_e != cudaSuccess)                                                                  \
            return fail(_e == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "%s: %s (%s:%d)", #x, \
                        cudaGetErrorString(_e), __FILE__, __LINE__);                            \
    } while (0)
#define OCTRY(x)                \
    do {                        \
        int _r = (x);           \
        if (_r != OC_OK) return _r; \
    } while (0)

extern "C" const char *oc_last_error(void) { return g_err; }
extern "C" int oc_version(void) { return 100; }
extern "C" void oc_abi_sizes(size_t out[4]) {
    out[0] = sizeof(oc_search_params); out[1] = sizeof(oc_timing); out[2] = sizeof(oc_emb_info_t); out[3] = sizeof(oc_str_info_t);
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is per (device, function): remember what was configured
// per device so several contexts on different GPUs in one process each get their kernels configured
static bool smem_cfg_needed(int device, const void *fn, size_t smem) {
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, size_t> done;
    std::lock_guard<std::mutex> g(mu);
    size_t &v = done[std::make_pair(device, fn)];
    if (smem <= v) return false;
    v = smem;
    return true;
}

// ------------------------------------------------------------------------------------ buffers
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes) {
        if (bytes <= cap) return OC_OK;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { e = cudaMalloc(&p, bytes); want = bytes; }
        if (e != cudaSuccess) return fail(OC_ERR_OOM, "cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e));
        cap = want;
        return OC_OK;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <typename T> T *as() { return reinterpret_cast<T *>(p); }
};
struct HostBuf {  // pinned staging
    void *p = nullptr;
    size_t cap = 0;
    int ensure(size_t bytes) {
        if (bytes <= cap) return OC_OK;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e != cudaSuccess) return fail(OC_ERR_OOM, "cudaMallocHost(%zu): %s", want, cudaGetErrorString(e));
        cap = want;
        return OC_OK;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
    template <typename T> T *as() { return reinterpret_cast<T *>(p); }
};

// lays several host arrays out in one pinned blob -> one H2D copy (sources are copied once,
// straight into the pinned staging buffer)
struct Packer {
    struct Seg { const void *src; size_t off, bytes; bool direct; };
    std::vector<Seg> segs;
    size_t total = 0;
    // direct = the source already lives in pinned host memory (oc_pinned_alloc / cudaHostRegister):
    // it is DMA'd straight from the caller's buffer instead of being staged
    size_t add(const void *src, size_t bytes, bool direct = false) {
        const size_t off = (total + 255) & ~size_t(255);
        segs.push_back({src, off, bytes, direct});
        total = off + bytes;
        return off;
    }
    void fill(void *dst) const {
        for (const Seg &g : segs) if (g.bytes && g.src && !g.direct) memcpy(static_cast<uint8_t *>(dst) + g.off, g.src, g.bytes);
    }
};
static bool is_pinned_host(const void *p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

enum { EV_START, EV_H2D, EV_DEV, EV_D2H, EV_SCAN0, EV_SCAN1, EV_BM0, EV_BM1, EV_FUSE0, EV_FUSE1, EV_COMM0, EV_COMM1, EV_SWEEP0, EV_SWEEP1, EV_RR0, EV_RR1, EV_GRP0, EV_GRP1, EV_N };

constexpr size_t P2P_WIN_BYTES = size_t(1) << 20;   // per (parity, source rank): a batch's records must fit (256 queries x 520 B = 133 KB)
constexpr uint32_t P2P_MAX_Q = 4096;
constexpr size_t P2P_FLAG_BYTES = size_t(2) * P2P_MAX_Q * 4;
constexpr uint32_t P2P_MAX_WORLD = 16;

struct oc_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t side = nullptr;      // descriptor upload + BM25 plan/precompute while the main stream sweeps the matrix
    cudaEvent_t ev_side = nullptr;
    bool sweep_timed = false;         // EV_SWEEP0/1 recorded in this call (tensor-core path)
    bool rerun_timed = false;         // EV_RR0/1 recorded: flagged queries were re-run through the exact sweep
    bool side_dirty = false;          // work was queued on the side stream and not yet joined (an error path returned early)
    cudaDeviceProp prop{};
    std::mutex mu;
    cudaEvent_t ev[EV_N]{};
    oc_timing timing{};
    uint64_t launches = 0;
    uint32_t call_launches = 0, call_scan_launches = 0;
    // workspaces
    DevBuf in_blob, in_blob0, q_pad, q_inv, eff_norm, filter_dev, scan_cand, v_doc, v_score, v_row, v_cnt, v_srow, v_ft, v_present, v_raw;
    DevBuf seg, df_dev, row_ok, tau, cand_key, cand_ft, cand_cnt, tile_cnt, tile_max, tile_min, min_hint;
    DevBuf out_blob, shard_send, shard_recv, work_ctr, flat_desc, mbits, dbits, facet_req, facet_out;
    bool gemm_pending = false; const float *gemm_inv_norm = nullptr;
    DevBuf row_ft, grp_vdoc, grp_vscore, grp_vn, grp_gmin, grp_den, grp_doc, grp_score, grp_n;   // oc_search_groups
    DevBuf pin_row, pin_ft, pin_ftp, pin_score, pin_present, pin_top_doc, pin_top_score, pin_top_n, pin_gdoc, pin_gscore, pin_gn;   // pins
    DevBuf srt_doc, srt_row, srt_n, srt_ft, srt_ftp, srt_score, srt_present, srt_zero;   // sortBy
    DevBuf q_bf16, q_rho, pre_post, dense_buf, g_thr, g_eps, g_ovf, g_ovfcnt, g_resc, g_cand, g_cnt, g_flag, g_max, r_qpad, r_qinv, r_map, r_doc, r_score, r_row, r_cnt, r_raw;
    // per-query where-filters (q_filters): the embedding rows' bitmap of every distinct handle, and the slots of the
    // queries the exact sweep re-runs; v_qslot / v_rowbits describe the vector stage of the current call (fix_unproven)
    DevBuf e_rowbits, r_slot;
    const uint32_t *v_rowbits = nullptr; uint64_t v_row_words = 0;
    std::vector<uint32_t> v_qslot;

    HostBuf h_in, h_out, h_in0;   // h_in0 / in_blob0: query vectors + filter, uploaded before the descriptors
    OcComm comm;
    // direct NVLink exchange of the shard records (oc_comm_p2p_*): one IPC-shared window per rank —
    // [2 parities][P2P_MAX_Q] arrival counters, then [2 parities][world source ranks][P2P_WIN_BYTES] records
    struct P2P {
        bool ready = false;
        uint8_t *local = nullptr;
        uint8_t *peer[16] = {};      // peer[rank] == local
        uint64_t seq = 0;            // exchanges done (all ranks run the same batches): parity = seq & 1
    } p2p;
};

static inline void launched(oc_ctx *c, bool scan = false) {
    c->launches++; c->call_launches++;
    if (scan) c->call_scan_launches++;
}

extern "C" int oc_init(int device_id, oc_ctx **out) {
    if (!out) return fail(OC_ERR_INVALID, "oc_init: out is NULL");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(OC_ERR_CUDA, "no CUDA device: %s (this library has no CPU fallback)", cudaGetErrorString(e));
    if (device_id < 0 || device_id >= n) return fail(OC_ERR_INVALID, "device %d out of range (%d devices)", device_id, n);
    CU(cudaSetDevice(device_id));
    oc_ctx *c = new oc_ctx();
    c->device = device_id;
    CU(cudaGetDeviceProperties(&c->prop, device_id));
    if (c->prop.major != 9 || c->prop.minor != 0) {   // sm_90a code (wgmma) runs on sm_90 devices only
        int mj = c->prop.major, mn = c->prop.minor;
        delete c;
        return fail(OC_ERR_CUDA, "device sm_%d%d is not sm_90; kernels are built for sm_90a only", mj, mn);
    }
    CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CU(cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&c->ev_side, cudaEventDisableTiming));
    for (int i = 0; i < EV_N; i++) CU(cudaEventCreate(&c->ev[i]));
    *out = c;
    return OC_OK;
}

extern "C" void oc_shutdown(oc_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (int r = 0; r < 16; r++) if (c->p2p.ready && c->p2p.peer[r] && c->p2p.peer[r] != c->p2p.local) cudaIpcCloseMemHandle(c->p2p.peer[r]);
    if (c->p2p.local) cudaFree(c->p2p.local);
    c->comm.destroy();
    DevBuf *bufs[] = {&c->in_blob, &c->q_pad, &c->q_inv, &c->eff_norm, &c->filter_dev, &c->scan_cand, &c->v_doc,
                      &c->v_score, &c->v_row, &c->v_cnt, &c->v_srow, &c->v_ft, &c->v_present, &c->v_raw, &c->seg, &c->df_dev,
                      &c->row_ok, &c->tau, &c->cand_key, &c->cand_ft, &c->cand_cnt, &c->tile_cnt, &c->tile_max,
                      &c->tile_min, &c->min_hint, &c->out_blob, &c->shard_send, &c->shard_recv, &c->work_ctr, &c->flat_desc, &c->mbits, &c->dbits, &c->facet_req, &c->facet_out, &c->q_bf16, &c->q_rho, &c->pre_post, &c->dense_buf, &c->g_thr, &c->g_eps, &c->g_ovf, &c->g_ovfcnt, &c->g_resc, &c->g_cand, &c->g_cnt, &c->g_max,
                      &c->g_flag, &c->r_qpad, &c->r_qinv, &c->r_map, &c->r_doc, &c->r_score, &c->r_row, &c->r_cnt, &c->r_raw,
                      &c->row_ft, &c->grp_vdoc, &c->grp_vscore, &c->grp_vn, &c->grp_gmin, &c->grp_den, &c->grp_doc, &c->grp_score, &c->grp_n,
                      &c->pin_row, &c->pin_ft, &c->pin_ftp, &c->pin_score, &c->pin_present, &c->pin_top_doc, &c->pin_top_score,
                      &c->pin_top_n, &c->pin_gdoc, &c->pin_gscore, &c->pin_gn,
                      &c->srt_doc, &c->srt_row, &c->srt_n, &c->srt_ft, &c->srt_ftp, &c->srt_score, &c->srt_present, &c->srt_zero,
                      &c->e_rowbits, &c->r_slot};
    for (DevBuf *b : bufs) b->release();
    c->h_in.release(); c->h_out.release();
    for (int i = 0; i < EV_N; i++) if (c->ev[i]) cudaEventDestroy(c->ev[i]);
    cudaStreamDestroy(c->stream);
    if (c->side) cudaStreamDestroy(c->side);
    if (c->ev_side) cudaEventDestroy(c->ev_side);
    delete c;
}

extern "C" int oc_device_info(oc_ctx *c, int *sm_count, size_t *hbm_bytes, char *name, size_t name_cap) {
    if (!c) return fail(OC_ERR_INVALID, "ctx is NULL");
    if (sm_count) *sm_count = c->prop.multiProcessorCount;
    if (hbm_bytes) *hbm_bytes = c->prop.totalGlobalMem;
    if (name && name_cap) { strncpy(name, c->prop.name, name_cap - 1); name[name_cap - 1] = 0; }
    return OC_OK;
}

extern "C" int oc_pinned_alloc(size_t bytes, void **out) {
    if (!out) return fail(OC_ERR_INVALID, "out is NULL");
    CU(cudaMallocHost(out, bytes ? bytes : 1));
    return OC_OK;
}
extern "C" void oc_pinned_free(void *p) { if (p) cudaFreeHost(p); }

extern "C" int oc_last_timing(oc_ctx *c, oc_timing *out) {
    if (!c || !out) return fail(OC_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> g(c->mu);
    *out = c->timing;
    return OC_OK;
}
extern "C" uint64_t oc_launch_count(oc_ctx *c) { return c ? c->launches : 0; }

extern "C" int oc_comm_unique_id(uint8_t out_id[OC_COMM_ID_BYTES]) {
    std::string err;
    if (!OcComm::unique_id(out_id, &err)) return fail(OC_ERR_COMM, "%s", err.c_str());
    return OC_OK;
}
extern "C" int oc_comm_init(oc_ctx *c, int world, int rank, const uint8_t id[OC_COMM_ID_BYTES]) {
    if (!c || world < 1 || rank < 0 || rank >= world) return fail(OC_ERR_INVALID, "bad comm arguments");
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    std::string err;
    if (!c->comm.init(world, rank, id, &err)) return fail(OC_ERR_COMM, "%s", err.c_str());
    return OC_OK;
}

// Direct NVLink exchange: rank r exports the IPC handle of its window, the host runtime all-gathers the blobs (like
// the NCCL unique id) and every rank maps all peers' windows.  Afterwards the sharded oc_search stores each query's
// shard record straight into every rank's window from the pack kernel and the merge kernel waits on arrival
// counters — no library collective on the data path (ncclAllGather stays the fallback for batches larger than a window).
extern "C" int oc_comm_p2p_export(oc_ctx *c, uint8_t out[OC_P2P_HANDLE_BYTES]) {
    if (!c || !out) return fail(OC_ERR_INVALID, "NULL argument");
    if (c->comm.world < 2 || c->comm.world > (int)P2P_MAX_WORLD) return fail(OC_ERR_INVALID, "oc_comm_init first (2..%u ranks)", P2P_MAX_WORLD);
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    if (!c->p2p.local) {
        const size_t bytes = P2P_FLAG_BYTES + size_t(2) * c->comm.world * P2P_WIN_BYTES;
        CU(cudaMalloc(&c->p2p.local, bytes));
        CU(cudaMemset(c->p2p.local, 0, bytes));
    }
    cudaIpcMemHandle_t h;
    CU(cudaIpcGetMemHandle(&h, c->p2p.local));
    static_assert(sizeof(h) <= OC_P2P_HANDLE_BYTES, "handle blob");
    memset(out, 0, OC_P2P_HANDLE_BYTES);
    memcpy(out, &h, sizeof(h));
    return OC_OK;
}
extern "C" int oc_comm_p2p_import(oc_ctx *c, const uint8_t *handles) {
    if (!c || !handles) return fail(OC_ERR_INVALID, "NULL argument");
    if (!c->p2p.local) return fail(OC_ERR_INVALID, "oc_comm_p2p_export first");
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    for (int r = 0; r < c->comm.world; r++) {
        if (r == c->comm.rank) { c->p2p.peer[r] = c->p2p.local; continue; }
        cudaIpcMemHandle_t h;
        memcpy(&h, handles + size_t(r) * OC_P2P_HANDLE_BYTES, sizeof(h));
        void *ptr = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return fail(OC_ERR_COMM, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
        c->p2p.peer[r] = static_cast<uint8_t *>(ptr);
    }
    c->p2p.seq = 0;
    c->p2p.ready = true;
    return OC_OK;
}

// ------------------------------------------------------------------------------------ embedding store
struct oc_emb {
    oc_ctx *ctx;
    uint32_t dim, stride;
    int dtype, e5;
    void *rows = nullptr;        // [cap][stride] fp32 or bf16
    uint32_t esz = 4;            // element bytes
    float *inv_norm = nullptr;   // [cap] (NaN = tombstone)
    uint64_t *row_doc = nullptr; // [cap]
    uint64_t n_rows = 0, cap = 0, n_live = 0;
    std::unordered_multimap<uint64_t, uint64_t> doc_rows;  // doc -> rows (for delete)
};

extern "C" int oc_emb_create(oc_ctx *c, uint32_t dim, int dtype, int rescale_e5, oc_emb **out) {
    if (!c || !out) return fail(OC_ERR_INVALID, "NULL argument");
    if (dim == 0 || dim > 1024) return fail(OC_ERR_UNSUPPORTED, "dim %u unsupported (1..1024)", dim);
    if (dtype != OC_DTYPE_F32 && dtype != OC_DTYPE_BF16) return fail(OC_ERR_UNSUPPORTED, "dtype %d unknown", dtype);
    oc_emb *e = new oc_emb();
    e->ctx = c; e->dim = dim; e->dtype = dtype; e->e5 = rescale_e5 ? 1 : 0;
    e->esz = dtype == OC_DTYPE_BF16 ? 2 : 4;
    e->stride = ((dim + 127) / 128) * 128;
    if (e->stride / 128 == 5 || e->stride / 128 == 7) e->stride += 128;  // instantiated widths: 1,2,3,4,6,8
    *out = e;
    return OC_OK;
}

extern "C" void oc_emb_destroy(oc_emb *e) {
    if (!e) return;
    cudaSetDevice(e->ctx->device);
    cudaStreamSynchronize(e->ctx->stream);
    cudaFree(e->rows); cudaFree(e->inv_norm); cudaFree(e->row_doc);
    delete e;
}

static int emb_grow(oc_emb *e, uint64_t want_rows) {
    if (want_rows <= e->cap) return OC_OK;
    oc_ctx *c = e->ctx;
    uint64_t ncap = std::max<uint64_t>(want_rows, e->cap + e->cap / 2);
    ncap = (ncap + 63) / 64 * 64;
    void *nr = nullptr; float *nn = nullptr; uint64_t *nd = nullptr;
    CU(cudaMalloc(&nr, ncap * e->stride * e->esz));
    CU(cudaMalloc(&nn, (ncap + 64) * sizeof(float)));
    CU(cudaMalloc(&nd, ncap * sizeof(uint64_t)));
    if (e->n_rows) {
        CU(cudaMemcpyAsync(nr, e->rows, e->n_rows * e->stride * e->esz, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(nn, e->inv_norm, e->n_rows * sizeof(float), cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(nd, e->row_doc, e->n_rows * sizeof(uint64_t), cudaMemcpyDeviceToDevice, c->stream));
    }
    CU(cudaStreamSynchronize(c->stream));
    cudaFree(e->rows); cudaFree(e->inv_norm); cudaFree(e->row_doc);
    e->rows = nr; e->inv_norm = nn; e->row_doc = nd; e->cap = ncap;
    return OC_OK;
}

extern "C" int oc_emb_reserve(oc_emb *e, uint64_t n_rows) {
    if (!e) return fail(OC_ERR_INVALID, "emb is NULL");
    std::lock_guard<std::mutex> g(e->ctx->mu);
    CU(cudaSetDevice(e->ctx->device));
    return emb_grow(e, n_rows);
}

extern "C" int oc_emb_insert(oc_emb *e, const uint64_t *doc_ids, const void *rows, uint64_t n) {
    if (!e || (!doc_ids && n) || (!rows && n)) return fail(OC_ERR_INVALID, "NULL argument");
    if (n == 0) return OC_OK;
    oc_ctx *c = e->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    if (e->n_rows + n > 0xfffffff0ull) return fail(OC_ERR_UNSUPPORTED, "more than 2^32 rows per store");
    OCTRY(emb_grow(e, e->n_rows + n));
    uint8_t *dst = static_cast<uint8_t *>(e->rows) + e->n_rows * e->stride * e->esz;
    if (e->stride != e->dim) CU(cudaMemsetAsync(dst, 0, n * e->stride * e->esz, c->stream));
    CU(cudaMemcpy2DAsync(dst, size_t(e->stride) * e->esz, rows, size_t(e->dim) * e->esz, size_t(e->dim) * e->esz, n,
                         cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(e->row_doc + e->n_rows, doc_ids, n * sizeof(uint64_t), cudaMemcpyHostToDevice, c->stream));
    const uint64_t warps_per_block = 8;
    const uint64_t blocks = (n + warps_per_block - 1) / warps_per_block;
    if (e->esz == 2) emb_inv_norm_kernel<bf16_t><<<(unsigned)blocks, 256, 0, c->stream>>>(e->rows, e->stride, e->n_rows, e->n_rows + n, e->inv_norm);
    else emb_inv_norm_kernel<float><<<(unsigned)blocks, 256, 0, c->stream>>>(e->rows, e->stride, e->n_rows, e->n_rows + n, e->inv_norm);
    launched(c);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    for (uint64_t i = 0; i < n; i++) e->doc_rows.emplace(doc_ids[i], e->n_rows + i);
    e->n_rows += n; e->n_live += n;
    return OC_OK;
}

__global__ void tombstone_rows_kernel(float *inv_norm, const uint64_t *rows, uint64_t n) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) inv_norm[rows[i]] = __int_as_float(0x7fc00000);
}

extern "C" int oc_emb_delete(oc_emb *e, const uint64_t *doc_ids, uint64_t n) {
    if (!e || (!doc_ids && n)) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = e->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    std::vector<uint64_t> rows;
    for (uint64_t i = 0; i < n; i++) {
        auto range = e->doc_rows.equal_range(doc_ids[i]);
        for (auto it = range.first; it != range.second; ++it) rows.push_back(it->second);
        e->doc_rows.erase(range.first, range.second);
    }
    if (rows.empty()) return OC_OK;
    OCTRY(c->in_blob.ensure(rows.size() * 8));
    CU(cudaMemcpyAsync(c->in_blob.p, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, c->stream));
    tombstone_rows_kernel<<<(unsigned)((rows.size() + 255) / 256), 256, 0, c->stream>>>(e->inv_norm, c->in_blob.as<uint64_t>(), rows.size());
    launched(c);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));
    e->n_live -= rows.size();
    return OC_OK;
}

extern "C" int oc_emb_info(oc_emb *e, oc_emb_info_t *out) {
    if (!e || !out) return fail(OC_ERR_INVALID, "NULL argument");
    out->num_embeddings = e->n_live; out->num_rows = e->n_rows; out->dimensions = e->dim; out->dtype = e->dtype;
    out->device_bytes = e->cap * (uint64_t(e->stride) * e->esz + 4 + 8);
    return OC_OK;
}

// ---- scan launch plumbing
template <int NCH, int QB, typename T>
static int launch_scan_t(oc_ctx *c, const ScanParams &sp, uint32_t grid, size_t smem) {
    if (smem_cfg_needed(c->device, (const void *)emb_scan_kernel<NCH, QB, T>, smem))
        CU(cudaFuncSetAttribute(emb_scan_kernel<NCH, QB, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    emb_scan_kernel<NCH, QB, T><<<grid, SCAN_THREADS, smem, c->stream>>>(sp);
    launched(c, true);
    CU(cudaGetLastError());
    return OC_OK;
}
template <int QB, typename T>
static int launch_scan_q(oc_ctx *c, const ScanParams &sp, uint32_t grid, size_t smem) {
    switch (sp.stride / 128) {
        case 1: return launch_scan_t<1, QB, T>(c, sp, grid, smem);
        case 2: return launch_scan_t<2, QB, T>(c, sp, grid, smem);
        case 3: return launch_scan_t<3, QB, T>(c, sp, grid, smem);
        case 4: return launch_scan_t<4, QB, T>(c, sp, grid, smem);
        case 6: return launch_scan_t<6, QB, T>(c, sp, grid, smem);
        case 8: return launch_scan_t<8, QB, T>(c, sp, grid, smem);
    }
    return fail(OC_ERR_UNSUPPORTED, "stride %u not instantiated", sp.stride);
}
template <int QB>
static int launch_scan_d(oc_ctx *c, const ScanParams &sp, uint32_t grid, size_t smem, uint32_t esz) {
    return esz == 2 ? launch_scan_q<QB, bf16_t>(c, sp, grid, smem) : launch_scan_q<QB, float>(c, sp, grid, smem);
}

struct ScanPlan {
    uint32_t rows_per_stage, n_stages, wcap, grid, qb_max;
};
static ScanPlan plan_scan(const oc_ctx *c, const oc_emb *e, uint32_t n_keep) {
    ScanPlan pl;
    uint32_t qb = 4;
    const uint32_t row_bytes = e->stride * e->esz;
    uint32_t R = (32768 / row_bytes) / 8 * 8;
    if (R < 8) R = 8;
    pl.rows_per_stage = R;
    pl.wcap = std::max<uint32_t>(32, next_pow2(2 * n_keep));
    const size_t budget = 227 * 1024 - 1024;
    while (qb > 1 && size_t(SCAN_CONSUMER_WARPS) * qb * pl.wcap * 8 > budget / 2) qb >>= 1;
    pl.qb_max = qb;
    const size_t fixed = size_t(SCAN_CONSUMER_WARPS) * qb * pl.wcap * 8 + 256;
    const size_t per_stage = size_t(R) * row_bytes + R * 4 + 16;
    uint32_t S = (uint32_t)std::min<size_t>(8, fixed < budget ? (budget - fixed) / per_stage : 0);
    pl.n_stages = S;
    const uint64_t tiles = (e->n_rows + R - 1) / R;
    pl.grid = (uint32_t)std::min<uint64_t>(c->prop.multiProcessorCount, std::max<uint64_t>(tiles, 1));
    return pl;
}

// ---- exact sweeps (K1) + merge for nq prepared queries; results into the given buffers
struct VecOut { uint64_t *doc; float *score; uint32_t *row; uint32_t *cnt; float *raw; };
// row_bits / q_slot: per-query where-filters (ScanParams), or NULL
static int run_exact_sweeps(oc_ctx *c, oc_emb *e, const float *inv_norm, const float *qpad, const float *qinv,
                            uint32_t nq, uint32_t limit, float similarity, const VecOut &o,
                            const uint32_t *row_bits = nullptr, uint64_t row_words = 0, const uint32_t *q_slot = nullptr) {
    ScanPlan pl = plan_scan(c, e, limit);
    if (pl.n_stages < 2) return fail(OC_ERR_UNSUPPORTED, "limit %u leaves no shared memory for the scan ring", limit);
    OCTRY(c->scan_cand.ensure(size_t(nq) * pl.grid * limit * 8));
    uint32_t q0 = 0;
    while (q0 < nq) {
        const uint32_t rem = nq - q0;
        const uint32_t qb = std::min<uint32_t>(pl.qb_max, rem >= 4 ? 4 : (rem >= 2 ? 2 : 1));
        ScanParams sp{};
        sp.rows = e->rows; sp.inv_norm = inv_norm; sp.n_rows = e->n_rows; sp.stride = e->stride;
        sp.queries = qpad + size_t(q0) * e->stride;
        sp.inv_qnorm = qinv + q0;
        sp.n_keep = limit; sp.wcap = pl.wcap; sp.rows_per_stage = pl.rows_per_stage; sp.n_stages = pl.n_stages;
        sp.n_ctas_total = pl.grid;
        sp.cand = c->scan_cand.as<uint64_t>() + size_t(q0) * pl.grid * limit;
        if (row_bits) { sp.row_bits = row_bits; sp.row_words = row_words; sp.q_slot = q_slot + q0; }
        const size_t smem = scan_smem_bytes(e->stride, pl.rows_per_stage, pl.n_stages, pl.wcap, qb, e->esz);
        if (qb == 4) OCTRY((launch_scan_d<4>(c, sp, pl.grid, smem, e->esz)));
        else if (qb == 2) OCTRY((launch_scan_d<2>(c, sp, pl.grid, smem, e->esz)));
        else OCTRY((launch_scan_d<1>(c, sp, pl.grid, smem, e->esz)));
        c->timing.scan_bytes += e->n_rows * (uint64_t(e->stride) * e->esz + 4);
        q0 += qb;
    }
    CU(cudaEventRecord(c->ev[EV_SCAN1], c->stream));
    ScanMergeParams mp{};
    mp.cand = c->scan_cand.as<uint64_t>(); mp.n_lists = pl.grid; mp.n_keep = limit; mp.limit = limit;
    mp.capb = std::max<uint32_t>(2048, next_pow2(2 * limit));
    mp.row_doc_ids = e->row_doc; mp.rescale_e5 = e->e5; mp.similarity = similarity;
    mp.out_doc = o.doc; mp.out_score = o.score; mp.out_row = o.row; mp.out_count = o.cnt; mp.out_raw = o.raw;
    if (smem_cfg_needed(c->device, (const void *)emb_scan_merge_kernel, size_t(mp.capb) * 8))
        CU(cudaFuncSetAttribute(emb_scan_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(mp.capb * 8)));
    emb_scan_merge_kernel<<<nq, 256, mp.capb * 8, c->stream>>>(mp);
    launched(c);
    CU(cudaGetLastError());
    return OC_OK;
}

// ---- TMA descriptors (tmap.cuh)
static int tmap_2d(CUtensorMap *m, const void *base, uint64_t n_rows, uint32_t stride, uint32_t box_rows, bool bf16) {
    const TmapStatus s = make_tmap_2d(m, base, n_rows, stride, box_rows, bf16);
    if (s.what) return fail(OC_ERR_CUDA, "%s failed: %d", s.what, s.code);
    return OC_OK;
}

static bool g_disable_gemm = false;   // OC_DISABLE_GEMM=1: force the exact sweep path (A/B testing)

// Per-query where-filters of one search (oc_search_params.q_filters), deduplicated by handle.
struct QFilterJob {
    std::vector<RowsOkSlot> slots;     // the K distinct handles, then {NULL, 0}: the fulltext slot of unfiltered queries
    std::vector<uint32_t> q_slot;      // [B] vector stage: index into slots, SLOT_NONE = unfiltered
    std::vector<uint32_t> q_slot_ft;   // [B] fulltext stage: index into slots, K = unfiltered (tombstones only)
    const RowsOkSlot *d_slots = nullptr;
    const uint32_t *d_q_slot = nullptr, *d_q_slot_ft = nullptr;
    uint32_t k() const { return (uint32_t)slots.size() - 1; }
};

// Runs prep + (tensor-core batched scan | exact sweeps) + merge for B queries already in device
// memory (q_dev: B x dim).  Leaves hits in c->v_doc / v_score / v_row / v_cnt / v_raw ([B][limit]).
// qf: per-query where-filters (device tables uploaded), or NULL.
static int run_vector_stage(oc_ctx *c, oc_emb *e, const float *q_dev, uint32_t B, uint32_t limit, float similarity,
                            const uint64_t *filter_dev, uint64_t filter_nbits, const QFilterJob *qf = nullptr) {
    OCTRY(c->v_doc.ensure(size_t(B) * limit * 8));
    OCTRY(c->v_score.ensure(size_t(B) * limit * 4));
    OCTRY(c->v_row.ensure(size_t(B) * limit * 4));
    OCTRY(c->v_cnt.ensure(size_t(B) * 4));
    OCTRY(c->v_raw.ensure(size_t(B) * limit * 4));
    if (e->n_rows == 0) {
        CU(cudaMemsetAsync(c->v_cnt.p, 0, size_t(B) * 4, c->stream));
        CU(cudaMemsetAsync(c->v_doc.p, 0, size_t(B) * limit * 8, c->stream));
        CU(cudaMemsetAsync(c->v_score.p, 0, size_t(B) * limit * 4, c->stream));
        CU(cudaMemsetAsync(c->v_row.p, 0xff, size_t(B) * limit * 4, c->stream));
        return OC_OK;
    }
    const uint32_t n_qgroups = (B + GEMM_M - 1) / GEMM_M, Bpad = n_qgroups * GEMM_M;
    OCTRY(c->q_pad.ensure(size_t(Bpad) * e->stride * 4));
    OCTRY(c->q_inv.ensure(size_t(Bpad) * 4));
    OCTRY(c->q_rho.ensure(size_t(Bpad) * 4));
    const char *env = getenv("OC_DISABLE_GEMM");
    g_disable_gemm = env && env[0] == '1';
    // tensor-core scan: a batch (the distance is a true GEMM), a store large enough that the threshold pass sees
    // at least `limit` row groups with data (its seeds are the limit-th largest group maximum; with fewer live groups
    // the threshold degenerates to "gather everything" and the query falls back to the exact sweep).  A group is the
    // 64 rows one list sees of its CTA's first 256-row tile: n_rows >= 256 limit leaves >= limit full tiles, i.e.
    // 4 min(ctas_per_group, limit) >= limit live groups whenever ctas_per_group >= limit / 4
    const bool use_gemm = !g_disable_gemm && B >= 8 && limit <= GEMM_MAX_LIMIT && e->n_rows >= std::max<uint64_t>(4096, uint64_t(limit) * 256);
    // (the prep kernel writes rows [0, B) whole, zero padded: only the rows of a partial last query group need clearing)
    if (use_gemm && Bpad != B) CU(cudaMemsetAsync(c->q_pad.as<float>() + size_t(B) * e->stride, 0, size_t(Bpad - B) * e->stride * 4, c->stream));
    emb_prep_queries_kernel<<<(B + 7) / 8, 256, 0, c->stream>>>(q_dev, e->dim, e->stride, B, c->q_pad.as<float>(), c->q_inv.as<float>(),
                                                                c->q_rho.as<float>());
    launched(c);
    const float *inv_norm = e->inv_norm;
    if (filter_dev) {
        OCTRY(c->eff_norm.ensure((e->n_rows + 64) * 4));
        emb_apply_filter_kernel<<<(unsigned)((e->n_rows + 255) / 256), 256, 0, c->stream>>>(
            e->inv_norm, e->row_doc, e->n_rows, filter_dev, filter_nbits, c->eff_norm.as<float>());
        launched(c);
        inv_norm = c->eff_norm.as<float>();
    }
    const uint32_t *row_bits = nullptr;
    uint64_t row_words = 0;
    if (qf) {   // one bitmap over the store's rows per distinct filter (whole 256-row tiles: K2 reads 8 words per tile)
        row_words = (e->n_rows + GEMM_N - 1) / GEMM_N * (GEMM_N / 32);
        OCTRY(c->e_rowbits.ensure(size_t(qf->k()) * row_words * 4));
        rows_ok_kernel<<<dim3((unsigned)((row_words + 255) / 256), qf->k()), 256, 0, c->stream>>>(
            e->row_doc, e->n_rows, nullptr, nullptr, 0, c->e_rowbits.as<uint32_t>(), row_words, qf->d_slots);
        launched(c);
        CU(cudaGetLastError());
        row_bits = c->e_rowbits.as<uint32_t>();
        c->v_rowbits = row_bits; c->v_row_words = row_words; c->v_qslot = qf->q_slot;
    }
    VecOut out{c->v_doc.as<uint64_t>(), c->v_score.as<float>(), c->v_row.as<uint32_t>(), c->v_cnt.as<uint32_t>(), c->v_raw.as<float>()};
    CU(cudaEventRecord(c->ev[EV_SCAN0], c->stream));
    if (!use_gemm)
        return run_exact_sweeps(c, e, inv_norm, c->q_pad.as<float>(), c->q_inv.as<float>(), B, limit, similarity, out, row_bits,
                                row_words, qf ? qf->d_q_slot : nullptr);

    // ---------------- K2: wgmma batched scan ----------------
    const bool bf16 = e->esz == 2;
    const void *sweep_fn = bf16 ? (const void *)emb_gemm_kernel<true> : (const void *)emb_gemm_kernel<false>;
    if (smem_cfg_needed(c->device, (const void *)emb_gemm_kernel<false>, gemm_smem_bytes())) {   // all sweep kernels at once
        CU(cudaFuncSetAttribute(emb_gemm_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gemm_smem_bytes()));
        CU(cudaFuncSetAttribute(emb_gemm_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gemm_smem_bytes()));
        CU(cudaFuncSetAttribute(emb_gemm_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gemm_merge_smem_bytes()));
    }
    // an even number of query groups runs in CTA pairs that share every row tile (emb_gemm.cuh)
    const bool paired = n_qgroups % GEMM_CLUSTER == 0;
    cudaLaunchAttribute cluster_attr{};
    cluster_attr.id = cudaLaunchAttributeClusterDimension;
    cluster_attr.val.clusterDim.x = paired ? GEMM_CLUSTER : 1;
    cluster_attr.val.clusterDim.y = cluster_attr.val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg{};
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = gemm_smem_bytes();
    cfg.stream = c->stream;
    cfg.attrs = &cluster_attr;
    cfg.numAttrs = paired ? 1 : 0;
    // one wave: one CTA per SM and query group, or as many pairs as can be resident at once (a GPC with an odd number
    // of free SMs leaves one idle; a second wave would double the sweep); the merge gathers at most 512 lists per query
    uint32_t resident = c->prop.multiProcessorCount;
    if (paired) {
        static std::mutex occ_mu;   // resident clusters per (device, kernel): queried once
        static std::map<std::pair<int, const void *>, int> occ;
        std::lock_guard<std::mutex> g(occ_mu);
        auto it = occ.find(std::make_pair(c->device, sweep_fn));
        int n_clusters = 0;
        if (it == occ.end()) {
            cfg.gridDim = dim3(GEMM_CLUSTER * c->prop.multiProcessorCount);
            CU(cudaOccupancyMaxActiveClusters(&n_clusters, sweep_fn, &cfg));
            occ[std::make_pair(c->device, sweep_fn)] = n_clusters;
        } else n_clusters = it->second;
        if (n_clusters < 1) return fail(OC_ERR_UNSUPPORTED, "no CTA pair of the K2 sweep fits on device %d", c->device);
        resident = GEMM_CLUSTER * uint32_t(n_clusters);
    }
    const uint32_t cpg = std::min<uint32_t>(512 / GEMM_LISTS_PER_CTA, std::max<uint32_t>(1, resident / n_qgroups));
    const uint32_t grid = cpg * n_qgroups;
    cfg.gridDim = dim3(grid);
    const uint32_t lists = cpg * GEMM_LISTS_PER_CTA;
    const uint32_t cap = GEMM_LIST_CAP;
    CUtensorMap tm_q, tm_x;
    const void *q_operand = c->q_pad.p;
    if (bf16) {   // the sweep's query operand in the store's dtype (the exact re-score keeps the fp32 query)
        OCTRY(c->q_bf16.ensure(size_t(Bpad) * e->stride * 2));
        const size_t nq_el = size_t(Bpad) * e->stride;
        f32_to_bf16_kernel<<<(unsigned)((nq_el + 255) / 256), 256, 0, c->stream>>>(c->q_pad.as<float>(), c->q_bf16.as<uint16_t>(), nq_el);
        launched(c);
        q_operand = c->q_bf16.p;
    }
    OCTRY(tmap_2d(&tm_q, q_operand, Bpad, e->stride, GEMM_M, bf16));
    OCTRY(tmap_2d(&tm_x, e->rows, e->n_rows, e->stride, GEMM_N / (paired ? GEMM_CLUSTER : 1), bf16));   // a CTA's share of a tile
    OCTRY(c->g_thr.ensure(size_t(B) * 4));
    OCTRY(c->g_eps.ensure(size_t(B) * 4));
    OCTRY(c->g_cand.ensure(size_t(Bpad) * lists * cap * 8));
    OCTRY(c->g_cnt.ensure(size_t(Bpad) * lists * 4));
    OCTRY(c->g_ovf.ensure(size_t(B) * GEMM_OVF_CAP * 8));
    OCTRY(c->g_ovfcnt.ensure(size_t(B) * 4));
    OCTRY(c->g_resc.ensure(size_t(B) * 4));
    OCTRY(c->g_flag.ensure(B));
    OCTRY(c->g_max.ensure(size_t(Bpad) * lists * 4));
    GemmParams gp{};
    gp.n_rows = e->n_rows; gp.n_kblocks = e->stride / (bf16 ? 2 * GEMM_KB : GEMM_KB); gp.inv_norm = inv_norm; gp.n_queries = B;
    gp.n_qgroups = n_qgroups; gp.ctas_per_group = cpg; gp.cap = cap; gp.lists_per_query = lists;
    gp.thr = c->g_thr.as<unsigned int>(); gp.eps_v = c->g_eps.as<float>(); gp.limit = limit; gp.cand = c->g_cand.as<uint64_t>(); gp.cand_cnt = c->g_cnt.as<uint32_t>();
    gp.gmax = c->g_max.as<float>();
    gp.ovf = c->g_ovf.as<uint64_t>(); gp.ovf_cnt = c->g_ovfcnt.as<uint32_t>(); gp.ovf_cap = GEMM_OVF_CAP;
    if (qf) { gp.row_bits = row_bits; gp.row_words = row_words; gp.q_slot = qf->d_q_slot; }
    auto launch_gemm = [&]() -> int {
        if (bf16) CU(cudaLaunchKernelEx(&cfg, emb_gemm_kernel<true>, tm_q, tm_x, gp));
        else CU(cudaLaunchKernelEx(&cfg, emb_gemm_kernel<false>, tm_q, tm_x, gp));
        launched(c, gp.max_mode == 0);   // the one-tile threshold pass is not counted as a sweep
        CU(cudaGetLastError());
        return OC_OK;
    };
    // threshold pass: one row tile per CTA, record per-list maxima; thr = (limit-th largest maximum) - 2 eps
    gp.max_mode = 1; gp.tile_limit = 1;
    OCTRY(launch_gemm());
    GemmThrParams tp{};
    tp.gmax = c->g_max.as<float>(); tp.lists = lists; tp.limit = limit; tp.inv_qnorm = c->q_inv.as<float>();
    tp.eps_const = bf16 ? GEMM_EPS_ACC : GEMM_EPS_TF32;
    tp.rho_q = bf16 ? c->q_rho.as<float>() : nullptr;             // bf16 store: the rows are exact, the query is rounded
    tp.thr = c->g_thr.as<unsigned int>(); tp.eps_v = c->g_eps.as<float>(); tp.ovf_cnt = c->g_ovfcnt.as<uint32_t>();
    gemm_thr_kernel<<<B, 256, 0, c->stream>>>(tp);
    launched(c);
    // the sweep
    gp.max_mode = 0; gp.tile_limit = 0;
    CU(cudaEventRecord(c->ev[EV_SWEEP0], c->stream));
    OCTRY(launch_gemm());
    CU(cudaEventRecord(c->ev[EV_SWEEP1], c->stream));
    c->sweep_timed = true;
    c->timing.scan_bytes += e->n_rows * (uint64_t(e->stride) * e->esz + 4);
    CU(cudaEventRecord(c->ev[EV_SCAN1], c->stream));
    GemmMergeParams mp{};
    mp.cand = gp.cand; mp.cand_cnt = gp.cand_cnt; mp.n_lists = lists; mp.cap = cap; mp.limit = limit;
    mp.ovf = gp.ovf; mp.ovf_cnt = gp.ovf_cnt; mp.ovf_cap = gp.ovf_cap; mp.eps_v = tp.eps_v;
    mp.rows = e->rows; mp.rows_bf16 = bf16 ? 1 : 0; mp.stride = e->stride; mp.inv_norm = inv_norm; mp.queries = c->q_pad.as<float>();
    mp.inv_qnorm = c->q_inv.as<float>(); mp.row_doc_ids = e->row_doc; mp.rescale_e5 = e->e5; mp.similarity = similarity;
    mp.out_doc = out.doc; mp.out_score = out.score; mp.out_row = out.row; mp.out_count = out.cnt; mp.out_raw = out.raw;
    mp.out_unproven = c->g_flag.as<uint8_t>(); mp.out_rescored = c->g_resc.as<uint32_t>();
    emb_gemm_merge_kernel<<<B, 512, gemm_merge_smem_bytes(), c->stream>>>(mp);
    launched(c);
    CU(cudaGetLastError());
    // the overflow flags travel back with the results; oc_*search re-runs flagged queries (fix_unproven)
    c->gemm_pending = true; c->gemm_inv_norm = inv_norm;
    c->timing.scan_tensor_core = 1;
    c->timing.scan_variant = bf16 ? OC_SCAN_TC_BF16 : OC_SCAN_TC_TF32;
    return OC_OK;
}

// Re-runs the queries whose tensor-core result failed the exactness proof through the exact
// K1 sweep and patches their slots of c->v_* (rare).  flags: host copy of g_flag.
static int fix_unproven(oc_ctx *c, oc_emb *e, const uint8_t *flags, uint32_t B, uint32_t limit, float similarity,
                        uint32_t *n_redone) {
    std::vector<uint32_t> redo;
    for (uint32_t q = 0; q < B; q++) if (flags[q]) redo.push_back(q);
    *n_redone = (uint32_t)redo.size();
    c->timing.scan_unproven = *n_redone;
    if (redo.empty()) return OC_OK;
    const float *inv_norm = c->gemm_inv_norm;
    VecOut out{c->v_doc.as<uint64_t>(), c->v_score.as<float>(), c->v_row.as<uint32_t>(), c->v_cnt.as<uint32_t>(), c->v_raw.as<float>()};
    const uint32_t nr = (uint32_t)redo.size();
    OCTRY(c->r_qpad.ensure(size_t(nr) * e->stride * 4));
    OCTRY(c->r_qinv.ensure(size_t(nr) * 4));
    OCTRY(c->r_map.ensure(size_t(nr) * 4));
    OCTRY(c->r_doc.ensure(size_t(nr) * limit * 8));
    OCTRY(c->r_score.ensure(size_t(nr) * limit * 4));
    OCTRY(c->r_row.ensure(size_t(nr) * limit * 4));
    OCTRY(c->r_cnt.ensure(size_t(nr) * 4));
    OCTRY(c->r_raw.ensure(size_t(nr) * limit * 4));
    for (uint32_t i = 0; i < nr; i++) {
        CU(cudaMemcpyAsync(c->r_qpad.as<float>() + size_t(i) * e->stride, c->q_pad.as<float>() + size_t(redo[i]) * e->stride,
                           size_t(e->stride) * 4, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(c->r_qinv.as<float>() + i, c->q_inv.as<float>() + redo[i], 4, cudaMemcpyDeviceToDevice, c->stream));
    }
    CU(cudaMemcpyAsync(c->r_map.p, redo.data(), size_t(nr) * 4, cudaMemcpyHostToDevice, c->stream));
    std::vector<uint32_t> rslot;   // per-query where-filters: each redone query keeps its own slot
    if (c->v_rowbits) {
        for (uint32_t q : redo) rslot.push_back(c->v_qslot[q]);
        OCTRY(c->r_slot.ensure(size_t(nr) * 4));
        CU(cudaMemcpyAsync(c->r_slot.p, rslot.data(), size_t(nr) * 4, cudaMemcpyHostToDevice, c->stream));
    }
    VecOut ro{c->r_doc.as<uint64_t>(), c->r_score.as<float>(), c->r_row.as<uint32_t>(), c->r_cnt.as<uint32_t>(), c->r_raw.as<float>()};
    OCTRY(run_exact_sweeps(c, e, inv_norm, c->r_qpad.as<float>(), c->r_qinv.as<float>(), nr, limit, similarity, ro, c->v_rowbits,
                           c->v_row_words, c->v_rowbits ? c->r_slot.as<uint32_t>() : nullptr));
    scatter_rows_kernel<<<nr, 64, 0, c->stream>>>(c->r_map.as<uint32_t>(), nr, limit, ro.doc, ro.score, ro.row, ro.cnt, ro.raw,
                                                   out.doc, out.score, out.row, out.cnt, out.raw);
    launched(c);
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(c->stream));   // redo vector lives on the stack
    return OC_OK;
}

static void begin_call(oc_ctx *c) {
    c->call_launches = 0; c->call_scan_launches = 0; c->gemm_pending = false; c->sweep_timed = false; c->rerun_timed = false;
    c->v_rowbits = nullptr; c->v_row_words = 0;
    memset(&c->timing, 0, sizeof(c->timing));
}
static int finish_timing(oc_ctx *c, bool scan, bool bm, bool fuse, bool comm) {
    auto el = [&](int a, int b) { float ms = 0; cudaEventElapsedTime(&ms, c->ev[a], c->ev[b]); return ms; };
    c->timing.h2d_ms = el(EV_START, EV_H2D);
    c->timing.rerun_ms = c->rerun_timed ? el(EV_RR0, EV_RR1) : 0.f;
    c->timing.device_ms = el(EV_H2D, EV_DEV) + c->timing.rerun_ms;   // a re-run is device work of this batch
    c->timing.d2h_ms = el(EV_DEV, EV_D2H);
    c->timing.scan_ms = scan ? el(EV_SCAN0, EV_SCAN1) : 0;
    c->timing.scan_sweep_ms = !scan ? 0 : (c->sweep_timed ? el(EV_SWEEP0, EV_SWEEP1) : c->timing.scan_ms);
    c->timing.bm25_ms = bm ? el(EV_BM0, EV_BM1) : 0;
    c->timing.fuse_ms = fuse ? el(EV_FUSE0, EV_FUSE1) : 0;
    c->timing.comm_ms = comm ? el(EV_COMM0, EV_COMM1) : 0;
    c->timing.kernel_launches = c->call_launches;
    c->timing.scan_launches = c->call_scan_launches;
    return OC_OK;
}

extern "C" int oc_emb_search(oc_emb *e, const float *queries, uint32_t B, uint32_t limit, float similarity,
                             const uint64_t *filter_bits, uint64_t filter_nbits, uint64_t *out_doc_ids,
                             float *out_scores, uint32_t *out_counts) {
    if (!e || !queries || !out_doc_ids || !out_scores || !out_counts) return fail(OC_ERR_INVALID, "NULL argument");
    if (B == 0) return OC_OK;
    if (limit == 0 || limit > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "limit %u outside 1..%u", limit, OC_MAX_TOPK);
    oc_ctx *c = e->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    begin_call(c);
    const size_t qbytes = size_t(B) * e->dim * 4;
    const size_t fwords = filter_bits ? (filter_nbits + 63) / 64 : 0;
    OCTRY(c->in_blob.ensure(qbytes));
    CU(cudaEventRecord(c->ev[EV_START], c->stream));
    CU(cudaMemcpyAsync(c->in_blob.p, queries, qbytes, cudaMemcpyHostToDevice, c->stream));
    if (fwords) {
        OCTRY(c->filter_dev.ensure(fwords * 8));
        CU(cudaMemcpyAsync(c->filter_dev.p, filter_bits, fwords * 8, cudaMemcpyHostToDevice, c->stream));
    }
    c->timing.h2d_bytes = qbytes + fwords * 8;
    CU(cudaEventRecord(c->ev[EV_H2D], c->stream));
    OCTRY(run_vector_stage(c, e, c->in_blob.as<float>(), B, limit, similarity,
                           fwords ? c->filter_dev.as<uint64_t>() : nullptr, filter_nbits));
    CU(cudaEventRecord(c->ev[EV_DEV], c->stream));
    const size_t ob = size_t(B) * limit * 12 + size_t(B) * 4;
    const size_t o_resc = ob + ((size_t(B) + 3) & ~size_t(3));
    OCTRY(c->h_out.ensure(o_resc + size_t(B) * 4));
    uint8_t *h = c->h_out.as<uint8_t>();
    auto fetch = [&]() -> int {
        CU(cudaMemcpyAsync(h, c->v_doc.p, size_t(B) * limit * 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(h + size_t(B) * limit * 8, c->v_score.p, size_t(B) * limit * 4, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(h + size_t(B) * limit * 12, c->v_cnt.p, size_t(B) * 4, cudaMemcpyDeviceToHost, c->stream));
        if (c->gemm_pending) {
            CU(cudaMemcpyAsync(h + ob, c->g_flag.p, B, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaMemcpyAsync(h + o_resc, c->g_resc.p, size_t(B) * 4, cudaMemcpyDeviceToHost, c->stream));
        }
        return OC_OK;
    };
    OCTRY(fetch());
    CU(cudaEventRecord(c->ev[EV_D2H], c->stream));
    CU(cudaStreamSynchronize(c->stream));
    if (c->gemm_pending) {
        uint64_t resc = 0;
        for (uint32_t q = 0; q < B; q++) resc += reinterpret_cast<const uint32_t *>(h + o_resc)[q];
        c->timing.scan_rescored = (uint32_t)(resc / B);
        uint32_t redone = 0;
        CU(cudaEventRecord(c->ev[EV_RR0], c->stream));
        OCTRY(fix_unproven(c, e, h + ob, B, limit, similarity, &redone));
        if (redone) {
            c->gemm_pending = false; OCTRY(fetch());
            CU(cudaEventRecord(c->ev[EV_RR1], c->stream));
            c->rerun_timed = true;
            CU(cudaStreamSynchronize(c->stream));
        }
    }
    c->timing.d2h_bytes = ob;
    memcpy(out_doc_ids, h, size_t(B) * limit * 8);
    memcpy(out_scores, h + size_t(B) * limit * 8, size_t(B) * limit * 4);
    memcpy(out_counts, h + size_t(B) * limit * 12, size_t(B) * 4);
    return finish_timing(c, e->n_rows > 0, false, false, false);
}

// ------------------------------------------------------------------------------------ string store
// Snapshot model (the reference keeps `CURRENT` + `versions/<n>` per field and swaps the pointer after
// compact(), embedding_field.rs:91-95 / string_field.rs:186-191): searches work on the published,
// immutable StrSnap they grabbed at call entry; oc_str_commit builds the next snapshot WITHOUT the
// ctx lock (host merge + upload on the store's own stream) and publishes it with a pointer swap, so
// searches keep running on the previous version while a commit is in flight.  Ops that arrive during
// a commit: inserts queue for the next one, deletes hit the old snapshot at once and are replayed on
// the new one before it is published.
struct StrField {
    float avg_len = 0;
    uint32_t n_terms = 0;
    std::vector<uint64_t> term_offsets;  // host copy (n_terms+1)
    std::vector<uint32_t> global_df;     // optional: per-term corpus df across all shards
    PostingRaw *raw = nullptr;           // device: (row, tf, field_len) as loaded
    Posting *post = nullptr;             // device: (row, tf') derived for b_cached
    float b_cached = -1.f;
    uint64_t n_post = 0;
    std::vector<PostingRaw> host_post;   // host copy of the committed postings (term-major), kept for oc_str_commit
};
struct StrSnap {
    int device = 0;
    uint64_t version = 0;
    std::vector<StrField> fields;
    uint64_t n_rows = 0, document_count = 0;
    std::vector<uint64_t> row_doc_host;  // empty => identity
    uint64_t *row_doc = nullptr;         // device or NULL
    uint32_t *alive = nullptr;           // device bitmap (allocated on first delete)
    std::vector<uint32_t> alive_host;
    uint64_t n_deleted = 0;
    ~StrSnap() {
        int dev = -1;
        cudaGetDevice(&dev);
        if (dev != device) cudaSetDevice(device);
        for (auto &f : fields) { cudaFree(f.post); cudaFree(f.raw); }
        cudaFree(row_doc); cudaFree(alive);
        if (dev >= 0 && dev != device) cudaSetDevice(dev);
    }
    // row of a DocumentId, or ~0ull
    uint64_t row_of(uint64_t doc) const {
        if (row_doc_host.empty()) return doc < n_rows ? doc : ~0ull;
        auto it = std::lower_bound(row_doc_host.begin(), row_doc_host.end(), doc);
        return (it == row_doc_host.end() || *it != doc) ? ~0ull : uint64_t(it - row_doc_host.begin());
    }
};
struct PendingPost { uint64_t doc, seq; uint32_t term; uint16_t tf, len; };   // term == ~0u: "document inserted with no term"
struct oc_str {
    oc_ctx *ctx = nullptr;
    std::mutex mu;                                   // cur / pending / logs (short critical sections; never held across device work of a search)
    std::shared_ptr<StrSnap> cur;                    // the published snapshot ("CURRENT")
    uint64_t version = 0;
    std::vector<std::vector<PendingPost>> pending;   // per field: StringFieldStorage::insert since the last commit
    uint64_t seq = 0;                                // op sequence: a delete only cancels inserts that came before it
    std::unordered_map<uint64_t, uint64_t> pending_deleted;   // doc -> seq of its latest delete
    bool committing = false;
    std::vector<uint64_t> deletes_during_commit;
    bool global_count = false, global_avg = false;   // document_count / avg_field_len are values owned by the caller (shard of a larger index; an
                                                     // Index whose document_count also counts documents without string fields): commit keeps them
    cudaStream_t load_stream = nullptr;
};
static std::shared_ptr<StrSnap> str_snapshot(oc_str *s) {
    std::lock_guard<std::mutex> g(s->mu);
    return s->cur;
}

extern "C" int oc_str_create(oc_ctx *c, uint32_t n_fields, oc_str **out) {
    if (!c || !out || n_fields == 0) return fail(OC_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    oc_str *s = new oc_str();
    s->ctx = c;
    s->cur = std::make_shared<StrSnap>();
    s->cur->device = c->device;
    s->cur->fields.resize(n_fields);
    s->pending.resize(n_fields);
    CU(cudaStreamCreateWithFlags(&s->load_stream, cudaStreamNonBlocking));
    *out = s;
    return OC_OK;
}
extern "C" void oc_str_destroy(oc_str *s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    cudaStreamSynchronize(s->ctx->stream);
    if (s->load_stream) { cudaStreamSynchronize(s->load_stream); cudaStreamDestroy(s->load_stream); }
    s->cur.reset();
    delete s;
}

// Bulk load (oc_str_set_rows + oc_str_load_field per field) starts a fresh snapshot; both run under the
// ctx lock, i.e. never concurrently with a search on this ctx.
extern "C" int oc_str_set_rows(oc_str *s, uint64_t n_rows, const uint64_t *row_doc_ids, uint64_t document_count) {
    if (!s) return fail(OC_ERR_INVALID, "str is NULL");
    if (n_rows > 0xfffffff0ull) return fail(OC_ERR_UNSUPPORTED, "more than 2^32 rows per store");
    oc_ctx *c = s->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    if (row_doc_ids)
        for (uint64_t i = 1; i < n_rows; i++)
            if (row_doc_ids[i] <= row_doc_ids[i - 1]) return fail(OC_ERR_INVALID, "row_doc_ids must be strictly ascending");
    auto ns = std::make_shared<StrSnap>();
    ns->device = c->device;
    ns->n_rows = n_rows; ns->document_count = document_count;
    if (row_doc_ids && n_rows) {
        ns->row_doc_host.assign(row_doc_ids, row_doc_ids + n_rows);
        CU(cudaMalloc(&ns->row_doc, n_rows * 8));
        CU(cudaMemcpy(ns->row_doc, row_doc_ids, n_rows * 8, cudaMemcpyHostToDevice));
    }
    std::lock_guard<std::mutex> g2(s->mu);
    if (s->committing) return fail(OC_ERR_INVALID, "oc_str_set_rows while a commit is in flight");
    ns->fields.resize(s->cur->fields.size());
    ns->version = ++s->version;
    s->cur = ns;
    // a document count that differs from the row count can only be a corpus-wide N (this store is a shard)
    s->global_count = s->global_avg = document_count != n_rows;
    for (auto &p : s->pending) p.clear();
    s->pending_deleted.clear();
    return OC_OK;
}

extern "C" int oc_str_set_global(oc_str *s, uint64_t document_count, const float *avg_field_len) {
    if (!s) return fail(OC_ERR_INVALID, "str is NULL");
    oc_ctx *c = s->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    std::lock_guard<std::mutex> g2(s->mu);
    StrSnap &S = *s->cur;
    S.document_count = document_count;
    if (avg_field_len)
        for (size_t i = 0; i < S.fields.size(); i++)
            if (S.fields[i].avg_len != avg_field_len[i]) { S.fields[i].avg_len = avg_field_len[i]; S.fields[i].b_cached = -1.f; }
    s->global_count = true;
    s->global_avg = avg_field_len != nullptr;
    return OC_OK;
}

extern "C" int oc_str_load_field(oc_str *s, uint32_t field, float avg_field_len, uint32_t n_terms,
                                 const uint64_t *term_offsets, const uint32_t *post_row, const uint16_t *post_tf,
                                 const uint16_t *post_len, const uint32_t *global_df) {
    if (!s || !term_offsets) return fail(OC_ERR_INVALID, "bad arguments");
    oc_ctx *c = s->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    std::shared_ptr<StrSnap> snap = str_snapshot(s);
    StrSnap &S = *snap;
    if (field >= S.fields.size()) return fail(OC_ERR_INVALID, "field %u out of range", field);
    StrField &f = S.fields[field];
    cudaFree(f.post); f.post = nullptr; cudaFree(f.raw); f.raw = nullptr; f.b_cached = -1.f;
    const uint64_t np = term_offsets[n_terms];
    if (np && (!post_row || !post_tf || !post_len)) return fail(OC_ERR_INVALID, "posting arrays are NULL");
    for (uint32_t t = 0; t < n_terms; t++) {
        if (term_offsets[t + 1] < term_offsets[t]) return fail(OC_ERR_INVALID, "term_offsets not monotone");
        if (term_offsets[t + 1] - term_offsets[t] > 0xffffffffull) return fail(OC_ERR_UNSUPPORTED, "posting list too long");
    }
    f.avg_len = avg_field_len; f.n_terms = n_terms; f.n_post = np;
    f.host_post.resize(np);
    for (uint64_t i = 0; i < np; i++) {
        if (post_row[i] >= S.n_rows && S.n_rows) return fail(OC_ERR_INVALID, "posting row %u >= n_rows", post_row[i]);
        f.host_post[i].row = post_row[i]; f.host_post[i].tf = post_tf[i]; f.host_post[i].len = post_len[i];
    }
    f.term_offsets.assign(term_offsets, term_offsets + n_terms + 1);
    f.global_df.clear();
    if (global_df) f.global_df.assign(global_df, global_df + n_terms);
    if (np) {
        CU(cudaMalloc(&f.post, (np + 4) * sizeof(Posting)));
        CU(cudaMalloc(&f.raw, (np + 4) * sizeof(PostingRaw)));
        CU(cudaMemcpyAsync(f.raw, f.host_post.data(), np * sizeof(PostingRaw), cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    return OC_OK;
}

// tombstones `rows` of snapshot S (host bitmap + device copy on stream st)
static int snap_tombstone(StrSnap &S, const std::vector<uint64_t> &rows, cudaStream_t st) {
    if (rows.empty() || S.n_rows == 0) return OC_OK;
    const uint64_t words = (S.n_rows + BM25_TILE - 1) / BM25_TILE * (BM25_TILE / 32);
    if (S.alive_host.empty()) {
        S.alive_host.assign(words, 0xffffffffu);
        CU(cudaMalloc(&S.alive, words * 4));
    }
    for (uint64_t r : rows)
        if (S.alive_host[r >> 5] & (1u << (r & 31))) { S.alive_host[r >> 5] &= ~(1u << (r & 31)); S.n_deleted++; }
    CU(cudaMemcpyAsync(S.alive, S.alive_host.data(), words * 4, cudaMemcpyHostToDevice, st));
    CU(cudaStreamSynchronize(st));
    return OC_OK;
}

// StringFieldStorage::delete (string_field.rs:180-182).  Ops apply in order, as the reference's compact
// does: a delete tombstones the committed rows of the document now and cancels its inserts that are
// still pending (inserted before this call); an insert after the delete is a new document.
extern "C" int oc_str_delete(oc_str *s, const uint64_t *doc_ids, uint64_t n) {
    if (!s || (!doc_ids && n)) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = s->ctx;
    std::lock_guard<std::mutex> g(c->mu);      // the device bitmap is read by searches on the ctx stream
    CU(cudaSetDevice(c->device));
    std::lock_guard<std::mutex> g2(s->mu);
    StrSnap &S = *s->cur;
    std::vector<uint64_t> rows;
    for (uint64_t i = 0; i < n; i++) {
        s->pending_deleted[doc_ids[i]] = ++s->seq;
        if (s->committing) s->deletes_during_commit.push_back(doc_ids[i]);
        const uint64_t r = S.row_of(doc_ids[i]);
        if (r != ~0ull) rows.push_back(r);
    }
    return snap_tombstone(S, rows, c->stream);
}

// StringFieldStorage::insert(DocumentId, IndexedValue{field_length, terms}) (string_field.rs:155-177):
// buffered on the host; visible to searches after oc_str_commit (== compact, :186-191).  Inserting a
// document again (before or after a commit) replaces its postings in that field: last insert wins.
extern "C" int oc_str_insert(oc_str *s, uint32_t field, uint64_t doc_id, uint16_t field_len, uint32_t n_terms,
                             const uint32_t *term_ids, const uint16_t *tfs) {
    if (!s || (n_terms && (!term_ids || !tfs))) return fail(OC_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> g(s->mu);
    if (field >= s->pending.size()) return fail(OC_ERR_INVALID, "field %u out of range", field);
    for (uint32_t i = 0; i < n_terms; i++)
        if (term_ids[i] == 0xffffffffu) return fail(OC_ERR_INVALID, "term id 0xffffffff is reserved");
    const uint64_t q = ++s->seq;
    auto &pv = s->pending[field];
    if (n_terms == 0) pv.push_back({doc_id, q, 0xffffffffu, 0, field_len});
    for (uint32_t i = 0; i < n_terms; i++) pv.push_back({doc_id, q, term_ids[i], tfs[i], field_len});
    return OC_OK;
}

// Merges pending inserts and deletes into the next snapshot: rows are the ascending doc ids, postings
// term-major / row-ascending, avg_field_len and document_count refreshed (unless the caller owns the
// corpus-wide values), tombstones dropped.  Everything is built in temporaries; the published snapshot
// is replaced only after every field validated and uploaded, so a failed commit changes nothing.
extern "C" int oc_str_commit(oc_str *s) {
    if (!s) return fail(OC_ERR_INVALID, "str is NULL");
    oc_ctx *c = s->ctx;
    std::shared_ptr<StrSnap> base;
    std::vector<std::vector<PendingPost>> pend;
    std::unordered_map<uint64_t, uint64_t> pdel;
    std::vector<uint32_t> base_alive;
    bool global_count, global_avg;
    {
        std::lock_guard<std::mutex> g(s->mu);
        if (s->committing) return fail(OC_ERR_INVALID, "a commit of this store is already in flight");
        s->committing = true;
        s->deletes_during_commit.clear();
        base = s->cur;
        pend.resize(s->pending.size());
        for (size_t i = 0; i < pend.size(); i++) pend[i].swap(s->pending[i]);
        pdel.swap(s->pending_deleted);
        base_alive = base->alive_host;
        global_count = s->global_count; global_avg = s->global_avg;
    }
    // on failure: put the taken ops back (in front of whatever arrived meanwhile) and leave `cur` alone
    auto abort_commit = [&](int rc) {
        std::lock_guard<std::mutex> g(s->mu);
        for (size_t i = 0; i < pend.size(); i++) {
            pend[i].insert(pend[i].end(), s->pending[i].begin(), s->pending[i].end());
            s->pending[i].swap(pend[i]);
        }
        for (auto &kv : pdel) { auto it = s->pending_deleted.find(kv.first); if (it == s->pending_deleted.end() || it->second < kv.second) s->pending_deleted[kv.first] = kv.second; }
        s->committing = false;
        return rc;
    };
    if (cudaSetDevice(c->device) != cudaSuccess) return abort_commit(fail(OC_ERR_CUDA, "cudaSetDevice failed"));
    const StrSnap &B = *base;
    const size_t nf = B.fields.size();
    // ---- pending ops in order: drop inserts cancelled by a later delete, keep the last insert per (field, doc)
    for (size_t fi = 0; fi < nf; fi++) {
        auto &pv = pend[fi];
        std::unordered_map<uint64_t, uint64_t> last;   // doc -> seq of its last surviving insert in this field
        for (auto &pn : pv) {
            auto d = pdel.find(pn.doc);
            if (d != pdel.end() && pn.seq < d->second) continue;
            uint64_t &l = last[pn.doc];
            if (pn.seq > l) l = pn.seq;
        }
        size_t w = 0;
        for (auto &pn : pv) {
            auto it = last.find(pn.doc);
            if (it != last.end() && it->second == pn.seq) pv[w++] = pn;
        }
        pv.resize(w);
    }
    // ---- row space of the next snapshot
    std::vector<uint64_t> docs;
    std::vector<uint8_t> old_alive(B.n_rows, 1);
    for (uint64_t r = 0; r < B.n_rows; r++) {
        const bool alive = base_alive.empty() || ((base_alive[r >> 5] >> (r & 31)) & 1u);
        old_alive[r] = alive;
        if (alive) docs.push_back(B.row_doc_host.empty() ? r : B.row_doc_host[r]);
    }
    for (auto &pv : pend) for (auto &pn : pv) docs.push_back(pn.doc);
    std::sort(docs.begin(), docs.end());
    docs.erase(std::unique(docs.begin(), docs.end()), docs.end());
    if (docs.size() > 0xfffffff0ull) return abort_commit(fail(OC_ERR_UNSUPPORTED, "more than 2^32 rows per store"));
    auto row_of = [&](uint64_t d) { return (uint32_t)(std::lower_bound(docs.begin(), docs.end(), d) - docs.begin()); };
    std::vector<uint32_t> remap(B.n_rows, 0xffffffffu);
    for (uint64_t r = 0; r < B.n_rows; r++) if (old_alive[r]) remap[r] = row_of(B.row_doc_host.empty() ? r : B.row_doc_host[r]);
    auto ns = std::make_shared<StrSnap>();
    ns->device = c->device;
    ns->fields.resize(nf);
    struct Rec { uint32_t term, row; uint16_t tf, len; };
    for (size_t fi = 0; fi < nf; fi++) {
        const StrField &of = B.fields[fi];
        StrField &f = ns->fields[fi];
        // the committed postings are already term-major / row-ascending and the row remap is monotone, so only the
        // PENDING postings are sorted; the next CSR is a per-term linear merge of (surviving old list, new list):
        // O(P_old + p log p) instead of a sort of everything
        std::vector<uint8_t> replaced(docs.size(), 0);   // a re-inserted document replaces its old postings in this field
        for (auto &pn : pend[fi]) replaced[row_of(pn.doc)] = 1;
        std::vector<Rec> add;
        add.reserve(pend[fi].size());
        uint32_t max_term = of.n_terms;
        for (auto &pn : pend[fi]) {
            if (pn.term == 0xffffffffu) continue;
            add.push_back({pn.term, row_of(pn.doc), pn.tf, pn.len});
            max_term = std::max(max_term, pn.term + 1);
        }
        std::sort(add.begin(), add.end(), [](const Rec &a, const Rec &b) { return a.term != b.term ? a.term < b.term : a.row < b.row; });
        for (size_t i = 1; i < add.size(); i++)
            if (add[i].term == add[i - 1].term && add[i].row == add[i - 1].row)
                return abort_commit(fail(OC_ERR_INVALID, "field %zu: term %u listed twice in one insert of a document", fi, add[i].term));
        f.n_terms = max_term;
        f.term_offsets.assign(size_t(max_term) + 1, 0);
        f.host_post.clear();
        f.host_post.reserve(of.host_post.size() + add.size());
        std::vector<uint16_t> len_of_row(docs.size(), 0);
        size_t ai = 0;
        for (uint32_t t = 0; t < max_term; t++) {
            f.term_offsets[t] = f.host_post.size();
            uint64_t oi = t < of.n_terms ? of.term_offsets[t] : 0, oe = t < of.n_terms ? of.term_offsets[t + 1] : 0;
            auto old_next = [&]() -> bool {   // advances oi to the next surviving old posting of this term
                while (oi < oe) {
                    const uint32_t nr = remap[of.host_post[oi].row];
                    if (nr != 0xffffffffu && !replaced[nr]) return true;
                    oi++;
                }
                return false;
            };
            for (;;) {
                const bool ho = old_next(), hn = ai < add.size() && add[ai].term == t;
                if (!ho && !hn) break;
                PostingRaw pr;
                if (ho && (!hn || remap[of.host_post[oi].row] < add[ai].row)) {
                    pr.row = remap[of.host_post[oi].row]; pr.tf = of.host_post[oi].tf; pr.len = of.host_post[oi].len; oi++;
                } else {   // (equal rows cannot happen: a row with a pending insert is `replaced`)
                    pr.row = add[ai].row; pr.tf = add[ai].tf; pr.len = add[ai].len; ai++;
                }
                f.host_post.push_back(pr);
                len_of_row[pr.row] = pr.len;
            }
        }
        f.term_offsets[max_term] = f.host_post.size();
        const size_t n_recs = f.host_post.size();
        f.avg_len = of.avg_len;
        if (!global_avg) {
            double sum = 0; uint64_t cnt = 0;
            for (uint16_t l : len_of_row) if (l) { sum += l; cnt++; }
            if (cnt) f.avg_len = (float)(sum / (double)cnt);   // info().avg_field_length
        }
        f.n_post = n_recs;
        // per-term corpus df of a shard cannot be refreshed locally: sharded searches on this snapshot count
        // df across ranks (OC_SHARD_COUNT_DF) until the caller loads new global tables
    }
    const bool identity = !docs.empty() && docs.front() == 0 && docs.back() == docs.size() - 1;
    ns->n_rows = docs.size();
    ns->document_count = global_count ? B.document_count : docs.size();
    // ---- upload on the store's own stream (searches keep the ctx stream)
    auto upload = [&]() -> int {
        if (!identity && !docs.empty()) {
            ns->row_doc_host = docs;
            CU(cudaMalloc(&ns->row_doc, docs.size() * 8));
            CU(cudaMemcpyAsync(ns->row_doc, docs.data(), docs.size() * 8, cudaMemcpyHostToDevice, s->load_stream));
        }
        for (auto &f : ns->fields) {
            const uint64_t np = f.host_post.size();
            if (!np) continue;
            CU(cudaMalloc(&f.post, (np + 4) * sizeof(Posting)));
            CU(cudaMalloc(&f.raw, (np + 4) * sizeof(PostingRaw)));
            CU(cudaMemcpyAsync(f.raw, f.host_post.data(), np * sizeof(PostingRaw), cudaMemcpyHostToDevice, s->load_stream));
        }
        CU(cudaStreamSynchronize(s->load_stream));
        return OC_OK;
    };
    const int urc = upload();
    if (urc != OC_OK) return abort_commit(urc);
    // ---- publish: replay the deletes that arrived while we were building, then swap the pointer
    {
        std::lock_guard<std::mutex> g(s->mu);
        std::vector<uint64_t> rows;
        for (uint64_t d : s->deletes_during_commit) { const uint64_t r = ns->row_of(d); if (r != ~0ull) rows.push_back(r); }
        const int trc = snap_tombstone(*ns, rows, s->load_stream);
        if (trc != OC_OK) { s->committing = false; return trc; }   // (pending ops were consumed; the old snapshot stays published)
        ns->version = ++s->version;
        s->cur = ns;
        s->deletes_during_commit.clear();
        s->committing = false;
    }
    return OC_OK;
}

extern "C" int oc_str_info(oc_str *s, oc_str_info_t *out) {
    if (!s || !out) return fail(OC_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> g(s->mu);
    const StrSnap &S = *s->cur;
    out->total_documents = S.n_rows - S.n_deleted; out->n_fields = (uint32_t)S.fields.size();
    out->total_postings = 0; out->unique_terms_count = 0;
    for (auto &f : S.fields) { out->total_postings += f.n_post; out->unique_terms_count += f.n_terms; }
    out->device_bytes = out->total_postings * 16 + (S.row_doc ? S.n_rows * 8 : 0);
    out->version = S.version;
    out->pending_postings = 0;
    for (auto &p : s->pending) out->pending_postings += p.size();
    return OC_OK;
}

// ------------------------------------------------------------------------------------ device-resident filters
struct oc_facets;
struct oc_filter {
    oc_ctx *ctx;
    uint64_t nbits, words;
    uint64_t *bits = nullptr;   // device
};
__global__ void filter_scatter_ids_kernel(const uint64_t *ids, uint64_t n, uint64_t nbits, unsigned long long *bits) {
    const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint64_t d = ids[i];
    if (d < nbits) atomicOr(bits + (d >> 6), 1ull << (d & 63));
}
// op: 0 and, 1 or, 2 not(a); the padding bits of the last word stay clear
__global__ void filter_combine_kernel(const uint64_t *a, const uint64_t *b, uint64_t words, uint64_t nbits, int op, uint64_t *out) {
    const uint64_t w = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w >= words) return;
    uint64_t v = op == 0 ? (a[w] & b[w]) : op == 1 ? (a[w] | b[w]) : ~a[w];
    if (w == words - 1 && (nbits & 63)) v &= (1ull << (nbits & 63)) - 1;
    out[w] = v;
}
__global__ void filter_popcount_kernel(const uint64_t *a, uint64_t words, unsigned long long *out) {
    uint64_t c = 0;
    for (uint64_t w = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; w < words; w += uint64_t(gridDim.x) * blockDim.x) c += __popcll(a[w]);
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}
static int filter_alloc(oc_ctx *c, uint64_t nbits, oc_filter **out) {
    oc_filter *f = new oc_filter();
    f->ctx = c; f->nbits = nbits; f->words = (nbits + 63) / 64;
    cudaError_t e = cudaMalloc(&f->bits, std::max<uint64_t>(f->words, 1) * 8);
    if (e != cudaSuccess) { delete f; return fail(OC_ERR_OOM, "cudaMalloc(filter): %s", cudaGetErrorString(e)); }
    *out = f;
    return OC_OK;
}
extern "C" void oc_filter_destroy(oc_filter *f) {
    if (!f) return;
    std::lock_guard<std::mutex> g(f->ctx->mu);
    cudaSetDevice(f->ctx->device);
    cudaStreamSynchronize(f->ctx->stream);
    cudaFree(f->bits);
    delete f;
}
extern "C" int oc_filter_from_ids(oc_ctx *c, const uint64_t *doc_ids, uint64_t n, uint64_t nbits, oc_filter **out) {
    if (!c || !out || (n && !doc_ids)) return fail(OC_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    oc_filter *f = nullptr;
    OCTRY(filter_alloc(c, nbits, &f));
    CU(cudaMemsetAsync(f->bits, 0, std::max<uint64_t>(f->words, 1) * 8, c->stream));
    if (n) {
        OCTRY(c->in_blob.ensure(n * 8));
        CU(cudaMemcpyAsync(c->in_blob.p, doc_ids, n * 8, cudaMemcpyHostToDevice, c->stream));
        filter_scatter_ids_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>(c->in_blob.as<uint64_t>(), n, nbits,
                                                                                    reinterpret_cast<unsigned long long *>(f->bits));
        launched(c);
        CU(cudaGetLastError());
    }
    CU(cudaStreamSynchronize(c->stream));
    *out = f;
    return OC_OK;
}
extern "C" int oc_filter_from_bits(oc_ctx *c, const uint64_t *bits, uint64_t nbits, oc_filter **out) {
    if (!c || !out || (nbits && !bits)) return fail(OC_ERR_INVALID, "bad arguments");
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    oc_filter *f = nullptr;
    OCTRY(filter_alloc(c, nbits, &f));
    if (f->words) CU(cudaMemcpy(f->bits, bits, f->words * 8, cudaMemcpyHostToDevice));
    *out = f;
    return OC_OK;
}
static int filter_combine(const oc_filter *a, const oc_filter *b, int op, oc_filter **out) {
    if (!a || !out || (op != 2 && !b)) return fail(OC_ERR_INVALID, "NULL argument");
    if (b && (b->ctx != a->ctx || b->nbits != a->nbits)) return fail(OC_ERR_INVALID, "filters of different contexts / sizes");
    oc_ctx *c = a->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    oc_filter *f = nullptr;
    OCTRY(filter_alloc(c, a->nbits, &f));
    if (f->words) {
        filter_combine_kernel<<<(unsigned)((f->words + 255) / 256), 256, 0, c->stream>>>(a->bits, b ? b->bits : nullptr, f->words, f->nbits, op, f->bits);
        launched(c);
        CU(cudaGetLastError());
        CU(cudaStreamSynchronize(c->stream));
    }
    *out = f;
    return OC_OK;
}
extern "C" int oc_filter_and(const oc_filter *a, const oc_filter *b, oc_filter **out) { return filter_combine(a, b, 0, out); }
extern "C" int oc_filter_or(const oc_filter *a, const oc_filter *b, oc_filter **out) { return filter_combine(a, b, 1, out); }
extern "C" int oc_filter_not(const oc_filter *a, oc_filter **out) { return filter_combine(a, nullptr, 2, out); }
extern "C" int oc_filter_count(const oc_filter *f, uint64_t *out) {
    if (!f || !out) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = f->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    OCTRY(c->work_ctr.ensure(8));
    CU(cudaMemsetAsync(c->work_ctr.p, 0, 8, c->stream));
    if (f->words) {
        filter_popcount_kernel<<<(unsigned)std::min<uint64_t>((f->words + 255) / 256, 1184), 256, 0, c->stream>>>(
            f->bits, f->words, c->work_ctr.as<unsigned long long>());
        launched(c);
    }
    unsigned long long v = 0;
    CU(cudaMemcpyAsync(&v, c->work_ctr.p, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    *out = v;
    return OC_OK;
}
extern "C" int oc_filter_read(const oc_filter *f, uint64_t *out_bits) {
    if (!f || !out_bits) return fail(OC_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> g(f->ctx->mu);
    CU(cudaSetDevice(f->ctx->device));
    CU(cudaStreamSynchronize(f->ctx->stream));
    if (f->words) CU(cudaMemcpy(out_bits, f->bits, f->words * 8, cudaMemcpyDeviceToHost));
    return OC_OK;
}

// ------------------------------------------------------------------------------------ multi-index union (host)
// k-way merge of query q's per-index lists, each sorted by (score desc, doc asc) (NaN never reaches a list): the first
// `take` entries of the union, as (doc, score)
static void merge_union_top(uint32_t n_indexes, uint32_t q, uint32_t in_stride, const uint64_t *const *doc_ids,
                            const float *const *scores, const uint32_t *const *n, uint32_t take,
                            std::vector<std::pair<uint64_t, float>> &out) {
    std::vector<uint32_t> head(n_indexes, 0u);
    out.clear();
    while (out.size() < take) {
        int best = -1;
        for (uint32_t i = 0; i < n_indexes; i++) {
            if (head[i] >= n[i][q]) continue;
            if (best < 0) { best = (int)i; continue; }
            const float sa = scores[i][size_t(q) * in_stride + head[i]], sb = scores[best][size_t(q) * in_stride + head[best]];
            const uint64_t da = doc_ids[i][size_t(q) * in_stride + head[i]], db = doc_ids[best][size_t(q) * in_stride + head[best]];
            if (sa > sb || (sa == sb && da < db)) best = (int)i;
        }
        if (best < 0) break;
        out.emplace_back(doc_ids[best][size_t(q) * in_stride + head[best]], scores[best][size_t(q) * in_stride + head[best]]);
        head[best]++;
    }
}
// skip(offset).take(limit) of `top` into row q of the outputs (zero-padded)
static void write_page(const std::vector<std::pair<uint64_t, float>> &top, uint32_t q, uint32_t limit, uint32_t offset,
                       uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n) {
    uint32_t written = 0;
    for (size_t i = offset; i < top.size() && written < limit; i++, written++) {
        out_doc_ids[size_t(q) * limit + written] = top[i].first;
        out_scores[size_t(q) * limit + written] = top[i].second;
    }
    for (uint32_t k = written; k < limit; k++) { out_doc_ids[size_t(q) * limit + k] = 0; out_scores[size_t(q) * limit + k] = 0.f; }
    out_n[q] = written;
}

extern "C" int oc_merge_results(uint32_t n_indexes, uint32_t B, uint32_t limit, uint32_t offset, uint32_t in_stride,
                                const uint64_t *const *doc_ids, const float *const *scores, const uint32_t *const *n,
                                const uint64_t *const *counts, uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n,
                                uint64_t *out_count) {
    if (!doc_ids || !scores || !n || !counts || !out_doc_ids || !out_scores || !out_n || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (limit == 0) return fail(OC_ERR_INVALID, "limit must be >= 1");
    std::vector<std::pair<uint64_t, float>> top;
    for (uint32_t q = 0; q < B; q++) {
        uint64_t cnt = 0;
        for (uint32_t i = 0; i < n_indexes; i++) {
            if (n[i][q] > in_stride) return fail(OC_ERR_INVALID, "index %u query %u: n > in_stride", i, q);
            cnt += counts[i][q];
        }
        merge_union_top(n_indexes, q, in_stride, doc_ids, scores, n, uint32_t(std::min<uint64_t>(uint64_t(limit) + offset, 0xffffffffu)), top);
        write_page(top, q, limit, offset, out_doc_ids, out_scores, out_n);
        out_count[q] = cnt;
    }
    return OC_OK;
}

// apply_pin_rules_internal (read/sort.rs:285-391) on the host for query q: drop the promoted documents from top, then
// insert the items, stably sorted by position, each with the score of the index that holds the document (else 0.0)
static void splice_pins_host(std::vector<std::pair<uint64_t, float>> &top, const oc_pins *pins, uint32_t q, uint32_t n_indexes,
                             const float *const *pin_scores, const uint8_t *const *pin_present) {
    const uint32_t *off = pins->q_pin_offsets;
    std::vector<std::pair<uint32_t, uint32_t>> items;   // (position, item), sorted stably by position
    std::vector<uint64_t> promoted;
    for (uint32_t j = off[q]; j < off[q + 1]; j++) { items.emplace_back(pins->positions[j], j); promoted.push_back(pins->doc_ids[j]); }
    std::sort(promoted.begin(), promoted.end());
    top.erase(std::remove_if(top.begin(), top.end(),
                             [&](const std::pair<uint64_t, float> &e) { return std::binary_search(promoted.begin(), promoted.end(), e.first); }),
              top.end());
    std::stable_sort(items.begin(), items.end(), [](const std::pair<uint32_t, uint32_t> &a, const std::pair<uint32_t, uint32_t> &b) {
        return a.first < b.first;
    });
    for (const auto &it : items) {
        float s = 0.f;   // the disjoint maps: the score from the one index that holds the document, else 0.0
        for (uint32_t i = 0; i < n_indexes; i++)
            if (pin_present[i][it.second]) { s = pin_scores[i][it.second]; break; }
        top.insert(top.begin() + std::min<size_t>(it.first, top.size()), std::make_pair(pins->doc_ids[it.second], s));
    }
}

// apply_pin_rules_internal (read/sort.rs:285-391) on the host: the union's top list of an active query, spliced
extern "C" int oc_merge_pinned(uint32_t n_indexes, uint32_t B, uint32_t limit, uint32_t offset, uint32_t in_stride,
                               const uint64_t *const *doc_ids, const float *const *scores, const uint32_t *const *n,
                               const uint64_t *const *counts, const oc_pins *pins, const float *const *pin_scores,
                               const uint8_t *const *pin_present, uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n,
                               uint64_t *out_count) {
    if (!doc_ids || !scores || !n || !counts || !pins || !pins->q_pin_offsets || !out_doc_ids || !out_scores || !out_n || !out_count)
        return fail(OC_ERR_INVALID, "NULL argument");
    if (limit == 0) return fail(OC_ERR_INVALID, "limit must be >= 1");
    const uint32_t *off = pins->q_pin_offsets;
    const uint64_t top_pinned = (uint64_t(limit) + offset) * 2;
    bool any = false;
    for (uint32_t q = 0; q < B; q++) {   // everything is checked before anything is written
        if (off[q + 1] < off[q]) return fail(OC_ERR_INVALID, "pins: q_pin_offsets is not monotone at query %u", q);
        any = any || (pins->apply && off[q + 1] > off[q]);
        for (uint32_t i = 0; i < n_indexes; i++)
            if (n[i][q] > in_stride) return fail(OC_ERR_INVALID, "index %u query %u: n > in_stride", i, q);
    }
    if (any && (!pins->doc_ids || !pins->positions || !pin_scores || !pin_present)) return fail(OC_ERR_INVALID, "NULL pin argument");
    if (any && in_stride < top_pinned)
        return fail(OC_ERR_INVALID, "pins: in_stride %u < 2 x (limit+offset) %llu", in_stride, (unsigned long long)top_pinned);
    std::vector<std::pair<uint64_t, float>> top;
    for (uint32_t q = 0; q < B; q++) {
        uint64_t cnt = 0;
        for (uint32_t i = 0; i < n_indexes; i++) cnt += counts[i][q];
        const bool active = pins->apply && off[q + 1] > off[q];
        merge_union_top(n_indexes, q, in_stride, doc_ids, scores, n, uint32_t(active ? top_pinned : uint64_t(limit) + offset), top);
        if (active) splice_pins_host(top, pins, q, n_indexes, pin_scores, pin_present);
        write_page(top, q, limit, offset, out_doc_ids, out_scores, out_n);
        out_count[q] = cnt;
    }
    return OC_OK;
}

// MergeSortedIterator (read/sort.rs:491-559) on the host: the per-index lists, each in field order, merged by sort value;
// on equal values the index listed first wins (strict comparison), then pins and skip/take as oc_merge_pinned
extern "C" int oc_merge_sorted(uint32_t n_indexes, uint32_t B, uint32_t limit, uint32_t offset, uint32_t in_stride, int order,
                               const uint64_t *const *doc_ids, const float *const *scores, const double *const *sort_values,
                               const uint32_t *const *n, const uint64_t *const *counts, const oc_pins *pins,
                               const float *const *pin_scores, const uint8_t *const *pin_present, uint64_t *out_doc_ids,
                               float *out_scores, double *out_sort_values, uint32_t *out_n, uint64_t *out_count) {
    if (!doc_ids || !scores || !sort_values || !n || !counts || !out_doc_ids || !out_scores || !out_n || !out_count)
        return fail(OC_ERR_INVALID, "NULL argument");
    if (limit == 0) return fail(OC_ERR_INVALID, "limit must be >= 1");
    if (order != OC_SORT_ASC && order != OC_SORT_DESC) return fail(OC_ERR_INVALID, "sort order %d is neither ASC nor DESC", order);
    if (pins && !pins->q_pin_offsets) return fail(OC_ERR_INVALID, "pins: q_pin_offsets is NULL");
    const uint32_t *off = pins ? pins->q_pin_offsets : nullptr;
    const uint64_t top_plain = uint64_t(limit) + offset, top_pinned = top_plain * 2;
    bool any = false;
    for (uint32_t q = 0; q < B; q++) {   // everything is checked before anything is written
        if (off && off[q + 1] < off[q]) return fail(OC_ERR_INVALID, "pins: q_pin_offsets is not monotone at query %u", q);
        any = any || (off && pins->apply && off[q + 1] > off[q]);
        for (uint32_t i = 0; i < n_indexes; i++)
            if (n[i][q] > in_stride) return fail(OC_ERR_INVALID, "index %u query %u: n > in_stride", i, q);
    }
    if (any && (!pins->doc_ids || !pins->positions || !pin_scores || !pin_present)) return fail(OC_ERR_INVALID, "NULL pin argument");
    if (any && in_stride < top_pinned)
        return fail(OC_ERR_INVALID, "pins: in_stride %u < 2 x (limit+offset) %llu", in_stride, (unsigned long long)top_pinned);
    std::vector<std::pair<uint64_t, float>> top;
    std::vector<std::pair<uint64_t, double>> placed;   // (doc, sort value) of the merged entries, by doc
    std::vector<uint32_t> head(n_indexes);
    for (uint32_t q = 0; q < B; q++) {
        uint64_t cnt = 0;
        for (uint32_t i = 0; i < n_indexes; i++) cnt += counts[i][q];
        const bool active = off && pins->apply && off[q + 1] > off[q];
        const uint64_t take = active ? top_pinned : top_plain;
        std::fill(head.begin(), head.end(), 0u);
        top.clear(); placed.clear();
        while (top.size() < take) {
            int best = -1;
            for (uint32_t i = 0; i < n_indexes; i++) {
                if (head[i] >= n[i][q]) continue;
                if (best < 0) { best = (int)i; continue; }
                const double va = sort_values[i][size_t(q) * in_stride + head[i]], vb = sort_values[best][size_t(q) * in_stride + head[best]];
                if (order == OC_SORT_ASC ? va < vb : va > vb) best = (int)i;
            }
            if (best < 0) break;
            const size_t at = size_t(q) * in_stride + head[best];
            top.emplace_back(doc_ids[best][at], scores[best][at]);
            placed.emplace_back(doc_ids[best][at], sort_values[best][at]);
            head[best]++;
        }
        if (active) splice_pins_host(top, pins, q, n_indexes, pin_scores, pin_present);
        write_page(top, q, limit, offset, out_doc_ids, out_scores, out_n);
        out_count[q] = cnt;
        if (!out_sort_values) continue;
        std::sort(placed.begin(), placed.end());
        for (uint32_t k = 0; k < limit; k++) {
            double v = 0.0;
            if (k < out_n[q]) {
                const uint64_t d = out_doc_ids[size_t(q) * limit + k];
                bool promoted = false;
                for (uint32_t j = active ? off[q] : 0; active && j < off[q + 1]; j++) promoted = promoted || pins->doc_ids[j] == d;
                auto it = std::lower_bound(placed.begin(), placed.end(), std::make_pair(d, -std::numeric_limits<double>::infinity()));
                v = (promoted || it == placed.end() || it->first != d) ? std::numeric_limits<double>::quiet_NaN() : it->second;
            }
            out_sort_values[size_t(q) * limit + k] = v;
        }
    }
    return OC_OK;
}

// ------------------------------------------------------------------------------------ search()
// bm25.rs:78-82, evaluated on the host with libm (the same log1pf the oracle uses)
static inline float host_idf(float total_documents, uint64_t corpus_df) {
    const float df = (float)corpus_df;
    const float ratio = (total_documents - df + 0.5f) / (df + 0.5f);
    return log1pf(ratio);
}

template <bool MULTI, bool THRESH, bool OMC, bool ROWFT>
static int launch_tile_t(oc_ctx *c, const Bm25Params &bp, uint32_t grid, size_t smem, cudaStream_t st) {
    // (static smem counts against the 227 KB cap)
    if (smem_cfg_needed(c->device, (const void *)bm25_tile_kernel<MULTI, THRESH, OMC, ROWFT>, smem))
        CU(cudaFuncSetAttribute(bm25_tile_kernel<MULTI, THRESH, OMC, ROWFT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    bm25_tile_kernel<MULTI, THRESH, OMC, ROWFT><<<grid, BM25_THREADS, smem, st>>>(bp);
    launched(c);
    CU(cudaGetLastError());
    return OC_OK;
}
template <bool THRESH, bool OMC, bool ROWFT>
static int launch_tile2_t(oc_ctx *c, const Bm25Params &bp, size_t smem, cudaStream_t st, const ItemTok *flat, unsigned int *counter) {
    if (smem_cfg_needed(c->device, (const void *)bm25_tile2_kernel<THRESH, OMC, ROWFT>, smem))
        CU(cudaFuncSetAttribute(bm25_tile2_kernel<THRESH, OMC, ROWFT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    static std::mutex occ_mu;                         // occupancy per (device, shared-memory size): queried once
    static std::map<std::pair<int, size_t>, int> occ;
    int per_sm = 1;
    {
        std::lock_guard<std::mutex> g(occ_mu);
        auto it = occ.find(std::make_pair(c->device, smem));
        if (it == occ.end()) {
            CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bm25_tile2_kernel<THRESH, OMC, ROWFT>, BM25_THREADS, smem));
            occ[std::make_pair(c->device, smem)] = per_sm;
        } else per_sm = it->second;
    }
    const uint64_t items = uint64_t(bp.n_tiles) * bp.n_queries;
    const uint32_t grid = (uint32_t)std::min<uint64_t>(items, uint64_t(std::max(per_sm, 1)) * c->prop.multiProcessorCount);
    bm25_tile2_kernel<THRESH, OMC, ROWFT><<<grid, BM25_THREADS, smem, st>>>(bp, flat, counter);
    launched(c);
    CU(cudaGetLastError());
    return OC_OK;
}
// multi == false (every token resolves to <= 1 term): the posting-centred persistent kernel; else the slot-scan kernel
static int launch_tile(oc_ctx *c, const Bm25Params &bp_in, uint32_t grid, bool multi, bool thr, bool omc, cudaStream_t st,
                       uint32_t max_tokens, unsigned int *counter /* zeroed by the caller */, bool counted_df) {
    const char *env = getenv("OC_BM25_TILE2");
    if (!multi && !(env && env[0] == '0')) {
        // one level of descriptors per (tile, query) item, prefetched by the kernel during the previous item
        const ItemTok *flat = nullptr;
        const char *fenv = getenv("OC_BM25_FLAT");
        const char *t3e = getenv("OC_BM25_TILE3");
        const bool can_flat = max_tokens <= BM25_FLAT_TOK && !(fenv && fenv[0] == '0');
        // counted_df (filter / tombstones / OC_SHARD_COUNT_DF): no token has a host-known idf, so nothing is shared or dense
        // and every hot term arrives as a long posting list — the accumulator kernel walks those at ~10 instructions per
        // posting, the register-folded scorers would fold each posting's row separately
        const bool use3 = can_flat && !thr && !omc && !counted_df && !bp_in.matched_bits && !(t3e && t3e[0] == '0');
        Bm25Params bp = bp_in;
        // OC_BM25_ORDER=1: deal the items of the dense-token queries first and the list-only queries last (a lighter
        // ragged end of the persistent schedule); measured 1-2 % SLOWER on both bench shapes (the tile-major order of
        // ALL queries keeps the posting ranges of a tile together in L2), so the natural order is the default
        const char *oenv = getenv("OC_BM25_ORDER");
        if (!use3 || !(oenv && oenv[0] == '1')) bp.perm = nullptr;
        if (can_flat) {
            const uint64_t n_it = uint64_t(bp.n_tiles) * bp.n_queries * BM25_FLAT_TOK;
            OCTRY(c->flat_desc.ensure(n_it * sizeof(ItemTok)));
            bm25_flatten_kernel<<<(unsigned)((n_it + 255) / 256), 256, 0, st>>>(bp, c->flat_desc.as<ItemTok>());
            launched(c);
            CU(cudaGetLastError());
            flat = c->flat_desc.as<ItemTok>();
        }
        if (use3) {
            // plain queries: the register-folded scorer (no accumulator arrays)
            const size_t smem3 = bm25_tile3_smem_bytes(bp.cap);
            if (smem_cfg_needed(c->device, (const void *)bm25_tile3_kernel, smem3))
                CU(cudaFuncSetAttribute(bm25_tile3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem3));
            static std::mutex occ3_mu;
            static std::map<std::pair<int, size_t>, int> occ3;
            int per_sm = 1;
            {
                std::lock_guard<std::mutex> g(occ3_mu);
                auto it = occ3.find(std::make_pair(c->device, smem3));
                if (it == occ3.end()) {
                    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bm25_tile3_kernel, BM25_THREADS, smem3));
                    occ3[std::make_pair(c->device, smem3)] = per_sm;
                } else per_sm = it->second;
            }
            const uint64_t items = uint64_t(bp.n_tiles) * bp.n_queries;
            const uint32_t g3 = (uint32_t)std::min<uint64_t>(items, uint64_t(std::max(per_sm, 1)) * c->prop.multiProcessorCount);
            const char *seed_env = getenv("OC_BM25_SEED");
            if (bp.n_keep <= 32 && bp.n_tiles > 1 && !(seed_env && seed_env[0] == '0')) {   // warm start of the candidate thresholds
                bm25_seed_kernel<<<(bp.n_queries * 32 + 255) / 256, 256, 0, st>>>(bp);
                launched(c);
            }
            const char *wenv = getenv("OC_BM25_WARP");
            if (bp.n_keep <= 32 && !(wenv && wenv[0] == '0')) {   // a warp per item: no block barriers
                const size_t smemw = size_t(BW_WARPS) * sizeof(WarpScratch);
                if (smem_cfg_needed(c->device, (const void *)bm25_warp_kernel, smemw))
                    CU(cudaFuncSetAttribute(bm25_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemw));
                static std::mutex occw_mu;
                static std::map<int, int> occw;
                int pw = 1;
                {
                    std::lock_guard<std::mutex> g(occw_mu);
                    auto it = occw.find(c->device);
                    if (it == occw.end()) {
                        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&pw, bm25_warp_kernel, BW_WARPS * 32, smemw));
                        occw[c->device] = pw;
                    } else pw = it->second;
                }
                const uint32_t gw = (uint32_t)std::min<uint64_t>((items + BW_WARPS - 1) / BW_WARPS, uint64_t(std::max(pw, 1)) * c->prop.multiProcessorCount);
                bm25_warp_kernel<<<gw, BW_WARPS * 32, smemw, st>>>(bp, flat, counter);
                launched(c);
                CU(cudaGetLastError());
                return OC_OK;
            }
            bm25_tile3_kernel<<<g3, BM25_THREADS, smem3, st>>>(bp, flat, counter);
            launched(c);
            CU(cudaGetLastError());
            return OC_OK;
        }
        const size_t smem = bm25_tile2_smem_bytes(thr, omc, bp.cap);
        const int sel = (thr ? 2 : 0) | (omc ? 1 : 0);
        if (bp.row_ft) switch (sel) {   // group mode: the matched rows' scores too
            case 0: return launch_tile2_t<false, false, true>(c, bp, smem, st, flat, counter);
            case 1: return launch_tile2_t<false, true, true>(c, bp, smem, st, flat, counter);
            case 2: return launch_tile2_t<true, false, true>(c, bp, smem, st, flat, counter);
            default: return launch_tile2_t<true, true, true>(c, bp, smem, st, flat, counter);
        }
        switch (sel) {
            case 0: return launch_tile2_t<false, false, false>(c, bp, smem, st, flat, counter);
            case 1: return launch_tile2_t<false, true, false>(c, bp, smem, st, flat, counter);
            case 2: return launch_tile2_t<true, false, false>(c, bp, smem, st, flat, counter);
            default: return launch_tile2_t<true, true, false>(c, bp, smem, st, flat, counter);
        }
    }
    Bm25Params bp = bp_in;
    bp.perm = nullptr;
    const size_t smem = bm25_smem_bytes(multi, thr, omc, bp.cap);
    const int sel = (multi ? 4 : 0) | (thr ? 2 : 0) | (omc ? 1 : 0);
    if (bp.row_ft) switch (sel) {   // group mode: the matched rows' scores too
        case 0: return launch_tile_t<false, false, false, true>(c, bp, grid, smem, st);
        case 1: return launch_tile_t<false, false, true, true>(c, bp, grid, smem, st);
        case 2: return launch_tile_t<false, true, false, true>(c, bp, grid, smem, st);
        case 3: return launch_tile_t<false, true, true, true>(c, bp, grid, smem, st);
        case 4: return launch_tile_t<true, false, false, true>(c, bp, grid, smem, st);
        case 5: return launch_tile_t<true, false, true, true>(c, bp, grid, smem, st);
        case 6: return launch_tile_t<true, true, false, true>(c, bp, grid, smem, st);
        default: return launch_tile_t<true, true, true, true>(c, bp, grid, smem, st);
    }
    switch (sel) {
        case 0: return launch_tile_t<false, false, false, false>(c, bp, grid, smem, st);
        case 1: return launch_tile_t<false, false, true, false>(c, bp, grid, smem, st);
        case 2: return launch_tile_t<false, true, false, false>(c, bp, grid, smem, st);
        case 3: return launch_tile_t<false, true, true, false>(c, bp, grid, smem, st);
        case 4: return launch_tile_t<true, false, false, false>(c, bp, grid, smem, st);
        case 5: return launch_tile_t<true, false, true, false>(c, bp, grid, smem, st);
        case 6: return launch_tile_t<true, true, false, false>(c, bp, grid, smem, st);
        default: return launch_tile_t<true, true, true, false>(c, bp, grid, smem, st);
    }
}

#include "shard.cuh"
#include "batcher.h"

struct FacetJob {   // oc_search_facets: count, per query, the matched documents of each requested variant
    oc_facets *fc;
    const oc_facet_req *reqs;
    uint32_t n_reqs;
    uint64_t *out_counts;   // [B][n_reqs]
};
static int run_facets(oc_ctx *c, const FacetJob &fj, uint32_t B, bool has_ft, bool has_v, const StrSnap *S, uint32_t n_tiles,
                      uint32_t vlimit);
struct GroupJob {   // oc_search_groups: the top max_results documents of every (query, group)
    oc_group_by *g;
    uint32_t max_results;
    uint64_t *out_doc;      // [B][G][max_results]
    float *out_score;
    uint32_t *out_n;        // [B][G]
    uint32_t stride = 0;    // oc_search_groups_pinned: row stride of the group arrays ([B][G][stride])
};
struct PinJob {   // oc_search_pinned / oc_search_groups_pinned: the promote items, padded to `stride` slots per query
    uint32_t stride = 0;                // most items of one query (0: no item in the batch)
    bool splice = false;                // pins apply and some query has items: top lists at twice the depth + the splice
    std::vector<uint64_t> doc;          // [B][stride]
    std::vector<uint32_t> pos, cnt;     // [B][stride], [B]
    const uint64_t *d_doc = nullptr;    // their device copies (set by search_impl)
    const uint32_t *d_pos = nullptr, *d_cnt = nullptr;
};
// Checks and pads the items of pins (NULL: none).  Nothing is written on failure.
static int pin_job_init(const oc_pins *pins, uint32_t B, PinJob &pj) {
    if (!pins) return OC_OK;
    const uint32_t *off = pins->q_pin_offsets;
    if (!off) return fail(OC_ERR_INVALID, "pins: q_pin_offsets is NULL");
    uint32_t most = 0;
    for (uint32_t q = 0; q < B; q++) {
        if (off[q + 1] < off[q]) return fail(OC_ERR_INVALID, "pins: q_pin_offsets is not monotone at query %u", q);
        most = std::max(most, off[q + 1] - off[q]);
    }
    if (most > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "pins: a query has %u items > %u", most, OC_MAX_TOPK);
    if (uint64_t(B) * most * 32 > 0x7fffffffull) return fail(OC_ERR_UNSUPPORTED, "pins: %u queries x %u items: pass smaller batches", B, most);
    if (most && (!pins->doc_ids || !pins->positions)) return fail(OC_ERR_INVALID, "pins: doc_ids / positions are NULL");
    pj.stride = most;
    pj.splice = pins->apply && most > 0;
    pj.doc.assign(size_t(B) * most, 0);
    pj.pos.assign(size_t(B) * most, 0);
    pj.cnt.assign(B, 0);
    for (uint32_t q = 0; q < B; q++) {
        pj.cnt[q] = off[q + 1] - off[q];
        for (uint32_t j = 0; j < pj.cnt[q]; j++) {
            pj.doc[size_t(q) * most + j] = pins->doc_ids[off[q] + j];
            pj.pos[size_t(q) * most + j] = pins->positions[off[q] + j];
        }
    }
    return OC_OK;
}
// ------------------------------------------------------------------------------------ sortBy (sort.cuh)
// A sort field, per order: the documents in rank order (value, then ascending id; each document once, at its first
// value in that order), the rank of every document id, and the string row of every rank for one snapshot of one string
// store (rebuilt when a search sees another snapshot, i.e. after a commit).  Host copies give the outputs' sort values.
struct SortOrder {
    uint64_t n = 0;
    uint64_t *rank_doc = nullptr;          // device [n]
    uint32_t *doc_rank = nullptr;          // device [nbits], RANK_NONE = no value
    uint32_t *rank_row = nullptr;          // device [n + 1]; rank_row[n] = RANK_NONE (the mapping kernel's count)
    std::weak_ptr<StrSnap> rows_of;        // the snapshot rank_row maps to
    std::vector<uint32_t> h_doc_rank;      // [nbits]
    std::vector<double> h_value;           // [n] value of each rank
};
struct oc_sort_field {
    oc_ctx *ctx;
    uint64_t nbits;
    SortOrder ord[2];                      // OC_SORT_ASC, OC_SORT_DESC
};
static void sort_field_free(oc_sort_field *f) {
    for (SortOrder &o : f->ord) { cudaFree(o.rank_doc); cudaFree(o.doc_rank); cudaFree(o.rank_row); }
    delete f;
}
struct SortJob {
    oc_sort_field *f;
    int order;
    double *out_values;                    // B x limit, may be NULL
    double *out_group_values;              // B x n_groups x group_stride, may be NULL
    uint32_t n_groups;
};
static int sort_job_init(oc_ctx *c, const oc_sort *s, SortJob &sj) {
    if (!s || !s->field) return fail(OC_ERR_INVALID, "NULL sort");
    if (s->order != OC_SORT_ASC && s->order != OC_SORT_DESC) return fail(OC_ERR_INVALID, "sort order %d is neither ASC nor DESC", s->order);
    if (s->field->ctx != c) return fail(OC_ERR_INVALID, "sort field belongs to another ctx");
    sj.f = const_cast<oc_sort_field *>(s->field);   // only its per-snapshot row map is refreshed, under the ctx lock
    sj.order = s->order;
    return OC_OK;
}
// the value a listed document was placed by: NaN for a document the (active) query promotes, else its value
static double sort_value_of(const SortJob &sj, const PinJob *pj, uint32_t q, uint64_t d) {
    if (pj && pj->splice)
        for (uint32_t j = 0; j < pj->cnt[q]; j++)
            if (pj->doc[size_t(q) * pj->stride + j] == d) return std::numeric_limits<double>::quiet_NaN();
    const SortOrder &o = sj.f->ord[sj.order];
    const uint32_t r = d < sj.f->nbits ? o.h_doc_rank[d] : RANK_NONE;
    return r == RANK_NONE ? std::numeric_limits<double>::quiet_NaN() : o.h_value[r];
}
// rank -> string row of snapshot S (kept until another snapshot is searched)
static int sort_rows_for(oc_ctx *c, SortOrder &o, const std::shared_ptr<StrSnap> &snap) {
    if (o.rows_of.lock() == snap) return OC_OK;
    constexpr uint64_t CH = 1ull << 30;
    for (uint64_t a = 0; a < o.n; a += CH) {
        const uint32_t len = (uint32_t)std::min<uint64_t>(CH, o.n - a);
        map_docs_to_rows_kernel<<<(len + 255) / 256, 256, 0, c->stream>>>(o.rank_doc + a, o.rank_row + o.n, len, 1, snap->row_doc,
                                                                          snap->n_rows, o.rank_row + a);
        launched(c);
        CU(cudaGetLastError());
    }
    o.rows_of = snap;
    return OC_OK;
}

static int run_groups(oc_ctx *c, const GroupJob &gj, uint32_t B, int mode, const StrSnap *S, uint32_t n_tiles, uint32_t vlimit,
                      const uint64_t *omc_doc, const float *omc_mult, uint32_t n_omc, const PinJob *pj, const SortJob *sj);

// gj != NULL: oc_search_groups.  Then limit == 0 is allowed: the hits are not written (out_doc_ids / out_scores / out_n
// may be NULL), the vector stage gets depth 0 and the fulltext stage runs with one candidate slot per tile.
// pj != NULL: the pinned calls; the items' score-map values go to out_pin_scores / out_pin_present (may be NULL).
// sj != NULL: the sorted calls (always with pj); the hits are the walk's in field order, K4's list only gives the count.
static int search_impl(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, uint64_t *out_doc_ids,
                       float *out_scores, uint32_t *out_n, uint64_t *out_count, const FacetJob *fj, const GroupJob *gj = nullptr,
                       PinJob *pj = nullptr, const oc_pins *pins = nullptr, float *out_pin_scores = nullptr,
                       uint8_t *out_pin_present = nullptr, const SortJob *sj = nullptr) {
    if (!c || !p || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    const bool write_hits = !gj || p->limit > 0;
    if (write_hits && (!out_doc_ids || !out_scores || !out_n)) return fail(OC_ERR_INVALID, "NULL argument");
    const uint32_t B = p->n_queries;
    if (B == 0) return OC_OK;
    const bool has_v = p->mode == OC_MODE_VECTOR || p->mode == OC_MODE_HYBRID;
    const bool has_ft = p->mode == OC_MODE_FULLTEXT || p->mode == OC_MODE_HYBRID;
    if (!has_v && !has_ft) return fail(OC_ERR_INVALID, "unknown mode %d", p->mode);
    if (has_v && (!emb || !p->q_vecs)) return fail(OC_ERR_INVALID, "vector/hybrid mode needs emb and q_vecs");
    if (has_ft && (!str || !p->q_token_offsets)) return fail(OC_ERR_INVALID, "fulltext/hybrid mode needs str and tokens");
    if (emb && emb->ctx != c) return fail(OC_ERR_INVALID, "emb belongs to another ctx");
    if (str && str->ctx != c) return fail(OC_ERR_INVALID, "str belongs to another ctx");
    // per-query where-filters: deduplicated by handle; all NULL = unfiltered, one handle for every query = p->filter
    const oc_filter *batch_filter = p->filter;
    QFilterJob qfj;
    bool per_q = false;
    if (p->q_filters) {
        if (gj || pj || sj) return fail(OC_ERR_UNSUPPORTED, "q_filters: per-query filters are supported by oc_search only");
        if (p->filter || p->filter_bits) return fail(OC_ERR_INVALID, "q_filters together with filter / filter_bits");
        if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "q_filters over a sharded search");
        std::unordered_map<const oc_filter *, uint32_t> idx;
        std::vector<const oc_filter *> distinct;
        bool any_none = false;
        qfj.q_slot.resize(B);
        for (uint32_t b = 0; b < B; b++) {
            const oc_filter *f = p->q_filters[b];
            if (!f) { any_none = true; qfj.q_slot[b] = SLOT_NONE; continue; }
            if (f->ctx != c) return fail(OC_ERR_INVALID, "q_filters[%u] belongs to another ctx", b);
            auto it = idx.emplace(f, (uint32_t)distinct.size()).first;
            if (it->second == distinct.size()) distinct.push_back(f);
            qfj.q_slot[b] = it->second;
        }
        if (distinct.size() > 65535) return fail(OC_ERR_UNSUPPORTED, "q_filters: %zu distinct handles > 65535", distinct.size());
        if (distinct.size() == 1 && !any_none) batch_filter = distinct[0];
        else if (!distinct.empty()) {
            per_q = true;
            const uint32_t K = (uint32_t)distinct.size();
            for (const oc_filter *f : distinct) qfj.slots.push_back(RowsOkSlot{f->bits, f->nbits});
            qfj.slots.push_back(RowsOkSlot{nullptr, 0});
            qfj.q_slot_ft.resize(B);
            for (uint32_t b = 0; b < B; b++) qfj.q_slot_ft[b] = qfj.q_slot[b] == SLOT_NONE ? K : qfj.q_slot[b];
        }
    }
    if (p->limit == 0 && !gj) return fail(OC_ERR_INVALID, "limit must be >= 1");
    const uint32_t limit = write_hits ? p->limit : 1;
    // sort_token_scores with pins selects the top 2 * (limit + offset) (sort.rs:25-34); the vector depth stays limit
    const bool pin_flat = pj && pj->splice && write_hits && !sj;
    const bool sort_flat = sj && write_hits;
    // sort_token_scores with sort_by: top_count keys in field order, twice as many for an active pinned query
    const uint32_t sort_top = sort_flat ? uint32_t((uint64_t(limit) + p->offset) * (pj->splice ? 2 : 1)) : 0u;
    const uint64_t n_keep64 = (uint64_t(limit) + p->offset) * (pin_flat ? 2 : 1);
    if (n_keep64 > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "limit+offset %llu > %u", (unsigned long long)n_keep64, OC_MAX_TOPK);
    const uint32_t n_keep = (uint32_t)n_keep64;
    // limit_hint = limit, NOT limit+offset (search.rs:330-336); vector_limit lets a multi-index caller keep that depth
    const uint32_t vlimit = !write_hits ? 0u : p->vector_limit ? p->vector_limit : limit;
    if (vlimit > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "vector_limit %u > %u", vlimit, OC_MAX_TOPK);
    if (p->sharded && !c->comm.ready()) return fail(OC_ERR_COMM, "sharded search without oc_comm_init");

    // the published snapshot of the string store: grabbed once, immutable for the whole call (a commit may
    // publish the next version meanwhile); declared before the lock so a last reference dies outside it
    std::shared_ptr<StrSnap> snap = str ? str_snapshot(str) : nullptr;
    StrSnap *S = snap.get();
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    begin_call(c);

    // staged segments go in one copy per contiguous run; pinned caller buffers are DMA'd directly
    auto upload = [&](const Packer &pk, HostBuf &hb, DevBuf &db, cudaStream_t st) -> int {
        OCTRY(hb.ensure(pk.total + 256));
        OCTRY(db.ensure(pk.total + 256));
        pk.fill(hb.p);
        size_t run0 = 0;
        for (size_t i = 0; i <= pk.segs.size(); i++) {
            const bool brk = i == pk.segs.size() || pk.segs[i].direct;
            if (brk) {
                const size_t end = i == pk.segs.size() ? pk.total : pk.segs[i].off;
                if (end > run0) CU(cudaMemcpyAsync(db.as<uint8_t>() + run0, hb.as<uint8_t>() + run0, end - run0, cudaMemcpyHostToDevice, st));
                if (i < pk.segs.size()) {
                    CU(cudaMemcpyAsync(db.as<uint8_t>() + pk.segs[i].off, pk.segs[i].src, pk.segs[i].bytes, cudaMemcpyHostToDevice, st));
                    run0 = pk.segs[i].off + pk.segs[i].bytes;
                }
            }
        }
        return OC_OK;
    };
    // ------------------------------------------------------------ vector stage first: the query vectors
    // (+ filter) go up alone and the matrix sweep starts; the host-side descriptor work below overlaps it
    if (batch_filter && batch_filter->ctx != c) return fail(OC_ERR_INVALID, "filter belongs to another ctx");
    const bool filter_h = !batch_filter && p->filter_bits != nullptr;     // host bitmap: uploaded with this call
    const bool filter = filter_h || batch_filter != nullptr;
    const uint64_t filter_nbits = batch_filter ? batch_filter->nbits : p->filter_nbits;
    const size_t fwords = filter_h ? (p->filter_nbits + 63) / 64 : 0;
    const uint64_t *filter_dev = batch_filter ? batch_filter->bits : nullptr;
    // per-query filters: the slot tables travel with the first upload of the call
    auto add_qf = [&](Packer &pk, size_t o[3]) {
        o[0] = pk.add(qfj.slots.data(), qfj.slots.size() * sizeof(RowsOkSlot));
        o[1] = pk.add(qfj.q_slot.data(), size_t(B) * 4);
        o[2] = pk.add(qfj.q_slot_ft.data(), size_t(B) * 4);
    };
    auto bind_qf = [&](uint8_t *base, const size_t o[3]) {
        qfj.d_slots = reinterpret_cast<const RowsOkSlot *>(base + o[0]);
        qfj.d_q_slot = reinterpret_cast<const uint32_t *>(base + o[1]);
        qfj.d_q_slot_ft = reinterpret_cast<const uint32_t *>(base + o[2]);
    };
    size_t h2d_early = 0;
    if (has_v) {
        Packer pk0;
        const size_t o_qv = pk0.add(p->q_vecs, size_t(B) * emb->dim * 4, is_pinned_host(p->q_vecs));
        const size_t o_flt = filter_h ? pk0.add(p->filter_bits, fwords * 8) : 0;
        size_t o_qf[3] = {0, 0, 0};
        if (per_q) add_qf(pk0, o_qf);
        CU(cudaEventRecord(c->ev[EV_START], c->stream));
        OCTRY(upload(pk0, c->h_in0, c->in_blob0, c->stream));
        CU(cudaEventRecord(c->ev[EV_H2D], c->stream));
        h2d_early = pk0.total;
        if (filter_h) filter_dev = reinterpret_cast<const uint64_t *>(c->in_blob0.as<uint8_t>() + o_flt);
        if (per_q) bind_qf(c->in_blob0.as<uint8_t>(), o_qf);
        if (vlimit) {
            OCTRY(run_vector_stage(c, emb, reinterpret_cast<const float *>(c->in_blob0.as<uint8_t>() + o_qv), B, vlimit, p->similarity,
                                   filter_dev, filter_nbits, per_q ? &qfj : nullptr));
        } else {   // limit_hint 0 (groups only): no vector hit
            OCTRY(c->v_cnt.ensure(size_t(B) * 4));
            CU(cudaMemsetAsync(c->v_cnt.p, 0, size_t(B) * 4, c->stream));
        }
    }

    // ------------------------------------------------------------ host: descriptors
    const bool multi_rank = p->sharded && c->comm.world > 1;
    // sharded: every rank must take the same df decisions (they drive a collective), so the
    // tombstone state is the caller's global flag (OC_SHARD_TOMBSTONES), not this shard's
    const bool tombs_local = has_ft && S->n_deleted > 0;
    if (multi_rank && tombs_local && !(p->sharded & OC_SHARD_TOMBSTONES))
        return fail(OC_ERR_INVALID, "sharded search: this shard holds tombstones, set OC_SHARD_TOMBSTONES on every rank");
    const bool tombs = has_ft && (multi_rank ? (p->sharded & OC_SHARD_TOMBSTONES) != 0 : tombs_local);
    const uint32_t n_tiles = has_ft ? (uint32_t)((S->n_rows + BM25_TILE - 1) / BM25_TILE) : 0;
    std::vector<TermDesc> terms;
    std::vector<uint32_t> term_token;
    std::vector<uint64_t> term_key;     // (field << 32 | term id) of each expanded term
    std::vector<TokenDesc> tokens;
    std::vector<QueryDesc> queries;
    std::vector<uint8_t> tok_need_df;
    std::vector<uint32_t> tok_slot;     // per-query filters: the fulltext slot of each token's query
    std::vector<PreDesc> pre_descs;
    std::vector<uint2> pre_items;
    bool any_multi = false, need_df = false, derived_now = false;
    uint32_t max_tokens = 0;    // tokens of the longest query of the batch
    uint64_t dense_bytes = 0;   // dense contribution arrays of this batch (zeroed before the precompute kernel fills them)
    // sharded: df comes from the replicated per-term table, or — OC_SHARD_COUNT_DF on every rank, e.g. after a
    // commit dropped the table — from counting + all-reduce.  A shard-local list length is never a corpus df.
    const bool count_df = multi_rank && (p->sharded & OC_SHARD_COUNT_DF) != 0;
    bool df_local_only = false;
    uint64_t postings_walked = 0;
    const bool thr = p->threshold >= 0.0f;
    if (has_ft) {
        for (auto &f : S->fields)   // streamed posting format depends on (avg_field_len, b): derive once
            if (f.n_post && f.b_cached != p->bm25_b) {
                bm25_derive_postings_kernel<<<(unsigned)((f.n_post + 255) / 256), 256, 0, c->stream>>>(f.raw, f.n_post, f.avg_len, p->bm25_b, f.post);
                launched(c);
                CU(cudaGetLastError());
                f.b_cached = p->bm25_b;
                derived_now = true;   // queued on the main stream: this call keeps the BM25 prologue there too
            }
        const float N = (float)S->document_count;  // token_score.rs:221
        queries.resize(B);
        // Per-query filters are routed as a filtered batch is: df is counted on the device (need_df), so nothing is shared
        // or dense and K3b / K3 score the batch, each (tile, query) item under its query's row bitmap.  A token keeps the
        // idf its query would get alone: counted under the query's filter, or — single term, no filter, no tombstones —
        // from the host's posting-list length (or corpus df table), as a plain oc_search does.  An unfiltered query runs
        // under the tombstone-only row bitmap (slot K), so it scores exactly the rows it would score alone.
        if (per_q) need_df = true;
        for (uint32_t q = 0; q < B; q++) {
            const uint32_t t0 = p->q_token_offsets[q], t1 = p->q_token_offsets[q + 1];
            const bool q_filter = filter || (per_q && qfj.q_slot[q] != SLOT_NONE);
            QueryDesc qd{};
            qd.token_begin = (uint32_t)tokens.size();
            const uint32_t ntok = t1 - t0;
            max_tokens = std::max(max_tokens, ntok);
            qd.required = thr ? (uint32_t)floorf((float)ntok * p->threshold) : 0;  // token_score.rs:211-218
            qd.flags = thr ? QF_THRESHOLD : 0;
            for (uint32_t t = t0; t < t1; t++) {
                TokenDesc tk{};
                tk.term_begin = (uint32_t)terms.size();
                tk.bit = 1u << ((t - t0) & 31u);
                uint64_t df_known = 0;
                for (uint32_t e = p->token_term_offsets[t]; e < p->token_term_offsets[t + 1]; e++) {
                    const uint32_t fi = p->term_field[e], ti = p->term_id[e];
                    if (fi >= S->fields.size()) return fail(OC_ERR_INVALID, "term field %u out of range", fi);
                    const StrField &f = S->fields[fi];
                    if (ti >= f.n_terms) continue;  // unknown term: no postings
                    TermDesc td{};
                    td.ptr = f.post + f.term_offsets[ti];
                    td.len = (uint32_t)(f.term_offsets[ti + 1] - f.term_offsets[ti]);
                    td.weight = p->term_weight ? p->term_weight[e] : 1.0f;
                    td.avg_len = f.avg_len;
                    df_known = f.global_df.empty() ? td.len : f.global_df[ti];
                    if (multi_rank && f.global_df.empty()) df_local_only = true;
                    postings_walked += td.len;
                    term_key.push_back((uint64_t(fi) << 32) | ti);
                    terms.push_back(td);
                    term_token.push_back((uint32_t)tokens.size());
                }
                tk.term_end = (uint32_t)terms.size();
                const uint32_t nt = tk.term_end - tk.term_begin;
                uint8_t need = 0;
                if (nt == 1 && !q_filter && !tombs && !count_df) tk.idf = host_idf(N, std::max<uint64_t>(1, df_known));
                else if (nt == 0) tk.idf = host_idf(N, 1);
                else { need = 1; need_df = true; tk.idf = 0.f; }
                if (nt != 1) { any_multi = any_multi || nt > 1; }
                tokens.push_back(tk);
                tok_need_df.push_back(need);
                if (per_q) tok_slot.push_back(qfj.q_slot_ft[q]);
            }
            qd.token_end = (uint32_t)tokens.size();
            queries[q] = qd;
        }
        if (df_local_only && !count_df)
            return fail(OC_ERR_INVALID, "sharded search: a field of this shard has no corpus-wide df table (dropped by a commit?): "
                                        "reload it or pass OC_SHARD_COUNT_DF on every rank");
        // ---- batch-level sharing of per-posting contributions (single-term tokens with a host-known idf); not with
        // per-query filters: the precomputed contributions and dense arrays are masked by ONE row bitmap
        if (!per_q) {
            struct U { uint32_t first_e; uint32_t uses; };
            struct K128 { uint64_t a, b; };            // (field, term) | (weight bits, idf bits)
            size_t cap_t = 64;
            while (cap_t < tokens.size() * 2) cap_t <<= 1;
            std::vector<K128> tab_k(cap_t);
            std::vector<uint32_t> tab_v(cap_t, 0xffffffffu);   // open addressing, linear probing
            std::vector<U> uniq;
            std::vector<uint32_t> e_to_u(terms.size(), 0xffffffffu);
            uint64_t walked = 0, distinct = 0;
            for (size_t t = 0; t < tokens.size(); t++) {
                const TokenDesc &tk = tokens[t];
                if (tk.term_end - tk.term_begin != 1 || tok_need_df[t]) continue;
                const uint32_t e = tk.term_begin;
                if (terms[e].len < 64) continue;
                uint32_t wb, ib;
                memcpy(&wb, &terms[e].weight, 4); memcpy(&ib, &tk.idf, 4);
                const K128 key{term_key[e], (uint64_t(wb) << 32) | ib};
                uint64_t h = (key.a * 0x9E3779B97F4A7C15ull) ^ (key.b * 0xC2B2AE3D27D4EB4Full);
                size_t slot = (h ^ (h >> 29)) & (cap_t - 1);
                while (tab_v[slot] != 0xffffffffu && !(tab_k[slot].a == key.a && tab_k[slot].b == key.b)) slot = (slot + 1) & (cap_t - 1);
                if (tab_v[slot] == 0xffffffffu) {
                    tab_k[slot] = key; tab_v[slot] = (uint32_t)uniq.size();
                    uniq.push_back({e, 0}); distinct += terms[e].len;
                }
                uniq[tab_v[slot]].uses++;
                e_to_u[e] = tab_v[slot];
                walked += terms[e].len;
            }
            const char *share_env = getenv("OC_BM25_SHARE");   // "off" / "force": A/B testing of the sharing pass
            const bool share_off = share_env && !strcmp(share_env, "off"), share_force = share_env && !strcmp(share_env, "force");
            // hot terms (a posting in at least every 16th row) go DENSE: their contributions are scattered once per batch
            // into a float[rows] array and every (query, tile) item adds 8192 floats with 128-bit loads instead of
            // walking ~thousands of postings (posting-centred kernel only: every token of the batch has <= 1 term)
            const char *dense_env = getenv("OC_BM25_DENSE");
            const char *t2_env = getenv("OC_BM25_TILE2");
            const bool dense_on = !any_multi && !(dense_env && dense_env[0] == '0') && !share_off && !(t2_env && t2_env[0] == '0');
            const uint64_t rows_pad = uint64_t(n_tiles) * BM25_TILE;
            const uint64_t dense_min = std::max<uint64_t>(512, S->n_rows / 16);
            std::vector<uint8_t> u_dense(uniq.size(), 0);
            uint64_t n_dense = 0;
            if (dense_on)
                for (size_t u = 0; u < uniq.size(); u++)
                    if (terms[uniq[u].first_e].len >= dense_min && (n_dense + 1) * rows_pad * 4 <= (size_t(8) << 30)) { u_dense[u] = 1; n_dense++; }
            uint64_t walked_l = 0, distinct_l = 0;   // what is left for the list form
            for (size_t e = 0; e < terms.size(); e++)
                if (e_to_u[e] != 0xffffffffu && !u_dense[e_to_u[e]]) walked_l += terms[e].len;
            for (size_t u = 0; u < uniq.size(); u++) if (!u_dense[u]) distinct_l += terms[uniq[u].first_e].len;
            const bool lists = distinct_l && !share_off && (share_force || (walked_l >= 2 * distinct_l && walked_l >= (64u << 20))) &&
                               distinct_l * 8 <= (size_t(6) << 30);
            if (lists || n_dense) {
                if (lists) OCTRY(c->pre_post.ensure(distinct_l * 8 + 64));
                if (n_dense) OCTRY(c->dense_buf.ensure(n_dense * rows_pad * 4));
                dense_bytes = n_dense * rows_pad * 4;
                uint64_t off = 0, doff = 0;
                std::vector<uint64_t> u_off(uniq.size());
                std::vector<uint8_t> u_used(uniq.size(), 0);
                for (size_t u = 0; u < uniq.size(); u++) {
                    if (!u_dense[u] && !lists) continue;
                    u_used[u] = 1;
                    const TermDesc &td = terms[uniq[u].first_e];
                    PreDesc pd{};
                    pd.src = td.ptr; pd.len = td.len; pd.weight = td.weight;
                    pd.idf = tokens[term_token[uniq[u].first_e]].idf;
                    if (u_dense[u]) { u_off[u] = doff; pd.dense = c->dense_buf.as<float>() + doff; doff += rows_pad; }
                    else { u_off[u] = off; pd.dst = c->pre_post.as<Posting>() + off; off += td.len; }
                    const uint32_t pi = (uint32_t)pre_descs.size();
                    pre_descs.push_back(pd);
                    for (uint32_t ch = 0; ch * PRE_CHUNK < td.len; ch++) pre_items.push_back(make_uint2(pi, ch));
                }
                for (size_t e = 0; e < terms.size(); e++) {
                    const uint32_t u = e_to_u[e];
                    if (u == 0xffffffffu || !u_used[u]) continue;
                    if (u_dense[u]) { terms[e].ptr = reinterpret_cast<const Posting *>(c->dense_buf.as<float>() + u_off[u]); terms[e].flags |= TD_DENSE; }
                    else { terms[e].ptr = c->pre_post.as<Posting>() + u_off[u]; terms[e].flags |= TD_PRE; }
                }
            }
        }
    }
    // OMC rows for the tile kernel (string rows, ascending)
    std::vector<uint32_t> omc_rows; std::vector<float> omc_row_mult;
    const uint32_t n_omc = (uint32_t)p->n_omc;
    if (n_omc && (!p->omc_doc_ids || !p->omc_mult)) return fail(OC_ERR_INVALID, "omc arrays are NULL");
    if (n_omc && has_ft) {
        for (uint32_t i = 0; i < n_omc; i++) {
            if (i && p->omc_doc_ids[i] <= p->omc_doc_ids[i - 1]) return fail(OC_ERR_INVALID, "omc_doc_ids must be ascending");
            uint64_t r;
            if (S->row_doc_host.empty()) { r = p->omc_doc_ids[i]; if (r >= S->n_rows) continue; }
            else {
                auto it = std::lower_bound(S->row_doc_host.begin(), S->row_doc_host.end(), p->omc_doc_ids[i]);
                if (it == S->row_doc_host.end() || *it != p->omc_doc_ids[i]) continue;
                r = uint64_t(it - S->row_doc_host.begin());
            }
            omc_rows.push_back((uint32_t)r); omc_row_mult.push_back(p->omc_mult[i]);
        }
    }
    const bool omc_tile = !omc_rows.empty();

    // ------------------------------------------------------------ H2D: descriptors in one packed blob
    Packer pk;
    const size_t o_flt = (filter_h && !has_v) ? pk.add(p->filter_bits, fwords * 8) : 0;
    const size_t o_terms = has_ft ? pk.add(terms.data(), terms.size() * sizeof(TermDesc)) : 0;
    const size_t o_tokens = has_ft ? pk.add(tokens.data(), tokens.size() * sizeof(TokenDesc)) : 0;
    const size_t o_ttok = has_ft ? pk.add(term_token.data(), term_token.size() * 4) : 0;
    const size_t o_pre = pre_descs.empty() ? 0 : pk.add(pre_descs.data(), pre_descs.size() * sizeof(PreDesc));
    const size_t o_pitems = pre_items.empty() ? 0 : pk.add(pre_items.data(), pre_items.size() * sizeof(uint2));
    const size_t o_queries = has_ft ? pk.add(queries.data(), queries.size() * sizeof(QueryDesc)) : 0;
    const size_t o_omcd = n_omc ? pk.add(p->omc_doc_ids, size_t(n_omc) * 8) : 0;
    const size_t o_omcm = n_omc ? pk.add(p->omc_mult, size_t(n_omc) * 4) : 0;
    const size_t o_omcr = omc_tile ? pk.add(omc_rows.data(), omc_rows.size() * 4) : 0;
    const size_t o_omcrm = omc_tile ? pk.add(omc_row_mult.data(), omc_row_mult.size() * 4) : 0;
    size_t o_qf[3] = {0, 0, 0};
    if (per_q && !has_v) add_qf(pk, o_qf);
    const size_t o_tslot = (per_q && !tok_slot.empty()) ? pk.add(tok_slot.data(), tok_slot.size() * 4) : 0;
    // item order of the register-folded scorers (Bm25Params::perm): queries by their number of dense tokens, descending
    std::vector<uint32_t> q_perm;
    uint32_t cls_nq[BM25_CLASSES] = {0, 0, 0, 0, 0};
    if (has_ft && !any_multi && max_tokens <= BM25_FLAT_TOK) {
        std::vector<uint8_t> nd_q(B, 0);
        for (uint32_t q = 0; q < B; q++) {
            uint32_t nd = 0;
            for (uint32_t t = queries[q].token_begin; t < queries[q].token_end; t++)
                if (tokens[t].term_end > tokens[t].term_begin && (terms[tokens[t].term_begin].flags & TD_DENSE) && terms[tokens[t].term_begin].len) nd++;
            nd_q[q] = (uint8_t)std::min<uint32_t>(nd, BM25_CLASSES - 1);
        }
        // (used with OC_BM25_ORDER=1 only.)  TWO classes: every query with a dense token (one tile-major pass over the dense
        // arrays: one class per dense-token count re-streamed those arrays once per class and cost the 10M-document
        // workload 20 %), then the list-only queries, whose items are cheap and touch no dense array.  Inside the first
        // class the queries are sorted by their number of dense tokens, descending.
        auto cls_of = [&](uint32_t q) { return nd_q[q] ? 0u : BM25_CLASSES - 1; };
        for (uint32_t q = 0; q < B; q++) cls_nq[cls_of(q)]++;
        q_perm.resize(B);
        uint32_t at[BM25_CLASSES], acc = 0;
        for (uint32_t g = 0; g < BM25_CLASSES; g++) { at[g] = acc; acc += cls_nq[g]; }
        for (int nd = BM25_CLASSES - 1; nd >= 0; nd--)
            for (uint32_t q = 0; q < B; q++) if (nd_q[q] == nd) q_perm[at[cls_of(q)]++] = q;
    }
    const size_t o_perm = q_perm.empty() ? 0 : pk.add(q_perm.data(), q_perm.size() * 4);
    const bool pin_items = pj && pj->stride;
    const size_t o_pdoc = pin_items ? pk.add(pj->doc.data(), pj->doc.size() * 8) : 0;
    const size_t o_ppos = pin_items ? pk.add(pj->pos.data(), pj->pos.size() * 4) : 0;
    const size_t o_pcnt = pin_items ? pk.add(pj->cnt.data(), pj->cnt.size() * 4) : 0;
    // hybrid: the descriptors, the shared-contribution precompute, the filter bitmap and the (term, tile) plan do
    // not depend on the vector results: they run on the side stream while the main stream sweeps the matrix
    // (OC_SIDE_STREAM=0 disables it: the step gets ~2.5 % longer, the sweep itself ~4 % shorter — A/B switch)
    const char *senv = getenv("OC_SIDE_STREAM");
    // (single-GPU only for now: the sharded path was measured and validated without it)
    const bool side = !(senv && senv[0] == '0') && has_v && has_ft && !need_df && !derived_now;
    if (!has_v) CU(cudaEventRecord(c->ev[EV_START], c->stream));
    if (c->side_dirty) { CU(cudaStreamSynchronize(c->side)); c->side_dirty = false; }   // leftover of a failed call
    if (side) { CU(cudaStreamWaitEvent(c->side, c->ev[EV_H2D], 0)); c->side_dirty = true; }   // the filter bitmap went up with the query vectors
    OCTRY(upload(pk, c->h_in, c->in_blob, side ? c->side : c->stream));
    if (!has_v) CU(cudaEventRecord(c->ev[EV_H2D], c->stream));   // hybrid/vector: this copy rides inside the device window
    c->timing.h2d_bytes = h2d_early + pk.total;
    uint8_t *din = c->in_blob.as<uint8_t>();
    if (filter_h && !has_v) filter_dev = reinterpret_cast<const uint64_t *>(din + o_flt);
    if (per_q && !has_v) bind_qf(din, o_qf);
    if (pin_items) {
        pj->d_doc = reinterpret_cast<const uint64_t *>(din + o_pdoc);
        pj->d_pos = reinterpret_cast<const uint32_t *>(din + o_ppos);
        pj->d_cnt = reinterpret_cast<const uint32_t *>(din + o_pcnt);
    }

    // ------------------------------------------------------------ fulltext stage + fusion (re-runnable)
    // arg-max selection (n_keep <= 32) needs no power-of-two buffer; the bitonic fallback does
    // (also >= BM25_SPARSE_MAX: the sparse finish of the posting-centred kernel pushes at most that many candidates)
    const uint32_t cap = n_keep <= 32 ? std::max<uint32_t>(n_keep + BM25_CHUNK, BM25_SPARSE_MAX) : next_pow2(std::max<uint32_t>(n_keep + BM25_CHUNK, BM25_SPARSE_MAX));
    Bm25Params bp{};
    float *min_hint_dev = nullptr;
    unsigned int *tile_counter = nullptr;
    const size_t o_doc = 0, o_sc = size_t(B) * limit * 8, o_n = o_sc + size_t(B) * limit * 4;
    const size_t o_cnt = (o_n + size_t(B) * 4 + 7) & ~size_t(7), o_min = o_cnt + size_t(B) * 8;
    const size_t o_gflag = o_min + size_t(B) * 4;                       // sharded: OR over the ranks of the per-query overflow flags
    const size_t out_bytes = o_gflag + ((size_t(B) + 3) & ~size_t(3));
    const size_t o_resc = out_bytes + ((size_t(B) + 3) & ~size_t(3));
    OCTRY(c->out_blob.ensure(out_bytes));
    OCTRY(c->h_out.ensure(o_resc + size_t(B) * 4));
    uint8_t *dout = c->out_blob.as<uint8_t>();
    FuseParams fp{};
    size_t fuse_smem = 0;
    bool did_comm = false;
    // The fulltext stage does not depend on the vector stage (the vector hits' fulltext scores are point lookups
    // afterwards): in hybrid mode it runs on the side stream, concurrently with the matrix sweep, and is joined
    // before the lookups and the fusion.  It runs ONCE per call; device_tail (lookups + fusion) is re-runnable.
    const uint32_t *row_ok = nullptr;
    auto bm25_stage = [&]() -> int {
        cudaStream_t ps = side ? c->side : c->stream;
        CU(cudaEventRecord(c->ev[EV_BM0], ps));
        const uint64_t ok_words = uint64_t(n_tiles) * (BM25_TILE / 32);
        if (per_q) {   // one row bitmap per distinct filter (tombstones AND filter), then the tombstone-only slot K
            OCTRY(c->row_ok.ensure(std::max<uint64_t>(ok_words, 1) * qfj.slots.size() * 4));
            if (ok_words) {
                rows_ok_kernel<<<dim3((unsigned)((ok_words + 255) / 256), (unsigned)qfj.slots.size()), 256, 0, ps>>>(
                    S->row_doc, S->n_rows, tombs ? S->alive : nullptr, nullptr, 0, c->row_ok.as<uint32_t>(), ok_words, qfj.d_slots);
                launched(c);
            }
            row_ok = c->row_ok.as<uint32_t>();
        } else if (filter || tombs) {
            OCTRY(c->row_ok.ensure(ok_words * 4));
            rows_ok_kernel<<<(unsigned)((ok_words + 255) / 256), 256, 0, ps>>>(
                S->row_doc, S->n_rows, tombs ? S->alive : nullptr, filter_dev, filter_nbits,
                c->row_ok.as<uint32_t>(), ok_words);
            launched(c);
            row_ok = c->row_ok.as<uint32_t>();
        }
        if (!pre_items.empty()) {
            if (dense_bytes) CU(cudaMemsetAsync(c->dense_buf.p, 0, dense_bytes, ps));
            bm25_precompute_kernel<<<(unsigned)pre_items.size(), 256, 0, ps>>>(
                reinterpret_cast<const PreDesc *>(din + o_pre), reinterpret_cast<const uint2 *>(din + o_pitems), p->bm25_k, row_ok);
            launched(c);
            CU(cudaGetLastError());
        }
        const size_t n_td = terms.size();
        OCTRY(c->seg.ensure((n_td * (size_t(n_tiles) + 1) + 1) * 4));
        if (n_td) {
            const uint64_t work = uint64_t(n_td) * (n_tiles + 1);
            bm25_plan_kernel<<<(unsigned)((work + 255) / 256), 256, 0, ps>>>(
                reinterpret_cast<const TermDesc *>(din + o_terms), (uint32_t)n_td, n_tiles, c->seg.as<uint32_t>());
            launched(c);
        }
        if (need_df) {   // (never on the side stream)
            // corpus_df by counting (token_score.rs:262-275), then idf on the host
            const size_t ntok = tokens.size();
            OCTRY(c->df_dev.ensure(ntok * 4));
            CU(cudaMemsetAsync(c->df_dev.p, 0, ntok * 4, c->stream));
            DfParams dp{};
            dp.terms = reinterpret_cast<const TermDesc *>(din + o_terms);
            dp.tokens = reinterpret_cast<const TokenDesc *>(din + o_tokens);
            dp.n_tokens = (uint32_t)ntok; dp.n_tiles = n_tiles; dp.seg = c->seg.as<uint32_t>();
            dp.row_ok_bits = row_ok; dp.df = c->df_dev.as<unsigned int>();
            if (per_q) { dp.tok_ok_slot = reinterpret_cast<const uint32_t *>(din + o_tslot); dp.ok_words = ok_words; }
            if (n_tiles && ntok) {
                bm25_df_kernel<<<(unsigned)(uint64_t(n_tiles) * ntok), BM25_THREADS, 0, c->stream>>>(dp);
                launched(c);
            }
            if (multi_rank) {   // corpus df = sum of the shards' counts (disjoint documents)
                std::string err;
                if (!c->comm.all_reduce_sum_u32(c->df_dev.p, c->df_dev.p, ntok, c->stream, &err)) return fail(OC_ERR_COMM, "%s", err.c_str());
            }
            std::vector<uint32_t> dfh(ntok);
            CU(cudaMemcpyAsync(dfh.data(), c->df_dev.p, ntok * 4, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaStreamSynchronize(c->stream));
            const float N = (float)S->document_count;
            for (size_t t = 0; t < ntok; t++)
                if (tok_need_df[t]) tokens[t].idf = host_idf(N, std::max<uint32_t>(1u, dfh[t]));
            CU(cudaMemcpyAsync(din + o_tokens, tokens.data(), ntok * sizeof(TokenDesc), cudaMemcpyHostToDevice, c->stream));
        }
        const size_t slots = size_t(B) * std::max<uint32_t>(n_tiles, 1);
        OCTRY(c->tau.ensure(size_t(B) * 16 + 16));   // [tau B x 8][min_hint B x 8][work counter]: one memset
        OCTRY(c->cand_key.ensure(slots * n_keep * 8));
        OCTRY(c->cand_ft.ensure(slots * n_keep * 4));
        OCTRY(c->cand_cnt.ensure(slots * 4));
        OCTRY(c->tile_cnt.ensure(slots * 4));
        OCTRY(c->tile_max.ensure(slots * 4));
        OCTRY(c->tile_min.ensure(slots * 4));
        min_hint_dev = reinterpret_cast<float *>(c->tau.as<uint8_t>() + size_t(B) * 8);
        tile_counter = reinterpret_cast<unsigned int *>(c->tau.as<uint8_t>() + size_t(B) * 16);
        CU(cudaMemsetAsync(c->tau.p, 0, size_t(B) * 16 + 16, ps));
        bp.terms = reinterpret_cast<const TermDesc *>(din + o_terms);
        bp.tokens = reinterpret_cast<const TokenDesc *>(din + o_tokens);
        bp.queries = reinterpret_cast<const QueryDesc *>(din + o_queries);
        bp.term_token = reinterpret_cast<const uint32_t *>(din + o_ttok);
        bp.seg = c->seg.as<uint32_t>();
        bp.n_queries = B; bp.n_tiles = n_tiles; bp.n_rows = S->n_rows;
        bp.k = p->bm25_k; bp.b = p->bm25_b;
        bp.row_ok_bits = row_ok;
        if (per_q) { bp.q_ok_slot = qfj.d_q_slot_ft; bp.ok_words = ok_words; }
        bp.omc_row = omc_tile ? reinterpret_cast<const uint32_t *>(din + o_omcr) : nullptr;
        bp.omc_mult = omc_tile ? reinterpret_cast<const float *>(din + o_omcrm) : nullptr;
        bp.n_omc = (uint32_t)omc_rows.size();
        bp.v_row = nullptr;            // the hybrid lookups are point lookups (bm25_point_kernel)
        bp.v_stride = vlimit;
        bp.v_ft = nullptr; bp.v_present = nullptr;
        bp.min_hint = min_hint_dev;
        bp.n_keep = n_keep; bp.cap = cap;
        bp.tau = c->tau.as<unsigned long long>();
        bp.cand_key = c->cand_key.as<uint64_t>(); bp.cand_ft = c->cand_ft.as<float>();
        bp.cand_cnt = c->cand_cnt.as<uint32_t>(); bp.tile_count = c->tile_cnt.as<uint32_t>();
        bp.tile_max = c->tile_max.as<float>(); bp.tile_min = c->tile_min.as<float>();
        bp.tile_first = 0;
        if (!q_perm.empty()) {
            bp.perm = reinterpret_cast<const uint32_t *>(din + o_perm);
            uint32_t off = 0, q0 = 0;
            for (uint32_t g = 0; g < BM25_CLASSES; g++) {
                bp.cls_off[g] = off; bp.cls_nq[g] = cls_nq[g]; bp.cls_q0[g] = q0;
                off += cls_nq[g] * n_tiles; q0 += cls_nq[g];
            }
        }
        if (fj || gj || sj) {   // facets / groups / sortBy: the tile kernels also emit the bitmap of matched rows (every (query, tile) item writes its 256 words)
            OCTRY(c->mbits.ensure(size_t(B) * std::max<uint32_t>(n_tiles, 1) * (BM25_TILE / 32) * 4));
            bp.matched_bits = c->mbits.as<uint32_t>();
        }
        if (gj && n_tiles) {   // groups: and the raw score of each matched row
            OCTRY(c->row_ft.ensure(size_t(B) * n_tiles * BM25_TILE * 4));
            bp.row_ft = c->row_ft.as<float>();
        }
        if (n_tiles) OCTRY(launch_tile(c, bp, n_tiles * B, any_multi, thr, omc_tile, ps, max_tokens, tile_counter, need_df));
        CU(cudaEventRecord(c->ev[EV_BM1], ps));
        c->timing.bm25_postings = postings_walked;
        if (side) {   // join: the lookups and the fusion need the vector hits (main stream) and the tiles (side stream)
            CU(cudaEventRecord(c->ev_side, c->side));
            CU(cudaStreamWaitEvent(c->stream, c->ev_side, 0));
            c->side_dirty = false;
        }
        return OC_OK;
    };
    if (has_ft) OCTRY(bm25_stage());

    const bool exports = gj || pj || sj;   // K4 exports the normalisation and the vector part of the score map
    // pins, after K4: the score-map value of every promoted document, then (pin_flat) the splice into K4's top list
    auto pin_tail = [&]() -> int {
        if (!pin_items) return OC_OK;
        const uint32_t ps = pj->stride;
        const uint64_t nslot = uint64_t(B) * ps;
        const unsigned warp_grid = (unsigned)((nslot * 32 + 255) / 256);
        OCTRY(c->pin_score.ensure(nslot * 4));
        OCTRY(c->pin_present.ensure(nslot));
        if (has_ft) {   // the promoted documents' string rows and their fulltext scores (the hybrid lookups' kernels)
            OCTRY(c->pin_row.ensure(nslot * 4));
            OCTRY(c->pin_ft.ensure(nslot * 4));
            OCTRY(c->pin_ftp.ensure(nslot));
            map_docs_to_rows_kernel<<<(unsigned)((nslot + 255) / 256), 256, 0, c->stream>>>(
                pj->d_doc, pj->d_cnt, ps, B, S->row_doc, S->n_rows, c->pin_row.as<uint32_t>());
            launched(c);
            PointParams pp{};
            pp.terms = bp.terms; pp.tokens = bp.tokens; pp.queries = bp.queries;
            pp.n_queries = B; pp.v_stride = ps; pp.v_row = c->pin_row.as<uint32_t>(); pp.row_ok_bits = row_ok;
            pp.k = p->bm25_k; pp.threshold = thr ? 1 : 0;
            pp.v_ft = c->pin_ft.as<float>(); pp.v_present = c->pin_ftp.as<uint8_t>();
            bm25_point_kernel<<<warp_grid, 256, 0, c->stream>>>(pp);
            launched(c);
        }
        PinScoreParams sp{};
        sp.n_queries = B; sp.stride = ps; sp.doc = pj->d_doc; sp.cnt = pj->d_cnt;
        sp.has_ft = has_ft; sp.hybrid = has_ft && has_v;
        sp.ft = c->pin_ft.as<float>(); sp.ft_present = c->pin_ftp.as<uint8_t>();
        sp.gmin = fp.out_gmin; sp.den = fp.out_den;
        sp.v_doc = fp.out_vdoc; sp.v_score = fp.out_vscore; sp.v_n = fp.out_vn; sp.v_stride = std::max<uint32_t>(vlimit, 1);
        sp.omc_doc = fp.omc_doc; sp.omc_mult = fp.omc_mult; sp.n_omc = n_omc;
        sp.out_score = c->pin_score.as<float>(); sp.out_present = c->pin_present.as<uint8_t>();
        pin_score_kernel<<<warp_grid, 256, 0, c->stream>>>(sp);
        launched(c);
        if (pin_flat) {
            PinSpliceParams xp{};
            xp.stride = ps; xp.kp2 = std::max<uint32_t>(32, next_pow2(ps));
            xp.doc = pj->d_doc; xp.pos = pj->d_pos; xp.score = c->pin_score.as<float>(); xp.cnt = pj->d_cnt;
            xp.n_top = n_keep; xp.limit = limit; xp.offset = p->offset;
            xp.top_doc = c->pin_top_doc.as<uint64_t>(); xp.top_score = c->pin_top_score.as<float>(); xp.top_n = c->pin_top_n.as<uint32_t>();
            xp.out_doc = reinterpret_cast<uint64_t *>(dout + o_doc); xp.out_score = reinterpret_cast<float *>(dout + o_sc);
            xp.out_n = reinterpret_cast<uint32_t *>(dout + o_n);
            const size_t smem = pin_splice_smem(xp.kp2, n_keep, limit + p->offset);
            pin_splice_kernel<<<B, PIN_THREADS, smem, c->stream>>>(xp);
            launched(c);
        }
        CU(cudaGetLastError());
        return OC_OK;
    };
    // sortBy, after K4 and the pins' scores: the first sort_top keys in field order, scored like promoted documents,
    // then paged with the pins spliced (pin_splice_kernel writes the hits over K4's)
    auto sort_tail = [&]() -> int {
        if (!sort_flat) return OC_OK;
        SortOrder &so = sj->f->ord[sj->order];
        const bool ft_map = has_ft && n_tiles > 0;
        if (ft_map) OCTRY(sort_rows_for(c, so, snap));
        const uint32_t top = sort_top;
        const uint64_t nslot = uint64_t(B) * top;
        const uint32_t vs = std::max<uint32_t>(vlimit, 1);
        OCTRY(c->srt_doc.ensure(nslot * 8));
        OCTRY(c->srt_row.ensure(nslot * 4));
        OCTRY(c->srt_n.ensure(size_t(B) * 4));
        OCTRY(c->srt_score.ensure(nslot * 4));
        OCTRY(c->srt_present.ensure(nslot));
        SortWalkParams wp{};
        wp.n_ranks = so.n; wp.rank_row = ft_map ? so.rank_row : nullptr; wp.doc_rank = so.doc_rank; wp.nbits = sj->f->nbits;
        wp.mbits = ft_map ? c->mbits.as<uint32_t>() : nullptr; wp.row_words = uint64_t(n_tiles) * (BM25_TILE / 32);
        wp.v_doc = fp.out_vdoc; wp.v_n = fp.out_vn; wp.v_stride = vs;
        wp.rank_doc = so.rank_doc; wp.top = top;
        wp.out_doc = c->srt_doc.as<uint64_t>(); wp.out_row = c->srt_row.as<uint32_t>(); wp.out_n = c->srt_n.as<uint32_t>();
        sort_walk_kernel<<<B, SORT_THREADS, size_t(vs) * 4, c->stream>>>(wp);
        launched(c);
        const unsigned warp_grid = (unsigned)((nslot * 32 + 255) / 256);
        if (has_ft) {   // the selected rows' fulltext scores (RANK_NONE rows: vector hits without a row, empty slots)
            OCTRY(c->srt_ft.ensure(nslot * 4));
            OCTRY(c->srt_ftp.ensure(nslot));
            PointParams pp{};
            pp.terms = bp.terms; pp.tokens = bp.tokens; pp.queries = bp.queries;
            pp.n_queries = B; pp.v_stride = top; pp.v_row = c->srt_row.as<uint32_t>(); pp.row_ok_bits = row_ok;
            pp.k = p->bm25_k; pp.threshold = thr ? 1 : 0;
            pp.v_ft = c->srt_ft.as<float>(); pp.v_present = c->srt_ftp.as<uint8_t>();
            bm25_point_kernel<<<warp_grid, 256, 0, c->stream>>>(pp);
            launched(c);
        }
        PinScoreParams sp{};
        sp.n_queries = B; sp.stride = top; sp.doc = c->srt_doc.as<uint64_t>(); sp.cnt = c->srt_n.as<uint32_t>();
        sp.has_ft = has_ft; sp.hybrid = has_ft && has_v;
        sp.ft = c->srt_ft.as<float>(); sp.ft_present = c->srt_ftp.as<uint8_t>();
        sp.gmin = fp.out_gmin; sp.den = fp.out_den;
        sp.v_doc = fp.out_vdoc; sp.v_score = fp.out_vscore; sp.v_n = fp.out_vn; sp.v_stride = vs;
        sp.omc_doc = fp.omc_doc; sp.omc_mult = fp.omc_mult; sp.n_omc = n_omc;
        sp.out_score = c->srt_score.as<float>(); sp.out_present = c->srt_present.as<uint8_t>();
        pin_score_kernel<<<warp_grid, 256, 0, c->stream>>>(sp);
        launched(c);
        PinSpliceParams xp{};
        if (pj->splice) {
            xp.stride = pj->stride; xp.kp2 = std::max<uint32_t>(32, next_pow2(pj->stride));
            xp.doc = pj->d_doc; xp.pos = pj->d_pos; xp.score = c->pin_score.as<float>(); xp.cnt = pj->d_cnt;
        } else {   // no item anywhere: every query takes the page of its list as it is
            OCTRY(c->srt_zero.ensure(size_t(B) * 4));
            CU(cudaMemsetAsync(c->srt_zero.p, 0, size_t(B) * 4, c->stream));
            xp.stride = 0; xp.kp2 = 32;
            xp.doc = c->srt_doc.as<uint64_t>(); xp.pos = c->srt_zero.as<uint32_t>(); xp.score = c->srt_score.as<float>();
            xp.cnt = c->srt_zero.as<uint32_t>();
        }
        xp.n_top = top; xp.limit = limit; xp.offset = p->offset;
        xp.top_doc = c->srt_doc.as<uint64_t>(); xp.top_score = c->srt_score.as<float>(); xp.top_n = c->srt_n.as<uint32_t>();
        xp.out_doc = reinterpret_cast<uint64_t *>(dout + o_doc); xp.out_score = reinterpret_cast<float *>(dout + o_sc);
        xp.out_n = reinterpret_cast<uint32_t *>(dout + o_n);
        pin_splice_kernel<<<B, PIN_THREADS, pin_splice_smem(xp.kp2, top, limit + p->offset), c->stream>>>(xp);
        launched(c);
        CU(cudaGetLastError());
        return OC_OK;
    };

    auto device_tail = [&]() -> int {
    if (has_ft && has_v) {
        // hybrid: vector hits -> string rows -> their fulltext scores (point lookups)
        OCTRY(c->v_srow.ensure(size_t(B) * vlimit * 4));
        OCTRY(c->v_ft.ensure(size_t(B) * vlimit * 4));
        OCTRY(c->v_present.ensure(size_t(B) * vlimit));
        if (vlimit) {
        map_docs_to_rows_kernel<<<(B * vlimit + 255) / 256, 256, 0, c->stream>>>(
            c->v_doc.as<uint64_t>(), c->v_cnt.as<uint32_t>(), vlimit, B, S->row_doc, S->n_rows, c->v_srow.as<uint32_t>());
        launched(c);
        PointParams pp{};
        pp.terms = bp.terms; pp.tokens = bp.tokens; pp.queries = bp.queries;
        pp.n_queries = B; pp.v_stride = vlimit; pp.v_row = c->v_srow.as<uint32_t>(); pp.row_ok_bits = row_ok;
        pp.q_ok_slot = per_q ? qfj.d_q_slot_ft : nullptr; pp.ok_words = uint64_t(n_tiles) * (BM25_TILE / 32);
        pp.k = p->bm25_k; pp.threshold = thr ? 1 : 0;
        pp.v_ft = c->v_ft.as<float>(); pp.v_present = c->v_present.as<uint8_t>();
        bm25_point_kernel<<<(B * vlimit * 32 + 255) / 256, 256, 0, c->stream>>>(pp);
        launched(c);
        CU(cudaGetLastError());
        }
    }

    // ------------------------------------------------------------ fusion + top-n (+ shard exchange)
    fp = FuseParams{};
    fp.mode = p->mode; fp.n_tiles = n_tiles; fp.n_keep = n_keep; fp.limit = limit; fp.offset = p->offset;
    {   // smallest power-of-two key buffer that takes the candidates in one round (sort cost ~ capb log^2 capb)
        const uint64_t total = (has_ft ? uint64_t(n_tiles) * n_keep : 0) + (has_v ? vlimit : 0);
        // up to 16 K keys (128 KB) stay in shared memory and go through one radix select; the streaming bitonic path behind
        // it is for larger candidate sets (the 10M-document fulltext workload has 1221 tiles x 10 candidate slots per query)
        fp.capb = next_pow2((uint32_t)std::min<uint64_t>(16384, std::max<uint64_t>(total, 2 * n_keep)));
        fp.capb = std::max<uint32_t>(fp.capb, std::max<uint32_t>(64, next_pow2(2 * n_keep)));
    }
    if (has_ft) {
        fp.cand_key = bp.cand_key; fp.cand_ft = bp.cand_ft; fp.cand_cnt = bp.cand_cnt; fp.tile_count = bp.tile_count;
        fp.tile_max = bp.tile_max; fp.tile_min = bp.tile_min; fp.str_row_doc_ids = S->row_doc;
    }
    if (has_v) {
        fp.v_doc = c->v_doc.as<uint64_t>(); fp.v_score = c->v_score.as<float>(); fp.v_count = c->v_cnt.as<uint32_t>();
        fp.v_row = has_ft ? c->v_srow.as<uint32_t>() : nullptr;
        fp.v_ft = c->v_ft.as<float>(); fp.v_present = c->v_present.as<uint8_t>();
    }
    fp.v_stride = vlimit;
    fp.omc_doc = n_omc ? reinterpret_cast<const uint64_t *>(din + o_omcd) : nullptr;
    fp.omc_mult = n_omc ? reinterpret_cast<const float *>(din + o_omcm) : nullptr;
    fp.n_omc = n_omc;
    fp.out_doc = reinterpret_cast<uint64_t *>(dout + o_doc); fp.out_score = reinterpret_cast<float *>(dout + o_sc);
    fp.out_n = reinterpret_cast<uint32_t *>(dout + o_n); fp.out_count = reinterpret_cast<unsigned long long *>(dout + o_cnt);
    fp.out_min = reinterpret_cast<float *>(dout + o_min);
    if (pin_flat) {   // K4 keeps its whole top n_keep for the splice, which writes the hits
        fp.limit = n_keep; fp.offset = 0;
        OCTRY(c->pin_top_doc.ensure(size_t(B) * n_keep * 8));
        OCTRY(c->pin_top_score.ensure(size_t(B) * n_keep * 4));
        OCTRY(c->pin_top_n.ensure(size_t(B) * 4));
        fp.out_doc = c->pin_top_doc.as<uint64_t>(); fp.out_score = c->pin_top_score.as<float>(); fp.out_n = c->pin_top_n.as<uint32_t>();
    }
    if (exports) {   // groups / pins: K4 also exports the normalisation and the vector part of the score map
        const uint32_t vs = std::max<uint32_t>(vlimit, 1);
        OCTRY(c->grp_vdoc.ensure(size_t(B) * vs * 8));
        OCTRY(c->grp_vscore.ensure(size_t(B) * vs * 4));
        OCTRY(c->grp_vn.ensure(size_t(B) * 4));
        OCTRY(c->grp_gmin.ensure(size_t(B) * 4));
        OCTRY(c->grp_den.ensure(size_t(B) * 4));
        fp.out_vdoc = c->grp_vdoc.as<uint64_t>(); fp.out_vscore = c->grp_vscore.as<float>(); fp.out_vn = c->grp_vn.as<uint32_t>();
        fp.out_gmin = c->grp_gmin.as<float>(); fp.out_den = c->grp_den.as<float>();
    }
    fuse_smem = size_t(fp.capb) * 8 + size_t(std::max<uint32_t>(32, next_pow2(n_keep))) * 8 + size_t(vlimit) * 8 + 64;
    if (smem_cfg_needed(c->device, exports ? (const void *)fuse_topk_kernel<true> : (const void *)fuse_topk_kernel<false>, fuse_smem))
        CU(cudaFuncSetAttribute(exports ? (const void *)fuse_topk_kernel<true> : (const void *)fuse_topk_kernel<false>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fuse_smem));

    if (p->sharded && c->comm.world > 1) {
        CU(cudaEventRecord(c->ev[EV_FUSE0], c->stream));
        OCTRY(run_sharded_merge(c, p, fp, has_ft ? (uint32_t)S->n_rows : 0, has_v ? (uint32_t)emb->n_rows : 0, B,
                                (has_v && c->gemm_pending) ? c->g_flag.as<uint8_t>() : nullptr, dout + o_gflag));
        CU(cudaEventRecord(c->ev[EV_FUSE1], c->stream));
        did_comm = true;
    } else {
        CU(cudaEventRecord(c->ev[EV_FUSE0], c->stream));
        if (exports) fuse_topk_kernel<true><<<B, 256, fuse_smem, c->stream>>>(fp);
        else fuse_topk_kernel<<<B, 256, fuse_smem, c->stream>>>(fp);
        launched(c);
        CU(cudaGetLastError());
        OCTRY(pin_tail());
        OCTRY(sort_tail());
        CU(cudaEventRecord(c->ev[EV_FUSE1], c->stream));
    }
    return OC_OK;
    };   // device_tail
    OCTRY(device_tail());
    CU(cudaEventRecord(c->ev[EV_DEV], c->stream));
    uint8_t *h = c->h_out.as<uint8_t>();
    CU(cudaMemcpyAsync(h, dout, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    if (c->gemm_pending) {
        CU(cudaMemcpyAsync(h + out_bytes, c->g_flag.p, B, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(h + o_resc, c->g_resc.p, size_t(B) * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaEventRecord(c->ev[EV_D2H], c->stream));
    CU(cudaStreamSynchronize(c->stream));
    {   // tensor-core scan: re-run the (rare) queries whose candidate buffers overflowed
        // sharded: every rank must enter the collective the same number of times, so the decision to re-run is
        // taken on the flags all ranks exchanged inside the shard records (no host sync before the collective),
        // by every rank — also one whose own shard was served by the exact sweep
        bool rerun = false;
        if (did_comm && has_v) for (uint32_t q = 0; q < B; q++) rerun = rerun || h[o_gflag + q] != 0;
        uint32_t redone = 0;
        if (c->gemm_pending || rerun) CU(cudaEventRecord(c->ev[EV_RR0], c->stream));
        if (c->gemm_pending) {
            uint64_t resc = 0;
            for (uint32_t q = 0; q < B; q++) resc += reinterpret_cast<const uint32_t *>(h + o_resc)[q];
            c->timing.scan_rescored = (uint32_t)(resc / B);
            OCTRY(fix_unproven(c, emb, h + out_bytes, B, vlimit, p->similarity, &redone));
        }
        if (redone || rerun) {
            c->gemm_pending = false;
            OCTRY(device_tail());
            CU(cudaMemcpyAsync(h, dout, out_bytes, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaEventRecord(c->ev[EV_RR1], c->stream));
            c->rerun_timed = true;
            CU(cudaStreamSynchronize(c->stream));
        }
    }

    // rank-proxy validation: with OMC multipliers the tile ranking assumed min == min_hint (0);
    // a negative global min changes the order of (ft - min) * omc -> rerun with the real min.
    if (!did_comm && p->mode == OC_MODE_HYBRID && omc_tile && n_tiles) {
        const float *mins = reinterpret_cast<const float *>(h + o_min);
        bool redo = false;
        for (uint32_t q = 0; q < B; q++) redo = redo || mins[q] < 0.f;
        if (redo) {
            CU(cudaMemcpyAsync(min_hint_dev, mins, size_t(B) * 4, cudaMemcpyHostToDevice, c->stream));
            CU(cudaMemsetAsync(c->tau.p, 0, size_t(B) * 8, c->stream));
            CU(cudaMemsetAsync(tile_counter, 0, 8, c->stream));
            OCTRY(launch_tile(c, bp, n_tiles * B, any_multi, thr, omc_tile, c->stream, max_tokens, tile_counter, need_df));
            if (exports) fuse_topk_kernel<true><<<B, 256, fuse_smem, c->stream>>>(fp);
            else fuse_topk_kernel<<<B, 256, fuse_smem, c->stream>>>(fp);
            launched(c);
            OCTRY(pin_tail());
            OCTRY(sort_tail());
            CU(cudaMemcpyAsync(c->h_out.p, dout, out_bytes, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaStreamSynchronize(c->stream));
        }
    }
    if (fj) OCTRY(run_facets(c, *fj, B, has_ft, has_v, S, n_tiles, vlimit));
    if (gj) {
        CU(cudaEventRecord(c->ev[EV_GRP0], c->stream));
        OCTRY(run_groups(c, *gj, B, p->mode, S, n_tiles, vlimit, fp.omc_doc, fp.omc_mult, n_omc, pj, sj));
        CU(cudaEventRecord(c->ev[EV_GRP1], c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    std::vector<float> pin_sc;
    std::vector<uint8_t> pin_pr;
    if (pin_items && (out_pin_scores || out_pin_present)) {
        pin_sc.resize(pj->doc.size());
        pin_pr.resize(pj->doc.size());
        CU(cudaMemcpyAsync(pin_sc.data(), c->pin_score.p, pin_sc.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(pin_pr.data(), c->pin_present.p, pin_pr.size(), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    c->timing.d2h_bytes = out_bytes;
    if (write_hits) {
        memcpy(out_doc_ids, h + o_doc, size_t(B) * limit * 8);
        memcpy(out_scores, h + o_sc, size_t(B) * limit * 4);
        memcpy(out_n, h + o_n, size_t(B) * 4);
    }
    memcpy(out_count, h + o_cnt, size_t(B) * 8);
    if (sort_flat && sj->out_values)
        for (uint32_t q = 0; q < B; q++)
            for (uint32_t i = 0; i < limit; i++) {
                const size_t o = size_t(q) * limit + i;
                sj->out_values[o] = i < out_n[q] ? sort_value_of(*sj, pj, q, out_doc_ids[o]) : 0.0;
            }
    if (sj && gj && sj->out_group_values) {   // run_groups' copies are complete (synchronised above)
        const uint32_t G = sj->n_groups;
        for (uint32_t q = 0; q < B; q++)
            for (uint32_t g = 0; g < G; g++)
                for (uint32_t i = 0; i < gj->stride; i++) {
                    const size_t o = (size_t(q) * G + g) * gj->stride + i;
                    sj->out_group_values[o] = i < gj->out_n[size_t(q) * G + g] ? sort_value_of(*sj, pj, q, gj->out_doc[o]) : 0.0;
                }
    }
    if (!pin_sc.empty())
        for (uint32_t q = 0; q < B; q++)
            for (uint32_t j = 0; j < pj->cnt[q]; j++) {
                const size_t i = size_t(pins->q_pin_offsets[q]) + j, s = size_t(q) * pj->stride + j;
                if (out_pin_scores) out_pin_scores[i] = pin_sc[s];
                if (out_pin_present) out_pin_present[i] = pin_pr[s];
            }
    OCTRY(finish_timing(c, has_v && vlimit && emb->n_rows > 0, has_ft, true, did_comm));
    if (gj) {   // the group stage is device work of this call too
        float ms = 0.f;
        CU(cudaEventElapsedTime(&ms, c->ev[EV_GRP0], c->ev[EV_GRP1]));
        c->timing.device_ms += ms;
    }
    return OC_OK;
}

extern "C" int oc_search(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, uint64_t *out_doc_ids,
                         float *out_scores, uint32_t *out_n, uint64_t *out_count) {
    return search_impl(c, emb, str, p, out_doc_ids, out_scores, out_n, out_count, nullptr);
}

// ------------------------------------------------------------------------------------ facets
// FacetContext::execute (read/index/facet.rs:147-209): for every requested variant of a filter field — bool
// true/false (bool_field.rs:182-208), a number range [from, to] inclusive (number_field.rs:368-387), a
// string_filter key (string_filter_field.rs:175-193) — count the documents of the variant that are keys of the
// score map.  On the device the score map's key set is a bitmap over DocumentId: the matched rows of the BM25
// tile kernels (+ the vector hits), and a variant is a slice of a device-resident document array.
struct FacetField {
    bool number = false;
    uint64_t n_docs = 0;
    uint64_t *docs = nullptr;              // device: variant-major (CSR) or value-sorted (number field)
    std::vector<uint64_t> offsets;         // host: n_variants + 1
    std::vector<double> values;            // host: ascending (number field)
};
struct oc_facets {
    oc_ctx *ctx;
    uint64_t nbits;                        // DocumentId space [0, nbits)
    std::vector<FacetField> fields;
};
struct FacetReqDev { const uint64_t *docs; uint64_t n; };

extern "C" int oc_facets_create(oc_ctx *c, uint64_t nbits, oc_facets **out) {
    if (!c || !out || nbits == 0) return fail(OC_ERR_INVALID, "bad arguments");
    oc_facets *f = new oc_facets();
    f->ctx = c; f->nbits = nbits;
    *out = f;
    return OC_OK;
}
extern "C" void oc_facets_destroy(oc_facets *f) {
    if (!f) return;
    {
        std::lock_guard<std::mutex> g(f->ctx->mu);
        cudaSetDevice(f->ctx->device);
        cudaStreamSynchronize(f->ctx->stream);
        for (auto &fl : f->fields) cudaFree(fl.docs);
    }
    delete f;
}
static int facets_add(oc_facets *f, FacetField &&fl, const uint64_t *doc_ids, uint32_t *out_field) {
    oc_ctx *c = f->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    if (fl.n_docs) {
        CU(cudaMalloc(&fl.docs, fl.n_docs * 8));
        CU(cudaMemcpy(fl.docs, doc_ids, fl.n_docs * 8, cudaMemcpyHostToDevice));
    }
    f->fields.push_back(std::move(fl));
    if (out_field) *out_field = (uint32_t)f->fields.size() - 1;
    return OC_OK;
}
extern "C" int oc_facets_add_field(oc_facets *f, uint32_t n_variants, const uint64_t *variant_offsets, const uint64_t *doc_ids,
                                   uint32_t *out_field) {
    if (!f || !variant_offsets || n_variants == 0) return fail(OC_ERR_INVALID, "bad arguments");
    for (uint32_t v = 0; v < n_variants; v++)
        if (variant_offsets[v + 1] < variant_offsets[v]) return fail(OC_ERR_INVALID, "variant_offsets not monotone");
    if (variant_offsets[n_variants] && !doc_ids) return fail(OC_ERR_INVALID, "doc_ids is NULL");
    FacetField fl;
    fl.n_docs = variant_offsets[n_variants];
    fl.offsets.assign(variant_offsets, variant_offsets + n_variants + 1);
    return facets_add(f, std::move(fl), doc_ids, out_field);
}
extern "C" int oc_facets_add_number_field(oc_facets *f, uint64_t n, const double *values_sorted, const uint64_t *doc_ids,
                                          uint32_t *out_field) {
    if (!f || (n && (!values_sorted || !doc_ids))) return fail(OC_ERR_INVALID, "bad arguments");
    for (uint64_t i = 1; i < n; i++)
        if (!(values_sorted[i] >= values_sorted[i - 1])) return fail(OC_ERR_INVALID, "values must be ascending (no NaN)");
    FacetField fl;
    fl.number = true; fl.n_docs = n;
    fl.values.assign(values_sorted, values_sorted + n);
    return facets_add(f, std::move(fl), doc_ids, out_field);
}

// where-filter leaves over a filter field (read/index/filter.rs:49-124).  A leaf is one slice [lo, hi) of the field's
// device document array, found on the host by `slice` (called under the ctx lock), scattered into a zeroed bitmap by
// filter_scatter_ids_kernel: nothing is copied from the host and an empty slice launches nothing.
template <typename F>
static int facet_leaf(const oc_facets *f, uint32_t field, bool number, oc_filter **out, F &&slice) {
    oc_ctx *c = f->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    if (field >= f->fields.size()) return fail(OC_ERR_INVALID, "field %u: the store has %zu fields", field, f->fields.size());
    const FacetField &fl = f->fields[field];
    if (fl.number != number)
        return fail(OC_ERR_INVALID, "field %u is a %s field", field, fl.number ? "number" : "bool / string_filter");
    uint64_t lo = 0, hi = 0;
    OCTRY(slice(fl, lo, hi));
    CU(cudaSetDevice(c->device));
    oc_filter *r = nullptr;
    OCTRY(filter_alloc(c, f->nbits, &r));
    cudaError_t e = cudaMemsetAsync(r->bits, 0, std::max<uint64_t>(r->words, 1) * 8, c->stream);
    if (e == cudaSuccess && hi > lo) {
        filter_scatter_ids_kernel<<<(unsigned)((hi - lo + 255) / 256), 256, 0, c->stream>>>(
            fl.docs + lo, hi - lo, f->nbits, reinterpret_cast<unsigned long long *>(r->bits));
        launched(c);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
        cudaFree(r->bits);
        delete r;
        return fail(OC_ERR_CUDA, "facet filter: %s", cudaGetErrorString(e));
    }
    *out = r;
    return OC_OK;
}

extern "C" int oc_filter_facet_variant(const oc_facets *f, uint32_t field, uint32_t variant, oc_filter **out) {
    if (!f || !out) return fail(OC_ERR_INVALID, "NULL argument");
    return facet_leaf(f, field, false, out, [&](const FacetField &fl, uint64_t &lo, uint64_t &hi) {
        if (variant + uint64_t(1) >= fl.offsets.size())
            return fail(OC_ERR_INVALID, "variant %u: field %u has %zu variants", variant, field, fl.offsets.size() - 1);
        lo = fl.offsets[variant];
        hi = fl.offsets[variant + 1];
        return int(OC_OK);
    });
}

extern "C" int oc_filter_facet_range(const oc_facets *f, uint32_t field, double lo, double hi, uint32_t flags, oc_filter **out) {
    if (!f || !out) return fail(OC_ERR_INVALID, "NULL argument");
    if (std::isnan(lo) || std::isnan(hi)) return fail(OC_ERR_INVALID, "NaN range bound");
    if (flags & ~(OC_RANGE_LO_OPEN | OC_RANGE_HI_OPEN)) return fail(OC_ERR_INVALID, "unknown range flags 0x%x", flags);
    return facet_leaf(f, field, true, out, [&](const FacetField &fl, uint64_t &a, uint64_t &b) {
        const auto &v = fl.values;   // ascending, no NaN
        a = (flags & OC_RANGE_LO_OPEN) ? std::upper_bound(v.begin(), v.end(), lo) - v.begin()
                                       : std::lower_bound(v.begin(), v.end(), lo) - v.begin();
        b = (flags & OC_RANGE_HI_OPEN) ? std::lower_bound(v.begin(), v.end(), hi) - v.begin()
                                       : std::upper_bound(v.begin(), v.end(), hi) - v.begin();
        b = std::max(a, b);   // lo > hi: empty
        return int(OC_OK);
    });
}

// row bitmap -> DocumentId bitmap when rows are not document ids
__global__ void facet_rows_to_docs_kernel(const uint32_t *row_bits, uint64_t row_stride_words, const uint64_t *row_doc, uint64_t n_rows,
                                          uint32_t *doc_bits, uint64_t doc_stride_words, uint64_t nbits) {
    const uint32_t q = blockIdx.y;
    const uint64_t w = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w * 32 >= n_rows) return;
    uint32_t v = row_bits[size_t(q) * row_stride_words + w];
    while (v) {
        const uint32_t b = __ffs(v) - 1;
        v &= v - 1;
        const uint64_t r = w * 32 + b;
        if (r < n_rows) { const uint64_t d = row_doc[r]; if (d < nbits) atomicOr(&doc_bits[size_t(q) * doc_stride_words + (d >> 5)], 1u << (d & 31)); }
    }
}
// the vector hits are keys of the score map too (token_score.rs:340-351, 416-419)
__global__ void facet_mark_hits_kernel(const uint64_t *v_doc, const uint32_t *v_cnt, uint32_t v_stride, uint32_t B, uint32_t *doc_bits,
                                       uint64_t doc_stride_words, uint64_t nbits_cap) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * v_stride) return;
    const uint32_t q = i / v_stride, j = i % v_stride;
    if (j >= v_cnt[q]) return;
    const uint64_t d = v_doc[i];
    if (d < nbits_cap) atomicOr(&doc_bits[size_t(q) * doc_stride_words + (d >> 5)], 1u << (d & 31));
}
// one block = 1024 documents of one variant, counted against every query's bitmap (the slice is read once)
__global__ void __launch_bounds__(256) facet_count_kernel(const FacetReqDev *reqs, uint32_t n_reqs, const uint32_t *bits,
                                                          uint64_t stride_words, uint64_t nbits_cap, uint32_t B,
                                                          unsigned long long *out) {
    const uint32_t r = blockIdx.y;
    const FacetReqDev rq = reqs[r];
    const uint64_t base = uint64_t(blockIdx.x) * 1024;
    if (base >= rq.n) return;
    uint64_t d[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const uint64_t i = base + threadIdx.x + u * 256;
        const uint64_t v = i < rq.n ? rq.docs[i] : ~0ull;
        d[u] = v < nbits_cap ? v : ~0ull;
    }
    __shared__ uint32_t s_c[8];
    for (uint32_t q = 0; q < B; q++) {
        const uint32_t *bq = bits + size_t(q) * stride_words;
        uint32_t c = 0;
#pragma unroll
        for (int u = 0; u < 4; u++)
            if (d[u] != ~0ull) c += (bq[d[u] >> 5] >> (d[u] & 31)) & 1u;
        c = __reduce_add_sync(0xffffffffu, c);
        if ((threadIdx.x & 31) == 0) s_c[threadIdx.x >> 5] = c;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t t = 0;
            for (int w = 0; w < 8; w++) t += s_c[w];
            if (t) atomicAdd(out + size_t(q) * n_reqs + r, (unsigned long long)t);
        }
        __syncthreads();
    }
}

static int run_facets(oc_ctx *c, const FacetJob &fj, uint32_t B, bool has_ft, bool has_v, const StrSnap *S, uint32_t n_tiles,
                      uint32_t vlimit) {
    oc_facets *fc = fj.fc;
    // resolve the requests to device slices
    std::vector<FacetReqDev> rd(fj.n_reqs);
    uint64_t max_n = 0;
    for (uint32_t i = 0; i < fj.n_reqs; i++) {
        const oc_facet_req &rq = fj.reqs[i];
        if (rq.field >= fc->fields.size()) return fail(OC_ERR_INVALID, "facet request %u: unknown field %u", i, rq.field);
        const FacetField &fl = fc->fields[rq.field];
        uint64_t lo, hi;
        if (fl.number) {   // NumberFilter::Between = inclusive on both ends (number_field.rs:376, 604-631)
            lo = uint64_t(std::lower_bound(fl.values.begin(), fl.values.end(), rq.from) - fl.values.begin());
            hi = uint64_t(std::upper_bound(fl.values.begin(), fl.values.end(), rq.to) - fl.values.begin());
            if (hi < lo) hi = lo;
        } else {
            if (rq.variant + 1 >= fl.offsets.size()) return fail(OC_ERR_INVALID, "facet request %u: unknown variant %u", i, rq.variant);
            lo = fl.offsets[rq.variant]; hi = fl.offsets[rq.variant + 1];
        }
        rd[i].docs = fl.docs + lo; rd[i].n = hi - lo;
        max_n = std::max(max_n, rd[i].n);
    }
    // the key set of each query's score map as a DocumentId bitmap
    const uint64_t row_words = uint64_t(n_tiles) * (BM25_TILE / 32);
    const uint64_t doc_words = (fc->nbits + 31) / 32;
    const bool identity = has_ft && S->row_doc == nullptr;
    const uint32_t *bits; uint64_t stride, cap_bits;
    if (identity && !has_v) {   // the row bitmap is the document bitmap
        bits = c->mbits.as<uint32_t>(); stride = row_words; cap_bits = S->n_rows;
    } else {
        OCTRY(c->dbits.ensure(size_t(B) * doc_words * 4));
        CU(cudaMemsetAsync(c->dbits.p, 0, size_t(B) * doc_words * 4, c->stream));
        if (has_ft && n_tiles) {
            if (identity) {
                const uint64_t wcopy = std::min(row_words, doc_words);
                CU(cudaMemcpy2DAsync(c->dbits.p, doc_words * 4, c->mbits.p, row_words * 4, wcopy * 4, B, cudaMemcpyDeviceToDevice, c->stream));
            } else {
                dim3 grid((unsigned)((row_words + 255) / 256), B);
                facet_rows_to_docs_kernel<<<grid, 256, 0, c->stream>>>(c->mbits.as<uint32_t>(), row_words, S->row_doc, S->n_rows,
                                                                      c->dbits.as<uint32_t>(), doc_words, fc->nbits);
                launched(c);
            }
        }
        if (has_v) {
            facet_mark_hits_kernel<<<(B * vlimit + 255) / 256, 256, 0, c->stream>>>(c->v_doc.as<uint64_t>(), c->v_cnt.as<uint32_t>(), vlimit, B,
                                                                                  c->dbits.as<uint32_t>(), doc_words, fc->nbits);
            launched(c);
        }
        bits = c->dbits.as<uint32_t>(); stride = doc_words; cap_bits = fc->nbits;
    }
    OCTRY(c->facet_req.ensure(size_t(fj.n_reqs) * sizeof(FacetReqDev)));
    OCTRY(c->facet_out.ensure(size_t(B) * fj.n_reqs * 8));
    CU(cudaMemcpyAsync(c->facet_req.p, rd.data(), size_t(fj.n_reqs) * sizeof(FacetReqDev), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemsetAsync(c->facet_out.p, 0, size_t(B) * fj.n_reqs * 8, c->stream));
    if (max_n) {
        dim3 grid((unsigned)((max_n + 1023) / 1024), fj.n_reqs);
        facet_count_kernel<<<grid, 256, 0, c->stream>>>(c->facet_req.as<FacetReqDev>(), fj.n_reqs, bits, stride, cap_bits, B,
                                                       c->facet_out.as<unsigned long long>());
        launched(c);
        CU(cudaGetLastError());
    }
    CU(cudaMemcpyAsync(fj.out_counts, c->facet_out.p, size_t(B) * fj.n_reqs * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));   // rd lives on this stack
    return OC_OK;
}

extern "C" int oc_search_facets(oc_ctx *c, oc_emb *emb, oc_str *str, oc_facets *facets, const oc_search_params *p,
                                const oc_facet_req *reqs, uint32_t n_reqs, uint64_t *out_counts) {
    if (!c || !p || !facets || !out_counts || (n_reqs && !reqs)) return fail(OC_ERR_INVALID, "NULL argument");
    if (facets->ctx != c) return fail(OC_ERR_INVALID, "facets belong to another ctx");
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "facets over a sharded search: count per shard and add the counts");
    if (n_reqs == 0) return OC_OK;
    // the reference computes facets on the score map re-scored WITHOUT the where-filter (search.rs:361-396: only the
    // uncommitted deletes stay excluded), so that the counts do not collapse onto the selected category
    oc_search_params q = *p;
    q.filter_bits = nullptr; q.filter_nbits = 0; q.filter = nullptr; q.q_filters = nullptr;
    const uint32_t B = p->n_queries;
    std::vector<uint64_t> docs(size_t(B) * p->limit), cnt(B);
    std::vector<float> scores(size_t(B) * p->limit);
    std::vector<uint32_t> n(B);
    FacetJob fj{facets, reqs, n_reqs, out_counts};
    return search_impl(c, emb, str, &q, docs.data(), scores.data(), n.data(), cnt.data(), &fj);
}

// ------------------------------------------------------------------------------------ groups
// GroupContext::execute (read/index/group.rs) + sort_groups (read/sort.rs:129-230): the group CSR is built once on
// the host; per call its documents are mapped to string rows and group_topk_kernel (group.cuh) runs one CTA per
// (group, query) over the score map the search left on the device.
struct oc_group_by {
    oc_ctx *ctx;
    uint32_t n_groups = 0;
    uint64_t n_docs = 0;           // entries of the CSR (a document counts once per group it belongs to)
    uint64_t *off = nullptr;       // device [n_groups + 1]
    uint64_t *docs = nullptr;      // device [n_docs]
    uint32_t *rows = nullptr;      // device [n_docs + 1]: string row of each entry, filled per call; rows[n_docs] = ~0
};
static void group_by_free(oc_group_by *g) {
    cudaFree(g->off); cudaFree(g->docs); cudaFree(g->rows);
    delete g;
}
extern "C" void oc_group_by_destroy(oc_group_by *g) {
    if (!g) return;
    {
        std::lock_guard<std::mutex> lk(g->ctx->mu);
        cudaSetDevice(g->ctx->device);
        cudaStreamSynchronize(g->ctx->stream);
    }
    group_by_free(g);
}
extern "C" int oc_group_by_create(oc_facets *f, const uint32_t *fields, uint32_t n_fields, oc_group_by **out, uint64_t *out_n_groups) {
    if (!f || !fields || n_fields == 0 || !out) return fail(OC_ERR_INVALID, "bad arguments");
    oc_ctx *c = f->ctx;
    constexpr uint64_t MAX_GROUPS = 1ull << 20, MAX_GROUP_DOCS = 0xfffffffeull;
    // per field: its (document, variant index) pairs, sorted and unique
    std::vector<std::vector<std::pair<uint64_t, uint32_t>>> dv(n_fields);
    std::vector<uint64_t> nv(n_fields);
    uint64_t G = 1;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        CU(cudaSetDevice(c->device));
        for (uint32_t i = 0; i < n_fields; i++) {
            if (fields[i] >= f->fields.size()) return fail(OC_ERR_INVALID, "group field %u: unknown field id %u", i, fields[i]);
            const FacetField &fl = f->fields[fields[i]];
            std::vector<uint64_t> docs(fl.n_docs);
            if (fl.n_docs) CU(cudaMemcpy(docs.data(), fl.docs, fl.n_docs * 8, cudaMemcpyDeviceToHost));
            auto &pairs = dv[i];
            pairs.reserve(fl.n_docs);
            if (fl.number) {   // variant = rank of the distinct value (values are ascending; == merges -0.0 and 0.0)
                uint32_t v = 0;
                for (uint64_t k = 0; k < fl.n_docs; k++) {
                    if (k && !(fl.values[k] == fl.values[k - 1])) v++;
                    if (docs[k] < f->nbits) pairs.emplace_back(docs[k], v);
                }
                nv[i] = fl.n_docs ? uint64_t(v) + 1 : 0;
            } else {
                nv[i] = fl.offsets.size() - 1;
                for (uint32_t v = 0; v + 1 < fl.offsets.size(); v++)
                    for (uint64_t k = fl.offsets[v]; k < fl.offsets[v + 1]; k++)
                        if (docs[k] < f->nbits) pairs.emplace_back(docs[k], v);
            }
            std::sort(pairs.begin(), pairs.end());
            pairs.erase(std::unique(pairs.begin(), pairs.end()), pairs.end());
            G *= nv[i];
            if (G > MAX_GROUPS) return fail(OC_ERR_UNSUPPORTED, "more than %llu groups", (unsigned long long)MAX_GROUPS);
        }
    }
    // memberships (group, doc), walked in ascending document order so every group's list comes out ascending
    std::vector<std::pair<uint32_t, uint64_t>> memb;
    std::vector<uint64_t> cnt(G + 1, 0);
    if (G) {
        std::vector<std::pair<size_t, size_t>> rng(n_fields);   // this document's pairs in each field
        std::vector<size_t> at(n_fields);
        const auto &f0 = dv[0];
        for (size_t a = 0; a < f0.size();) {
            const uint64_t d = f0[a].first;
            size_t b = a;
            while (b < f0.size() && f0[b].first == d) b++;
            rng[0] = {a, b};
            bool all = true;
            for (uint32_t i = 1; i < n_fields && all; i++) {
                auto lo = std::lower_bound(dv[i].begin(), dv[i].end(), std::make_pair(d, 0u));
                auto hi = std::upper_bound(lo, dv[i].end(), std::make_pair(d, 0xffffffffu));
                rng[i] = {size_t(lo - dv[i].begin()), size_t(hi - dv[i].begin())};
                all = hi != lo;
            }
            if (all) {   // every combination of this document's variants (odometer, last field fastest)
                for (uint32_t i = 0; i < n_fields; i++) at[i] = rng[i].first;
                for (;;) {
                    uint64_t gid = 0;
                    for (uint32_t i = 0; i < n_fields; i++) gid = gid * nv[i] + dv[i][at[i]].second;
                    memb.emplace_back((uint32_t)gid, d);
                    if (++cnt[gid + 1] > MAX_GROUP_DOCS)
                        return fail(OC_ERR_UNSUPPORTED, "group %llu holds more than %llu documents", (unsigned long long)gid,
                                    (unsigned long long)MAX_GROUP_DOCS);
                    int i = int(n_fields) - 1;
                    while (i >= 0 && ++at[i] == rng[i].second) { at[i] = rng[i].first; i--; }
                    if (i < 0) break;
                }
            }
            a = b;
        }
    }
    for (uint64_t g = 0; g < G; g++) cnt[g + 1] += cnt[g];
    std::vector<uint64_t> csr(memb.size());
    {
        std::vector<uint64_t> pos(cnt.begin(), cnt.end() - 1);
        for (const auto &e : memb) csr[pos[e.first]++] = e.second;   // stable: documents stay ascending
    }
    oc_group_by *g = new oc_group_by();
    g->ctx = c; g->n_groups = (uint32_t)G; g->n_docs = csr.size();
    auto fail_free = [&](int code) { group_by_free(g); return code; };
    std::lock_guard<std::mutex> lk(c->mu);
    if (cudaSetDevice(c->device) != cudaSuccess) return fail_free(fail(OC_ERR_CUDA, "cudaSetDevice failed"));
    const uint32_t none = 0xffffffffu;
    cudaError_t e = cudaMalloc(&g->off, (G + 1) * 8);
    if (e == cudaSuccess) e = cudaMalloc(&g->docs, std::max<size_t>(csr.size(), 1) * 8);
    if (e == cudaSuccess) e = cudaMalloc(&g->rows, (csr.size() + 1) * 4);
    if (e == cudaSuccess) e = cudaMemcpy(g->off, cnt.data(), (G + 1) * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && !csr.empty()) e = cudaMemcpy(g->docs, csr.data(), csr.size() * 8, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(g->rows + csr.size(), &none, 4, cudaMemcpyHostToDevice);
    if (e != cudaSuccess)
        return fail_free(fail(e == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "group CSR upload: %s", cudaGetErrorString(e)));
    *out = g;
    if (out_n_groups) *out_n_groups = G;
    return OC_OK;
}

static int run_groups(oc_ctx *c, const GroupJob &gj, uint32_t B, int mode, const StrSnap *S, uint32_t n_tiles, uint32_t vlimit,
                      const uint64_t *omc_doc, const float *omc_mult, uint32_t n_omc, const PinJob *pj, const SortJob *sj) {
    oc_group_by *g = gj.g;
    // sort_groups with pins takes every group's top 2 * max_results (sort.rs:137-142)
    const bool pin_grp = pj && pj->splice;
    const uint32_t G = g->n_groups, m = gj.max_results * (pin_grp ? 2 : 1);
    if (G == 0) return OC_OK;
    const bool has_ft = mode != OC_MODE_VECTOR && n_tiles > 0;
    if (has_ft && g->n_docs) {   // the CSR's documents -> string rows (identity, or a binary search over the ascending row_doc)
        constexpr uint64_t CH = 1ull << 30;
        for (uint64_t a = 0; a < g->n_docs; a += CH) {
            const uint32_t len = (uint32_t)std::min<uint64_t>(CH, g->n_docs - a);
            // counts = rows[n_docs] (~0): every entry of the chunk is mapped
            map_docs_to_rows_kernel<<<(len + 255) / 256, 256, 0, c->stream>>>(g->docs + a, g->rows + g->n_docs, len, 1, S->row_doc,
                                                                              S->n_rows, g->rows + a);
            launched(c);
            CU(cudaGetLastError());
        }
    }
    const size_t n_out = size_t(B) * G * m;
    OCTRY(c->grp_doc.ensure(std::max<size_t>(n_out, 1) * 8));
    OCTRY(c->grp_score.ensure(std::max<size_t>(n_out, 1) * 4));
    OCTRY(c->grp_n.ensure(size_t(B) * G * 4));
    GroupParams gp{};
    gp.n_groups = G; gp.max_results = m;
    gp.kp2 = std::max<uint32_t>(32, next_pow2(m));
    gp.vp2 = next_pow2(std::max<uint32_t>(vlimit, 1));
    gp.g_off = g->off; gp.g_doc = g->docs; gp.g_row = has_ft ? g->rows : nullptr;
    gp.has_ft = has_ft; gp.hybrid = mode == OC_MODE_HYBRID;
    gp.mbits = c->mbits.as<uint32_t>(); gp.row_words = uint64_t(n_tiles) * (BM25_TILE / 32);
    gp.row_ft = c->row_ft.as<float>();
    gp.gmin = c->grp_gmin.as<float>(); gp.den = c->grp_den.as<float>();
    gp.v_doc = c->grp_vdoc.as<uint64_t>(); gp.v_score = c->grp_vscore.as<float>(); gp.v_n = c->grp_vn.as<uint32_t>();
    gp.v_stride = std::max<uint32_t>(vlimit, 1);
    gp.omc_doc = omc_doc; gp.omc_mult = omc_mult; gp.n_omc = n_omc;
    gp.out_doc = c->grp_doc.as<uint64_t>(); gp.out_score = c->grp_score.as<float>(); gp.out_n = c->grp_n.as<uint32_t>();
    if (sj) { gp.doc_rank = sj->f->ord[sj->order].doc_rank; gp.rank_nbits = sj->f->nbits; }
    const void *kern = sj ? (const void *)group_sort_topk_kernel : (const void *)group_topk_kernel;
    const size_t smem = (size_t(GROUP_BUF) + gp.kp2 + gp.vp2) * 8 + size_t(gp.vp2) * 4;
    if (smem_cfg_needed(c->device, kern, smem))
        CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (sj) group_sort_topk_kernel<<<dim3(G, B), GROUP_THREADS, smem, c->stream>>>(gp);
    else group_topk_kernel<<<dim3(G, B), GROUP_THREADS, smem, c->stream>>>(gp);
    launched(c);
    CU(cudaGetLastError());
    if (pj) {   // oc_search_groups_pinned: every group's list at the caller's stride, spliced for the queries with items
        const size_t n_res = size_t(B) * G * gj.stride;
        OCTRY(c->pin_gdoc.ensure(std::max<size_t>(n_res, 1) * 8));
        OCTRY(c->pin_gscore.ensure(std::max<size_t>(n_res, 1) * 4));
        OCTRY(c->pin_gn.ensure(size_t(B) * G * 4));
        GroupPinParams xp{};
        xp.n_groups = G; xp.max_results = gj.max_results; xp.stride = gj.stride; xp.n_top = m;
        xp.kp2 = std::max<uint32_t>(32, next_pow2(pj->stride));
        xp.g_off = g->off; xp.g_doc = g->docs;
        xp.doc = pj->d_doc; xp.pos = pj->d_pos; xp.score = c->pin_score.as<float>();
        xp.cnt = pin_grp ? pj->d_cnt : nullptr; xp.item_stride = pj->stride;
        xp.top_doc = gp.out_doc; xp.top_score = gp.out_score; xp.top_n = gp.out_n;
        xp.out_doc = c->pin_gdoc.as<uint64_t>(); xp.out_score = c->pin_gscore.as<float>(); xp.out_n = c->pin_gn.as<uint32_t>();
        const size_t psmem = pin_splice_smem(xp.kp2, m, std::min<uint32_t>(gj.stride, m + pj->stride));
        group_pin_splice_kernel<<<dim3(G, B), PIN_THREADS, psmem, c->stream>>>(xp);
        launched(c);
        CU(cudaGetLastError());
        if (n_res) {
            CU(cudaMemcpyAsync(gj.out_doc, xp.out_doc, n_res * 8, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaMemcpyAsync(gj.out_score, xp.out_score, n_res * 4, cudaMemcpyDeviceToHost, c->stream));
        }
        CU(cudaMemcpyAsync(gj.out_n, xp.out_n, size_t(B) * G * 4, cudaMemcpyDeviceToHost, c->stream));
        return OC_OK;
    }
    if (n_out) {
        CU(cudaMemcpyAsync(gj.out_doc, gp.out_doc, n_out * 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(gj.out_score, gp.out_score, n_out * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaMemcpyAsync(gj.out_n, gp.out_n, size_t(B) * G * 4, cudaMemcpyDeviceToHost, c->stream));
    return OC_OK;
}

extern "C" int oc_search_groups(oc_ctx *c, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                                uint32_t max_results, uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n, uint64_t *out_count,
                                uint64_t *out_group_doc_ids, float *out_group_scores, uint32_t *out_group_n) {
    if (!c || !p || !groups || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (groups->n_groups && (!out_group_n || (max_results && (!out_group_doc_ids || !out_group_scores))))
        return fail(OC_ERR_INVALID, "NULL group output");
    if (groups->ctx != c) return fail(OC_ERR_INVALID, "group_by belongs to another ctx");
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "groups over a sharded search: hybrid normalisation and the vector set are global");
    if (max_results > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "max_results %u > %u", max_results, OC_MAX_TOPK);
    if (p->n_queries > 65535) return fail(OC_ERR_UNSUPPORTED, "groups: n_queries %u > 65535", p->n_queries);
    GroupJob gj{groups, max_results, out_group_doc_ids, out_group_scores, out_group_n};
    return search_impl(c, emb, str, p, out_doc_ids, out_scores, out_n, out_count, nullptr, &gj);
}

// ------------------------------------------------------------------------------------ pin rules (pins.cuh)
static int pins_check_flat(const oc_search_params *p, const PinJob &pj) {
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "pins over a sharded search: scores and the hybrid normalisation are global");
    if (pj.splice && (uint64_t(p->limit) + p->offset) * 2 > OC_MAX_TOPK)
        return fail(OC_ERR_UNSUPPORTED, "pins: 2 x (limit+offset) %llu > %u", (unsigned long long)(uint64_t(p->limit) + p->offset) * 2,
                    OC_MAX_TOPK);
    return OC_OK;
}

extern "C" int oc_search_pinned(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_pins *pins,
                                uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n, uint64_t *out_count,
                                float *out_pin_scores, uint8_t *out_pin_present) {
    if (!c || !p) return fail(OC_ERR_INVALID, "NULL argument");
    PinJob pj;
    OCTRY(pin_job_init(pins, p->n_queries, pj));
    OCTRY(pins_check_flat(p, pj));
    return search_impl(c, emb, str, p, out_doc_ids, out_scores, out_n, out_count, nullptr, nullptr, &pj, pins, out_pin_scores,
                       out_pin_present);
}

extern "C" int oc_search_groups_pinned(oc_ctx *c, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                                       uint32_t max_results, const oc_pins *pins, uint32_t group_stride, uint64_t *out_doc_ids,
                                       float *out_scores, uint32_t *out_n, uint64_t *out_count, uint64_t *out_group_doc_ids,
                                       float *out_group_scores, uint32_t *out_group_n) {
    if (!c || !p || !groups || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (groups->n_groups && (!out_group_n || (group_stride && (!out_group_doc_ids || !out_group_scores))))
        return fail(OC_ERR_INVALID, "NULL group output");
    if (groups->ctx != c) return fail(OC_ERR_INVALID, "group_by belongs to another ctx");
    if (max_results > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "max_results %u > %u", max_results, OC_MAX_TOPK);
    if (p->n_queries > 65535) return fail(OC_ERR_UNSUPPORTED, "groups: n_queries %u > 65535", p->n_queries);
    PinJob pj;
    OCTRY(pin_job_init(pins, p->n_queries, pj));
    OCTRY(pins_check_flat(p, pj));
    if (pj.splice && 2 * max_results > OC_MAX_TOPK)
        return fail(OC_ERR_UNSUPPORTED, "pins: 2 x max_results %u > %u", 2 * max_results, OC_MAX_TOPK);
    const uint64_t need = pj.splice ? 2ull * max_results + pj.stride : max_results;
    if (group_stride < need) return fail(OC_ERR_INVALID, "group_stride %u < %llu", group_stride, (unsigned long long)need);
    GroupJob gj{groups, max_results, out_group_doc_ids, out_group_scores, out_group_n};
    gj.stride = group_stride;
    return search_impl(c, emb, str, p, out_doc_ids, out_scores, out_n, out_count, nullptr, &gj, &pj, pins);
}

// ------------------------------------------------------------------------------------ sortBy (sort.cuh)
extern "C" int oc_sort_field_create(oc_ctx *c, uint64_t nbits, uint64_t n, const uint64_t *doc_ids, const double *values,
                                    oc_sort_field **out) {
    if (!c || !out || nbits == 0 || (n && (!doc_ids || !values))) return fail(OC_ERR_INVALID, "bad arguments");
    if (nbits >= RANK_NONE) return fail(OC_ERR_INVALID, "nbits %llu >= 2^32 - 1", (unsigned long long)nbits);
    std::vector<std::pair<double, uint64_t>> e;
    e.reserve(n);
    for (uint64_t i = 0; i < n; i++) {
        if (values[i] != values[i]) return fail(OC_ERR_INVALID, "sort value %llu is NaN", (unsigned long long)i);
        if (doc_ids[i] < nbits) e.emplace_back(values[i] + 0.0, doc_ids[i]);   // -0.0 ties with 0.0
    }
    oc_sort_field *f = new oc_sort_field();
    f->ctx = c; f->nbits = nbits;
    auto fail_free = [&](int code) { sort_field_free(f); return code; };
    std::lock_guard<std::mutex> lk(c->mu);
    if (cudaSetDevice(c->device) != cudaSuccess) return fail_free(fail(OC_ERR_CUDA, "cudaSetDevice failed"));
    std::vector<uint64_t> rank_doc;
    for (int ord = OC_SORT_ASC; ord <= OC_SORT_DESC; ord++) {
        // value in the requested order, ties by ascending id; a document keeps its first position
        std::sort(e.begin(), e.end(), [ord](const std::pair<double, uint64_t> &a, const std::pair<double, uint64_t> &b) {
            if (a.first != b.first) return ord == OC_SORT_ASC ? a.first < b.first : a.first > b.first;
            return a.second < b.second;
        });
        SortOrder &o = f->ord[ord];
        o.h_doc_rank.assign(nbits, RANK_NONE);
        rank_doc.clear();
        for (const auto &x : e)
            if (o.h_doc_rank[x.second] == RANK_NONE) {
                o.h_doc_rank[x.second] = (uint32_t)rank_doc.size();
                rank_doc.push_back(x.second);
                o.h_value.push_back(x.first);
            }
        o.n = rank_doc.size();
        const uint32_t none = RANK_NONE;
        cudaError_t err = cudaMalloc(&o.rank_doc, std::max<size_t>(o.n, 1) * 8);
        if (err == cudaSuccess) err = cudaMalloc(&o.doc_rank, nbits * 4);
        if (err == cudaSuccess) err = cudaMalloc(&o.rank_row, (o.n + 1) * 4);
        if (err == cudaSuccess && o.n) err = cudaMemcpy(o.rank_doc, rank_doc.data(), o.n * 8, cudaMemcpyHostToDevice);
        if (err == cudaSuccess) err = cudaMemcpy(o.doc_rank, o.h_doc_rank.data(), nbits * 4, cudaMemcpyHostToDevice);
        if (err == cudaSuccess) err = cudaMemcpy(o.rank_row + o.n, &none, 4, cudaMemcpyHostToDevice);
        if (err != cudaSuccess)
            return fail_free(fail(err == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "sort field upload: %s", cudaGetErrorString(err)));
    }
    *out = f;
    return OC_OK;
}

extern "C" void oc_sort_field_destroy(oc_sort_field *f) {
    if (!f) return;
    {
        std::lock_guard<std::mutex> lk(f->ctx->mu);
        cudaSetDevice(f->ctx->device);
        cudaStreamSynchronize(f->ctx->stream);
    }
    sort_field_free(f);
}

extern "C" int oc_search_sorted(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_sort *sort,
                                const oc_pins *pins, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                                uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present) {
    if (!c || !p) return fail(OC_ERR_INVALID, "NULL argument");
    SortJob sj{};
    OCTRY(sort_job_init(c, sort, sj));
    sj.out_values = out_sort_values;
    PinJob pj;
    OCTRY(pin_job_init(pins, p->n_queries, pj));
    OCTRY(pins_check_flat(p, pj));
    return search_impl(c, emb, str, p, out_doc_ids, out_scores, out_n, out_count, nullptr, nullptr, &pj, pins, out_pin_scores,
                       out_pin_present, &sj);
}

extern "C" int oc_search_groups_sorted(oc_ctx *c, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                                       uint32_t max_results, const oc_sort *sort, const oc_pins *pins, uint32_t group_stride,
                                       uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                                       uint64_t *out_count, uint64_t *out_group_doc_ids, float *out_group_scores,
                                       double *out_group_sort_values, uint32_t *out_group_n) {
    if (!c || !p || !groups || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (groups->n_groups && (!out_group_n || (group_stride && (!out_group_doc_ids || !out_group_scores))))
        return fail(OC_ERR_INVALID, "NULL group output");
    if (groups->ctx != c) return fail(OC_ERR_INVALID, "group_by belongs to another ctx");
    SortJob sj{};
    OCTRY(sort_job_init(c, sort, sj));
    sj.out_values = out_sort_values; sj.out_group_values = out_group_sort_values; sj.n_groups = groups->n_groups;
    if (max_results > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "max_results %u > %u", max_results, OC_MAX_TOPK);
    if (p->n_queries > 65535) return fail(OC_ERR_UNSUPPORTED, "groups: n_queries %u > 65535", p->n_queries);
    PinJob pj;
    OCTRY(pin_job_init(pins, p->n_queries, pj));
    OCTRY(pins_check_flat(p, pj));
    if (pj.splice && 2 * max_results > OC_MAX_TOPK)
        return fail(OC_ERR_UNSUPPORTED, "pins: 2 x max_results %u > %u", 2 * max_results, OC_MAX_TOPK);
    const uint64_t need = pj.splice ? 2ull * max_results + pj.stride : max_results;
    if (group_stride < need) return fail(OC_ERR_INVALID, "group_stride %u < %llu", group_stride, (unsigned long long)need);
    GroupJob gj{groups, max_results, out_group_doc_ids, out_group_scores, out_group_n};
    gj.stride = group_stride;
    return search_impl(c, emb, str, p, out_doc_ids, out_scores, out_n, out_count, nullptr, &gj, &pj, pins, nullptr, nullptr, &sj);
}

// ------------------------------------------------------------------------------------ geopoint where-filter leaves (geo.cuh)
static_assert(OC_GEO_MAX_VERTICES == GEO_MAX_VERTICES, "the header's vertex cap is the kernel's staging size");
constexpr double GEO_PI = 3.14159265358979323846;

struct oc_geo_field {
    oc_ctx *ctx;
    uint64_t nbits, n;
    void *blob = nullptr;   // device: x, y, z, lat, lon (f64) then doc (u64), n entries each
    GeoPoints pts() const {
        const double *d = static_cast<const double *>(blob);
        return GeoPoints{d, d + n, d + 2 * n, d + 3 * n, d + 4 * n, reinterpret_cast<const uint64_t *>(d + 5 * n), n};
    }
};

static bool geo_valid(double lat, double lon) {
    return std::isfinite(lat) && std::isfinite(lon) && lat >= -90.0 && lat <= 90.0 && lon >= -180.0 && lon <= 180.0;
}
static void geo_unit(double lat, double lon, double u[3]) {
    const double la = lat * (GEO_PI / 180.0), lo = lon * (GEO_PI / 180.0);
    u[0] = std::cos(la) * std::cos(lo); u[1] = std::cos(la) * std::sin(lo); u[2] = std::sin(la);
}

extern "C" int oc_geo_field_create(oc_ctx *c, uint64_t nbits, uint64_t n, const uint64_t *doc_ids, const double *lat,
                                   const double *lon, oc_geo_field **out) {
    if (!c || !out || (n && (!doc_ids || !lat || !lon))) return fail(OC_ERR_INVALID, "bad arguments");
    for (uint64_t i = 0; i < n; i++)
        if (!geo_valid(lat[i], lon[i]))
            return fail(OC_ERR_INVALID, "geopoint %llu: invalid coordinates (%g, %g)", (unsigned long long)i, lat[i], lon[i]);
    std::vector<uint64_t> order;
    order.reserve(n);
    for (uint64_t i = 0; i < n; i++) if (doc_ids[i] < nbits) order.push_back(i);
    std::stable_sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return doc_ids[a] < doc_ids[b]; });
    const uint64_t m = order.size();
    std::vector<double> h(6 * m);
    for (uint64_t k = 0; k < m; k++) {
        const uint64_t i = order[k];
        double u[3];
        geo_unit(lat[i], lon[i], u);
        h[k] = u[0]; h[m + k] = u[1]; h[2 * m + k] = u[2]; h[3 * m + k] = lat[i]; h[4 * m + k] = lon[i];
        memcpy(&h[5 * m + k], &doc_ids[i], 8);
    }
    oc_geo_field *g = new oc_geo_field();
    g->ctx = c; g->nbits = nbits; g->n = m;
    std::lock_guard<std::mutex> lk(c->mu);
    cudaError_t e = cudaSetDevice(c->device);
    if (e == cudaSuccess && m) e = cudaMalloc(&g->blob, h.size() * 8);
    if (e == cudaSuccess && m) e = cudaMemcpy(g->blob, h.data(), h.size() * 8, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        if (g->blob) cudaFree(g->blob);
        delete g;
        return fail(e == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "geo field upload: %s", cudaGetErrorString(e));
    }
    *out = g;
    return OC_OK;
}

extern "C" void oc_geo_field_destroy(oc_geo_field *g) {
    if (!g) return;
    {
        std::lock_guard<std::mutex> lk(g->ctx->mu);
        cudaSetDevice(g->ctx->device);
        cudaStreamSynchronize(g->ctx->stream);
        if (g->blob) cudaFree(g->blob);
    }
    delete g;
}

// a zeroed leaf over [0, nbits) of g's ctx, filled by `launch` (called under the ctx lock when g has points)
template <typename F>
static int geo_leaf(const oc_geo_field *g, oc_filter **out, F &&launch) {
    oc_ctx *c = g->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    CU(cudaSetDevice(c->device));
    oc_filter *f = nullptr;
    OCTRY(filter_alloc(c, g->nbits, &f));
    auto fail_free = [&](int code) { cudaFree(f->bits); delete f; return code; };
    cudaError_t e = cudaMemsetAsync(f->bits, 0, std::max<uint64_t>(f->words, 1) * 8, c->stream);
    if (e == cudaSuccess && g->n) {
        const int r = launch(c, reinterpret_cast<unsigned long long *>(f->bits),
                             (unsigned)std::min<uint64_t>((g->n + GEO_THREADS - 1) / GEO_THREADS, uint64_t(c->prop.multiProcessorCount) * 8));
        if (r != OC_OK) return fail_free(r);
        launched(c);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return fail_free(fail(OC_ERR_CUDA, "geo filter: %s", cudaGetErrorString(e)));
    *out = f;
    return OC_OK;
}

extern "C" int oc_filter_geo_radius(const oc_geo_field *g, double lat, double lon, double radius_m, int inside, oc_filter **out) {
    if (!g || !out) return fail(OC_ERR_INVALID, "NULL argument");
    if (!geo_valid(lat, lon)) return fail(OC_ERR_INVALID, "radius centre: invalid coordinates (%g, %g)", lat, lon);
    if (!(std::isfinite(radius_m) && radius_m >= 0.0)) return fail(OC_ERR_INVALID, "radius %g m: not finite and >= 0", radius_m);
    double u[3];
    geo_unit(lat, lon, u);
    const double half = radius_m / (2.0 * OC_GEO_EARTH_RADIUS_M);   // half the central angle
    const double s = std::sin(half);
    const double thr = half >= GEO_PI / 2 ? std::numeric_limits<double>::infinity() : 4.0 * s * s;
    return geo_leaf(g, out, [&](oc_ctx *c, unsigned long long *bits, unsigned grid) {
        geo_radius_kernel<<<grid, GEO_THREADS, 0, c->stream>>>(g->pts(), u[0], u[1], u[2], thr, inside, bits);
        return OC_OK;
    });
}

extern "C" int oc_filter_geo_polygon(const oc_geo_field *g, const double *lat, const double *lon, uint32_t n_vertices,
                                     int inside, oc_filter **out) {
    if (!g || !out || (n_vertices && (!lat || !lon))) return fail(OC_ERR_INVALID, "NULL argument");
    if (n_vertices < 3 || n_vertices > OC_GEO_MAX_VERTICES)
        return fail(OC_ERR_INVALID, "polygon of %u vertices: 3 to %u are supported", n_vertices, OC_GEO_MAX_VERTICES);
    double4 bb = make_double4(lon[0], lon[0], lat[0], lat[0]);
    for (uint32_t k = 0; k < n_vertices; k++) {
        if (!geo_valid(lat[k], lon[k])) return fail(OC_ERR_INVALID, "polygon vertex %u: invalid coordinates (%g, %g)", k, lat[k], lon[k]);
        bb.x = std::min(bb.x, lon[k]); bb.y = std::max(bb.y, lon[k]); bb.z = std::min(bb.z, lat[k]); bb.w = std::max(bb.w, lat[k]);
    }
    bb.x -= GEO_BBOX_MARGIN; bb.y += GEO_BBOX_MARGIN;
    return geo_leaf(g, out, [&](oc_ctx *c, unsigned long long *bits, unsigned grid) {
        OCTRY(c->in_blob.ensure(size_t(2) * n_vertices * 8));
        double *v = c->in_blob.as<double>();
        CU(cudaMemcpyAsync(v, lon, size_t(n_vertices) * 8, cudaMemcpyHostToDevice, c->stream));
        CU(cudaMemcpyAsync(v + n_vertices, lat, size_t(n_vertices) * 8, cudaMemcpyHostToDevice, c->stream));
        geo_polygon_kernel<<<grid, GEO_THREADS, 0, c->stream>>>(g->pts(), v, v + n_vertices, n_vertices, bb, inside, bits);
        return OC_OK;
    });
}

// ------------------------------------------------------------------------------------ micro-batching front
struct OcSearchExec {
    oc_ctx *c; oc_emb *e; oc_str *s;
    int operator()(const oc_search_params *p, uint64_t *docs, float *scores, uint32_t *n, uint64_t *count) const {
        return oc_search(c, e, s, p, docs, scores, n, count);
    }
};
struct oc_batcher {
    ocb::Batcher<OcSearchExec> q;
    oc_ctx *ctx;
    oc_batcher(OcSearchExec x, uint32_t dim, uint32_t mb, uint32_t mw) : q(x, dim, mb, mw, x.e != nullptr, x.s != nullptr), ctx(x.c) {}
};
extern "C" int oc_batcher_create(oc_ctx *c, oc_emb *emb, oc_str *str, uint32_t max_batch, uint32_t max_wait_us, oc_batcher **out) {
    if (!c || !out || (!emb && !str)) return fail(OC_ERR_INVALID, "bad arguments");
    if ((emb && emb->ctx != c) || (str && str->ctx != c)) return fail(OC_ERR_INVALID, "store belongs to another ctx");
    if (max_batch == 0 || max_batch > 4096) return fail(OC_ERR_INVALID, "max_batch %u outside 1..4096", max_batch);
    *out = new oc_batcher(OcSearchExec{c, emb, str}, emb ? emb->dim : 0, max_batch, max_wait_us);
    return OC_OK;
}
extern "C" void oc_batcher_destroy(oc_batcher *b) { delete b; }
extern "C" int oc_batcher_search(oc_batcher *b, const oc_search_params *p, uint64_t *out_doc_ids, float *out_scores,
                                 uint32_t *out_n, uint64_t *out_count) {
    if (!b || !p || !out_doc_ids || !out_scores || !out_n || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (p->n_queries != 1) return fail(OC_ERR_INVALID, "oc_batcher_search takes one query per call (n_queries = %u)", p->n_queries);
    // a device filter joins a batch as that query's q_filters entry: one of another ctx would fail the whole batch
    if (p->filter && p->filter->ctx != b->ctx) return fail(OC_ERR_INVALID, "filter belongs to another ctx");
    g_err[0] = 0;
    const int rc = b->q.submit(p, out_doc_ids, out_scores, out_n, out_count);
    // the batch ran on its leader's thread: that is where oc_last_error() holds the detail
    if (rc != OC_OK && g_err[0] == 0) return fail(rc, "the coalesced oc_search of this query's batch failed (detail on the leading caller's thread)");
    return rc;
}
extern "C" int oc_batcher_stats(oc_batcher *b, uint64_t *n_queries, uint64_t *n_batches, uint64_t *n_direct) {
    if (!b) return fail(OC_ERR_INVALID, "NULL argument");
    b->q.stats(n_queries, n_batches, n_direct);
    return OC_OK;
}

// ------------------------------------------------------------------------------------ term dictionary / query resolution
// Host only (no device): the step the reference performs before the posting walk — tokenize_and_stem
// (token_score.rs:196-209) and the FST term expansion inside StringStorage (string_field.rs:208-225).
struct oc_dict { ocd::Dict d; explicit oc_dict(uint32_t n) : d(n) {} };
struct oc_resolved { ocd::Resolved r; };

extern "C" int oc_dict_create(uint32_t n_fields, oc_dict **out) {
    if (!out || n_fields == 0) return fail(OC_ERR_INVALID, "bad arguments");
    *out = new oc_dict(n_fields);
    return OC_OK;
}
extern "C" void oc_dict_destroy(oc_dict *d) { delete d; }
extern "C" int oc_dict_add_terms(oc_dict *d, uint32_t field, const char *const *terms, uint32_t n, uint32_t *out_ids) {
    if (!d || field >= d->d.n_fields() || (n && !terms)) return fail(OC_ERR_INVALID, "bad arguments");
    for (uint32_t i = 0; i < n; i++) if (!terms[i]) return fail(OC_ERR_INVALID, "term %u is NULL", i);
    d->d.add_terms(field, terms, n, out_ids);
    return OC_OK;
}
extern "C" int oc_dict_lookup(oc_dict *d, uint32_t field, const char *term, uint32_t *out_id) {
    if (!d || field >= d->d.n_fields() || !term || !out_id) return fail(OC_ERR_INVALID, "bad arguments");
    if (!d->d.lookup(field, term, out_id)) *out_id = 0xffffffffu;
    return OC_OK;
}
extern "C" uint32_t oc_dict_size(oc_dict *d, uint32_t field) { return (d && field < d->d.n_fields()) ? d->d.size(field) : 0; }
// Snowball English (Porter2), restated in csrc/stem_en.h: an oc_stem_fn a host without its own parser can install
extern "C" size_t oc_stem_english(const char *tok, size_t len, char *out, size_t cap, void *user) {
    (void)user;
    if (!tok || !out) return 0;
    const std::string st = ocs::stem_english(std::string(tok, len));
    if (st.size() > cap) return 0;
    memcpy(out, st.data(), st.size());
    return st.size();
}
extern "C" int oc_dict_set_stemmer(oc_dict *d, oc_stem_fn fn, void *user) {
    if (!d) return fail(OC_ERR_INVALID, "dict is NULL");
    d->d.set_stemmer(fn, user);
    return OC_OK;
}
extern "C" int oc_dict_resolve(oc_dict *d, const oc_resolve_params *p, oc_resolved **out) {
    if (!d || !p || !out || (p->n_queries && !p->texts)) return fail(OC_ERR_INVALID, "bad arguments");
    for (uint32_t i = 0; i < p->n_queries; i++) if (!p->texts[i]) return fail(OC_ERR_INVALID, "text %u is NULL", i);
    if (p->tolerance > 8) return fail(OC_ERR_UNSUPPORTED, "tolerance %d > 8", p->tolerance);
    ocd::ResolveOpts o;
    o.exact = p->exact != 0; o.tolerance = p->tolerance; o.field_boost = p->field_boost; o.field_mask = p->field_mask;
    o.exact_match_boost = p->exact_match_boost > 0.f ? p->exact_match_boost : 2.0f;
    oc_resolved *r = new oc_resolved();
    d->d.resolve(p->texts, p->n_queries, o, &r->r);
    *out = r;
    return OC_OK;
}
extern "C" void oc_resolved_arrays(const oc_resolved *r, const uint32_t **q_token_offsets, const uint32_t **token_term_offsets,
                                   const uint32_t **term_field, const uint32_t **term_id, const float **term_weight,
                                   uint32_t *n_tokens, uint32_t *n_terms) {
    if (!r) return;
    static const uint32_t zero_u = 0; static const float one_f = 1.0f;   // empty arrays still get valid pointers
    if (q_token_offsets) *q_token_offsets = r->r.q_token_offsets.data();
    if (token_term_offsets) *token_term_offsets = r->r.token_term_offsets.data();
    if (term_field) *term_field = r->r.term_field.empty() ? &zero_u : r->r.term_field.data();
    if (term_id) *term_id = r->r.term_id.empty() ? &zero_u : r->r.term_id.data();
    if (term_weight) *term_weight = r->r.term_weight.empty() ? &one_f : r->r.term_weight.data();
    if (n_tokens) *n_tokens = (uint32_t)r->r.token_term_offsets.size() - 1;
    if (n_terms) *n_terms = (uint32_t)r->r.term_id.size();
}
extern "C" void oc_resolved_fill(const oc_resolved *r, oc_search_params *p) {
    if (!r || !p) return;
    oc_resolved_arrays(r, &p->q_token_offsets, &p->token_term_offsets, &p->term_field, &p->term_id, &p->term_weight, nullptr, nullptr);
    p->n_queries = (uint32_t)r->r.q_token_offsets.size() - 1;
}
extern "C" void oc_resolved_free(oc_resolved *r) { delete r; }
