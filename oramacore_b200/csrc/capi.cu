// capi.cu — host side of liboramacore_b200.so: the C ABI declared in
// include/oramacore_b200.h over the sm_90a kernels (emb_scan.cuh, bm25.cuh, fuse.cuh).
// No torch, no CPU fallback: every entry point needs a live CUDA device.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <atomic>
#include <chrono>
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
#include <tuple>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "bm25.cuh"
#include "comm.h"
#include "dense_cache.h"
#include "dict.h"
#include "dict_dev.cuh"
#include "stem_en.h"
#include "emb_compact.cuh"
#include "str_commit.cuh"
#include "facet_commit.cuh"
#include "emb_gemm.cuh"
#include "emb_scan.cuh"
#include "fuse.cuh"
#include "geo.cuh"
#include "group.cuh"
#include "pins.cuh"
#include "sort.cuh"
#include "index_merge.cuh"
#include "sort_build.cuh"
#include "omc.cuh"
#include "tmap.cuh"
#include "where.cuh"
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
// per device so several contexts on different GPUs in one process each get their kernels configured.  The attribute
// is set under the lock: a context sharing the device with another must not launch before the size it relies on is set.
static cudaError_t smem_cfg(int device, const void *fn, size_t smem) {
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, size_t> done;
    std::lock_guard<std::mutex> g(mu);
    size_t &v = done[std::make_pair(device, fn)];
    if (smem <= v) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) v = smem;
    return e;
}

// ------------------------------------------------------------------------------------ buffers
// workspaces grow on demand and free themselves
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
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
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }   // a large workspace of a rare call goes back at once
    template <typename T> T *as() { return reinterpret_cast<T *>(p); }
};
struct HostBuf {  // pinned staging
    void *p = nullptr;
    size_t cap = 0;
    HostBuf() = default;
    HostBuf(const HostBuf &) = delete;
    HostBuf &operator=(const HostBuf &) = delete;
    ~HostBuf() { if (p) cudaFreeHost(p); }
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
    template <typename T> T *as() { return reinterpret_cast<T *>(p); }
};

// an array's place in a packed upload; at(blob) is its device copy once the blob is up (NULL: never added)
template <typename T> struct Slot {
    size_t off = 0;
    bool added = false;
    const T *at(const DevBuf &blob) const {
        return added ? reinterpret_cast<const T *>(static_cast<const uint8_t *>(blob.p) + off) : nullptr;
    }
};
// lays several host arrays out in one pinned blob -> one H2D copy (sources are copied once,
// straight into the pinned staging buffer)
struct Packer {
    struct Seg { const void *src; size_t off, bytes; bool direct; };
    std::vector<Seg> segs;
    size_t total = 0;
    // n elements of src; direct = the source already lives in pinned host memory (oc_pinned_alloc /
    // cudaHostRegister): it is DMA'd straight from the caller's buffer instead of being staged
    template <typename T> Slot<T> add(const T *src, size_t n, bool direct = false) {
        const size_t off = (total + 255) & ~size_t(255);
        segs.push_back({src, off, n * sizeof(T), direct});
        total = off + n * sizeof(T);
        return Slot<T>{off, true};
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
constexpr uint32_t LOCAL_MAX_WORLD = 16;   // oc_comm_init_local: = SHARD_MAX_WORLD (shard.cuh), the merge's largest world

struct oc_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t side = nullptr;      // descriptor upload + BM25 plan/precompute while the main stream sweeps the matrix
    cudaEvent_t ev_side = nullptr;    // the side stream's fulltext stage is complete
    cudaEvent_t ev_side_in = nullptr; // the side stream has put up what the hybrid point lookups read (see bm25_stage)
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
    DevBuf seg, df_dev, row_ok, tau, cand_key, cand_ft, cand_cnt, tile_cnt, tile_max, tile_min;
    DevBuf out_blob, shard_send, shard_recv, work_ctr, flat_desc, mbits, dbits, facet_out;
    bool gemm_pending = false; const float *gemm_inv_norm = nullptr;
    DevBuf row_ft, grp_vdoc, grp_vscore, grp_vn, grp_gmin, grp_den, grp_doc, grp_score, grp_n;   // oc_search_groups
    DevBuf pin_row, pin_ft, pin_ftp, pin_score, pin_present, pin_top_doc, pin_top_score, pin_top_n, pin_gdoc, pin_gscore, pin_gn;   // pins
    DevBuf srt_doc, srt_row, srt_n, srt_ft, srt_ftp, srt_score, srt_present, srt_zero;   // sortBy
    DevBuf mi_doc, mi_score, mi_val, mi_n, mi_cnt, mi_pscore, mi_ppresent, mi_out;   // oc_search_indexes: per-index lists, page
    DevBuf mg_doc, mg_score, mg_val, mg_n;   // oc_search_indexes_ex: per-index group lists
    DevBuf sfb_ws;                    // sort field build (sort_build.cuh), released before the call returns
    DevBuf q_bf16, q_f16, q_scale, q_rho, pre_post, dense_buf, g_thr, g_eps, g_ovf, g_ovfcnt, g_resc, g_cand, g_cnt, g_flag, g_max, r_qpad, r_qinv, r_map, r_doc, r_score, r_row, r_cnt, r_raw;
    // per-query where-filters (q_filters): the embedding rows' bitmap of every distinct handle, and the slots of the
    // queries the exact sweep re-runs; v_qslot / v_rowbits describe the vector stage of the current call (fix_unproven)
    DevBuf e_rowbits, r_slot;
    const uint32_t *v_rowbits = nullptr; uint64_t v_row_words = 0;
    std::vector<uint32_t> v_qslot;
    // per-query parameters (q_params): the vector stage sweeps the sub-batch of queries with a vector part, each cut to
    // its own depth (v_qlim) and similarity (v_qsim); v_qmap: the batch query of each sub-batch query (empty: the
    // whole batch).  vq_*: the sub-batch's hits before they are scattered to their queries' rows.
    std::vector<uint32_t> v_qlim, v_qmap;
    std::vector<float> v_qsim;
    DevBuf vq_doc, vq_score, vq_row, vq_cnt, vq_raw, r_lim, r_sim;
    // where programs (q_where): the leaf and result bitmaps of the call, and its plan tables (h_where: their staging)
    DevBuf w_bits, w_blob;
    HostBuf h_where;
    // oc_emb_compact: the dead-row bitmap with its scan, and the staging window the rows move through (held for the
    // call only: a compaction is rare and its window is large)
    DevBuf cmp_scan, cmp_stage;
    // oc_str_sync_global: the staging of its small gathers (header, term counts, length sums)
    DevBuf sync_buf;
    // the dense contribution arrays of hot terms, kept across calls (dense_cache.h)
    DenseCache dense_cache;
    // oc_dict_resolve_q: the mirror of each dictionary resolved on this ctx, by dictionary serial (dict_dev.cuh), and
    // the call's pair descriptors, per-chunk counts and output
    std::unordered_map<uint64_t, std::unique_ptr<ocdd::DictMirror>> dict_mirrors;
    DevBuf fz_in, fz_cnt, fz_out;

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
    ~oc_ctx() {   // the workspaces free themselves after this
        for (int r = 0; r < 16; r++) if (p2p.ready && p2p.peer[r] && p2p.peer[r] != p2p.local) cudaIpcCloseMemHandle(p2p.peer[r]);
        if (p2p.local) cudaFree(p2p.local);
        comm.destroy();
        if (stream) { dense_cache.clear(stream); cudaStreamSynchronize(stream); }
        for (int i = 0; i < EV_N; i++) if (ev[i]) cudaEventDestroy(ev[i]);
        if (stream) cudaStreamDestroy(stream);
        if (side) cudaStreamDestroy(side);
        if (ev_side) cudaEventDestroy(ev_side);
        if (ev_side_in) cudaEventDestroy(ev_side_in);
    }
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
    CU(cudaEventCreateWithFlags(&c->ev_side_in, cudaEventDisableTiming));
    for (int i = 0; i < EV_N; i++) CU(cudaEventCreate(&c->ev[i]));
    *out = c;
    return OC_OK;
}

#ifdef OC_BM25_PHASE_PROFILE
// (phase-profile library only: where bm25_warp_kernel appends its records, device pointers; counters NULL: none)
extern "C" int oc_bm25_phase_profile(void *items, uint32_t cap_items, void *warps, uint32_t cap_warps, void *counters) {
    BwProf g{};
    g.items = static_cast<BwProfItem *>(items); g.warps = static_cast<BwProfWarp *>(warps);
    g.n_items = static_cast<unsigned int *>(counters); g.n_warps = g.n_items + 1;
    g.cap_items = cap_items; g.cap_warps = cap_warps;
    CU(cudaMemcpyToSymbol(g_bw_prof, &g, sizeof(g)));
    return OC_OK;
}
#endif

extern "C" void oc_shutdown(oc_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
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
extern "C" int oc_comm_init_local(oc_ctx *const *ctxs, int world) {
    if (!ctxs || world < 1 || world > (int)LOCAL_MAX_WORLD) return fail(OC_ERR_INVALID, "oc_comm_init_local: 1..%u contexts", LOCAL_MAX_WORLD);
    for (int r = 0; r < world; r++) {
        if (!ctxs[r]) return fail(OC_ERR_INVALID, "oc_comm_init_local: ctxs[%d] is NULL", r);
        for (int s = 0; s < r; s++)
            if (ctxs[s] == ctxs[r]) return fail(OC_ERR_INVALID, "oc_comm_init_local: ctxs[%d] == ctxs[%d]", s, r);
    }
    auto g = std::make_shared<LocalGroup>(world);
    for (int r = 0; r < world; r++) {
        std::lock_guard<std::mutex> lk(ctxs[r]->mu);
        ctxs[r]->comm.init_local(g, r);
    }
    return OC_OK;
}

// Direct NVLink exchange: rank r exports the IPC handle of its window, the host runtime all-gathers the blobs (like
// the NCCL unique id) and every rank maps all peers' windows.  Afterwards the sharded oc_search stores each query's
// shard record straight into every rank's window from the pack kernel and the merge kernel waits on arrival
// counters — no library collective on the data path (ncclAllGather stays the fallback for batches larger than a window).
extern "C" int oc_comm_p2p_export(oc_ctx *c, uint8_t out[OC_P2P_HANDLE_BYTES]) {
    if (!c || !out) return fail(OC_ERR_INVALID, "NULL argument");
    if (c->comm.local) return fail(OC_ERR_INVALID, "oc_comm_p2p_export: the ranks of a local group exchange through the host");
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
    // fp32 stores: the operand of the fp16 tensor-core sweep (emb_gemm.cuh, GEMM_F16).  f16 is false for bf16 stores,
    // when OC_EMB_F16=0 at creation, and from the first time the copy could not be allocated on (the store is then
    // swept through tf32)
    bool f16 = false;
    uint16_t *rows_f16 = nullptr; // [cap][stride] each row times 2^s, s putting its largest |x_i| in [2^14, 2^15)
    float *row_scale = nullptr;   // [cap] 2^-s (NaN: a non-finite element)
    uint64_t n_rows = 0, cap = 0, n_live = 0;
    std::unordered_multimap<uint64_t, uint64_t> doc_rows;  // doc -> rows (for delete)
    std::vector<uint64_t> dead;   // the rows tombstoned since the last compaction (n_rows - n_live of them), unsorted
};

// OC_EMB_F16=0: no fp16 copy for stores created while it is set, and searches use the tf32 sweep (A/B testing)
static bool env_emb_f16_off() {
    const char *v = getenv("OC_EMB_F16");
    return v && v[0] == '0';
}

extern "C" int oc_emb_create(oc_ctx *c, uint32_t dim, int dtype, int rescale_e5, oc_emb **out) {
    if (!c || !out) return fail(OC_ERR_INVALID, "NULL argument");
    if (dim == 0 || dim > 1024) return fail(OC_ERR_UNSUPPORTED, "dim %u unsupported (1..1024)", dim);
    if (dtype != OC_DTYPE_F32 && dtype != OC_DTYPE_BF16) return fail(OC_ERR_UNSUPPORTED, "dtype %d unknown", dtype);
    oc_emb *e = new oc_emb();
    e->ctx = c; e->dim = dim; e->dtype = dtype; e->e5 = rescale_e5 ? 1 : 0;
    e->esz = dtype == OC_DTYPE_BF16 ? 2 : 4;
    e->f16 = dtype == OC_DTYPE_F32 && !env_emb_f16_off();
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
    cudaFree(e->rows_f16); cudaFree(e->row_scale);
    delete e;
}

// Moves the store into fresh allocations of ncap >= n_rows rows.  An fp16 copy that finds no room is dropped (the
// store stays whole and is swept through tf32 from now on) unless keep_f16: then the call fails and changes nothing.
static int emb_realloc(oc_emb *e, uint64_t ncap, bool keep_f16) {
    oc_ctx *c = e->ctx;
    void *nr = nullptr; float *nn = nullptr; uint64_t *nd = nullptr;
    uint16_t *nh = nullptr; float *ns = nullptr;
    auto undo = [&](int rc) { cudaFree(nr); cudaFree(nn); cudaFree(nd); cudaFree(nh); cudaFree(ns); return rc; };
    if (cudaMalloc(&nr, ncap * e->stride * e->esz) != cudaSuccess || cudaMalloc(&nn, (ncap + 64) * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&nd, ncap * sizeof(uint64_t)) != cudaSuccess) {
        (void)cudaGetLastError();
        return undo(fail(OC_ERR_OOM, "embedding store: no room for %llu rows", (unsigned long long)ncap));
    }
    if (e->f16 && (cudaMalloc(&nh, ncap * e->stride * 2) != cudaSuccess || cudaMalloc(&ns, ncap * sizeof(float)) != cudaSuccess)) {
        (void)cudaGetLastError();
        if (keep_f16) return undo(fail(OC_ERR_OOM, "embedding store: no room for the fp16 copy of %llu rows", (unsigned long long)ncap));
        cudaFree(nh); cudaFree(ns); nh = nullptr; ns = nullptr;
        cudaFree(e->rows_f16); cudaFree(e->row_scale); e->rows_f16 = nullptr; e->row_scale = nullptr;
        e->f16 = false;
    }
    cudaError_t ce = cudaSuccess;
    auto copy = [&](void *dst, const void *src, size_t bytes) {
        if (ce == cudaSuccess) ce = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c->stream);
    };
    if (e->n_rows) {
        copy(nr, e->rows, e->n_rows * e->stride * e->esz);
        copy(nn, e->inv_norm, e->n_rows * sizeof(float));
        copy(nd, e->row_doc, e->n_rows * sizeof(uint64_t));
        if (nh) {
            copy(nh, e->rows_f16, e->n_rows * e->stride * 2);
            copy(ns, e->row_scale, e->n_rows * sizeof(float));
        }
    }
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(c->stream);
    if (ce != cudaSuccess) return undo(fail(OC_ERR_CUDA, "embedding store: copy to the new allocation: %s", cudaGetErrorString(ce)));
    cudaFree(e->rows); cudaFree(e->inv_norm); cudaFree(e->row_doc);
    e->rows = nr; e->inv_norm = nn; e->row_doc = nd; e->cap = ncap;
    if (nh) {
        cudaFree(e->rows_f16); cudaFree(e->row_scale);
        e->rows_f16 = nh; e->row_scale = ns;
    }
    return OC_OK;
}

// the capacity a store grown from empty to want_rows rows gets
static uint64_t emb_round_cap(uint64_t want_rows) { return (want_rows + 63) / 64 * 64; }

static int emb_grow(oc_emb *e, uint64_t want_rows) {
    if (want_rows <= e->cap) return OC_OK;
    return emb_realloc(e, emb_round_cap(std::max<uint64_t>(want_rows, e->cap + e->cap / 2)), false);
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
    if (e->f16) {
        emb_f16_rows_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(static_cast<const float *>(e->rows), e->stride, e->n_rows,
                                                                     e->n_rows + n, e->rows_f16, e->row_scale);
        launched(c);
    }
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
    e->dead.insert(e->dead.end(), rows.begin(), rows.end());
    return OC_OK;
}

extern "C" int oc_emb_info(oc_emb *e, oc_emb_info_t *out) {
    if (!e || !out) return fail(OC_ERR_INVALID, "NULL argument");
    out->num_embeddings = e->n_live; out->num_rows = e->n_rows; out->dimensions = e->dim; out->dtype = e->dtype;
    out->device_bytes = e->cap * (uint64_t(e->stride) * e->esz + 4 + 8);
    if (e->f16) out->device_bytes += e->cap * (uint64_t(e->stride) * 2 + 4);
    return OC_OK;
}

// ---- compaction (emb_compact.cuh)
// OC_EMB_COMPACT_WINDOW=<bytes>: the staging window of oc_emb_compact (tests use a small one to span many windows)
static size_t compact_window_bytes() {
    const char *v = getenv("OC_EMB_COMPACT_WINDOW");
    const unsigned long long b = v ? strtoull(v, nullptr, 10) : 0;
    return b ? (size_t)std::min<unsigned long long>(b, 128ull << 20) : size_t(32) << 20;
}

extern "C" int oc_emb_compact(oc_emb *e, uint32_t flags, oc_emb_compact_t *out) {
    if (!e) return fail(OC_ERR_INVALID, "emb is NULL");
    if (flags & ~OC_EMB_COMPACT_SHRINK) return fail(OC_ERR_INVALID, "oc_emb_compact: unknown flags 0x%x", flags);
    oc_ctx *c = e->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    struct Release {   // every way out of the call gives the workspace back
        oc_ctx *c;
        ~Release() { cudaStreamSynchronize(c->stream); c->cmp_scan.release(); c->cmp_stage.release(); }
    } release{c};
    oc_emb_compact_t st{};
    oc_emb_info_t inf{};
    oc_emb_info(e, &inf);
    st.rows_before = st.rows_after = e->n_rows;
    st.device_bytes_before = st.device_bytes_after = inf.device_bytes;
    if (!e->dead.empty()) {
        std::vector<uint64_t> &dead = e->dead;
        std::sort(dead.begin(), dead.end());
        const uint64_t n = e->n_rows, first = dead[0];
        const uint64_t n_words = (n + 31) / 32, n_blocks = (n_words + COMPACT_SCAN_WORDS - 1) / COMPACT_SCAN_WORDS;
        std::vector<uint32_t> bits(n_words, 0);
        for (uint64_t r : dead) bits[r >> 5] |= 1u << (r & 31);
        // row windows of the matrix (W rows) and of the per-row arrays (16 B per row: Ws rows), one staging buffer
        const size_t win = compact_window_bytes(), row_bytes = size_t(e->stride) * e->esz;
        const uint64_t W = std::max<uint64_t>(1, win / row_bytes), Ws = std::max<uint64_t>(1, win / 16);
        const size_t stage_bytes = std::max<size_t>(std::min<uint64_t>(W, n - first) * row_bytes, std::min<uint64_t>(Ws, n - first) * 16);
        const size_t o_pre = (n_words * 4 + 255) & ~size_t(255), o_blk = o_pre * 2;
        // everything that can fail for want of memory happens before the first row moves
        OCTRY(c->cmp_scan.ensure(o_blk + n_blocks * 4));
        OCTRY(c->cmp_stage.ensure(stage_bytes));
        st.workspace_bytes = c->cmp_scan.cap + c->cmp_stage.cap;
        uint32_t *d_bits = c->cmp_scan.as<uint32_t>(), *d_pre = d_bits + o_pre / 4, *d_blk = d_bits + o_blk / 4;
        CU(cudaMemcpyAsync(d_bits, bits.data(), n_words * 4, cudaMemcpyHostToDevice, c->stream));
        CU(cudaEventRecord(c->ev[EV_START], c->stream));
        compact_scan_words_kernel<<<(unsigned)n_blocks, COMPACT_SCAN_WORDS, 0, c->stream>>>(d_bits, n_words, d_pre, d_blk);
        launched(c);
        compact_scan_blocks_kernel<<<1, COMPACT_SCAN_WORDS, 0, c->stream>>>(d_blk, (uint32_t)n_blocks);
        launched(c);
        CU(cudaGetLastError());
        const unsigned max_grid = (unsigned)c->prop.multiProcessorCount * 8;
        auto grid_for = [&](uint64_t items, uint64_t per_block) {
            return (unsigned)std::min<uint64_t>(max_grid, std::max<uint64_t>(1, (items + per_block - 1) / per_block));
        };
        auto dead_below = [&](uint64_t r) { return uint64_t(std::lower_bound(dead.begin(), dead.end(), r) - dead.begin()); };
        // Windows of source rows [a, b) in ascending order on one stream, starting at the first dead row (the rows
        // below it keep their place).  A window's live rows go to [dst, dst + live) with dst = a - dead_below(a) <= a
        // and live <= b - a, so the store ends at or below b: it overwrites only rows of this window, which the
        // gather before it has read in full, and rows of earlier windows, which have been stored already.  Nothing of
        // a later window is touched before its own gather reads it.
        auto move = [&](uint64_t w_rows, auto &&gather, auto &&store) -> int {
            for (uint64_t a = first; a < n; a += w_rows) {
                const uint64_t b = std::min(n, a + w_rows), below = dead_below(a), live = (b - a) - (dead_below(b) - below);
                if (!live) continue;
                gather(a, b, a - below);
                store(a - below, live);
                CU(cudaGetLastError());
            }
            return OC_OK;
        };
        auto move_rows = [&](void *rows, uint32_t esz) -> int {   // the matrix or its fp16 copy, same stride
            const uint64_t row_vec = uint64_t(e->stride) * esz / 16;
            return move(W,
                [&](uint64_t a, uint64_t b, uint64_t dst) {
                    const unsigned grid = grid_for(b - a, COMPACT_THREADS / 32);
                    if (esz == 2) compact_gather_kernel<2><<<grid, COMPACT_THREADS, 0, c->stream>>>(
                        rows, e->stride, a, b, dst, d_bits, d_pre, d_blk, c->cmp_stage.as<uint4>());
                    else compact_gather_kernel<4><<<grid, COMPACT_THREADS, 0, c->stream>>>(
                        rows, e->stride, a, b, dst, d_bits, d_pre, d_blk, c->cmp_stage.as<uint4>());
                    launched(c);
                },
                [&](uint64_t dst, uint64_t live) {
                    compact_store_kernel<<<grid_for(live * row_vec, COMPACT_THREADS * 4), COMPACT_THREADS, 0, c->stream>>>(
                        c->cmp_stage.as<uint4>(), static_cast<uint4 *>(rows) + dst * row_vec, live * row_vec);
                    launched(c);
                });
        };
        OCTRY(move_rows(e->rows, e->esz));
        if (e->f16) OCTRY(move_rows(e->rows_f16, 2));
        const uint64_t ws_rows = std::min<uint64_t>(Ws, n - first);
        uint64_t *st_doc = c->cmp_stage.as<uint64_t>();
        float *st_inv = reinterpret_cast<float *>(st_doc + ws_rows), *st_scale = e->f16 ? st_inv + ws_rows : nullptr;
        float *row_scale = e->f16 ? e->row_scale : nullptr;
        OCTRY(move(Ws,
            [&](uint64_t a, uint64_t b, uint64_t dst) {
                compact_small_gather_kernel<<<(unsigned)((b - a + COMPACT_THREADS - 1) / COMPACT_THREADS), COMPACT_THREADS, 0, c->stream>>>(
                    e->inv_norm, e->row_doc, row_scale, a, b, dst, d_bits, d_pre, d_blk, st_doc, st_inv, st_scale);
                launched(c);
            },
            [&](uint64_t dst, uint64_t live) {
                compact_small_store_kernel<<<(unsigned)((live + COMPACT_THREADS - 1) / COMPACT_THREADS), COMPACT_THREADS, 0, c->stream>>>(
                    st_doc, st_inv, st_scale, live, e->row_doc + dst, e->inv_norm + dst, row_scale ? row_scale + dst : nullptr);
                launched(c);
            }));
        CU(cudaEventRecord(c->ev[EV_DEV], c->stream));
        CU(cudaStreamSynchronize(c->stream));
        cudaEventElapsedTime(&st.device_ms, c->ev[EV_START], c->ev[EV_DEV]);
        for (auto &dr : e->doc_rows) dr.second -= dead_below(dr.second);
        st.rows_moved = e->n_live - first;
        e->n_rows = e->n_live;
        dead.clear();
        st.rows_after = e->n_rows;
    }
    if ((flags & OC_EMB_COMPACT_SHRINK) && e->cap > emb_round_cap(e->n_rows)) {
        if (e->n_rows == 0) {
            CU(cudaStreamSynchronize(c->stream));
            cudaFree(e->rows); cudaFree(e->inv_norm); cudaFree(e->row_doc); cudaFree(e->rows_f16); cudaFree(e->row_scale);
            e->rows = nullptr; e->inv_norm = nullptr; e->row_doc = nullptr; e->rows_f16 = nullptr; e->row_scale = nullptr;
            e->cap = 0;
        } else if (emb_realloc(e, emb_round_cap(e->n_rows), true) == OC_ERR_CUDA) {
            return OC_ERR_CUDA;   // (no room for the smaller allocation: the store stays compacted at its old capacity)
        }
        oc_emb_info(e, &inf);
        st.device_bytes_after = inf.device_bytes;
    }
    if (out) *out = st;
    return OC_OK;
}

// ---- scan launch plumbing
template <int NCH, int QB, typename T>
static int launch_scan_t(oc_ctx *c, const ScanParams &sp, uint32_t grid, size_t smem) {
    CU(smem_cfg(c->device, (const void *)emb_scan_kernel<NCH, QB, T>, smem));
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
// q_lim / q_sim: per-query depth and similarity (ScanMergeParams), or NULL
static int run_exact_sweeps(oc_ctx *c, oc_emb *e, const float *inv_norm, const float *qpad, const float *qinv,
                            uint32_t nq, uint32_t limit, float similarity, const VecOut &o,
                            const uint32_t *row_bits = nullptr, uint64_t row_words = 0, const uint32_t *q_slot = nullptr,
                            const uint32_t *q_lim = nullptr, const float *q_sim = nullptr) {
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
    mp.q_limit = q_lim; mp.q_sim = q_sim;
    CU(smem_cfg(c->device, (const void *)emb_scan_merge_kernel, size_t(mp.capb) * 8));
    emb_scan_merge_kernel<<<nq, 256, mp.capb * 8, c->stream>>>(mp);
    launched(c);
    CU(cudaGetLastError());
    return OC_OK;
}

// ---- TMA descriptors (tmap.cuh)
static int tmap_2d(CUtensorMap *m, const void *base, uint64_t n_rows, uint32_t stride, uint32_t box_rows, int op) {
    const TmapStatus s = make_tmap_2d(m, base, n_rows, stride, box_rows, op);
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
// qf: per-query where-filters (device tables uploaded), or NULL.  q_lim / q_sim: per-query depth (<= limit) and
// similarity, or NULL.
static int run_vector_stage(oc_ctx *c, oc_emb *e, const float *q_dev, uint32_t B, uint32_t limit, float similarity,
                            const uint64_t *filter_dev, uint64_t filter_nbits, const QFilterJob *qf = nullptr,
                            const uint32_t *q_lim = nullptr, const float *q_sim = nullptr) {
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
                                row_words, qf ? qf->d_q_slot : nullptr, q_lim, q_sim);

    // ---------------- K2: wgmma batched scan ----------------
    const bool bf16 = e->esz == 2;
    // an fp32 store is swept through its fp16 copy when it has one (GEMM_F16), else through tf32 on the fp32 rows
    const bool f16 = !bf16 && e->f16 && !env_emb_f16_off();
    const int op = bf16 ? GEMM_BF16 : f16 ? GEMM_F16 : GEMM_TF32;
    const void *sweep_fn = bf16  ? (const void *)emb_gemm_kernel<GEMM_BF16>
                           : f16 ? (const void *)emb_gemm_kernel<GEMM_F16>
                                 : (const void *)emb_gemm_kernel<GEMM_TF32>;
    CU(smem_cfg(c->device, sweep_fn, gemm_smem_bytes()));
    CU(smem_cfg(c->device, (const void *)emb_gemm_merge_kernel, gemm_merge_smem_bytes()));
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
    } else if (f16) {   // power-of-two scaled fp16 query; its scale turns eps into the sweep's units (gemm_thr_kernel)
        OCTRY(c->q_f16.ensure(size_t(Bpad) * e->stride * 2));
        OCTRY(c->q_scale.ensure(size_t(Bpad) * 4));
        emb_f16_queries_kernel<<<(Bpad + 7) / 8, 256, 0, c->stream>>>(c->q_pad.as<float>(), e->stride, Bpad, c->q_f16.as<uint16_t>(),
                                                                      c->q_scale.as<float>());
        launched(c);
        q_operand = c->q_f16.p;
    }
    OCTRY(tmap_2d(&tm_q, q_operand, Bpad, e->stride, GEMM_M, op));
    OCTRY(tmap_2d(&tm_x, f16 ? (const void *)e->rows_f16 : e->rows, e->n_rows, e->stride, GEMM_N / (paired ? GEMM_CLUSTER : 1),
                  op));   // a CTA's share of a tile
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
    gp.n_rows = e->n_rows; gp.n_kblocks = e->stride / (op == GEMM_TF32 ? GEMM_KB : 2 * GEMM_KB); gp.inv_norm = inv_norm; gp.n_queries = B;
    gp.n_qgroups = n_qgroups; gp.ctas_per_group = cpg; gp.cap = cap; gp.lists_per_query = lists;
    gp.thr = c->g_thr.as<unsigned int>(); gp.eps_v = c->g_eps.as<float>(); gp.limit = limit; gp.cand = c->g_cand.as<uint64_t>(); gp.cand_cnt = c->g_cnt.as<uint32_t>();
    gp.gmax = c->g_max.as<float>();
    gp.ovf = c->g_ovf.as<uint64_t>(); gp.ovf_cnt = c->g_ovfcnt.as<uint32_t>(); gp.ovf_cap = GEMM_OVF_CAP;
    if (qf) { gp.row_bits = row_bits; gp.row_words = row_words; gp.q_slot = qf->d_q_slot; }
    auto launch_gemm = [&]() -> int {
        if (bf16) CU(cudaLaunchKernelEx(&cfg, emb_gemm_kernel<GEMM_BF16>, tm_q, tm_x, gp));
        else if (f16) {
            GemmF16Params fp{};
            static_cast<GemmParams &>(fp) = gp;
            fp.row_scale = e->row_scale;
            CU(cudaLaunchKernelEx(&cfg, emb_gemm_kernel<GEMM_F16>, tm_q, tm_x, fp));
        }
        else CU(cudaLaunchKernelEx(&cfg, emb_gemm_kernel<GEMM_TF32>, tm_q, tm_x, gp));
        launched(c, gp.max_mode == 0);   // the one-tile threshold pass is not counted as a sweep
        CU(cudaGetLastError());
        return OC_OK;
    };
    // threshold pass: one row tile per CTA, record per-list maxima; thr = (limit-th largest maximum) - 2 eps
    gp.max_mode = 1; gp.tile_limit = 1;
    OCTRY(launch_gemm());
    GemmThrParams tp{};
    tp.gmax = c->g_max.as<float>(); tp.lists = lists; tp.limit = limit; tp.inv_qnorm = c->q_inv.as<float>();
    tp.eps_const = bf16 ? GEMM_EPS_ACC : f16 ? GEMM_EPS_F16 : GEMM_EPS_TF32;
    tp.rho_q = bf16 ? c->q_rho.as<float>() : nullptr;             // bf16 store: the rows are exact, the query is rounded
    tp.q_scale = f16 ? c->q_scale.as<float>() : nullptr;
    tp.thr = c->g_thr.as<unsigned int>(); tp.eps_v = c->g_eps.as<float>(); tp.ovf_cnt = c->g_ovfcnt.as<uint32_t>();
    gemm_thr_kernel<<<B, 256, 0, c->stream>>>(tp);
    launched(c);
    // the sweep
    gp.max_mode = 0; gp.tile_limit = 0;
    CU(cudaEventRecord(c->ev[EV_SWEEP0], c->stream));
    OCTRY(launch_gemm());
    CU(cudaEventRecord(c->ev[EV_SWEEP1], c->stream));
    c->sweep_timed = true;
    // the fp16 sweep reads the copy, the inverse norms and the row scales
    c->timing.scan_bytes += f16 ? e->n_rows * (uint64_t(e->stride) * 2 + 4 + 4) : e->n_rows * (uint64_t(e->stride) * e->esz + 4);
    CU(cudaEventRecord(c->ev[EV_SCAN1], c->stream));
    GemmMergeParams mp{};
    mp.cand = gp.cand; mp.cand_cnt = gp.cand_cnt; mp.n_lists = lists; mp.cap = cap; mp.limit = limit;
    mp.ovf = gp.ovf; mp.ovf_cnt = gp.ovf_cnt; mp.ovf_cap = gp.ovf_cap; mp.eps_v = tp.eps_v;
    mp.rows = e->rows; mp.rows_bf16 = bf16 ? 1 : 0; mp.stride = e->stride; mp.inv_norm = inv_norm; mp.queries = c->q_pad.as<float>();
    mp.inv_qnorm = c->q_inv.as<float>(); mp.row_doc_ids = e->row_doc; mp.rescale_e5 = e->e5; mp.similarity = similarity;
    mp.out_doc = out.doc; mp.out_score = out.score; mp.out_row = out.row; mp.out_count = out.cnt; mp.out_raw = out.raw;
    mp.out_unproven = c->g_flag.as<uint8_t>(); mp.out_rescored = c->g_resc.as<uint32_t>();
    mp.q_limit = q_lim; mp.q_sim = q_sim;
    emb_gemm_merge_kernel<<<B, 512, gemm_merge_smem_bytes(), c->stream>>>(mp);
    launched(c);
    CU(cudaGetLastError());
    // the overflow flags travel back with the results; oc_*search re-runs flagged queries (fix_unproven)
    c->gemm_pending = true; c->gemm_inv_norm = inv_norm;
    c->timing.scan_tensor_core = 1;
    c->timing.scan_variant = bf16 ? OC_SCAN_TC_BF16 : f16 ? OC_SCAN_TC_F16 : OC_SCAN_TC_TF32;
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
    // the slot a redone query's result goes to: its batch row (a sub-batch of per-query parameters scattered its hits there)
    std::vector<uint32_t> rmap(redo);
    if (!c->v_qmap.empty()) for (uint32_t &q : rmap) q = c->v_qmap[q];
    CU(cudaMemcpyAsync(c->r_map.p, rmap.data(), size_t(nr) * 4, cudaMemcpyHostToDevice, c->stream));
    std::vector<uint32_t> rslot;   // per-query where-filters: each redone query keeps its own slot
    if (c->v_rowbits) {
        for (uint32_t q : redo) rslot.push_back(c->v_qslot[q]);
        OCTRY(c->r_slot.ensure(size_t(nr) * 4));
        CU(cudaMemcpyAsync(c->r_slot.p, rslot.data(), size_t(nr) * 4, cudaMemcpyHostToDevice, c->stream));
    }
    std::vector<uint32_t> rlim;    // per-query parameters: each redone query keeps its own depth and similarity
    std::vector<float> rsim;
    if (!c->v_qlim.empty()) {
        for (uint32_t q : redo) { rlim.push_back(c->v_qlim[q]); rsim.push_back(c->v_qsim[q]); }
        OCTRY(c->r_lim.ensure(size_t(nr) * 4));
        OCTRY(c->r_sim.ensure(size_t(nr) * 4));
        CU(cudaMemcpyAsync(c->r_lim.p, rlim.data(), size_t(nr) * 4, cudaMemcpyHostToDevice, c->stream));
        CU(cudaMemcpyAsync(c->r_sim.p, rsim.data(), size_t(nr) * 4, cudaMemcpyHostToDevice, c->stream));
    }
    VecOut ro{c->r_doc.as<uint64_t>(), c->r_score.as<float>(), c->r_row.as<uint32_t>(), c->r_cnt.as<uint32_t>(), c->r_raw.as<float>()};
    OCTRY(run_exact_sweeps(c, e, inv_norm, c->r_qpad.as<float>(), c->r_qinv.as<float>(), nr, limit, similarity, ro, c->v_rowbits,
                           c->v_row_words, c->v_rowbits ? c->r_slot.as<uint32_t>() : nullptr,
                           rlim.empty() ? nullptr : c->r_lim.as<uint32_t>(), rsim.empty() ? nullptr : c->r_sim.as<float>()));
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
    c->v_qlim.clear(); c->v_qsim.clear(); c->v_qmap.clear();
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
// ctx lock (device merge on the store's own stream, str_commit.cuh) and publishes it with a pointer swap, so
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
};
// a process-wide identity per snapshot state: a new snapshot takes one, and so does every change made to a published
// snapshot in place (a field load, corpus-wide values, tombstones).  Keys the dense-array cache (dense_cache.h).
static uint64_t next_snap_ident() {
    static std::atomic<uint64_t> n{0};
    return ++n;
}
struct StrSnap {
    int device = 0;
    uint64_t version = 0;
    uint64_t ident = next_snap_ident();
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
    cudaEvent_t ev[4] = {};                          // oc_str_commit_ex: device time of its two device phases
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
    for (auto &e : s->ev) CU(cudaEventCreate(&e));
    *out = s;
    return OC_OK;
}
extern "C" void oc_str_destroy(oc_str *s) {
    if (!s) return;
    cudaSetDevice(s->ctx->device);
    cudaStreamSynchronize(s->ctx->stream);
    if (s->load_stream) { cudaStreamSynchronize(s->load_stream); cudaStreamDestroy(s->load_stream); }
    for (auto &e : s->ev) if (e) cudaEventDestroy(e);
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
    S.ident = next_snap_ident();
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
    // held for the whole load: a commit reads the published snapshot's posting arrays on the device, so it may
    // neither be running now nor start before this field is in place
    std::lock_guard<std::mutex> g2(s->mu);
    if (s->committing) return fail(OC_ERR_INVALID, "oc_str_load_field while a commit is in flight");
    StrSnap &S = *s->cur;
    if (field >= S.fields.size()) return fail(OC_ERR_INVALID, "field %u out of range", field);
    StrField &f = S.fields[field];
    S.ident = next_snap_ident();
    cudaFree(f.post); f.post = nullptr; cudaFree(f.raw); f.raw = nullptr; f.b_cached = -1.f;
    const uint64_t np = term_offsets[n_terms];
    if (np && (!post_row || !post_tf || !post_len)) return fail(OC_ERR_INVALID, "posting arrays are NULL");
    for (uint32_t t = 0; t < n_terms; t++) {
        if (term_offsets[t + 1] < term_offsets[t]) return fail(OC_ERR_INVALID, "term_offsets not monotone");
        if (term_offsets[t + 1] - term_offsets[t] > 0xffffffffull) return fail(OC_ERR_UNSUPPORTED, "posting list too long");
    }
    f.avg_len = avg_field_len; f.n_terms = n_terms; f.n_post = np;
    std::vector<PostingRaw> stage(np);   // interleaved for the upload only: the store keeps no host copy
    for (uint64_t i = 0; i < np; i++) {
        if (post_row[i] >= S.n_rows && S.n_rows) return fail(OC_ERR_INVALID, "posting row %u >= n_rows", post_row[i]);
        stage[i].row = post_row[i]; stage[i].tf = post_tf[i]; stage[i].len = post_len[i];
    }
    f.term_offsets.assign(term_offsets, term_offsets + n_terms + 1);
    f.global_df.clear();
    if (global_df) f.global_df.assign(global_df, global_df + n_terms);
    if (np) {
        CU(cudaMalloc(&f.post, (np + 4) * sizeof(Posting)));
        CU(cudaMalloc(&f.raw, (np + 4) * sizeof(PostingRaw)));
        CU(cudaMemcpyAsync(f.raw, stage.data(), np * sizeof(PostingRaw), cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    return OC_OK;
}

// tombstones `rows` of snapshot S (host bitmap + device copy on stream st)
static int snap_tombstone(StrSnap &S, const std::vector<uint64_t> &rows, cudaStream_t st) {
    if (rows.empty() || S.n_rows == 0) return OC_OK;
    S.ident = next_snap_ident();
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
// corpus-wide values), tombstones dropped.  The host filters the pending ops; the merge of the committed postings
// runs on the device (str_commit.cuh) on the store's own stream, reading the base snapshot's immutable arrays and
// the alive bitmap as it was when the commit started.  Everything is built in temporaries; the published snapshot
// is replaced only after every field validated and was built, so a failed commit changes nothing.
extern "C" int oc_str_commit(oc_str *s) { return oc_str_commit_ex(s, nullptr); }

extern "C" int oc_str_commit_ex(oc_str *s, oc_str_commit_t *out) {
    if (!s) return fail(OC_ERR_INVALID, "str is NULL");
    const auto wall0 = std::chrono::steady_clock::now();
    oc_ctx *c = s->ctx;
    std::shared_ptr<StrSnap> base;
    std::vector<std::vector<PendingPost>> pend;
    std::unordered_map<uint64_t, uint64_t> pdel;
    std::vector<uint32_t> base_alive;
    uint64_t base_deleted;
    bool global_avg;
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
        base_deleted = base->n_deleted;
        global_avg = s->global_avg;
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
    // ---- row space of the next snapshot, as far as the pending documents decide it (O(pending)): the new rows are
    // the alive old documents merged with the pending documents that are not one of them, ascending
    const uint64_t n_old = B.n_rows;
    auto old_doc = [&](uint64_t r) { return B.row_doc_host.empty() ? r : B.row_doc_host[r]; };
    auto old_alive = [&](uint64_t r) { return base_alive.empty() || ((base_alive[r >> 5] >> (r & 31)) & 1u); };
    std::vector<uint64_t> pdoc;
    for (auto &pv : pend) for (auto &pn : pv) pdoc.push_back(pn.doc);
    std::sort(pdoc.begin(), pdoc.end());
    pdoc.erase(std::unique(pdoc.begin(), pdoc.end()), pdoc.end());
    if (pdoc.size() > 0xfffffff0ull) return abort_commit(fail(OC_ERR_UNSUPPORTED, "more than 2^32 rows per store"));
    const uint32_t n_pdoc = (uint32_t)pdoc.size();
    std::vector<uint32_t> p_lbold(n_pdoc), p_newbelow(size_t(n_pdoc) + 1);
    uint32_t n_new_p = 0;
    for (uint32_t j = 0; j < n_pdoc; j++) {
        const uint64_t d = pdoc[j];
        const uint64_t lb = B.row_doc_host.empty() ? std::min(d, n_old)
                                                   : uint64_t(std::lower_bound(B.row_doc_host.begin(), B.row_doc_host.end(), d) - B.row_doc_host.begin());
        p_lbold[j] = (uint32_t)lb;
        p_newbelow[j] = n_new_p;
        if (!(lb < n_old && old_doc(lb) == d && old_alive(lb))) n_new_p++;
    }
    p_newbelow[n_pdoc] = n_new_p;
    const uint64_t n_new = (n_old - base_deleted) + n_new_p;
    if (n_new > 0xfffffff0ull) return abort_commit(fail(OC_ERR_UNSUPPORTED, "more than 2^32 rows per store"));
    uint64_t max_doc = n_pdoc ? pdoc.back() : 0;
    for (uint64_t r = n_old; r-- > 0;)
        if (old_alive(r)) { max_doc = std::max(max_doc, old_doc(r)); break; }
    const bool identity = n_new > 0 && max_doc == n_new - 1;   // n_new distinct ascending ids ending at n_new - 1

    // ---- the upload, packed: per-field result slots first (len sums, duplicate flags: their initial values), then
    // the row-space arrays and the per-field pending postings
    struct FieldPlan {
        uint32_t n_terms_old, n_terms, n_pend, n_repl, end_bit;
        size_t o_off, o_term, o_doc, o_tf, o_len, o_repl;              // in the upload
        size_t o_keep, o_kpre, o_kblk, o_keys, o_vals, o_newoff, o_tblk, o_slo, o_plo;   // in the workspace
        uint64_t n_kw, n_kb, n_tb;
    };
    struct FieldRes { unsigned long long len_sum, len_cnt; uint32_t dup, dup_term; };
    std::vector<FieldPlan> plan(nf);
    std::vector<uint8_t> up;
    auto put = [&](const void *src, size_t bytes) {
        const size_t o = up.size();
        up.resize(o + ((bytes + 15) & ~size_t(15)), 0);
        if (bytes) memcpy(up.data() + o, src, bytes);
        return o;
    };
    std::vector<FieldRes> res(nf, FieldRes{0, 0, 0, 0xffffffffu});
    const size_t o_res = put(res.data(), nf * sizeof(FieldRes));
    const size_t o_pdoc = put(pdoc.data(), pdoc.size() * 8), o_lbold = put(p_lbold.data(), p_lbold.size() * 4),
                 o_newbelow = put(p_newbelow.data(), p_newbelow.size() * 4);
    size_t o_alive = 0;
    const uint64_t n_aw = base_alive.empty() ? 0 : base_alive.size() + 1;   // + a zero word: alive_below(n_old) reads it
    if (n_aw) { base_alive.push_back(0); o_alive = put(base_alive.data(), n_aw * 4); }
    uint64_t pend_total = 0, post_before = 0;
    for (size_t fi = 0; fi < nf; fi++) {
        const StrField &of = B.fields[fi];
        FieldPlan &P = plan[fi];
        std::vector<uint32_t> term, doc, repl;
        std::vector<uint16_t> tf, len;
        uint32_t max_term = 0;
        for (size_t i = 0; i < pend[fi].size(); i++) {
            const PendingPost &pn = pend[fi][i];
            const uint32_t j = (uint32_t)(std::lower_bound(pdoc.begin(), pdoc.end(), pn.doc) - pdoc.begin());
            if (i == 0 || pn.doc != pend[fi][i - 1].doc) repl.push_back(j);   // one insert's postings are adjacent
            if (pn.term == 0xffffffffu) continue;
            term.push_back(pn.term); doc.push_back(j); tf.push_back(pn.tf); len.push_back(pn.len);
            max_term = std::max(max_term, pn.term);
        }
        P.n_terms_old = of.n_terms;
        P.n_pend = (uint32_t)term.size();
        P.n_repl = (uint32_t)repl.size();
        P.n_terms = P.n_pend ? std::max(of.n_terms, max_term + 1) : of.n_terms;
        int tb = 0;
        while (tb < 32 && (uint64_t(max_term) >> tb)) tb++;
        P.end_bit = 32 + tb;
        P.o_off = put(of.term_offsets.data(), of.n_terms ? (size_t(of.n_terms) + 1) * 8 : 0);
        P.o_term = put(term.data(), term.size() * 4); P.o_doc = put(doc.data(), doc.size() * 4);
        P.o_tf = put(tf.data(), tf.size() * 2); P.o_len = put(len.data(), len.size() * 2);
        P.o_repl = put(repl.data(), repl.size() * 4);
        pend_total += P.n_pend; post_before += of.n_post;
    }
    // ---- the workspace, one allocation: upload | alive scan | remap | prow | replaced bits | row keys | CUB temp |
    // per field: survivor bits + scan, sorted keys / values, term counts and offsets
    size_t ws = 0;
    auto take = [&](size_t bytes) { const size_t o = ws; ws += (bytes + 255) & ~size_t(255); return o; };
    const size_t w_up = take(up.size());
    const uint64_t n_ab = (n_aw + COMPACT_SCAN_WORDS - 1) / COMPACT_SCAN_WORDS;
    const size_t w_apre = take(n_aw * 4), w_ablk = take(n_ab * 4);
    const size_t w_remap = take(n_old * 4), w_prow = take(size_t(n_pdoc) * 4);
    const uint64_t n_rw = n_new / 32 + 1;
    const size_t w_repl = take(n_rw * 4);
    const size_t w_rowkey = take(global_avg ? 0 : n_new * 8);
    size_t cub_bytes = 0;
    for (size_t fi = 0; fi < nf; fi++) {
        FieldPlan &P = plan[fi];
        const uint64_t np = B.fields[fi].n_post;
        P.n_kw = np ? np / 32 + 1 : 0;
        P.n_kb = (P.n_kw + COMPACT_SCAN_WORDS - 1) / COMPACT_SCAN_WORDS;
        P.n_tb = P.n_terms ? (uint64_t(P.n_terms) + 1 + COMPACT_SCAN_WORDS - 1) / COMPACT_SCAN_WORDS : 0;
        P.o_keep = take(P.n_kw * 4); P.o_kpre = take(P.n_kw * 4); P.o_kblk = take(P.n_kb * 4);
        P.o_keys = take(size_t(P.n_pend) * 16); P.o_vals = take(size_t(P.n_pend) * 8);
        P.o_newoff = take(P.n_terms ? (size_t(P.n_terms) + 1) * 8 : 0); P.o_tblk = take(P.n_tb * 8);
        P.o_slo = take(size_t(P.n_terms) * 4); P.o_plo = take(P.n_terms ? (size_t(P.n_terms) + 1) * 4 : 0);
        if (P.n_pend) {
            size_t b = 0;
            if (cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const uint32_t *)nullptr,
                                                (uint32_t *)nullptr, P.n_pend, 0, P.end_bit, s->load_stream) != cudaSuccess)
                return abort_commit(fail(OC_ERR_CUDA, "DeviceRadixSort temp size"));
            cub_bytes = std::max(cub_bytes, b);
        }
    }
    const size_t w_cub = take(cub_bytes);
    auto ns = std::make_shared<StrSnap>();   // declared before wsp: on failure its arrays are freed after the stream is idle
    ns->device = c->device;
    ns->fields.resize(nf);
    ns->n_rows = n_new;
    ns->document_count = n_new;             // or the caller's N, taken at the swap below
    struct Workspace {   // every way out of the call waits for the load stream, then gives the workspace back
        oc_str *s; uint8_t *p = nullptr;
        ~Workspace() { cudaStreamSynchronize(s->load_stream); cudaFree(p); }
    } wsp{s};
    auto merge = [&]() -> int {
        CU(cudaMalloc(&wsp.p, std::max<size_t>(ws, 256)));
        uint8_t *W = wsp.p;
        auto at = [&](size_t o) { return static_cast<void *>(W + o); };
        const uint8_t *U = W + w_up;
        auto up_at = [&](size_t o) { return static_cast<const void *>(U + o); };
        FieldRes *d_res = (FieldRes *)(W + w_up + o_res);
        if (!identity && n_new) CU(cudaMalloc(&ns->row_doc, n_new * 8));
        cudaStream_t st = s->load_stream;
        const unsigned max_grid = (unsigned)c->prop.multiProcessorCount * 8;
        auto blocks = [](uint64_t n, uint64_t per) { return (unsigned)std::max<uint64_t>(1, (n + per - 1) / per); };
        CU(cudaEventRecord(s->ev[0], st));
        CU(cudaMemcpyAsync(W + w_up, up.data(), up.size(), cudaMemcpyHostToDevice, st));
        // 1. row space
        const uint32_t *alive = n_aw ? (const uint32_t *)up_at(o_alive) : nullptr;
        uint32_t *a_pre = (uint32_t *)at(w_apre), *a_blk = (uint32_t *)at(w_ablk);
        if (n_aw) {
            compact_scan_words_kernel<<<(unsigned)n_ab, COMPACT_SCAN_WORDS, 0, st>>>(alive, n_aw, a_pre, a_blk);
            compact_scan_blocks_kernel<uint32_t><<<1, COMPACT_SCAN_WORDS, 0, st>>>(a_blk, (uint32_t)n_ab);
        }
        uint32_t *remap = (uint32_t *)at(w_remap), *prow = (uint32_t *)at(w_prow);
        const uint64_t *d_pdoc = (const uint64_t *)up_at(o_pdoc);
        const uint32_t *d_lbold = (const uint32_t *)up_at(o_lbold), *d_newbelow = (const uint32_t *)up_at(o_newbelow);
        if (n_old)
            sc_old_rows_kernel<<<blocks(n_old, SC_THREADS), SC_THREADS, 0, st>>>(n_old, alive, a_pre, a_blk, B.row_doc, d_pdoc,
                                                                               n_pdoc, d_newbelow, remap, ns->row_doc);
        if (n_pdoc)
            sc_pending_rows_kernel<<<blocks(n_pdoc, SC_THREADS), SC_THREADS, 0, st>>>(n_pdoc, d_pdoc, d_lbold, d_newbelow, alive, a_pre,
                                                                                    a_blk, remap, prow, ns->row_doc);
        // 2-4. per field: survivors, sorted pending postings, new term offsets
        uint32_t *repl_bits = (uint32_t *)at(w_repl);
        for (size_t fi = 0; fi < nf; fi++) {
            const FieldPlan &P = plan[fi];
            const StrField &of = B.fields[fi];
            StrField &f = ns->fields[fi];
            f.n_terms = P.n_terms;
            f.term_offsets.assign(size_t(P.n_terms) + 1, 0);
            CU(cudaMemsetAsync(repl_bits, 0, n_rw * 4, st));
            if (P.n_repl)
                sc_replaced_kernel<<<blocks(P.n_repl, SC_THREADS), SC_THREADS, 0, st>>>(P.n_repl, (const uint32_t *)up_at(P.o_repl),
                                                                                      prow, repl_bits);
            uint32_t *keep = (uint32_t *)at(P.o_keep), *kpre = (uint32_t *)at(P.o_kpre), *kblk = (uint32_t *)at(P.o_kblk);
            if (P.n_kw) {
                sc_survive_kernel<<<blocks(P.n_kw * 32, SC_THREADS), SC_THREADS, 0, st>>>(of.n_post, P.n_kw, of.raw, n_old, remap, repl_bits, keep);
                compact_scan_words_kernel<<<(unsigned)P.n_kb, COMPACT_SCAN_WORDS, 0, st>>>(keep, P.n_kw, kpre, kblk);
                compact_scan_blocks_kernel<uint32_t><<<1, COMPACT_SCAN_WORDS, 0, st>>>(kblk, (uint32_t)P.n_kb);
            }
            uint64_t *keys = (uint64_t *)at(P.o_keys);
            uint32_t *vals = (uint32_t *)at(P.o_vals);
            if (P.n_pend) {
                sc_pending_keys_kernel<<<blocks(P.n_pend, SC_THREADS), SC_THREADS, 0, st>>>(
                    P.n_pend, (const uint32_t *)up_at(P.o_term), (const uint32_t *)up_at(P.o_doc), prow, keys + P.n_pend, vals + P.n_pend);
                size_t b = cub_bytes;
                CU(cub::DeviceRadixSort::SortPairs(at(w_cub), b, keys + P.n_pend, keys, vals + P.n_pend, vals, P.n_pend, 0,
                                                   (int)P.end_bit, st));
                sc_duplicate_kernel<<<blocks(P.n_pend, SC_THREADS), SC_THREADS, 0, st>>>(P.n_pend, keys, &d_res[fi].dup);
            }
            if (P.n_terms) {
                uint64_t *new_off = (uint64_t *)at(P.o_newoff), *tblk = (uint64_t *)at(P.o_tblk);
                sc_term_counts_kernel<<<(unsigned)P.n_tb, COMPACT_SCAN_WORDS, 0, st>>>(
                    P.n_terms, of.n_post ? P.n_terms_old : 0, (const uint64_t *)up_at(P.o_off), keep, kpre, kblk, keys, P.n_pend,
                    (uint32_t *)at(P.o_slo), (uint32_t *)at(P.o_plo), new_off, tblk);
                compact_scan_blocks_kernel<uint64_t><<<1, COMPACT_SCAN_WORDS, 0, st>>>(tblk, (uint32_t)P.n_tb);
                sc_add_block_kernel<<<blocks(uint64_t(P.n_terms) + 1, SC_THREADS), SC_THREADS, 0, st>>>(P.n_terms + 1, tblk, new_off);
                CU(cudaMemcpyAsync(f.term_offsets.data(), new_off, (size_t(P.n_terms) + 1) * 8, cudaMemcpyDeviceToHost, st));
            }
        }
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(res.data(), d_res, nf * sizeof(FieldRes), cudaMemcpyDeviceToHost, st));
        CU(cudaEventRecord(s->ev[1], st));
        CU(cudaStreamSynchronize(st));
        for (size_t fi = 0; fi < nf; fi++)
            if (res[fi].dup) return fail(OC_ERR_INVALID, "field %zu: term %u listed twice in one insert of a document", fi, res[fi].dup_term);
        // 5. the new posting arrays at their exact size, and the scatter-merge into them
        for (size_t fi = 0; fi < nf; fi++) {
            StrField &f = ns->fields[fi];
            f.n_post = f.term_offsets.back();
            if (!f.n_post) continue;
            CU(cudaMalloc(&f.post, (f.n_post + 4) * sizeof(Posting)));
            CU(cudaMalloc(&f.raw, (f.n_post + 4) * sizeof(PostingRaw)));
        }
        CU(cudaEventRecord(s->ev[2], st));
        unsigned long long *row_key = global_avg ? nullptr : (unsigned long long *)at(w_rowkey);
        for (size_t fi = 0; fi < nf; fi++) {
            const FieldPlan &P = plan[fi];
            const StrField &of = B.fields[fi];
            StrField &f = ns->fields[fi];
            if (!f.n_post) continue;
            if (row_key) CU(cudaMemsetAsync(row_key, 0, n_new * 8, st));
            const uint32_t *keep = (const uint32_t *)at(P.o_keep), *kpre = (const uint32_t *)at(P.o_kpre), *kblk = (const uint32_t *)at(P.o_kblk);
            const uint64_t *old_off = (const uint64_t *)up_at(P.o_off), *new_off = (const uint64_t *)at(P.o_newoff), *keys = (const uint64_t *)at(P.o_keys);
            const uint32_t *slo = (const uint32_t *)at(P.o_slo), *plo = (const uint32_t *)at(P.o_plo);
            if (of.n_post)
                sc_scatter_old_kernel<<<blocks(of.n_post, SC_TILE), SC_THREADS, 0, st>>>(of.n_post, of.raw, remap, keep, kpre, kblk,
                                                                                       P.n_terms_old, old_off, new_off, slo, plo, keys, f.raw, row_key);
            if (P.n_pend)
                sc_scatter_pending_kernel<<<blocks(P.n_pend, SC_THREADS), SC_THREADS, 0, st>>>(
                    P.n_pend, keys, (const uint32_t *)at(P.o_vals), (const uint32_t *)up_at(P.o_doc), (const uint16_t *)up_at(P.o_tf),
                    (const uint16_t *)up_at(P.o_len), d_lbold, of.raw, of.n_post ? P.n_terms_old : 0, old_off, keep, kpre, kblk, new_off, slo, plo, f.raw, row_key);
            if (row_key)
                sc_len_sum_kernel<<<(unsigned)std::min<uint64_t>(max_grid, blocks(n_new, SC_THREADS)), SC_THREADS, 0, st>>>(
                    (uint32_t)n_new, row_key, &d_res[fi].len_sum);
        }
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(res.data(), d_res, nf * sizeof(FieldRes), cudaMemcpyDeviceToHost, st));
        if (ns->row_doc) {
            ns->row_doc_host.resize(n_new);
            CU(cudaMemcpyAsync(ns->row_doc_host.data(), ns->row_doc, n_new * 8, cudaMemcpyDeviceToHost, st));
        }
        CU(cudaEventRecord(s->ev[3], st));
        CU(cudaStreamSynchronize(st));
        return OC_OK;
    };
    const int mrc = merge();
    if (mrc != OC_OK) return abort_commit(mrc);
    uint64_t post_after = 0;
    for (size_t fi = 0; fi < nf; fi++) {
        StrField &f = ns->fields[fi];
        f.avg_len = B.fields[fi].avg_len;
        if (!global_avg && res[fi].len_cnt) f.avg_len = (float)((double)res[fi].len_sum / (double)res[fi].len_cnt);   // info().avg_field_length
        post_after += f.n_post;
        // per-term corpus df of a shard cannot be refreshed locally: sharded searches on this snapshot count
        // df across ranks (OC_SHARD_COUNT_DF) until the caller loads new global tables
    }
    if (out) {
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, s->ev[0], s->ev[1]);
        cudaEventElapsedTime(&b, s->ev[2], s->ev[3]);
        *out = oc_str_commit_t{};
        out->rows_before = n_old; out->rows_after = n_new;
        out->postings_before = post_before; out->postings_after = post_after;
        out->pending_postings = pend_total;
        out->workspace_bytes = ws;
        out->device_ms = a + b;
    }
    // ---- publish: replay the deletes that arrived while we were building, then swap the pointer
    {
        std::lock_guard<std::mutex> g(s->mu);
        std::vector<uint64_t> rows;
        for (uint64_t d : s->deletes_during_commit) { const uint64_t r = ns->row_of(d); if (r != ~0ull) rows.push_back(r); }
        const int trc = snap_tombstone(*ns, rows, s->load_stream);
        if (trc != OC_OK) { s->committing = false; return trc; }   // (pending ops were consumed; the old snapshot stays published)
        // the corpus-wide values the caller owns are taken now, not when the commit started, so that an
        // oc_str_set_global made while the merge ran is not lost with the old snapshot.  They are on `cur`: while a
        // commit is in flight only oc_str_set_global and tombstones change it (set_rows / load_field are refused).
        if (s->global_count) ns->document_count = s->cur->document_count;
        if (s->global_avg)
            for (size_t fi = 0; fi < nf; fi++) ns->fields[fi].avg_len = s->cur->fields[fi].avg_len;
        ns->version = ++s->version;
        s->cur = ns;
        s->deletes_during_commit.clear();
        s->committing = false;
    }
    if (out) out->wall_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    return OC_OK;
}

// Read-back of the published snapshot (the inverse of oc_str_set_rows + oc_str_load_field).
extern "C" int oc_str_read_rows(oc_str *s, uint64_t *n_rows, uint64_t *row_doc_ids, uint64_t *document_count, uint64_t *version) {
    if (!s || !n_rows) return fail(OC_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> g(s->mu);
    const StrSnap &S = *s->cur;
    const uint64_t cap = *n_rows;
    *n_rows = S.n_rows;
    if (document_count) *document_count = S.document_count;
    if (version) *version = S.version;
    if (!row_doc_ids) return OC_OK;
    if (cap < S.n_rows) return fail(OC_ERR_INVALID, "row_doc_ids holds %llu rows, the snapshot has %llu",
                                    (unsigned long long)cap, (unsigned long long)S.n_rows);
    if (S.row_doc_host.empty()) for (uint64_t r = 0; r < S.n_rows; r++) row_doc_ids[r] = r;
    else std::copy(S.row_doc_host.begin(), S.row_doc_host.end(), row_doc_ids);
    return OC_OK;
}

extern "C" int oc_str_read_field(oc_str *s, uint32_t field, float *avg_field_len, uint32_t *n_terms, uint64_t *n_postings,
                                 uint64_t *term_offsets, uint32_t *post_row, uint16_t *post_tf, uint16_t *post_len) {
    if (!s || !n_terms || !n_postings) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = s->ctx;
    std::lock_guard<std::mutex> g(c->mu);   // oc_str_load_field replaces a published field's arrays under this lock
    CU(cudaSetDevice(c->device));
    std::shared_ptr<StrSnap> snap = str_snapshot(s);
    if (field >= snap->fields.size()) return fail(OC_ERR_INVALID, "field %u out of range", field);
    const StrField &f = snap->fields[field];
    const uint32_t cap_t = *n_terms;
    const uint64_t cap_p = *n_postings;
    *n_terms = f.n_terms; *n_postings = f.n_post;
    if (avg_field_len) *avg_field_len = f.avg_len;
    if ((term_offsets && cap_t < f.n_terms) || ((post_row || post_tf || post_len) && cap_p < f.n_post))
        return fail(OC_ERR_INVALID, "arrays too small for field %u (%u terms, %llu postings)", field, f.n_terms,
                    (unsigned long long)f.n_post);
    if (term_offsets) {
        if (f.term_offsets.empty()) term_offsets[0] = 0;
        else std::copy(f.term_offsets.begin(), f.term_offsets.end(), term_offsets);
    }
    if ((post_row || post_tf || post_len) && f.n_post) {
        std::vector<PostingRaw> h(f.n_post);
        CU(cudaMemcpyAsync(h.data(), f.raw, f.n_post * sizeof(PostingRaw), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        for (uint64_t i = 0; i < f.n_post; i++) {
            if (post_row) post_row[i] = h[i].row;
            if (post_tf) post_tf[i] = h[i].tf;
            if (post_len) post_len[i] = h[i].len;
        }
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

// The corpus-wide df tables and averages of a sharded store, rebuilt by a collective over the ctx's comm group (see the
// header for the steps).  Every rank decides from gathered facts only, so all ranks return the same code and call the
// same collectives.  The installed values change host fields of the snapshot a commit in flight may be reading as its
// base: the df table (no commit reads it), avg_len (as oc_str_set_global does) and the identity; never term_offsets.
extern "C" int oc_str_sync_global(oc_str *s, oc_str_sync_t *out) {
    if (!s) return fail(OC_ERR_INVALID, "str is NULL");
    const auto wall0 = std::chrono::steady_clock::now();
    oc_ctx *c = s->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    if (!c->comm.comm && !c->comm.local) return fail(OC_ERR_COMM, "oc_str_sync_global without oc_comm_init");
    const int W = c->comm.world;
    std::shared_ptr<StrSnap> snap = str_snapshot(s);
    const StrSnap &S = *snap;
    const uint32_t nf = (uint32_t)S.fields.size();
    std::string err;
    auto gather = [&](const void *mine, void *all, size_t bytes) -> int {   // through c->sync_buf: [send | W recv]
        uint8_t *d = c->sync_buf.as<uint8_t>();
        CU(cudaMemcpyAsync(d, mine, bytes, cudaMemcpyHostToDevice, c->stream));
        if (!c->comm.all_gather(d, d + bytes, bytes, c->stream, &err)) return fail(OC_ERR_COMM, "%s", err.c_str());
        CU(cudaMemcpyAsync(all, d + bytes, bytes * W, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        return OC_OK;
    };
    // 1. handshake: the exchange buffer is sized for the largest of the three gathers at this rank's n_fields (a rank
    // with another n_fields leaves after the handshake, before the gathers that depend on it)
    struct Hdr { uint32_t n_fields, pad; uint64_t rows, version; };
    const size_t max_bytes = std::max<size_t>(sizeof(Hdr), 8 + size_t(nf) * 16);
    CU(cudaSetDevice(c->device));
    OCTRY(c->sync_buf.ensure(max_bytes * (W + 1)));
    Hdr me{nf, 0, S.n_rows, S.version};
    std::vector<Hdr> hdr(W);
    OCTRY(gather(&me, hdr.data(), sizeof(Hdr)));
    uint64_t rows_global = 0;
    bool same_nf = true;
    for (int r = 0; r < W; r++) {
        same_nf = same_nf && hdr[r].n_fields == nf;
        rows_global += hdr[r].rows;
    }
    if (!same_nf) return fail(OC_ERR_INVALID, "oc_str_sync_global: the ranks' stores have different numbers of fields");
    if (rows_global > 0xffffffffull) return fail(OC_ERR_INVALID, "oc_str_sync_global: %llu rows in all: df is 32-bit",
                                                 (unsigned long long)rows_global);
    // 2. term spaces
    std::vector<uint32_t> nt(nf), nt_all(size_t(W) * nf);
    for (uint32_t fi = 0; fi < nf; fi++) nt[fi] = S.fields[fi].n_terms;
    if (nf) OCTRY(gather(nt.data(), nt_all.data(), size_t(nf) * 4));
    std::vector<uint64_t> df_off(size_t(nf) + 1, 0);   // field fi's table in the df buffer
    for (uint32_t fi = 0; fi < nf; fi++) {
        uint32_t t = 0;
        for (int r = 0; r < W; r++) t = std::max(t, nt_all[size_t(r) * nf + fi]);
        df_off[fi + 1] = df_off[fi] + t;
    }
    const uint64_t n_df = df_off[nf];
    // 3. this rank's list lengths and length sums; the status of this part travels with the sums
    struct Pair { unsigned long long len_sum, len_cnt; };
    std::vector<uint32_t> df(n_df, 0);
    for (uint32_t fi = 0; fi < nf; fi++) {
        const StrField &f = S.fields[fi];
        for (uint32_t t = 0; t < f.n_terms; t++) df[df_off[fi] + t] = (uint32_t)(f.term_offsets[t + 1] - f.term_offsets[t]);
    }
    std::vector<uint8_t> mine(8 + size_t(nf) * 16, 0);   // {status, pad, Pair[nf]}
    Pair *pairs = reinterpret_cast<Pair *>(mine.data() + 8);
    uint8_t *ws = nullptr;   // [df u32 x n_df | Pair x nf | row lengths u64 x n_rows]
    struct Free { uint8_t *&p; oc_ctx *c; ~Free() { if (p) { cudaStreamSynchronize(c->stream); cudaFree(p); } } } wfree{ws, c};
    const size_t o_pair = (n_df * 4 + 255) & ~size_t(255), o_row = o_pair + ((size_t(nf) * 16 + 255) & ~size_t(255));
    auto local = [&]() -> int {
        CU(cudaMalloc(&ws, o_row + S.n_rows * 8 + 8));
        unsigned long long *d_pair = reinterpret_cast<unsigned long long *>(ws + o_pair), *row_key = reinterpret_cast<unsigned long long *>(ws + o_row);
        CU(cudaEventRecord(c->ev[EV_BM0], c->stream));
        if (n_df) CU(cudaMemcpyAsync(ws, df.data(), n_df * 4, cudaMemcpyHostToDevice, c->stream));
        CU(cudaMemsetAsync(d_pair, 0, size_t(nf) * 16, c->stream));
        const unsigned max_grid = (unsigned)c->prop.multiProcessorCount * 8;
        auto blocks = [&](uint64_t n) { return (unsigned)std::min<uint64_t>(max_grid, std::max<uint64_t>(1, (n + SC_THREADS - 1) / SC_THREADS)); };
        for (uint32_t fi = 0; fi < nf; fi++) {
            const StrField &f = S.fields[fi];
            if (!f.n_post || !S.n_rows) continue;
            CU(cudaMemsetAsync(row_key, 0, S.n_rows * 8, c->stream));
            sc_row_len_kernel<<<blocks(f.n_post), SC_THREADS, 0, c->stream>>>(f.n_post, f.raw, row_key);
            sc_len_sum_kernel<<<blocks(S.n_rows), SC_THREADS, 0, c->stream>>>((uint32_t)S.n_rows, row_key, d_pair + 2 * fi);
            launched(c); launched(c);
        }
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(pairs, d_pair, size_t(nf) * 16, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaEventRecord(c->ev[EV_BM1], c->stream));
        CU(cudaStreamSynchronize(c->stream));
        return OC_OK;
    };
    const int32_t st = local();
    const std::string local_err = st == OC_OK ? "" : oc_last_error();
    memcpy(mine.data(), &st, 4);
    // 4. collectives: the statuses and sums first, so that a failed rank stops every rank before the all-reduce
    std::vector<uint8_t> all(mine.size() * W);
    OCTRY(gather(mine.data(), all.data(), mine.size()));
    std::vector<Pair> tot(nf, Pair{0, 0});
    for (int r = 0; r < W; r++) {
        int32_t rs;
        memcpy(&rs, all.data() + r * mine.size(), 4);
        if (rs != OC_OK) return fail(rs, "oc_str_sync_global: rank %d: %s", r, r == c->comm.rank ? local_err.c_str() : "its device work failed");
        const Pair *pr = reinterpret_cast<const Pair *>(all.data() + r * mine.size() + 8);
        for (uint32_t fi = 0; fi < nf; fi++) { tot[fi].len_sum += pr[fi].len_sum; tot[fi].len_cnt += pr[fi].len_cnt; }
    }
    CU(cudaEventRecord(c->ev[EV_COMM0], c->stream));
    if (n_df) {
        if (!c->comm.all_reduce_sum_u32(ws, ws, n_df, c->stream, &err)) return fail(OC_ERR_COMM, "%s", err.c_str());
        CU(cudaMemcpyAsync(df.data(), ws, n_df * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaEventRecord(c->ev[EV_COMM1], c->stream));
    CU(cudaStreamSynchronize(c->stream));
    // 5. install
    {
        std::lock_guard<std::mutex> g2(s->mu);
        StrSnap &D = *snap;
        D.ident = next_snap_ident();
        for (uint32_t fi = 0; fi < nf; fi++) {
            StrField &f = D.fields[fi];
            f.global_df.assign(df.begin() + df_off[fi], df.begin() + df_off[fi + 1]);
            if (!tot[fi].len_cnt) continue;
            const float avg = (float)((double)tot[fi].len_sum / (double)tot[fi].len_cnt);   // as oc_str_commit_ex
            if (f.avg_len != avg) { f.avg_len = avg; f.b_cached = -1.f; }
        }
    }
    if (out) {
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, c->ev[EV_BM0], c->ev[EV_BM1]);
        cudaEventElapsedTime(&b, c->ev[EV_COMM0], c->ev[EV_COMM1]);
        *out = oc_str_sync_t{};
        out->version = S.version;
        out->rows_global = rows_global;
        out->bytes_reduced = n_df * 4 + uint64_t(nf) * 16;
        out->device_ms = a + b;
        out->wall_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    }
    return OC_OK;
}

extern "C" int oc_str_read_global_df(oc_str *s, uint32_t field, uint32_t *n_terms, uint32_t *df) {
    if (!s || !n_terms) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = s->ctx;
    std::lock_guard<std::mutex> g(c->mu);   // oc_str_sync_global / oc_str_load_field replace a table under this lock
    std::shared_ptr<StrSnap> snap = str_snapshot(s);
    if (field >= snap->fields.size()) return fail(OC_ERR_INVALID, "field %u out of range", field);
    const std::vector<uint32_t> &t = snap->fields[field].global_df;
    const uint32_t cap = *n_terms;
    *n_terms = (uint32_t)t.size();
    if (!df) return OC_OK;
    if (cap < t.size()) return fail(OC_ERR_INVALID, "df holds %u entries, the table has %zu", cap, t.size());
    std::copy(t.begin(), t.end(), df);
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
extern "C" int oc_filter_nbits(const oc_filter *f, uint64_t *out) {
    if (!f || !out) return fail(OC_ERR_INVALID, "NULL argument");
    *out = f->nbits;
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
    CU(smem_cfg(c->device, (const void *)bm25_tile_kernel<MULTI, THRESH, OMC, ROWFT>, smem));
    bm25_tile_kernel<MULTI, THRESH, OMC, ROWFT><<<grid, BM25_THREADS, smem, st>>>(bp);
    launched(c);
    CU(cudaGetLastError());
    return OC_OK;
}
// The grid of a persistent scorer launch, whose blocks pull (tile, query) items from a counter: one block per
// items_per_block items, but no more blocks than the device holds at once.  Occupancy is queried once per
// (device, kernel, block size, shared memory).
static cudaError_t persistent_grid(oc_ctx *c, const void *fn, int threads, size_t smem, uint32_t items_per_block,
                                   uint64_t items, uint32_t *grid) {
    static std::mutex mu;
    static std::map<std::tuple<int, const void *, int, size_t>, int> occ;
    const auto key = std::make_tuple(c->device, fn, threads, smem);
    int per_sm = 1;
    {
        std::lock_guard<std::mutex> g(mu);
        auto it = occ.find(key);
        if (it == occ.end()) {
            const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, smem);
            if (e != cudaSuccess) return e;
            occ[key] = per_sm;
        } else per_sm = it->second;
    }
    *grid = (uint32_t)std::min<uint64_t>((items + items_per_block - 1) / items_per_block,
                                         uint64_t(std::max(per_sm, 1)) * c->prop.multiProcessorCount);
    return cudaSuccess;
}
template <bool THRESH, bool OMC, bool ROWFT>
static int launch_tile2_t(oc_ctx *c, const Bm25Params &bp, size_t smem, cudaStream_t st, const ItemTok *flat, unsigned int *counter) {
    const void *fn = (const void *)bm25_tile2_kernel<THRESH, OMC, ROWFT>;
    CU(smem_cfg(c->device, fn, smem));
    uint32_t grid;
    CU(persistent_grid(c, fn, BM25_THREADS, smem, 1, uint64_t(bp.n_tiles) * bp.n_queries, &grid));
    bm25_tile2_kernel<THRESH, OMC, ROWFT><<<grid, BM25_THREADS, smem, st>>>(bp, flat, counter);
    launched(c);
    CU(cudaGetLastError());
    return OC_OK;
}
// multi == false (every token resolves to <= 1 term): the posting-centred persistent kernel; else the slot-scan kernel
static int launch_tile(oc_ctx *c, const Bm25Params &bp, uint32_t grid, bool multi, bool thr, bool omc, cudaStream_t st,
                       uint32_t max_tokens, unsigned int *counter /* zeroed by the caller */, bool counted_df) {
    const char *env = getenv("OC_BM25_TILE2");
    if (!multi && !(env && env[0] == '0')) {
        // one level of descriptors per (tile, query) item, prefetched by the kernel during the previous item
        const ItemTok *flat = nullptr;
        const char *t3e = getenv("OC_BM25_TILE3");
        const bool can_flat = max_tokens <= BM25_FLAT_TOK;
        // counted_df (filter / tombstones / OC_SHARD_COUNT_DF): no token has a host-known idf, so nothing is shared or dense
        // and every hot term arrives as a long posting list — the accumulator kernel walks those at ~10 instructions per
        // posting, the register-folded scorers would fold each posting's row separately
        const bool use3 = can_flat && !thr && !omc && !counted_df && !bp.matched_bits && !(t3e && t3e[0] == '0');
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
            const uint64_t items = uint64_t(bp.n_tiles) * bp.n_queries;
            const char *seed_env = getenv("OC_BM25_SEED");
            if (bp.n_keep <= 32 && bp.n_tiles > 1 && !(seed_env && seed_env[0] == '0')) {   // warm start of the candidate thresholds
                bm25_seed_kernel<<<(bp.n_queries * 32 + 255) / 256, 256, 0, st>>>(bp);
                launched(c);
            }
            const char *wenv = getenv("OC_BM25_WARP");
            if (bp.n_keep <= 32 && !(wenv && wenv[0] == '0')) {   // a warp per item: no block barriers
                const size_t smemw = size_t(BW_WARPS) * sizeof(WarpScratch);
                CU(smem_cfg(c->device, (const void *)bm25_warp_kernel, smemw));
                uint32_t gw;
                CU(persistent_grid(c, (const void *)bm25_warp_kernel, BW_WARPS * 32, smemw, BW_WARPS, items, &gw));
                bm25_warp_kernel<<<gw, BW_WARPS * 32, smemw, st>>>(bp, flat, counter);
                launched(c);
                CU(cudaGetLastError());
                return OC_OK;
            }
            const size_t smem3 = bm25_tile3_smem_bytes(bp.cap);
            CU(smem_cfg(c->device, (const void *)bm25_tile3_kernel, smem3));
            uint32_t g3;
            CU(persistent_grid(c, (const void *)bm25_tile3_kernel, BM25_THREADS, smem3, 1, items, &g3));
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

// The facet counts of one search: count k is the number of documents of request reqs[r[k]] that are keys of query
// q[k]'s score map, written to out_counts[o[k]].  oc_search_facets asks every query for the same list.
struct FacetJob {
    oc_facets *fc = nullptr;
    const oc_facet_req *reqs = nullptr;
    std::vector<uint32_t> q, r;
    std::vector<size_t> o;
    uint64_t *out_counts = nullptr;
    const uint32_t *q_off = nullptr;   // oc_search_q_facets: its q_facet_offsets (a query with facets may run at limit 0)
    bool hits_optional = false;        // limit 0 allowed: the hits are not written, the vector stage runs at depth 0
    unsigned long long *d_out = nullptr;   // oc_search_indexes_ex: device counts at o[k], added to in place (the indexes'
                                           // counts sum there): no zeroing, no copy, no synchronise
};
struct FacetSliceDev {   // one distinct document slice and the counts that want it
    const uint64_t *docs;
    uint64_t n;
    uint32_t block0;                   // its first block: it takes ceil(n / 1024) blocks
    uint32_t pair0, n_pairs;           // its (bitmap row, count) pairs
};
struct FacetPlan {
    std::vector<FacetSliceDev> slices;
    std::vector<uint2> pairs;          // (bitmap row, count index k)
    uint32_t n_blocks = 0;
    const FacetSliceDev *d_slices = nullptr;
    const uint2 *d_pairs = nullptr;
};
static int facet_plan(const FacetJob &fj, FacetPlan &pl);
static int run_facets(oc_ctx *c, const FacetJob &fj, const FacetPlan &pl, uint32_t B, bool has_ft, bool has_v, const StrSnap *S,
                      uint32_t n_tiles, uint32_t vlimit);
// A groupBy handle: the CSR of its groups, built once by oc_group_by_create (below).
struct oc_group_by {
    oc_ctx *ctx;
    uint32_t n_groups = 0;
    uint64_t n_docs = 0;           // entries of the CSR (a document counts once per group it belongs to)
    uint64_t *off = nullptr;       // device [n_groups + 1]
    uint64_t *docs = nullptr;      // device [n_docs]
    uint32_t *rows = nullptr;      // device [n_docs + 1]: string row of each entry, filled per call; rows[n_docs] = ~0
};
// The grouped calls: per query its oc_group_by (or none) and max_results.  Query q's groups are the output rows
// [q_row[q], q_row[q] + n_groups), each of `stride` entries.
constexpr uint32_t GROUP_NONE = 0xffffffffu;
struct GroupJob {
    std::vector<oc_group_by *> h;           // the batch's distinct handles
    std::vector<uint32_t> q_h;              // [B] index into h, GROUP_NONE: no groups
    std::vector<uint32_t> q_m;              // [B] max_results
    std::vector<uint32_t> q_row;            // [B]
    uint32_t rows = 0;                      // sum of the queries' n_groups
    uint32_t stride = 0;
    uint64_t *out_doc = nullptr;            // [rows][stride]
    float *out_score = nullptr;
    uint32_t *out_n = nullptr;              // [rows]
    double *out_values = nullptr;           // [rows][stride] sort values, may be NULL
    // the work list (set by search_impl): spans of the score-order queries first, then those in field order
    uint32_t n_spans = 0, n_score_spans = 0, n_score_items = 0, top = 0;
    bool direct = false;                    // no splice and every depth == stride: the top lists are the outputs
    const GroupHandle *d_hand = nullptr;
    const GroupSpan *d_spans = nullptr;
    const SortEntry *d_ents = nullptr;
    // oc_search_indexes_ex: the top lists stay on the device (c->grp_*, row stride top) for the group merge, with no splice
    // and no copy; q_deep[q] gives query q depth 2 x max_results without a splice (an active pinned query of the merge)
    bool keep_top = false;
    std::vector<uint8_t> q_deep;
};
struct PinJob {   // oc_search_pinned / oc_search_groups_pinned: the promote items, padded to `stride` slots per query
    const oc_pins *pins = nullptr;      // the caller's items (NULL: none)
    float *out_scores = nullptr;        // per item of pins: its score-map value and presence (each may be NULL)
    uint8_t *out_present = nullptr;
    uint32_t stride = 0;                // most items of one query (0: no item in the batch)
    bool splice = false;                // pins apply and some query has items: top lists at twice the depth + the splice
    std::vector<uint64_t> doc;          // [B][stride]
    std::vector<uint32_t> pos, cnt;     // [B][stride], [B]
    const uint64_t *d_doc = nullptr;    // their device copies (set by search_impl)
    const uint32_t *d_pos = nullptr, *d_cnt = nullptr;
};
// Checks and pads the items of pins (NULL: none).  Nothing is written on failure.
static int pin_job_init(const oc_pins *pins, uint32_t B, PinJob &pj) {
    pj.pins = pins;
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
    double *rank_value = nullptr;          // device [n]: h_value, built by the first oc_search_indexes that needs it
};
struct oc_sort_field {
    oc_ctx *ctx;
    uint64_t nbits;
    uint64_t facets_version = 0;           // oc_sort_field_from_facets: the facet-store version it was built from
    SortOrder ord[2];                      // OC_SORT_ASC, OC_SORT_DESC
};
static void sort_field_free(oc_sort_field *f) {
    for (SortOrder &o : f->ord) { cudaFree(o.rank_doc); cudaFree(o.doc_rank); cudaFree(o.rank_row); cudaFree(o.rank_value); }
    delete f;
}
// The sorts of one batch: its distinct (field, order) pairs and, per query, the index of its pair or SORT_BY_SCORE
// (oc_search_q_sorted: that query is oc_search_pinned's).  oc_search_sorted is the batch whose queries share entry 0.
struct SortJob {
    std::vector<oc_sort_field *> f;        // [entries]
    std::vector<int> order;                // [entries]
    std::vector<uint32_t> q_ent;           // [B]
    bool by_score = false;                 // some query is in score order
    SortOrder &ord(uint32_t e) const { return f[e]->ord[order[e]]; }
};
// Appends one query's sort (field NULL: score order).  Nothing is written on failure.
static int sort_job_add(oc_ctx *c, const oc_sort &s, SortJob &sj) {
    if (!s.field) { sj.q_ent.push_back(SORT_BY_SCORE); sj.by_score = true; return OC_OK; }
    if (s.order != OC_SORT_ASC && s.order != OC_SORT_DESC) return fail(OC_ERR_INVALID, "sort order %d is neither ASC nor DESC", s.order);
    if (s.field->ctx != c) return fail(OC_ERR_INVALID, "sort field belongs to another ctx");
    oc_sort_field *f = const_cast<oc_sort_field *>(s.field);   // only its per-snapshot row map is refreshed, under the ctx lock
    uint32_t e = 0;
    while (e < sj.f.size() && !(sj.f[e] == f && sj.order[e] == s.order)) e++;
    if (e == sj.f.size()) { sj.f.push_back(f); sj.order.push_back(s.order); }
    sj.q_ent.push_back(e);
    return OC_OK;
}
// one sort for every query of the batch
static int sort_job_init(oc_ctx *c, const oc_sort *s, uint32_t B, SortJob &sj) {
    if (!s || !s->field) return fail(OC_ERR_INVALID, "NULL sort");
    OCTRY(sort_job_add(c, *s, sj));
    sj.q_ent.assign(B, 0);
    return OC_OK;
}
// the value a listed document was placed by: NaN for a document the (active) query promotes or a query in score order,
// else its value
static double sort_value_of(const SortJob &sj, const PinJob *pj, uint32_t q, uint64_t d) {
    const uint32_t e = sj.q_ent[q];
    if (e == SORT_BY_SCORE) return std::numeric_limits<double>::quiet_NaN();
    if (pj && pj->splice)
        for (uint32_t j = 0; j < pj->cnt[q]; j++)
            if (pj->doc[size_t(q) * pj->stride + j] == d) return std::numeric_limits<double>::quiet_NaN();
    const SortOrder &o = sj.ord(e);
    const uint32_t r = d < sj.f[e]->nbits ? o.h_doc_rank[d] : RANK_NONE;
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

static int run_groups(oc_ctx *c, const GroupJob &gj, int mode, const StrSnap *S, uint32_t n_tiles, uint32_t vlimit,
                      const uint64_t *omc_doc, const float *omc_mult, uint32_t n_omc, const PinJob &pj, const QueryPlan *q_plan);

// ------------------------------------------------------------------------------------ OMC store (omc.cuh)
// The published version is replaced only by a commit, under the ctx lock once the ctx stream has drained; every search
// reads it under the ctx lock.  The queue is guarded by `mu`.  The row-list cache belongs to the searches (ctx lock).
struct oc_omc {
    oc_ctx *ctx = nullptr;
    uint64_t *doc = nullptr;               // device: the published version, doc ascending
    float *mult = nullptr;
    uint64_t n = 0, version = 0;
    std::mutex mu;
    bool committing = false;
    std::vector<uint64_t> q_doc;           // the queue, in call order
    std::vector<float> q_mult;
    std::vector<uint8_t> q_del;
    cudaStream_t stream = nullptr;         // the commit's merge
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    // the tile scorers' list of the version's string rows, ascending, for (rows_version, rows_snap): a cache the
    // searches (which see the handle as const) build on their own stream
    mutable cudaStream_t rows_stream = nullptr;
    mutable uint64_t rows_version = 0, rows_snap = 0;   // rows_snap: StrSnap::ident (0: none built)
    mutable uint32_t n_rows = 0;
    mutable uint64_t rows_cap = 0;
    mutable uint32_t *row = nullptr;
    mutable float *row_mult = nullptr;
};

extern "C" int oc_omc_create(oc_ctx *c, oc_omc **out) {
    if (!c || !out) return fail(OC_ERR_INVALID, "NULL argument");
    oc_omc *o = new oc_omc();
    o->ctx = c;
    *out = o;
    return OC_OK;
}
extern "C" void oc_omc_destroy(oc_omc *o) {
    if (!o) return;
    {
        std::lock_guard<std::mutex> g(o->ctx->mu);
        cudaSetDevice(o->ctx->device);
        cudaStreamSynchronize(o->ctx->stream);
        if (o->stream) { cudaStreamSynchronize(o->stream); cudaStreamDestroy(o->stream); }
        if (o->rows_stream) { cudaStreamSynchronize(o->rows_stream); cudaStreamDestroy(o->rows_stream); }
        for (cudaEvent_t e : o->ev) if (e) cudaEventDestroy(e);
        cudaFree(o->doc); cudaFree(o->mult); cudaFree(o->row); cudaFree(o->row_mult);
    }
    delete o;
}
extern "C" int oc_omc_set(oc_omc *o, const uint64_t *doc_ids, const float *mults, uint64_t n) {
    if (!o || (n && (!doc_ids || !mults))) return fail(OC_ERR_INVALID, "NULL argument");
    for (uint64_t i = 0; i < n; i++)
        if (!std::isfinite(mults[i])) return fail(OC_ERR_INVALID, "entry %llu: multiplier is not finite", (unsigned long long)i);
    std::lock_guard<std::mutex> g(o->mu);
    o->q_doc.insert(o->q_doc.end(), doc_ids, doc_ids + n);
    o->q_mult.insert(o->q_mult.end(), mults, mults + n);
    o->q_del.insert(o->q_del.end(), n, uint8_t(0));
    return OC_OK;
}
extern "C" int oc_omc_delete(oc_omc *o, const uint64_t *doc_ids, uint64_t n) {
    if (!o || (n && !doc_ids)) return fail(OC_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> g(o->mu);
    o->q_doc.insert(o->q_doc.end(), doc_ids, doc_ids + n);
    o->q_mult.insert(o->q_mult.end(), n, 0.f);
    o->q_del.insert(o->q_del.end(), n, uint8_t(1));
    return OC_OK;
}

// The merge of the n_b queued ops into the version (a_doc, a_mult, n_a), on `st` (omc.cuh).  Two device phases timed by
// ev[0..1] (upload .. scans) and ev[2..3] (scatter).
struct OmcMergeOut { uint64_t n = 0, kept = 0, added = 0, ws = 0; float device_ms = 0; uint64_t *doc = nullptr; float *mult = nullptr; };
static int omc_merge(cudaStream_t st, cudaEvent_t *ev, const uint64_t *a_doc, const float *a_mult, uint64_t n_a,
                     const std::vector<uint64_t> &q_doc, const std::vector<float> &q_mult, const std::vector<uint8_t> &q_del,
                     OmcMergeOut &o) {
    const uint64_t n_b = q_doc.size();
    if (n_a + n_b >= uint64_t(INT32_MAX)) return fail(OC_ERR_UNSUPPORTED, "OMC commit: %llu entries >= 2^31 - 1",
                                                      (unsigned long long)(n_a + n_b));   // cub counts in int
    size_t sort_b = 0, scan_a = 0, scan_b = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const uint32_t *)nullptr,
                                        (uint32_t *)nullptr, (int)n_b, 0, 64, st) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, scan_a, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)(n_a + 1), st) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)(n_b + 1), st) != cudaSuccess)
        return fail(OC_ERR_CUDA, "OMC commit: temp storage size");
    // workspace: [uploaded: q_doc | q_mult | q_del | idx] [b_doc | b_idx | a_keep | a_rank | b_keep | b_rank | temp]
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t o_qd = 0, o_qm = o_qd + al(n_b * 8), o_qx = o_qm + al(n_b * 4), o_ix = o_qx + al(n_b), up = o_ix + al(n_b * 4);
    const size_t o_bd = up, o_bi = o_bd + al(n_b * 8), o_ak = o_bi + al(n_b * 4), o_ar = o_ak + al((n_a + 1) * 4),
                 o_bk = o_ar + al((n_a + 1) * 4), o_br = o_bk + al((n_b + 1) * 4), o_tmp = o_br + al((n_b + 1) * 4),
                 total = o_tmp + al(std::max(sort_b, std::max(scan_a, scan_b)));
    std::vector<uint8_t> h(up, 0);
    memcpy(h.data() + o_qd, q_doc.data(), n_b * 8);
    memcpy(h.data() + o_qm, q_mult.data(), n_b * 4);
    memcpy(h.data() + o_qx, q_del.data(), n_b);
    uint32_t *idx = reinterpret_cast<uint32_t *>(h.data() + o_ix);
    for (uint64_t i = 0; i < n_b; i++) idx[i] = uint32_t(i);
    uint8_t *w = nullptr;
    if (cudaMallocAsync(&w, total, st) != cudaSuccess) return fail(OC_ERR_OOM, "OMC commit: %zu B of workspace", total);
    o.ws = total;
    auto done = [&](int r) { cudaFreeAsync(w, st); if (r != OC_OK) { cudaFree(o.doc); cudaFree(o.mult); o.doc = nullptr; o.mult = nullptr; } return r; };
    const uint64_t *qd = reinterpret_cast<const uint64_t *>(w + o_qd);
    const float *qm = reinterpret_cast<const float *>(w + o_qm);
    const uint8_t *qx = w + o_qx;
    const uint32_t *ix = reinterpret_cast<const uint32_t *>(w + o_ix);
    uint64_t *bd = reinterpret_cast<uint64_t *>(w + o_bd);
    uint32_t *bi = reinterpret_cast<uint32_t *>(w + o_bi), *ak = reinterpret_cast<uint32_t *>(w + o_ak);
    uint32_t *ar = reinterpret_cast<uint32_t *>(w + o_ar), *bk = reinterpret_cast<uint32_t *>(w + o_bk);
    uint32_t *br = reinterpret_cast<uint32_t *>(w + o_br);
    const uint64_t n_max = std::max(n_a, n_b) + 1;
    cudaError_t e = cudaMemcpyAsync(w, h.data(), up, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaEventRecord(ev[0], st);
    // stable: each document's ops keep their call order
    if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(w + o_tmp, sort_b, qd, bd, ix, bi, (int)n_b, 0, 64, st);
    if (e == cudaSuccess) {
        om_keep_kernel<<<(unsigned)((n_max + OM_THREADS - 1) / OM_THREADS), OM_THREADS, 0, st>>>(a_doc, n_a, bd, bi, qx, n_b, ak, bk);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(w + o_tmp, scan_a, ak, ar, (int)(n_a + 1), st);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(w + o_tmp, scan_b, bk, br, (int)(n_b + 1), st);
    uint32_t tot[2] = {0, 0};
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tot[0], ar + n_a, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaEventRecord(ev[1], st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tot[1], br + n_b, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&o.device_ms, ev[0], ev[1]);
    if (e != cudaSuccess) return done(fail(OC_ERR_CUDA, "OMC commit: %s", cudaGetErrorString(e)));
    o.kept = tot[0]; o.added = tot[1]; o.n = o.kept + o.added;
    if (o.n && (e = cudaMalloc(&o.doc, o.n * 8)) == cudaSuccess) e = cudaMalloc(&o.mult, o.n * 4);
    if (e != cudaSuccess) return done(fail(e == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "OMC commit: %llu entries: %s",
                                          (unsigned long long)o.n, cudaGetErrorString(e)));
    e = cudaEventRecord(ev[2], st);
    if (e == cudaSuccess && o.n) {
        if (n_a) om_scatter_a_kernel<<<(unsigned)((n_a + OM_THREADS - 1) / OM_THREADS), OM_THREADS, 0, st>>>(a_doc, a_mult, n_a, ar, bd, n_b, br, o.doc, o.mult);
        om_scatter_b_kernel<<<(unsigned)((n_b + OM_THREADS - 1) / OM_THREADS), OM_THREADS, 0, st>>>(bd, bi, qm, n_b, br, a_doc, n_a, ar, o.doc, o.mult);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev[3], st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    float ms2 = 0;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms2, ev[2], ev[3]);
    o.device_ms += ms2;
    return done(e == cudaSuccess ? OC_OK : fail(OC_ERR_CUDA, "OMC commit: %s", cudaGetErrorString(e)));
}

extern "C" int oc_omc_commit_ex(oc_omc *o, oc_filter_commit_t *out) {
    if (!o) return fail(OC_ERR_INVALID, "NULL argument");
    const auto wall0 = std::chrono::steady_clock::now();
    oc_ctx *c = o->ctx;
    std::vector<uint64_t> q_doc;
    std::vector<float> q_mult;
    std::vector<uint8_t> q_del;
    {
        std::lock_guard<std::mutex> g(o->mu);
        if (o->committing) return fail(OC_ERR_INVALID, "a commit of this handle is already in flight");
        if (cudaSetDevice(c->device) != cudaSuccess) return fail(OC_ERR_CUDA, "cudaSetDevice failed");
        if (!o->stream) {
            CU(cudaStreamCreateWithFlags(&o->stream, cudaStreamNonBlocking));
            for (cudaEvent_t &e : o->ev) CU(cudaEventCreate(&e));
        }
        o->committing = true;
        q_doc = o->q_doc; q_mult = o->q_mult; q_del = o->q_del;
    }
    // the published version is replaced only by a commit, so it is read without the ctx lock
    oc_filter_commit_t st{};
    OmcMergeOut res;
    int rc = OC_OK;
    if (!q_doc.empty()) {
        rc = omc_merge(o->stream, o->ev, o->doc, o->mult, o->n, q_doc, q_mult, q_del, res);
        st.device_ms = res.device_ms; st.workspace_bytes = res.ws;
        st.rows_kept = res.kept; st.rows_dropped = o->n - res.kept; st.rows_added = res.added;
    } else {
        st.rows_kept = o->n;
    }
    if (rc != OC_OK) {
        std::lock_guard<std::mutex> g(o->mu);
        o->committing = false;
        return rc;
    }
    {   // publish: every reader holds the ctx lock and works on the ctx stream (see oc_facets_commit_ex)
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        if (!q_doc.empty()) {
            cudaStreamSynchronize(c->stream);
            cudaFree(o->doc); cudaFree(o->mult);
            o->doc = res.doc; o->mult = res.mult; o->n = res.n;
        }
        std::lock_guard<std::mutex> gq(o->mu);
        o->q_doc.erase(o->q_doc.begin(), o->q_doc.begin() + q_doc.size());
        o->q_mult.erase(o->q_mult.begin(), o->q_mult.begin() + q_doc.size());
        o->q_del.erase(o->q_del.begin(), o->q_del.begin() + q_doc.size());
        o->committing = false;
        st.version = ++o->version;
    }
    st.wall_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    if (out) *out = st;
    return OC_OK;
}

extern "C" int oc_omc_read(oc_omc *o, uint64_t *n, uint64_t *doc_ids, float *mults, uint64_t *version) {
    if (!o || !n) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = o->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    const uint64_t cap = *n;
    *n = o->n;
    if (version) *version = o->version;
    if (!doc_ids && !mults) return OC_OK;
    if (cap < o->n) return fail(OC_ERR_INVALID, "capacity %llu < %llu entries", (unsigned long long)cap, (unsigned long long)o->n);
    CU(cudaSetDevice(c->device));
    if (o->n && doc_ids) CU(cudaMemcpy(doc_ids, o->doc, o->n * 8, cudaMemcpyDeviceToHost));
    if (o->n && mults) CU(cudaMemcpy(mults, o->mult, o->n * 4, cudaMemcpyDeviceToHost));
    return OC_OK;
}

// The tile scorers' row list of the published version over snapshot S, built on the device when the version or the
// snapshot changed since the last build (under the ctx lock).  Ends with the list's length on the host.
static int omc_rows_for(oc_ctx *c, const oc_omc *o, const StrSnap *S) {
    if (o->rows_snap == S->ident && o->rows_version == o->version) return OC_OK;
    const uint64_t n = o->n;
    o->n_rows = 0;
    o->rows_snap = 0;
    if (n) {
        if (!o->rows_stream) CU(cudaStreamCreateWithFlags(&o->rows_stream, cudaStreamNonBlocking));
        cudaStream_t st = o->rows_stream;
        if (n > o->rows_cap) {
            cudaFree(o->row); cudaFree(o->row_mult);
            o->row = nullptr; o->row_mult = nullptr; o->rows_cap = 0;
            CU(cudaMalloc(&o->row, n * 4));
            CU(cudaMalloc(&o->row_mult, n * 4));
            o->rows_cap = n;
        }
        size_t scan = 0;
        CU(cub::DeviceScan::ExclusiveSum(nullptr, scan, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)(n + 1), st));
        auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
        const size_t o_has = al(n * 4), o_pos = o_has + al((n + 1) * 4), o_tmp = o_pos + al((n + 1) * 4), total = o_tmp + al(scan);
        uint8_t *w = nullptr;
        if (cudaMallocAsync(&w, total, st) != cudaSuccess) return fail(OC_ERR_OOM, "OMC rows: %zu B of workspace", total);
        uint32_t *row = reinterpret_cast<uint32_t *>(w), *has = reinterpret_cast<uint32_t *>(w + o_has);
        uint32_t *pos = reinterpret_cast<uint32_t *>(w + o_pos);
        om_rows_kernel<<<(unsigned)((n + OM_THREADS) / OM_THREADS), OM_THREADS, 0, st>>>(o->doc, n, S->row_doc, S->n_rows, row, has);
        launched(c);
        cudaError_t e = cudaGetLastError();
        if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(w + o_tmp, scan, has, pos, (int)(n + 1), st);
        if (e == cudaSuccess) {
            om_rows_scatter_kernel<<<(unsigned)((n + OM_THREADS - 1) / OM_THREADS), OM_THREADS, 0, st>>>(row, o->mult, n, pos, o->row, o->row_mult);
            launched(c);
            e = cudaGetLastError();
        }
        uint32_t cnt = 0;
        if (e == cudaSuccess) e = cudaMemcpyAsync(&cnt, pos + n, 4, cudaMemcpyDeviceToHost, st);
        cudaFreeAsync(w, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return fail(OC_ERR_CUDA, "OMC rows: %s", cudaGetErrorString(e));
        o->n_rows = cnt;
    }
    o->rows_snap = S->ident; o->rows_version = o->version;
    return OC_OK;
}

// One search as an entry point asks for it.  fj: the facet counts.  gj: the grouped calls (always with pj); then
// limit == 0 is allowed: the hits are not written (out_doc_ids / out_scores / out_n may be NULL), the vector stage gets
// depth 0 and the fulltext stage runs with one candidate slot per tile.  pj: the pinned calls.  sj: the sorted calls
// (always with pj); the hits are the walk's in field order, K4's list only gives the count.
struct SearchReq {
    const oc_search_params *p;
    uint64_t *out_doc_ids; float *out_scores; uint32_t *out_n; uint64_t *out_count;
    SearchReq(const oc_search_params *p_, uint64_t *doc, float *score, uint32_t *n, uint64_t *count)
        : p(p_), out_doc_ids(doc), out_scores(score), out_n(n), out_count(count) {}
    double *out_sort_values = nullptr;   // [B][limit] the hits' sort values (NaN in score order), may be NULL
    const FacetJob *fj = nullptr;
    GroupJob *gj = nullptr;
    PinJob *pj = nullptr;
    const SortJob *sj = nullptr;
    bool q_filters_ok = false;           // the entry point takes per-query filters (p->q_filters)
    bool q_params_ok = false;            // ... and per-query parameters (p->q_params)
};

// What one search derives once, filled in by the stages of search_impl in order.
struct SearchCall {
    oc_ctx *c; oc_emb *emb; oc_str *str;
    const SearchReq &r;
    const oc_search_params *p;
    SearchCall(oc_ctx *c_, oc_emb *e, oc_str *s, const SearchReq &r_) : c(c_), emb(e), str(s), r(r_), p(r_.p) {}
    // shape and path.  mode: p->mode, or with per-query parameters the union of the entries' parts
    uint32_t B = 0, limit = 0, n_keep = 0, vlimit = 0, cap = 0, sort_top = 0;
    int mode = OC_MODE_FULLTEXT;
    // per-query parameters (p->q_params): K4's plan and the page of each query, the largest offset + limit, and the
    // sub-batch of queries with a vector part with each one's depth and similarity (v_rows: their packed vectors,
    // vqf: their filter slots, when the sub-batch is not the whole batch).  Bv: the queries the vector stage sweeps.
    bool qp = false;
    uint32_t page_max = 0, Bv = 0;
    std::vector<QueryPlan> q_plan;
    std::vector<uint2> q_page;
    std::vector<uint32_t> v_sub, v_lim;
    std::vector<float> v_sim, v_rows;
    QFilterJob vqf;
    Slot<QueryPlan> s_plan;
    Slot<uint2> s_page;
    Slot<uint32_t> s_vsub, s_vlim, s_vqslot;
    Slot<float> s_vsim;
    bool has_v = false, has_ft = false, per_q = false, facets = false, write_hits = false, pin_flat = false, sort_flat = false;
    bool k4_top = false, exports = false, pin_items = false, side = false;
    // inputs; filter_h: the filter is a host bitmap, uploaded with this call
    std::shared_ptr<StrSnap> snap;
    StrSnap *S = nullptr;
    QFilterJob qfj;
    // where programs (p->q_where): a handle over each distinct result bitmap in c->w_bits, and each query's handle
    std::vector<oc_filter> w_handles;
    std::vector<const oc_filter *> w_qf;
    FacetPlan fpl;
    const oc_filter *batch_filter = nullptr;
    bool filter_h = false, filter = false;
    uint64_t filter_nbits = 0;
    size_t fwords = 0;
    const uint64_t *filter_dev = nullptr;
    // fulltext descriptors.  max_tokens: tokens of the longest query; dense_bytes: the dense contribution arrays of the
    // batch in c->dense_buf, dense_new: those built into the ctx's dense-array cache (both zeroed before the precompute
    // kernel fills them); dense_seen: the snapshots the cache's sweep looked at (released after the ctx lock);
    // term_key: (field << 32 | term id) of each expanded term;
    // tok_slot: per-query filters, the fulltext slot of each token's query
    bool multi_rank = false, tombs = false, thr = false, count_df = false, any_multi = false, need_df = false, derived_now = false;
    uint32_t n_tiles = 0, max_tokens = 0;
    uint64_t dense_bytes = 0, postings_walked = 0;
    std::vector<DenseEntry *> dense_new;
    std::vector<std::shared_ptr<StrSnap>> dense_seen;
    std::vector<TermDesc> terms;
    std::vector<TokenDesc> tokens;
    std::vector<QueryDesc> queries;
    std::vector<uint64_t> term_key;
    std::vector<uint32_t> term_token, tok_slot;
    std::vector<uint8_t> tok_need_df;
    std::vector<PreDesc> pre_descs;
    std::vector<uint2> pre_items;
    // OMC: the documents and multipliers K4, the shard merge, groups and pins read (n_omc entries), and the tile
    // kernel's string rows, ascending (n_omc_rows).  Array path: uploaded with the call; store path (p->omc): the
    // version's device arrays and the handle's row list
    uint32_t n_omc = 0, n_omc_rows = 0;
    bool omc_tile = false;
    std::vector<uint32_t> omc_rows;
    std::vector<float> omc_row_mult;
    const uint64_t *omc_doc = nullptr;
    const float *omc_mult = nullptr;
    const uint32_t *omc_row_dev = nullptr;
    const float *omc_row_mult_dev = nullptr;
    // sortBy entries and per-query walks, group handles and spans
    std::vector<SortEntry> s_ents;
    std::vector<SortQuery> s_q;
    std::vector<uint8_t> s_alt;
    std::vector<GroupHandle> g_hand;
    std::vector<GroupSpan> g_spans;
    // the two uploads: pk0 (vector modes: the query vectors, sent before the descriptors are built) and pk; `first` is
    // the one the filter bitmap, the per-query filter tables and the facet work list ride in
    Packer pk0, pk, *first = nullptr;
    DevBuf *first_blob = nullptr;
    Slot<uint64_t> s_flt, s_omcd;
    Slot<uint32_t> s_qslot, s_qslot_ft, s_ttok, s_tslot, s_omcr;
    Slot<float> s_omcm, s_omcrm;
    Slot<uint2> s_fpairs, s_pitems;
    Slot<RowsOkSlot> s_qslots;
    Slot<FacetSliceDev> s_fslices;
    Slot<TermDesc> s_terms;
    Slot<TokenDesc> s_tokens;
    Slot<QueryDesc> s_queries;
    Slot<PreDesc> s_pre;
    Slot<SortEntry> s_sent;
    Slot<SortQuery> s_sq;
    Slot<uint8_t> s_salt;
    // device state of the stages
    Bm25Params bp{};
    FuseParams fp{};
    size_t fuse_smem = 0;
    const uint32_t *row_ok = nullptr;
    float *min_hint_dev = nullptr;
    unsigned int *tile_counter = nullptr;
    bool did_comm = false;
    // the output blob: [doc B x limit][score B x limit][n B][count B][min B][gflag B]; the host copy adds [g_flag B][rescored B]
    size_t o_sc = 0, o_n = 0, o_cnt = 0, o_min = 0, o_gflag = 0, out_bytes = 0, o_resc = 0, o_dstat = 0;
    uint8_t *dout = nullptr;
    uint64_t *d_doc = nullptr;
    float *d_score = nullptr;
    uint32_t *d_n = nullptr;
};

// staged segments go in one copy per contiguous run; pinned caller buffers are DMA'd directly
static int upload(const Packer &pk, HostBuf &hb, DevBuf &db, cudaStream_t st) {
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
}

// per-query where-filters: deduplicated by handle; all NULL = unfiltered, one handle for every query = p->filter
static int qfilter_slots(SearchCall &k, const oc_filter *const *q_filters);
static int qfilter_plan(SearchCall &k) {
    const oc_search_params *p = k.p;
    if (!k.r.q_filters_ok)
        return fail(OC_ERR_UNSUPPORTED, "q_filters: per-query filters are supported by oc_search, oc_search_q_sorted and "
                                        "oc_search_q_groups only");
    if (p->filter || p->filter_bits) return fail(OC_ERR_INVALID, "q_filters together with filter / filter_bits");
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "q_filters over a sharded search");
    return qfilter_slots(k, p->q_filters);
}
// the slots of the per-query filter handles q_filters[B] (p->q_filters, or the results of the call's where programs)
static int qfilter_slots(SearchCall &k, const oc_filter *const *q_filters) {
    const uint32_t B = k.B;
    QFilterJob &qfj = k.qfj;
    std::unordered_map<const oc_filter *, uint32_t> idx;
    std::vector<const oc_filter *> distinct;
    bool any_none = false;
    qfj.q_slot.resize(B);
    for (uint32_t b = 0; b < B; b++) {
        const oc_filter *f = q_filters[b];
        if (!f) { any_none = true; qfj.q_slot[b] = SLOT_NONE; continue; }
        if (f->ctx != k.c) return fail(OC_ERR_INVALID, "q_filters[%u] belongs to another ctx", b);
        auto it = idx.emplace(f, (uint32_t)distinct.size()).first;
        if (it->second == distinct.size()) distinct.push_back(f);
        qfj.q_slot[b] = it->second;
    }
    if (distinct.size() > 65535) return fail(OC_ERR_UNSUPPORTED, "q_filters: %zu distinct handles > 65535", distinct.size());
    if (distinct.size() == 1 && !any_none) k.batch_filter = distinct[0];
    else if (!distinct.empty()) {
        k.per_q = true;
        const uint32_t K = (uint32_t)distinct.size();
        for (const oc_filter *f : distinct) qfj.slots.push_back(RowsOkSlot{f->bits, f->nbits});
        qfj.slots.push_back(RowsOkSlot{nullptr, 0});
        qfj.q_slot_ft.resize(B);
        for (uint32_t b = 0; b < B; b++) qfj.q_slot_ft[b] = qfj.q_slot[b] == SLOT_NONE ? K : qfj.q_slot[b];
    }
    return OC_OK;
}

// Per-query parameters: each entry gets the checks its scalars get alone, and the table of what every stage does for it.
// The batch runs at the largest depths: n_keep = the largest (limit + offset) x (2 for an active pinned query), the
// vector depth = the largest of the vector entries' own depths, sort_top = the largest top_count.
static int qparams_plan(SearchCall &k) {
    const SearchReq &r = k.r; const oc_search_params *p = k.p;
    const PinJob *pj = r.pj;
    const bool limit0_ok = r.gj || (r.fj && r.fj->hits_optional);   // (oc_search_q_groups checks the queries without groups)
    k.q_page.resize(k.B);
    k.sort_top = 0;
    for (uint32_t b = 0; b < k.B; b++) {
        const oc_query_params &e = p->q_params[b];
        if (e.limit > p->limit) return fail(OC_ERR_INVALID, "q_params[%u]: limit %u > p->limit %u (the row stride)", b, e.limit, p->limit);
        if (e.limit == 0 && !limit0_ok) return fail(OC_ERR_INVALID, "q_params[%u]: limit must be >= 1", b);
        const bool hits = k.write_hits && e.limit > 0;   // as alone: limit 0 writes no hit and gives the vector stage depth 0
        const uint32_t lim = hits ? e.limit : 1;
        const bool active = pj && pj->splice && pj->cnt[b] > 0;
        if (active && (uint64_t(e.limit) + e.offset) * 2 > OC_MAX_TOPK)
            return fail(OC_ERR_UNSUPPORTED, "q_params[%u]: pins: 2 x (limit+offset) %llu > %u", b,
                        (unsigned long long)(uint64_t(e.limit) + e.offset) * 2, OC_MAX_TOPK);
        const uint64_t nk = (uint64_t(lim) + e.offset) * (active && hits ? 2 : 1);
        if (nk > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "q_params[%u]: limit+offset %llu > %u", b, (unsigned long long)nk, OC_MAX_TOPK);
        const uint32_t vl = !hits ? 0u : e.vector_limit ? e.vector_limit : e.limit;
        if (vl > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "q_params[%u]: vector_limit %u > %u", b, vl, OC_MAX_TOPK);
        const uint32_t page_lim = hits ? e.limit : 0u;
        k.q_page[b] = make_uint2(e.offset, page_lim);
        QueryPlan &qp = k.q_plan[b];
        qp.n_keep = (uint32_t)nk;
        qp.limit = k.k4_top ? qp.n_keep : page_lim;     // a splice pages K4's whole top n_keep afterwards
        qp.offset = k.k4_top ? 0u : e.offset;
        k.n_keep = std::max(k.n_keep, qp.n_keep);
        k.page_max = std::max(k.page_max, e.offset + page_lim);
        if (k.sort_flat) k.sort_top = std::max(k.sort_top, uint32_t((uint64_t(page_lim) + e.offset) * (active ? 2 : 1)));
        if (qp.mode != OC_MODE_FULLTEXT) {
            k.v_sub.push_back(b); k.v_lim.push_back(vl); k.v_sim.push_back(e.similarity);
            k.vlimit = std::max(k.vlimit, vl);
        }
    }
    if (k.sort_flat) k.sort_top = std::max(k.sort_top, 1u);
    return OC_OK;
}

// The checks that need no device, and the call's shape and path.  B == 0 stops here.
static int search_check(SearchCall &k) {
    oc_ctx *c = k.c; const SearchReq &r = k.r;
    const oc_search_params *p = r.p;
    if (!c || !p || !r.out_count) return fail(OC_ERR_INVALID, "NULL argument");
    k.write_hits = !(r.gj || (r.fj && r.fj->hits_optional)) || p->limit > 0;
    if (k.write_hits && (!r.out_doc_ids || !r.out_scores || !r.out_n)) return fail(OC_ERR_INVALID, "NULL argument");
    if (p->omc && p->n_omc) return fail(OC_ERR_INVALID, "omc together with omc_doc_ids / omc_mult / n_omc");
    if (p->omc && p->omc->ctx != c) return fail(OC_ERR_INVALID, "omc belongs to another ctx");
    const uint32_t B = k.B = p->n_queries;
    k.qp = p->q_params != nullptr;
    if (k.qp && !r.q_params_ok)
        return fail(OC_ERR_UNSUPPORTED, "q_params: per-query parameters are supported by oc_search, oc_search_q_sorted, "
                                        "oc_search_q_groups and oc_search_q_facets only");
    if (k.qp && p->sharded) return fail(OC_ERR_UNSUPPORTED, "q_params over a sharded search");
    if (B == 0) return OC_OK;
    if (k.qp) {   // each entry's mode; the batch has the union of their parts
        k.q_plan.resize(B);
        for (uint32_t b = 0; b < B; b++) {
            const int m = p->q_params[b].mode;
            if (m != OC_MODE_FULLTEXT && m != OC_MODE_VECTOR && m != OC_MODE_HYBRID)
                return fail(OC_ERR_INVALID, "q_params[%u]: unknown mode %d", b, m);
            k.q_plan[b].mode = m;
            k.has_v = k.has_v || m != OC_MODE_FULLTEXT;
            k.has_ft = k.has_ft || m != OC_MODE_VECTOR;
        }
        k.mode = k.has_v && k.has_ft ? OC_MODE_HYBRID : k.has_v ? OC_MODE_VECTOR : OC_MODE_FULLTEXT;
    } else {
        k.has_v = p->mode == OC_MODE_VECTOR || p->mode == OC_MODE_HYBRID;
        k.has_ft = p->mode == OC_MODE_FULLTEXT || p->mode == OC_MODE_HYBRID;
        if (!k.has_v && !k.has_ft) return fail(OC_ERR_INVALID, "unknown mode %d", p->mode);
        k.mode = p->mode;
    }
    if (k.has_v && (!k.emb || !p->q_vecs)) return fail(OC_ERR_INVALID, "vector/hybrid mode needs emb and q_vecs");
    if (k.has_ft && (!k.str || !p->q_token_offsets)) return fail(OC_ERR_INVALID, "fulltext/hybrid mode needs str and tokens");
    if (k.emb && k.emb->ctx != c) return fail(OC_ERR_INVALID, "emb belongs to another ctx");
    if (k.str && k.str->ctx != c) return fail(OC_ERR_INVALID, "str belongs to another ctx");
    k.batch_filter = p->filter;
    if (p->q_where) {   // the programs themselves are checked and planned under the ctx lock (where_stage)
        if (!r.q_filters_ok)
            return fail(OC_ERR_UNSUPPORTED, "q_where: per-query where programs are supported by oc_search, oc_search_q_sorted, "
                                            "oc_search_q_groups and oc_search_q_facets only");
        if (p->filter || p->filter_bits || p->q_filters) return fail(OC_ERR_INVALID, "q_where together with filter / filter_bits / q_filters");
        if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "q_where over a sharded search");
        if (!p->q_where->q_node_offsets) return fail(OC_ERR_INVALID, "q_where: q_node_offsets is NULL");
    }
    if (p->q_filters) OCTRY(qfilter_plan(k));
    if (p->limit == 0 && k.write_hits) return fail(OC_ERR_INVALID, "limit must be >= 1");
    const PinJob *pj = r.pj; const SortJob *sj = r.sj;
    const uint32_t limit = k.limit = k.write_hits ? p->limit : 1;
    // sort_token_scores with pins selects the top 2 * (limit + offset) (sort.rs:25-34); the vector depth stays limit
    k.pin_flat = pj && pj->splice && k.write_hits && !sj;
    k.sort_flat = sj && k.write_hits;
    // sort_token_scores with sort_by: top_count keys in field order, twice as many for an active pinned query
    k.sort_top = k.sort_flat ? uint32_t((uint64_t(limit) + p->offset) * (pj->splice ? 2 : 1)) : 0u;
    // oc_search_q_sorted: the queries in score order take K4's list, spliced as pin_flat does
    bool score_active = false;
    if (k.sort_flat && sj->by_score && pj->splice)
        for (uint32_t q = 0; q < B; q++) score_active = score_active || (sj->q_ent[q] == SORT_BY_SCORE && pj->cnt[q] > 0);
    k.k4_top = k.pin_flat || (k.sort_flat && sj->by_score);   // K4 writes its top n_keep (offset 0) for a splice
    if (k.qp) {
        OCTRY(qparams_plan(k));
    } else {
        const uint64_t n_keep64 = (uint64_t(limit) + p->offset) * (k.pin_flat || score_active ? 2 : 1);
        if (n_keep64 > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "limit+offset %llu > %u", (unsigned long long)n_keep64, OC_MAX_TOPK);
        k.n_keep = (uint32_t)n_keep64;
        // limit_hint = limit, NOT limit+offset (search.rs:330-336); vector_limit lets a multi-index caller keep that depth
        k.vlimit = !k.write_hits ? 0u : p->vector_limit ? p->vector_limit : limit;
        if (k.vlimit > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "vector_limit %u > %u", k.vlimit, OC_MAX_TOPK);
    }
    if (p->sharded && !c->comm.ready()) return fail(OC_ERR_COMM, "sharded search without oc_comm_init");
    k.exports = r.gj || pj || sj;   // K4 exports the normalisation and the vector part of the score map
    k.pin_items = pj && pj->stride;
    k.facets = r.fj && !r.fj->q.empty();
    return OC_OK;
}

// per-query filters and the facet work list travel with the call's first upload
static void add_first_tables(SearchCall &k) {
    Packer &pk = *k.first;
    if (k.per_q) {
        k.s_qslots = pk.add(k.qfj.slots.data(), k.qfj.slots.size());
        k.s_qslot = pk.add(k.qfj.q_slot.data(), k.B);
        k.s_qslot_ft = pk.add(k.qfj.q_slot_ft.data(), k.B);
    }
    if (k.facets) {
        k.s_fslices = pk.add(k.fpl.slices.data(), k.fpl.slices.size());
        k.s_fpairs = pk.add(k.fpl.pairs.data(), k.fpl.pairs.size());
    }
}
static void bind_first_tables(SearchCall &k) {
    const DevBuf &b = *k.first_blob;
    if (k.filter_h) k.filter_dev = k.s_flt.at(b);
    k.qfj.d_slots = k.s_qslots.at(b);
    k.qfj.d_q_slot = k.s_qslot.at(b);
    k.qfj.d_q_slot_ft = k.s_qslot_ft.at(b);
    k.fpl.d_slices = k.s_fslices.at(b);
    k.fpl.d_pairs = k.s_fpairs.at(b);
}

static void swap_buf(DevBuf &a, DevBuf &b) { std::swap(a.p, b.p); std::swap(a.cap, b.cap); }

// The sub-batch's vector hits ([Bv][vlimit] in c->v_*) to their queries' rows of [B][vlimit]; a query without a vector
// part gets no hit.  The buffers are swapped afterwards, so every later stage reads c->v_* in the batch's layout, and
// fix_unproven patches the batch rows through c->v_qmap.
static int scatter_sub_hits(SearchCall &k) {
    oc_ctx *c = k.c;
    const size_t n = size_t(k.B) * k.vlimit;
    OCTRY(c->vq_doc.ensure(n * 8));
    OCTRY(c->vq_score.ensure(n * 4));
    OCTRY(c->vq_row.ensure(n * 4));
    OCTRY(c->vq_cnt.ensure(size_t(k.B) * 4));
    OCTRY(c->vq_raw.ensure(n * 4));
    CU(cudaMemsetAsync(c->vq_cnt.p, 0, size_t(k.B) * 4, c->stream));
    scatter_rows_kernel<<<k.Bv, 64, 0, c->stream>>>(k.s_vsub.at(c->in_blob0), k.Bv, k.vlimit, c->v_doc.as<uint64_t>(), c->v_score.as<float>(),
                                                    c->v_row.as<uint32_t>(), c->v_cnt.as<uint32_t>(), c->v_raw.as<float>(),
                                                    c->vq_doc.as<uint64_t>(), c->vq_score.as<float>(), c->vq_row.as<uint32_t>(),
                                                    c->vq_cnt.as<uint32_t>(), c->vq_raw.as<float>());
    launched(c);
    CU(cudaGetLastError());
    swap_buf(c->v_doc, c->vq_doc); swap_buf(c->v_score, c->vq_score); swap_buf(c->v_row, c->vq_row);
    swap_buf(c->v_cnt, c->vq_cnt); swap_buf(c->v_raw, c->vq_raw);
    c->v_qmap = k.v_sub;
    return OC_OK;
}

// Vector stage first: the query vectors (+ filter) go up alone and the matrix sweep starts; the host-side descriptor
// work of the next stages overlaps it.
static int vector_first(SearchCall &k) {
    oc_ctx *c = k.c; const oc_search_params *p = k.p;
    const uint32_t B = k.B;
    if (k.batch_filter && k.batch_filter->ctx != c) return fail(OC_ERR_INVALID, "filter belongs to another ctx");
    k.filter_h = !k.batch_filter && p->filter_bits != nullptr;
    k.filter = k.filter_h || k.batch_filter != nullptr;
    k.filter_nbits = k.batch_filter ? k.batch_filter->nbits : p->filter_nbits;
    k.fwords = k.filter_h ? (p->filter_nbits + 63) / 64 : 0;
    k.filter_dev = k.batch_filter ? k.batch_filter->bits : nullptr;
    k.first = k.has_v ? &k.pk0 : &k.pk;
    k.first_blob = k.has_v ? &c->in_blob0 : &c->in_blob;
    // per-query parameters: the vector stage sweeps the sub-batch of queries with a vector part (their rows packed when it
    // is not the whole batch), each with its own depth and similarity
    k.Bv = k.qp ? (uint32_t)k.v_sub.size() : B;
    const bool sub = k.Bv < B;
    Slot<float> s_qv;
    if (k.has_v && sub) {
        const size_t dim = k.emb->dim;
        k.v_rows.resize(size_t(k.Bv) * dim);
        for (uint32_t i = 0; i < k.Bv; i++) memcpy(k.v_rows.data() + i * dim, p->q_vecs + size_t(k.v_sub[i]) * dim, dim * 4);
        s_qv = k.pk0.add(k.v_rows.data(), k.v_rows.size());
    } else if (k.has_v) {
        s_qv = k.pk0.add(p->q_vecs, size_t(B) * k.emb->dim, is_pinned_host(p->q_vecs));
    }
    if (k.filter_h) k.s_flt = k.first->add(p->filter_bits, k.fwords);
    if (!k.has_v) return OC_OK;
    add_first_tables(k);
    if (k.qp) {
        k.s_vlim = k.pk0.add(k.v_lim.data(), k.Bv);
        k.s_vsim = k.pk0.add(k.v_sim.data(), k.Bv);
        if (sub) k.s_vsub = k.pk0.add(k.v_sub.data(), k.Bv);
        if (sub && k.per_q) {   // the sub-batch's filter slots
            for (uint32_t b : k.v_sub) k.vqf.q_slot.push_back(k.qfj.q_slot[b]);
            k.s_vqslot = k.pk0.add(k.vqf.q_slot.data(), k.Bv);
        }
    }
    CU(cudaEventRecord(c->ev[EV_START], c->stream));
    OCTRY(upload(k.pk0, c->h_in0, c->in_blob0, c->stream));
    CU(cudaEventRecord(c->ev[EV_H2D], c->stream));
    bind_first_tables(k);
    if (k.vlimit) {
        const QFilterJob *qf = k.per_q ? &k.qfj : nullptr;
        if (sub && k.per_q) {
            k.vqf.slots = k.qfj.slots;
            k.vqf.d_slots = k.qfj.d_slots;
            k.vqf.d_q_slot = k.s_vqslot.at(c->in_blob0);
            qf = &k.vqf;
        }
        OCTRY(run_vector_stage(c, k.emb, s_qv.at(c->in_blob0), k.Bv, k.vlimit, p->similarity, k.filter_dev, k.filter_nbits, qf,
                               k.s_vlim.at(c->in_blob0), k.s_vsim.at(c->in_blob0)));
        if (k.qp) { c->v_qlim = k.v_lim; c->v_qsim = k.v_sim; }
        if (sub) OCTRY(scatter_sub_hits(k));
    } else {   // limit_hint 0 (groups only): no vector hit
        OCTRY(c->v_cnt.ensure(size_t(B) * 4));
        CU(cudaMemsetAsync(c->v_cnt.p, 0, size_t(B) * 4, c->stream));
    }
    return OC_OK;
}

// OC_BM25_DENSE_CACHE_MB (default 2048, enough for the hot terms of a 10M-row store): the device memory a ctx keeps
// dense arrays of hot terms in across calls; 0 builds every call's arrays from scratch into c->dense_buf
static uint64_t dense_cache_budget() {
    const char *v = getenv("OC_BM25_DENSE_CACHE_MB");
    return (v && *v ? strtoull(v, nullptr, 10) : 2048ull) << 20;
}

// Frees the kept arrays no call can read any more: their snapshot is gone or has changed (its ident moved on), or the
// call that was to build them failed first.  The snapshots looked at are held by the call until it has left the ctx
// lock, so a last reference never frees a snapshot under it.
static void dense_cache_sweep(SearchCall &k) {
    oc_ctx *c = k.c; DenseCache &dc = c->dense_cache;
    cudaStream_t ps = k.side ? c->side : c->stream;
    for (auto it = dc.map.begin(); it != dc.map.end();) {
        std::shared_ptr<StrSnap> s = it->second.snap.lock();
        const bool live = s && s->ident == it->first.snap && it->second.ready;
        if (s) k.dense_seen.push_back(std::move(s));
        it = live ? std::next(it) : dc.drop(it, ps);
    }
}

// The kept array of each of the call's dense terms (keys[i], `bytes` each).  A hit is read as it is (arr[i], build[i]
// = 0).  A miss gets a new array that this call builds (build[i] = 1) while the budget allows, evicting the least
// recently used arrays this call does not read.  arr[i] = NULL: the term's array goes in c->dense_buf, as every one
// does when a row bitmap masks the call's arrays (filter, tombstones, df counted on the device) or the budget is 0.
static void dense_cache_bind(SearchCall &k, const std::vector<DenseKey> &keys, uint64_t bytes, std::vector<float *> &arr,
                             std::vector<uint8_t> &build) {
    oc_ctx *c = k.c; DenseCache &dc = c->dense_cache;
    cudaStream_t ps = k.side ? c->side : c->stream;
    const uint64_t budget = dense_cache_budget();
    arr.assign(keys.size(), nullptr);
    build.assign(keys.size(), 0);
    if (!budget || k.filter || k.tombs || k.need_df) return;
    dc.tick++;
    dc.in_call = 0;
    for (size_t i = 0; i < keys.size(); i++) {
        auto it = dc.map.find(keys[i]);
        if (it != dc.map.end()) { it->second.last_use = dc.tick; dc.in_call += bytes; arr[i] = it->second.p; continue; }
        if (dc.in_call + bytes > budget) continue;
        while (dc.used + bytes > budget && dc.evict_one(ps)) {}
        float *p = nullptr;
        if (cudaMallocAsync(reinterpret_cast<void **>(&p), bytes, ps) != cudaSuccess) { cudaGetLastError(); continue; }   // device full: c->dense_buf
        DenseEntry &e = dc.map[keys[i]];
        e.p = p; e.bytes = bytes; e.last_use = dc.tick; e.snap = k.snap;
        dc.used += bytes; dc.in_call += bytes;
        arr[i] = p; build[i] = 1;
        k.dense_new.push_back(&e);
    }
}

// Batch-level sharing of per-posting contributions (single-term tokens with a host-known idf) and the dense form of
// hot terms.  Not with per-query filters: the precomputed contributions and dense arrays are masked by ONE row bitmap.
static int ft_share_dense(SearchCall &k) {
    oc_ctx *c = k.c;
    if (!c->dense_cache.map.empty()) dense_cache_sweep(k);
    std::vector<TermDesc> &terms = k.terms;
    const std::vector<TokenDesc> &tokens = k.tokens;
    struct K128 { uint64_t a, b; };            // (field, term) | (weight bits, idf bits)
    struct U { uint32_t first_e; uint32_t uses; K128 key; };
    size_t cap_t = 64;
    while (cap_t < tokens.size() * 2) cap_t <<= 1;
    std::vector<K128> tab_k(cap_t);
    std::vector<uint32_t> tab_v(cap_t, 0xffffffffu);   // open addressing, linear probing
    std::vector<U> uniq;
    std::vector<uint32_t> e_to_u(terms.size(), 0xffffffffu);
    uint64_t walked = 0, distinct = 0;
    for (size_t t = 0; t < tokens.size(); t++) {
        const TokenDesc &tk = tokens[t];
        if (tk.term_end - tk.term_begin != 1 || k.tok_need_df[t]) continue;
        const uint32_t e = tk.term_begin;
        if (terms[e].len < 64) continue;
        uint32_t wb, ib;
        memcpy(&wb, &terms[e].weight, 4); memcpy(&ib, &tk.idf, 4);
        const K128 key{k.term_key[e], (uint64_t(wb) << 32) | ib};
        uint64_t h = (key.a * 0x9E3779B97F4A7C15ull) ^ (key.b * 0xC2B2AE3D27D4EB4Full);
        size_t slot = (h ^ (h >> 29)) & (cap_t - 1);
        while (tab_v[slot] != 0xffffffffu && !(tab_k[slot].a == key.a && tab_k[slot].b == key.b)) slot = (slot + 1) & (cap_t - 1);
        if (tab_v[slot] == 0xffffffffu) {
            tab_k[slot] = key; tab_v[slot] = (uint32_t)uniq.size();
            uniq.push_back({e, 0, key}); distinct += terms[e].len;
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
    const bool dense_on = !k.any_multi && !(dense_env && dense_env[0] == '0') && !share_off && !(t2_env && t2_env[0] == '0');
    const uint64_t dbytes = bm25_dense_bytes(k.n_tiles);   // float[n_tiles * TILE] and its summary (bitmap, tile bounds)
    const uint64_t dense_min = std::max<uint64_t>(512, k.S->n_rows / 16);
    std::vector<uint8_t> u_dense(uniq.size(), 0);
    uint64_t n_dense = 0;
    if (dense_on)
        for (size_t u = 0; u < uniq.size(); u++)
            if (terms[uniq[u].first_e].len >= dense_min && (n_dense + 1) * dbytes <= (size_t(8) << 30)) { u_dense[u] = 1; n_dense++; }
    uint64_t walked_l = 0, distinct_l = 0;   // what is left for the list form
    for (size_t e = 0; e < terms.size(); e++)
        if (e_to_u[e] != 0xffffffffu && !u_dense[e_to_u[e]]) walked_l += terms[e].len;
    for (size_t u = 0; u < uniq.size(); u++) if (!u_dense[u]) distinct_l += terms[uniq[u].first_e].len;
    const bool lists = distinct_l && !share_off && (share_force || (walked_l >= 2 * distinct_l && walked_l >= (64u << 20))) &&
                       distinct_l * 8 <= (size_t(6) << 30);
    if (!lists && !n_dense) return OC_OK;
    // each dense term's array: a kept one of the ctx's cache (read as it is on a hit, built by this call on a miss), or
    // one in this call's c->dense_buf
    std::vector<float *> u_arr(uniq.size(), nullptr);
    std::vector<uint8_t> u_kept(uniq.size(), 0);
    if (n_dense) {
        std::vector<DenseKey> keys;
        std::vector<uint32_t> key_u;
        uint32_t kb, bb;
        memcpy(&kb, &k.p->bm25_k, 4); memcpy(&bb, &k.p->bm25_b, 4);
        for (size_t u = 0; u < uniq.size(); u++)
            if (u_dense[u]) {
                keys.push_back(DenseKey{k.S->ident, uniq[u].key.a, uint32_t(uniq[u].key.b >> 32), uint32_t(uniq[u].key.b), kb, bb});
                key_u.push_back((uint32_t)u);
            }
        std::vector<float *> arr;
        std::vector<uint8_t> build;
        dense_cache_bind(k, keys, dbytes, arr, build);
        for (size_t i = 0; i < keys.size(); i++) { u_arr[key_u[i]] = arr[i]; u_kept[key_u[i]] = arr[i] && !build[i]; }
    }
    uint64_t n_buf = 0;
    for (size_t u = 0; u < uniq.size(); u++) n_buf += u_dense[u] && !u_arr[u];
    if (lists) OCTRY(c->pre_post.ensure(distinct_l * 8 + 64));
    if (n_buf) OCTRY(c->dense_buf.ensure(n_buf * dbytes));
    k.dense_bytes = n_buf * dbytes;
    uint64_t off = 0, doff = 0;
    std::vector<uint64_t> u_off(uniq.size());
    std::vector<uint8_t> u_used(uniq.size(), 0);
    for (size_t u = 0; u < uniq.size(); u++) {
        if (!u_dense[u] && !lists) continue;
        u_used[u] = 1;
        if (u_dense[u] && !u_arr[u]) { u_arr[u] = c->dense_buf.as<float>() + doff; doff += dbytes / 4; }
        if (u_kept[u]) continue;   // a cache hit: nothing to build, its summary included
        const TermDesc &td = terms[uniq[u].first_e];
        PreDesc pd{};
        pd.src = td.ptr; pd.len = td.len; pd.weight = td.weight;
        pd.idf = tokens[k.term_token[uniq[u].first_e]].idf;
        if (u_dense[u]) { pd.dense = u_arr[u]; pd.n_tiles = k.n_tiles; }
        else { u_off[u] = off; pd.dst = c->pre_post.as<Posting>() + off; off += td.len; }
        const uint32_t pi = (uint32_t)k.pre_descs.size();
        k.pre_descs.push_back(pd);
        for (uint32_t ch = 0; ch * PRE_CHUNK < td.len; ch++) k.pre_items.push_back(make_uint2(pi, ch));
    }
    for (size_t e = 0; e < terms.size(); e++) {
        const uint32_t u = e_to_u[e];
        if (u == 0xffffffffu || !u_used[u]) continue;
        if (u_dense[u]) { terms[e].ptr = reinterpret_cast<const Posting *>(u_arr[u]); terms[e].flags |= TD_DENSE; }
        else { terms[e].ptr = c->pre_post.as<Posting>() + u_off[u]; terms[e].flags |= TD_PRE; }
    }
    return OC_OK;
}

// The fulltext descriptors: terms, tokens and queries, and each token's idf where the host knows it.
static int ft_descriptors(SearchCall &k) {
    oc_ctx *c = k.c; const oc_search_params *p = k.p;
    const uint32_t B = k.B; StrSnap *S = k.S;
    k.multi_rank = p->sharded && c->comm.world > 1;
    // sharded: every rank must take the same df decisions (they drive a collective), so the
    // tombstone state is the caller's global flag (OC_SHARD_TOMBSTONES), not this shard's
    const bool tombs_local = k.has_ft && S->n_deleted > 0;
    if (k.multi_rank && tombs_local && !(p->sharded & OC_SHARD_TOMBSTONES))
        return fail(OC_ERR_INVALID, "sharded search: this shard holds tombstones, set OC_SHARD_TOMBSTONES on every rank");
    k.tombs = k.has_ft && (k.multi_rank ? (p->sharded & OC_SHARD_TOMBSTONES) != 0 : tombs_local);
    k.n_tiles = k.has_ft ? (uint32_t)((S->n_rows + BM25_TILE - 1) / BM25_TILE) : 0;
    // sharded: df comes from the replicated per-term table, or — OC_SHARD_COUNT_DF on every rank, e.g. after a
    // commit dropped the table — from counting + all-reduce.  A shard-local list length is never a corpus df.
    k.count_df = k.multi_rank && (p->sharded & OC_SHARD_COUNT_DF) != 0;
    k.thr = p->threshold >= 0.0f;
    if (k.qp) {   // per-query parameters: the threshold scorer when some query with a text part has a threshold
        k.thr = false;
        for (uint32_t q = 0; q < B; q++) k.thr = k.thr || (k.q_plan[q].mode != OC_MODE_VECTOR && p->q_params[q].threshold >= 0.0f);
    }
    if (!k.has_ft) return OC_OK;
    bool df_local_only = false;
    for (auto &f : S->fields)   // streamed posting format depends on (avg_field_len, b): derive once
        if (f.n_post && f.b_cached != p->bm25_b) {
            bm25_derive_postings_kernel<<<(unsigned)((f.n_post + 255) / 256), 256, 0, c->stream>>>(f.raw, f.n_post, f.avg_len, p->bm25_b, f.post);
            launched(c);
            CU(cudaGetLastError());
            f.b_cached = p->bm25_b;
            k.derived_now = true;   // queued on the main stream: this call keeps the BM25 prologue there too
        }
    const float N = (float)S->document_count;  // token_score.rs:221
    k.queries.resize(B);
    // Per-query filters are routed as a filtered batch is: df is counted on the device (need_df), so nothing is shared
    // or dense and K3b / K3 score the batch, each (tile, query) item under its query's row bitmap.  A token keeps the
    // idf its query would get alone: counted under the query's filter, or — single term, no filter, no tombstones —
    // from the host's posting-list length (or corpus df table), as a plain oc_search does.  An unfiltered query runs
    // under the tombstone-only row bitmap (slot K), so it scores exactly the rows it would score alone.
    if (k.per_q) k.need_df = true;
    for (uint32_t q = 0; q < B; q++) {
        // per-query parameters: a vector query has no token, a query's threshold is its own
        const bool text = !k.qp || k.q_plan[q].mode != OC_MODE_VECTOR;
        const uint32_t t0 = text ? p->q_token_offsets[q] : 0, t1 = text ? p->q_token_offsets[q + 1] : 0;
        const float threshold = k.qp ? p->q_params[q].threshold : p->threshold;
        const bool thr = k.qp ? text && threshold >= 0.0f : k.thr;
        const bool q_filter = k.filter || (k.per_q && k.qfj.q_slot[q] != SLOT_NONE);
        QueryDesc qd{};
        qd.token_begin = (uint32_t)k.tokens.size();
        const uint32_t ntok = t1 - t0;
        k.max_tokens = std::max(k.max_tokens, ntok);
        qd.required = thr ? (uint32_t)floorf((float)ntok * threshold) : 0;  // token_score.rs:211-218
        qd.flags = thr ? QF_THRESHOLD : 0;
        for (uint32_t t = t0; t < t1; t++) {
            TokenDesc tk{};
            tk.term_begin = (uint32_t)k.terms.size();
            tk.bit = 1u << ((t - t0) & 31u);
            uint64_t df_known = 0;
            for (uint32_t e = p->token_term_offsets[t]; e < p->token_term_offsets[t + 1]; e++) {
                const uint32_t fi = p->term_field[e], ti = p->term_id[e];
                if (fi >= S->fields.size()) return fail(OC_ERR_INVALID, "term field %u out of range", fi);
                const StrField &f = S->fields[fi];
                // unknown term: no postings.  A term of the synced df table (oc_str_sync_global) that this shard has
                // never seen is an empty list, so that every rank takes the same df decisions.
                const bool local = ti < f.n_terms;
                if (!local && ti >= f.global_df.size()) continue;
                TermDesc td{};
                const uint64_t off = local ? f.term_offsets[ti] : f.n_post;
                td.ptr = f.post + off;
                td.len = local ? (uint32_t)(f.term_offsets[ti + 1] - off) : 0u;
                td.weight = p->term_weight ? p->term_weight[e] : 1.0f;
                td.avg_len = f.avg_len;
                df_known = f.global_df.empty() ? td.len : f.global_df[ti];
                if (k.multi_rank && f.global_df.empty()) df_local_only = true;
                k.postings_walked += td.len;
                k.term_key.push_back((uint64_t(fi) << 32) | ti);
                k.terms.push_back(td);
                k.term_token.push_back((uint32_t)k.tokens.size());
            }
            tk.term_end = (uint32_t)k.terms.size();
            const uint32_t nt = tk.term_end - tk.term_begin;
            uint8_t need = 0;
            if (nt == 1 && !q_filter && !k.tombs && !k.count_df) tk.idf = host_idf(N, std::max<uint64_t>(1, df_known));
            else if (nt == 0) tk.idf = host_idf(N, 1);
            else { need = 1; k.need_df = true; tk.idf = 0.f; }
            if (nt != 1) { k.any_multi = k.any_multi || nt > 1; }
            k.tokens.push_back(tk);
            k.tok_need_df.push_back(need);
            if (k.per_q) k.tok_slot.push_back(k.qfj.q_slot_ft[q]);
        }
        qd.token_end = (uint32_t)k.tokens.size();
        k.queries[q] = qd;
    }
    // K3b holds a query's tokens in a BM25_MAX_TOK-entry shared table: a batch with a longer query goes to the
    // accumulator kernel (K3), which walks any number of tokens, like a batch with multi-term tokens
    if (k.max_tokens > BM25_MAX_TOK) k.any_multi = true;
    if (df_local_only && !k.count_df)
        return fail(OC_ERR_INVALID, "sharded search: a field of this shard has no corpus-wide df table (dropped by a commit?): "
                                    "reload it or pass OC_SHARD_COUNT_DF on every rank");
    return OC_OK;
}

// The stream of the fulltext stage.  Hybrid: the descriptors, the shared-contribution precompute, the filter bitmap
// and the (term, tile) plan do not depend on the vector results: they run on the side stream while the main stream
// sweeps the matrix (OC_SIDE_STREAM=0 disables it: the step gets ~2.5 % longer, the sweep itself ~4 % shorter — A/B
// switch).  Chosen before the dense arrays are: kept arrays are allocated and freed on it.
static int ft_stream(SearchCall &k) {
    oc_ctx *c = k.c;
    const char *senv = getenv("OC_SIDE_STREAM");
    // (single-GPU only for now: the sharded path was measured and validated without it)
    k.side = !(senv && senv[0] == '0') && k.has_v && k.has_ft && !k.need_df && !k.derived_now;
    if (c->side_dirty) { CU(cudaStreamSynchronize(c->side)); c->side_dirty = false; }   // leftover of a failed call
    if (k.side) { CU(cudaStreamWaitEvent(c->side, c->ev[EV_H2D], 0)); c->side_dirty = true; }   // the filter bitmap went up with the query vectors
    return OC_OK;
}

// OMC rows for the tile kernel: the documents' string rows, ascending
static int omc_plan(SearchCall &k) {
    const oc_search_params *p = k.p; const StrSnap *S = k.S;
    if (const oc_omc *o = p->omc) {   // the published version (replaced only under the ctx lock this call holds)
        k.n_omc = (uint32_t)o->n;
        k.omc_doc = o->doc; k.omc_mult = o->mult;
        if (k.n_omc && k.has_ft) {
            OCTRY(omc_rows_for(k.c, o, S));
            k.n_omc_rows = o->n_rows; k.omc_row_dev = o->row; k.omc_row_mult_dev = o->row_mult;
        }
        k.omc_tile = k.n_omc_rows > 0;
        return OC_OK;
    }
    const uint32_t n_omc = k.n_omc = (uint32_t)p->n_omc;
    if (n_omc && (!p->omc_doc_ids || !p->omc_mult)) return fail(OC_ERR_INVALID, "omc arrays are NULL");
    if (n_omc && k.has_ft) {
        for (uint32_t i = 0; i < n_omc; i++) {
            if (i && p->omc_doc_ids[i] <= p->omc_doc_ids[i - 1]) return fail(OC_ERR_INVALID, "omc_doc_ids must be ascending");
            uint64_t r;
            if (S->row_doc_host.empty()) { r = p->omc_doc_ids[i]; if (r >= S->n_rows) continue; }
            else {
                auto it = std::lower_bound(S->row_doc_host.begin(), S->row_doc_host.end(), p->omc_doc_ids[i]);
                if (it == S->row_doc_host.end() || *it != p->omc_doc_ids[i]) continue;
                r = uint64_t(it - S->row_doc_host.begin());
            }
            k.omc_rows.push_back((uint32_t)r); k.omc_row_mult.push_back(p->omc_mult[i]);
        }
    }
    k.n_omc_rows = (uint32_t)k.omc_rows.size();
    k.omc_tile = k.n_omc_rows > 0;
    return OC_OK;
}

// sortBy: the batch's entries and each query's entry and top_count (doubled for an active query).  Groups: the batch's
// distinct handles and the work list of (query, group) items, one span per query with groups: the queries in score
// order first, then those in field order (one launch of group_topk_kernel / group_sort_topk_kernel each).
static void sort_group_plan(SearchCall &k) {
    const SortJob *sj = k.r.sj; const PinJob *pj = k.r.pj;
    GroupJob *gj = k.r.gj; const uint32_t B = k.B;
    const bool rows = k.has_ft && k.n_tiles > 0;
    if (sj)
        for (uint32_t e = 0; e < sj->f.size(); e++) {
            const SortOrder &o = sj->ord(e);
            k.s_ents.push_back(SortEntry{o.n, rows ? o.rank_row : nullptr, o.doc_rank, sj->f[e]->nbits, o.rank_doc});
        }
    if (k.sort_flat) {
        k.s_q.resize(B);
        k.s_alt.resize(B);
        for (uint32_t q = 0; q < B; q++) {
            const bool active = pj->splice && pj->cnt[q] > 0;
            const uint64_t page = k.qp ? uint64_t(k.q_page[q].y) + k.q_page[q].x : uint64_t(k.limit) + k.p->offset;
            k.s_q[q] = SortQuery{sj->q_ent[q], uint32_t(page * (active ? 2 : 1))};
            k.s_alt[q] = sj->q_ent[q] == SORT_BY_SCORE;
        }
    }
    if (!gj) return;
    for (const oc_group_by *g : gj->h) k.g_hand.push_back(GroupHandle{g->off, g->docs, rows ? g->rows : nullptr, g->n_groups});
    uint32_t first = 0;
    gj->top = 0;
    gj->direct = !pj->splice;
    for (int by_field = 0; by_field < 2; by_field++) {
        for (uint32_t q = 0; q < B; q++) {
            const uint32_t h = gj->q_h[q];
            const uint32_t ent = sj ? sj->q_ent[q] : SORT_BY_SCORE;
            if (h == GROUP_NONE || gj->h[h]->n_groups == 0 || (ent != SORT_BY_SCORE) != bool(by_field)) continue;
            // sort_groups with pins takes every group's top 2 * max_results for an active query (sort.rs:137-142)
            const bool deep = (pj->splice && pj->cnt[q] > 0) || (!gj->q_deep.empty() && gj->q_deep[q]);
            const uint32_t m = gj->q_m[q], depth = m * (deep ? 2 : 1);
            k.g_spans.push_back(GroupSpan{first, q, h, depth, m, ent, gj->q_row[q]});
            first += gj->h[h]->n_groups;
            gj->top = std::max(gj->top, depth);
            gj->direct = gj->direct && depth == gj->stride;
        }
        if (!by_field) { gj->n_score_spans = (uint32_t)k.g_spans.size(); gj->n_score_items = first; }
    }
    gj->n_spans = (uint32_t)k.g_spans.size();
}

// H2D: the descriptors in one packed blob (segment order is the upload's byte layout), then the output blob's layout.
static int main_upload(SearchCall &k) {
    oc_ctx *c = k.c; const oc_search_params *p = k.p;
    const uint32_t B = k.B; const SortJob *sj = k.r.sj;
    PinJob *pj = k.r.pj; GroupJob *gj = k.r.gj;
    Packer &pk = k.pk;
    if (k.has_ft) {
        k.s_terms = pk.add(k.terms.data(), k.terms.size());
        k.s_tokens = pk.add(k.tokens.data(), k.tokens.size());
        k.s_ttok = pk.add(k.term_token.data(), k.term_token.size());
    }
    if (!k.pre_descs.empty()) k.s_pre = pk.add(k.pre_descs.data(), k.pre_descs.size());
    if (!k.pre_items.empty()) k.s_pitems = pk.add(k.pre_items.data(), k.pre_items.size());
    if (k.has_ft) k.s_queries = pk.add(k.queries.data(), k.queries.size());
    if (k.n_omc && !p->omc) {
        k.s_omcd = pk.add(p->omc_doc_ids, k.n_omc);
        k.s_omcm = pk.add(p->omc_mult, k.n_omc);
    }
    if (k.omc_tile && !p->omc) {
        k.s_omcr = pk.add(k.omc_rows.data(), k.omc_rows.size());
        k.s_omcrm = pk.add(k.omc_row_mult.data(), k.omc_row_mult.size());
    }
    if (!k.has_v) add_first_tables(k);
    if (k.per_q && !k.tok_slot.empty()) k.s_tslot = pk.add(k.tok_slot.data(), k.tok_slot.size());
    Slot<uint64_t> s_pdoc;
    Slot<uint32_t> s_ppos, s_pcnt;
    if (k.pin_items) {
        s_pdoc = pk.add(pj->doc.data(), pj->doc.size());
        s_ppos = pk.add(pj->pos.data(), pj->pos.size());
        s_pcnt = pk.add(pj->cnt.data(), pj->cnt.size());
    }
    if (sj) k.s_sent = pk.add(k.s_ents.data(), k.s_ents.size());
    Slot<GroupHandle> s_ghand;
    Slot<GroupSpan> s_gspan;
    if (gj) {
        s_ghand = pk.add(k.g_hand.data(), k.g_hand.size());
        s_gspan = pk.add(k.g_spans.data(), k.g_spans.size());
    }
    if (k.sort_flat) k.s_sq = pk.add(k.s_q.data(), k.s_q.size());
    if (k.sort_flat && sj->by_score) k.s_salt = pk.add(k.s_alt.data(), k.s_alt.size());
    if (k.qp) {
        k.s_plan = pk.add(k.q_plan.data(), B);
        k.s_page = pk.add(k.q_page.data(), B);
    }
    // (the stream of the fulltext stage, k.side, was chosen by ft_stream)
    if (!k.has_v) CU(cudaEventRecord(c->ev[EV_START], c->stream));
    OCTRY(upload(pk, c->h_in, c->in_blob, k.side ? c->side : c->stream));
    if (!k.has_v) CU(cudaEventRecord(c->ev[EV_H2D], c->stream));   // hybrid/vector: this copy rides inside the device window
    c->timing.h2d_bytes = k.pk0.total + pk.total;
    const DevBuf &din = c->in_blob;
    if (!k.has_v) bind_first_tables(k);
    if (gj) {
        gj->d_hand = s_ghand.at(din);
        gj->d_spans = s_gspan.at(din);
        gj->d_ents = k.s_sent.at(din);
    }
    if (k.pin_items) {
        pj->d_doc = s_pdoc.at(din);
        pj->d_pos = s_ppos.at(din);
        pj->d_cnt = s_pcnt.at(din);
    }
    // arg-max selection (n_keep <= 32) needs no power-of-two buffer; the bitonic fallback does
    // (also >= BM25_SPARSE_MAX: the sparse finish of the posting-centred kernel pushes at most that many candidates)
    const uint32_t n_keep = k.n_keep;
    k.cap = n_keep <= 32 ? std::max<uint32_t>(n_keep + BM25_CHUNK, BM25_SPARSE_MAX)
                         : next_pow2(std::max<uint32_t>(n_keep + BM25_CHUNK, BM25_SPARSE_MAX));
    k.o_sc = size_t(B) * k.limit * 8;
    k.o_n = k.o_sc + size_t(B) * k.limit * 4;
    k.o_cnt = (k.o_n + size_t(B) * 4 + 7) & ~size_t(7);
    k.o_min = k.o_cnt + size_t(B) * 8;
    k.o_gflag = k.o_min + size_t(B) * 4;                       // sharded: OR over the ranks of the per-query overflow flags
    k.out_bytes = k.o_gflag + ((size_t(B) + 3) & ~size_t(3));
    k.o_resc = k.out_bytes + ((size_t(B) + 3) & ~size_t(3));
    k.o_dstat = k.o_resc + size_t(B) * 4;
    OCTRY(c->out_blob.ensure(k.out_bytes));
    OCTRY(c->h_out.ensure(k.o_dstat + 8));
    k.dout = c->out_blob.as<uint8_t>();
    k.d_doc = c->out_blob.as<uint64_t>();
    k.d_score = reinterpret_cast<float *>(k.dout + k.o_sc);
    k.d_n = reinterpret_cast<uint32_t *>(k.dout + k.o_n);
    return OC_OK;
}

// The fulltext stage.  It does not depend on the vector stage (the vector hits' fulltext scores are point lookups
// afterwards): in hybrid mode it runs on the side stream, concurrently with the matrix sweep; the lookups wait only for
// its inputs, and the fusion joins it.  It runs ONCE per call; device_tail (lookups + fusion) is re-runnable.
static int bm25_stage(SearchCall &k) {
    oc_ctx *c = k.c; const oc_search_params *p = k.p;
    const uint32_t B = k.B, n_tiles = k.n_tiles, n_keep = k.n_keep; const StrSnap *S = k.S;
    const DevBuf &din = c->in_blob; cudaStream_t ps = k.side ? c->side : c->stream;
    CU(cudaEventRecord(c->ev[EV_BM0], ps));
    const uint64_t ok_words = uint64_t(n_tiles) * (BM25_TILE / 32);
    if (k.per_q) {   // one row bitmap per distinct filter (tombstones AND filter), then the tombstone-only slot K
        OCTRY(c->row_ok.ensure(std::max<uint64_t>(ok_words, 1) * k.qfj.slots.size() * 4));
        if (ok_words) {
            rows_ok_kernel<<<dim3((unsigned)((ok_words + 255) / 256), (unsigned)k.qfj.slots.size()), 256, 0, ps>>>(
                S->row_doc, S->n_rows, k.tombs ? S->alive : nullptr, nullptr, 0, c->row_ok.as<uint32_t>(), ok_words, k.qfj.d_slots);
            launched(c);
        }
        k.row_ok = c->row_ok.as<uint32_t>();
    } else if (k.filter || k.tombs) {
        OCTRY(c->row_ok.ensure(std::max<uint64_t>(ok_words, 1) * 4));
        if (ok_words) {   // (a shard without string rows still takes part in the df all-reduce below)
            rows_ok_kernel<<<(unsigned)((ok_words + 255) / 256), 256, 0, ps>>>(
                S->row_doc, S->n_rows, k.tombs ? S->alive : nullptr, k.filter_dev, k.filter_nbits,
                c->row_ok.as<uint32_t>(), ok_words);
            launched(c);
        }
        k.row_ok = c->row_ok.as<uint32_t>();
    }
    if (!k.pre_items.empty()) {
        if (k.dense_bytes) CU(cudaMemsetAsync(c->dense_buf.p, 0, k.dense_bytes, ps));
        for (const DenseEntry *e : k.dense_new) CU(cudaMemsetAsync(e->p, 0, e->bytes, ps));
        bm25_precompute_kernel<<<(unsigned)k.pre_items.size(), 256, 0, ps>>>(k.s_pre.at(din), k.s_pitems.at(din), p->bm25_k, k.row_ok);
        launched(c);
        CU(cudaGetLastError());
        for (DenseEntry *e : k.dense_new) e->ready = true;   // later calls may read them (after this stream's work)
    }
    // the hybrid point lookups read the descriptors, the row bitmap and the dense / precomputed contributions, all on
    // the device from here: device_tail starts them under the tile scorer instead of behind it
    if (k.side) CU(cudaEventRecord(c->ev_side_in, c->side));
    const size_t n_td = k.terms.size();
    OCTRY(c->seg.ensure((n_td * (size_t(n_tiles) + 1) + 1) * 4));
    if (n_td) {
        const uint64_t work = uint64_t(n_td) * (n_tiles + 1);
        bm25_plan_kernel<<<(unsigned)((work + 255) / 256), 256, 0, ps>>>(k.s_terms.at(din), (uint32_t)n_td, n_tiles, c->seg.as<uint32_t>());
        launched(c);
    }
    if (k.need_df) {   // (never on the side stream)
        // corpus_df by counting (token_score.rs:262-275), then idf on the host
        const size_t ntok = k.tokens.size();
        OCTRY(c->df_dev.ensure(ntok * 4));
        CU(cudaMemsetAsync(c->df_dev.p, 0, ntok * 4, c->stream));
        DfParams dp{};
        dp.terms = k.s_terms.at(din);
        dp.tokens = k.s_tokens.at(din);
        dp.n_tokens = (uint32_t)ntok; dp.n_tiles = n_tiles; dp.seg = c->seg.as<uint32_t>();
        dp.row_ok_bits = k.row_ok; dp.df = c->df_dev.as<unsigned int>();
        if (k.per_q) { dp.tok_ok_slot = k.s_tslot.at(din); dp.ok_words = ok_words; }
        if (n_tiles && ntok) {
            bm25_df_kernel<<<(unsigned)(uint64_t(n_tiles) * ntok), BM25_THREADS, 0, c->stream>>>(dp);
            launched(c);
        }
        if (k.multi_rank) {   // corpus df = sum of the shards' counts (disjoint documents)
            std::string err;
            if (!c->comm.all_reduce_sum_u32(c->df_dev.p, c->df_dev.p, ntok, c->stream, &err)) return fail(OC_ERR_COMM, "%s", err.c_str());
        }
        std::vector<uint32_t> dfh(ntok);
        CU(cudaMemcpyAsync(dfh.data(), c->df_dev.p, ntok * 4, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        const float N = (float)S->document_count;
        for (size_t t = 0; t < ntok; t++)
            if (k.tok_need_df[t]) k.tokens[t].idf = host_idf(N, std::max<uint32_t>(1u, dfh[t]));
        CU(cudaMemcpyAsync(const_cast<TokenDesc *>(k.s_tokens.at(din)), k.tokens.data(), ntok * sizeof(TokenDesc),
                           cudaMemcpyHostToDevice, c->stream));
    }
    const size_t slots = size_t(B) * std::max<uint32_t>(n_tiles, 1);
    OCTRY(c->tau.ensure(size_t(B) * 16 + 16));   // [tau B x 8][min_hint B x 8][work counter]: one memset
    OCTRY(c->cand_key.ensure(slots * n_keep * 8));
    OCTRY(c->cand_ft.ensure(slots * n_keep * 4));
    OCTRY(c->cand_cnt.ensure(slots * 4));
    OCTRY(c->tile_cnt.ensure(slots * 4));
    OCTRY(c->tile_max.ensure(slots * 4));
    OCTRY(c->tile_min.ensure(slots * 4));
    k.min_hint_dev = reinterpret_cast<float *>(c->tau.as<uint8_t>() + size_t(B) * 8);
    k.tile_counter = reinterpret_cast<unsigned int *>(c->tau.as<uint8_t>() + size_t(B) * 16);
    CU(cudaMemsetAsync(c->tau.p, 0, size_t(B) * 16 + 16, ps));
    Bm25Params &bp = k.bp;
    bp.terms = k.s_terms.at(din);
    bp.tokens = k.s_tokens.at(din);
    bp.queries = k.s_queries.at(din);
    bp.term_token = k.s_ttok.at(din);
    bp.seg = c->seg.as<uint32_t>();
    bp.n_queries = B; bp.n_tiles = n_tiles; bp.n_rows = S->n_rows;
    bp.k = p->bm25_k;
    bp.row_ok_bits = k.row_ok;
    if (k.per_q) { bp.q_ok_slot = k.qfj.d_q_slot_ft; bp.ok_words = ok_words; }
    bp.omc_row = p->omc ? k.omc_row_dev : k.s_omcr.at(din);
    bp.omc_mult = p->omc ? k.omc_row_mult_dev : k.s_omcrm.at(din);
    bp.n_omc = k.n_omc_rows;
    bp.min_hint = k.min_hint_dev;
    bp.n_keep = n_keep; bp.cap = k.cap;
    bp.tau = c->tau.as<unsigned long long>();
    bp.cand_key = c->cand_key.as<uint64_t>(); bp.cand_ft = c->cand_ft.as<float>();
    bp.cand_cnt = c->cand_cnt.as<uint32_t>(); bp.tile_count = c->tile_cnt.as<uint32_t>();
    bp.tile_max = c->tile_max.as<float>(); bp.tile_min = c->tile_min.as<float>();
    bp.dense_stat = k.tile_counter + 2;   // (zeroed with the thresholds)
    const SearchReq &r = k.r;
    if (r.fj || r.gj || r.sj) {   // facets / groups / sortBy: the tile kernels also emit the bitmap of matched rows (every (query, tile) item writes its 256 words)
        OCTRY(c->mbits.ensure(size_t(B) * std::max<uint32_t>(n_tiles, 1) * (BM25_TILE / 32) * 4));
        bp.matched_bits = c->mbits.as<uint32_t>();
    }
    if (r.gj && n_tiles) {   // groups: and the raw score of each matched row
        OCTRY(c->row_ft.ensure(size_t(B) * n_tiles * BM25_TILE * 4));
        bp.row_ft = c->row_ft.as<float>();
    }
    if (n_tiles) OCTRY(launch_tile(c, bp, n_tiles * B, k.any_multi, k.thr, k.omc_tile, ps, k.max_tokens, k.tile_counter, k.need_df));
    CU(cudaEventRecord(c->ev[EV_BM1], ps));
    c->timing.bm25_postings = k.postings_walked;
    if (k.side) CU(cudaEventRecord(c->ev_side, c->side));   // (joined in device_tail, after the point lookups)
    return OC_OK;
}

// The fulltext scores of n_slots string rows ([B][stride], RANK_NONE: none), by point lookups into the postings.
static void point_lookup(SearchCall &k, const uint32_t *rows, uint32_t stride, float *out_ft, uint8_t *out_present, uint64_t n_slots) {
    PointParams pp{};
    pp.terms = k.bp.terms; pp.tokens = k.bp.tokens; pp.queries = k.bp.queries;
    pp.n_queries = k.B; pp.v_stride = stride; pp.v_row = rows; pp.row_ok_bits = k.row_ok;
    pp.q_ok_slot = k.per_q ? k.qfj.d_q_slot_ft : nullptr; pp.ok_words = uint64_t(k.n_tiles) * (BM25_TILE / 32);
    pp.k = k.p->bm25_k; pp.threshold = k.thr ? 1 : 0;
    pp.v_ft = out_ft; pp.v_present = out_present;
    bm25_point_kernel<<<(unsigned)((n_slots * 32 + 255) / 256), 256, 0, k.c->stream>>>(pp);
    launched(k.c);
}

// The score-map values of [B][stride] documents (cnt[q] per query), from K4's exports and their fulltext scores.
static void pin_scores(SearchCall &k, uint32_t stride, const uint64_t *doc, const uint32_t *cnt, const float *ft,
                       const uint8_t *ft_present, float *out_score, uint8_t *out_present) {
    const FuseParams &fp = k.fp;
    PinScoreParams sp{};
    sp.n_queries = k.B; sp.stride = stride; sp.doc = doc; sp.cnt = cnt;
    sp.has_ft = k.has_ft; sp.hybrid = k.has_ft && k.has_v;
    sp.ft = ft; sp.ft_present = ft_present;
    sp.gmin = fp.out_gmin; sp.den = fp.out_den;
    sp.v_doc = fp.out_vdoc; sp.v_score = fp.out_vscore; sp.v_n = fp.out_vn; sp.v_stride = std::max<uint32_t>(k.vlimit, 1);
    sp.omc_doc = fp.omc_doc; sp.omc_mult = fp.omc_mult; sp.n_omc = k.n_omc;
    sp.out_score = out_score; sp.out_present = out_present;
    sp.q_plan = k.s_plan.at(k.c->in_blob);
    pin_score_kernel<<<(unsigned)((uint64_t(k.B) * stride * 32 + 255) / 256), 256, 0, k.c->stream>>>(sp);
    launched(k.c);
}

// pins, after K4: the score-map value of every promoted document, then (pin_flat) the splice into K4's top list
static int pin_tail(SearchCall &k) {
    if (!k.pin_items) return OC_OK;
    oc_ctx *c = k.c; const PinJob *pj = k.r.pj;
    const uint32_t B = k.B, ps = pj->stride;
    const uint64_t nslot = uint64_t(B) * ps;
    OCTRY(c->pin_score.ensure(nslot * 4));
    OCTRY(c->pin_present.ensure(nslot));
    if (k.has_ft) {   // the promoted documents' string rows and their fulltext scores (the hybrid lookups' kernels)
        OCTRY(c->pin_row.ensure(nslot * 4));
        OCTRY(c->pin_ft.ensure(nslot * 4));
        OCTRY(c->pin_ftp.ensure(nslot));
        map_docs_to_rows_kernel<<<(unsigned)((nslot + 255) / 256), 256, 0, c->stream>>>(
            pj->d_doc, pj->d_cnt, ps, B, k.S->row_doc, k.S->n_rows, c->pin_row.as<uint32_t>());
        launched(c);
        point_lookup(k, c->pin_row.as<uint32_t>(), ps, c->pin_ft.as<float>(), c->pin_ftp.as<uint8_t>(), nslot);
    }
    pin_scores(k, ps, pj->d_doc, pj->d_cnt, c->pin_ft.as<float>(), c->pin_ftp.as<uint8_t>(), c->pin_score.as<float>(),
               c->pin_present.as<uint8_t>());
    if (k.pin_flat) {
        PinSpliceParams xp{};
        xp.stride = ps; xp.kp2 = std::max<uint32_t>(32, next_pow2(ps));
        xp.doc = pj->d_doc; xp.pos = pj->d_pos; xp.score = c->pin_score.as<float>(); xp.cnt = pj->d_cnt;
        xp.n_top = k.n_keep; xp.limit = k.limit; xp.offset = k.p->offset;
        xp.top_doc = c->pin_top_doc.as<uint64_t>(); xp.top_score = c->pin_top_score.as<float>(); xp.top_n = c->pin_top_n.as<uint32_t>();
        xp.out_doc = k.d_doc; xp.out_score = k.d_score; xp.out_n = k.d_n;
        xp.q_page = k.s_page.at(c->in_blob);
        const size_t smem = pin_splice_smem(xp.kp2, k.n_keep, k.qp ? k.page_max : k.limit + k.p->offset);
        pin_splice_kernel<<<B, PIN_THREADS, smem, c->stream>>>(xp);
        launched(c);
    }
    CU(cudaGetLastError());
    return OC_OK;
}

// sortBy, after K4 and the pins' scores: the first sort_top keys in field order, scored like promoted documents,
// then paged with the pins spliced (pin_splice_kernel writes the hits over K4's)
static int sort_tail(SearchCall &k) {
    if (!k.sort_flat) return OC_OK;
    oc_ctx *c = k.c; const SortJob *sj = k.r.sj;
    const PinJob *pj = k.r.pj;
    const uint32_t B = k.B, n_tiles = k.n_tiles, n_keep = k.n_keep, limit = k.limit, offset = k.p->offset;
    const DevBuf &din = c->in_blob;
    if (k.has_ft && n_tiles > 0)
        for (uint32_t e = 0; e < sj->f.size(); e++) OCTRY(sort_rows_for(c, sj->ord(e), k.snap));
    const uint32_t top = k.sort_top;
    const uint64_t nslot = uint64_t(B) * top;
    const uint32_t vs = std::max<uint32_t>(k.vlimit, 1);
    OCTRY(c->srt_doc.ensure(nslot * 8));
    OCTRY(c->srt_row.ensure(nslot * 4));
    OCTRY(c->srt_n.ensure(size_t(B) * 4));
    OCTRY(c->srt_score.ensure(nslot * 4));
    OCTRY(c->srt_present.ensure(nslot));
    SortWalkParams wp{};
    wp.ents = k.s_sent.at(din); wp.q = k.s_sq.at(din);
    wp.mbits = k.has_ft && n_tiles > 0 ? c->mbits.as<uint32_t>() : nullptr; wp.row_words = uint64_t(n_tiles) * (BM25_TILE / 32);
    wp.v_doc = k.fp.out_vdoc; wp.v_n = k.fp.out_vn; wp.v_stride = vs;
    wp.top = top;
    wp.out_doc = c->srt_doc.as<uint64_t>(); wp.out_row = c->srt_row.as<uint32_t>(); wp.out_n = c->srt_n.as<uint32_t>();
    sort_walk_kernel<<<B, SORT_THREADS, size_t(vs) * 4, c->stream>>>(wp);
    launched(c);
    if (k.has_ft) {   // the selected rows' fulltext scores (RANK_NONE rows: vector hits without a row, empty slots)
        OCTRY(c->srt_ft.ensure(nslot * 4));
        OCTRY(c->srt_ftp.ensure(nslot));
        point_lookup(k, c->srt_row.as<uint32_t>(), top, c->srt_ft.as<float>(), c->srt_ftp.as<uint8_t>(), nslot);
    }
    pin_scores(k, top, c->srt_doc.as<uint64_t>(), c->srt_n.as<uint32_t>(), c->srt_ft.as<float>(), c->srt_ftp.as<uint8_t>(),
               c->srt_score.as<float>(), c->srt_present.as<uint8_t>());
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
    xp.n_top = top; xp.limit = limit; xp.offset = offset;
    xp.top_doc = c->srt_doc.as<uint64_t>(); xp.top_score = c->srt_score.as<float>(); xp.top_n = c->srt_n.as<uint32_t>();
    xp.out_doc = k.d_doc; xp.out_score = k.d_score; xp.out_n = k.d_n;
    if (sj->by_score) {   // the queries in score order splice K4's top n_keep
        xp.q_alt = k.s_salt.at(din); xp.alt_n_top = n_keep;
        xp.alt_doc = c->pin_top_doc.as<uint64_t>(); xp.alt_score = c->pin_top_score.as<float>(); xp.alt_n = c->pin_top_n.as<uint32_t>();
    }
    xp.q_page = k.s_page.at(din);
    pin_splice_kernel<<<B, PIN_THREADS, pin_splice_smem(xp.kp2, sj->by_score ? std::max(top, n_keep) : top, k.qp ? k.page_max : limit + offset),
                        c->stream>>>(xp);
    launched(c);
    CU(cudaGetLastError());
    return OC_OK;
}

// K4 (fusion + top-n), then the pins and the sortBy walk that read its exports
static int fuse_and_tails(SearchCall &k) {
    void (*fuse)(const FuseParams) = k.exports ? fuse_topk_kernel<true> : fuse_topk_kernel<false>;
    fuse<<<k.B, 256, k.fuse_smem, k.c->stream>>>(k.fp);
    launched(k.c);
    CU(cudaGetLastError());
    OCTRY(pin_tail(k));
    return sort_tail(k);
}

// K4 and its tails, or on a sharded search the pack, the exchange of the shard records and the merge
static int fuse_or_merge(SearchCall &k) {
    oc_ctx *c = k.c;
    if (!(k.p->sharded && c->comm.world > 1)) return fuse_and_tails(k);
    const bool has_v = k.has_v;
    OCTRY(run_sharded_merge(c, k.p, k.fp, k.has_ft ? (uint32_t)k.S->n_rows : 0, has_v ? (uint32_t)k.emb->n_rows : 0, k.B,
                            (has_v && c->gemm_pending) ? c->g_flag.as<uint8_t>() : nullptr, k.dout + k.o_gflag));
    k.did_comm = true;
    return OC_OK;
}

// The hybrid lookups, the fusion and what follows it (+ the shard exchange).  Re-runnable.
static int device_tail(SearchCall &k) {
    oc_ctx *c = k.c; const oc_search_params *p = k.p;
    const uint32_t B = k.B, vlimit = k.vlimit, n_keep = k.n_keep; const bool has_ft = k.has_ft, has_v = k.has_v;
    const StrSnap *S = k.S;
    if (has_ft && has_v) {
        // hybrid: vector hits -> string rows -> their fulltext scores (point lookups)
        OCTRY(c->v_srow.ensure(size_t(B) * vlimit * 4));
        OCTRY(c->v_ft.ensure(size_t(B) * vlimit * 4));
        OCTRY(c->v_present.ensure(size_t(B) * vlimit));
        if (vlimit) {
            // side stream: the lookups' inputs are up (ev_side_in), the tile scorer may still run; they do not read its
            // outputs, so they run under it rather than after the join below
            if (k.side) CU(cudaStreamWaitEvent(c->stream, c->ev_side_in, 0));
            map_docs_to_rows_kernel<<<(B * vlimit + 255) / 256, 256, 0, c->stream>>>(
                c->v_doc.as<uint64_t>(), c->v_cnt.as<uint32_t>(), vlimit, B, S->row_doc, S->n_rows, c->v_srow.as<uint32_t>());
            launched(c);
            point_lookup(k, c->v_srow.as<uint32_t>(), vlimit, c->v_ft.as<float>(), c->v_present.as<uint8_t>(), uint64_t(B) * vlimit);
            CU(cudaGetLastError());
        }
    }
    if (k.side) {   // join: the fusion needs the tiles (side stream); a re-run waits again on the same, complete, record
        CU(cudaStreamWaitEvent(c->stream, c->ev_side, 0));
        c->side_dirty = false;
    }
    FuseParams &fp = k.fp;
    fp = FuseParams{};
    fp.mode = k.mode; fp.n_tiles = k.n_tiles; fp.n_keep = n_keep; fp.limit = k.limit; fp.offset = p->offset;
    fp.q_plan = k.s_plan.at(c->in_blob);
    {   // smallest power-of-two key buffer that takes the candidates in one round (sort cost ~ capb log^2 capb)
        const uint64_t total = (has_ft ? uint64_t(k.n_tiles) * n_keep : 0) + (has_v ? vlimit : 0);
        // up to 16 K keys (128 KB) stay in shared memory and go through one radix select; the streaming bitonic path behind
        // it is for larger candidate sets (the 10M-document fulltext workload has 1221 tiles x 10 candidate slots per query)
        fp.capb = next_pow2((uint32_t)std::min<uint64_t>(16384, std::max<uint64_t>(total, 2 * n_keep)));
        fp.capb = std::max<uint32_t>(fp.capb, std::max<uint32_t>(64, next_pow2(2 * n_keep)));
    }
    if (has_ft) {
        const Bm25Params &bp = k.bp;
        fp.cand_key = bp.cand_key; fp.cand_ft = bp.cand_ft; fp.cand_cnt = bp.cand_cnt; fp.tile_count = bp.tile_count;
        fp.tile_max = bp.tile_max; fp.tile_min = bp.tile_min; fp.str_row_doc_ids = S->row_doc;
    }
    if (has_v) {
        fp.v_doc = c->v_doc.as<uint64_t>(); fp.v_score = c->v_score.as<float>(); fp.v_count = c->v_cnt.as<uint32_t>();
        fp.v_row = has_ft ? c->v_srow.as<uint32_t>() : nullptr;
        fp.v_ft = c->v_ft.as<float>(); fp.v_present = c->v_present.as<uint8_t>();
    }
    fp.v_stride = vlimit;
    fp.omc_doc = p->omc ? k.omc_doc : k.s_omcd.at(c->in_blob);
    fp.omc_mult = p->omc ? k.omc_mult : k.s_omcm.at(c->in_blob);
    fp.n_omc = k.n_omc;
    fp.out_doc = k.d_doc; fp.out_score = k.d_score; fp.out_n = k.d_n;
    fp.out_count = reinterpret_cast<unsigned long long *>(k.dout + k.o_cnt);
    fp.out_min = reinterpret_cast<float *>(k.dout + k.o_min);
    if (k.k4_top) {   // K4 keeps its whole top n_keep for the splice, which writes the hits
        fp.limit = n_keep; fp.offset = 0;
        OCTRY(c->pin_top_doc.ensure(size_t(B) * n_keep * 8));
        OCTRY(c->pin_top_score.ensure(size_t(B) * n_keep * 4));
        OCTRY(c->pin_top_n.ensure(size_t(B) * 4));
        fp.out_doc = c->pin_top_doc.as<uint64_t>(); fp.out_score = c->pin_top_score.as<float>(); fp.out_n = c->pin_top_n.as<uint32_t>();
    }
    if (k.exports) {   // groups / pins: K4 also exports the normalisation and the vector part of the score map
        const uint32_t vs = std::max<uint32_t>(vlimit, 1);
        OCTRY(c->grp_vdoc.ensure(size_t(B) * vs * 8));
        OCTRY(c->grp_vscore.ensure(size_t(B) * vs * 4));
        OCTRY(c->grp_vn.ensure(size_t(B) * 4));
        OCTRY(c->grp_gmin.ensure(size_t(B) * 4));
        OCTRY(c->grp_den.ensure(size_t(B) * 4));
        fp.out_vdoc = c->grp_vdoc.as<uint64_t>(); fp.out_vscore = c->grp_vscore.as<float>(); fp.out_vn = c->grp_vn.as<uint32_t>();
        fp.out_gmin = c->grp_gmin.as<float>(); fp.out_den = c->grp_den.as<float>();
    }
    k.fuse_smem = size_t(fp.capb) * 8 + size_t(std::max<uint32_t>(32, next_pow2(n_keep))) * 8 + size_t(vlimit) * 16 + 64;
    const void *fuse = k.exports ? (const void *)fuse_topk_kernel<true> : (const void *)fuse_topk_kernel<false>;
    CU(smem_cfg(c->device, fuse, k.fuse_smem));
    CU(cudaEventRecord(c->ev[EV_FUSE0], c->stream));
    OCTRY(fuse_or_merge(k));
    CU(cudaEventRecord(c->ev[EV_FUSE1], c->stream));
    return OC_OK;
}

// The results (and the tensor-core scan's overflow flags) to the host, then the re-runs they ask for: the tensor-core
// scan's overflowed queries, and the hybrid rank proxy.
static int rerun_checks(SearchCall &k) {
    oc_ctx *c = k.c; const oc_search_params *p = k.p;
    const uint32_t B = k.B; uint8_t *h = c->h_out.as<uint8_t>();
    CU(cudaEventRecord(c->ev[EV_DEV], c->stream));
    CU(cudaMemcpyAsync(h, k.dout, k.out_bytes, cudaMemcpyDeviceToHost, c->stream));
    if (c->gemm_pending) {   // (per the Bv queries the vector stage swept)
        CU(cudaMemcpyAsync(h + k.out_bytes, c->g_flag.p, k.Bv, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(h + k.o_resc, c->g_resc.p, size_t(k.Bv) * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    const bool dstat = k.has_ft && k.n_tiles;   // the scorer's dense-pass counters (Bm25Params::dense_stat)
    if (dstat) CU(cudaMemcpyAsync(h + k.o_dstat, k.tile_counter + 2, 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaEventRecord(c->ev[EV_D2H], c->stream));
    CU(cudaStreamSynchronize(c->stream));
    c->timing.bm25_dense_items = dstat ? reinterpret_cast<const uint32_t *>(h + k.o_dstat)[0] : 0u;
    c->timing.bm25_dense_skipped = dstat ? reinterpret_cast<const uint32_t *>(h + k.o_dstat)[1] : 0u;
    {   // tensor-core scan: re-run the (rare) queries whose candidate buffers overflowed
        // sharded: every rank must enter the collective the same number of times, so the decision to re-run is
        // taken on the flags all ranks exchanged inside the shard records (no host sync before the collective),
        // by every rank — also one whose own shard was served by the exact sweep
        bool rerun = false;
        if (k.did_comm && k.has_v) for (uint32_t q = 0; q < B; q++) rerun = rerun || h[k.o_gflag + q] != 0;
        uint32_t redone = 0;
        if (c->gemm_pending || rerun) CU(cudaEventRecord(c->ev[EV_RR0], c->stream));
        if (c->gemm_pending) {
            const uint32_t Bv = k.Bv;
            uint64_t resc = 0;
            for (uint32_t q = 0; q < Bv; q++) resc += reinterpret_cast<const uint32_t *>(h + k.o_resc)[q];
            c->timing.scan_rescored = (uint32_t)(resc / Bv);
            OCTRY(fix_unproven(c, k.emb, h + k.out_bytes, Bv, k.vlimit, p->similarity, &redone));
        }
        if (redone || rerun) {
            c->gemm_pending = false;
            OCTRY(device_tail(k));
            CU(cudaMemcpyAsync(h, k.dout, k.out_bytes, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaEventRecord(c->ev[EV_RR1], c->stream));
            c->rerun_timed = true;
            CU(cudaStreamSynchronize(c->stream));
        }
    }
    // rank-proxy validation: with OMC multipliers the tile ranking assumed min == min_hint (0);
    // a negative global min changes the order of (ft - min) * omc -> rerun with the real min.
    // The hybrid point lookups do not depend on the tiles: they are not redone.
    // Sharded: the re-run re-enters the collective, so every rank decides on what all ranks share — the merged min,
    // the batch's mode and whether it carries OMC — never on its own shard's OMC rows or tiles.  A rank whose shard
    // has neither re-launches no tile, but packs, exchanges and merges again.
    const bool proxy = k.mode == OC_MODE_HYBRID && (k.did_comm ? k.n_omc > 0 : k.omc_tile && k.n_tiles);
    if (proxy) {
        const float *mins = reinterpret_cast<const float *>(h + k.o_min);
        std::vector<float> hyb_mins;   // per-query parameters: only the hybrid queries rank by (ft - min)
        if (k.qp) {
            hyb_mins.assign(mins, mins + B);
            for (uint32_t q = 0; q < B; q++) if (k.q_plan[q].mode != OC_MODE_HYBRID) hyb_mins[q] = 0.f;
            mins = hyb_mins.data();
        }
        bool redo = false;
        for (uint32_t q = 0; q < B; q++) redo = redo || mins[q] < 0.f;
        if (redo) {
            if (k.omc_tile && k.n_tiles) {
                CU(cudaMemcpyAsync(k.min_hint_dev, mins, size_t(B) * 4, cudaMemcpyHostToDevice, c->stream));
                CU(cudaMemsetAsync(c->tau.p, 0, size_t(B) * 8, c->stream));
                CU(cudaMemsetAsync(k.tile_counter, 0, 8, c->stream));
                OCTRY(launch_tile(c, k.bp, k.n_tiles * B, k.any_multi, k.thr, k.omc_tile, c->stream, k.max_tokens, k.tile_counter, k.need_df));
            }
            OCTRY(fuse_or_merge(k));
            CU(cudaMemcpyAsync(h, k.dout, k.out_bytes, cudaMemcpyDeviceToHost, c->stream));
            CU(cudaStreamSynchronize(c->stream));
        }
    }
    return OC_OK;
}

// the value a listed document was placed by: its sort value, NaN in score order
static double value_of(const SearchCall &k, uint32_t q, uint64_t d) {
    return k.r.sj ? sort_value_of(*k.r.sj, k.r.pj, q, d) : std::numeric_limits<double>::quiet_NaN();
}

// Facets and groups (on the final score map), then every output to the caller, and the call's timing.
static int copy_out(SearchCall &k) {
    oc_ctx *c = k.c; const SearchReq &r = k.r;
    const PinJob *pj = r.pj; GroupJob *gj = r.gj;
    const uint32_t B = k.B, limit = k.limit; const uint8_t *h = c->h_out.as<uint8_t>();
    if (k.facets) OCTRY(run_facets(c, *r.fj, k.fpl, B, k.has_ft, k.has_v, k.S, k.n_tiles, k.vlimit));
    if (gj) {
        CU(cudaEventRecord(c->ev[EV_GRP0], c->stream));
        OCTRY(run_groups(c, *gj, k.mode, k.S, k.n_tiles, k.vlimit, k.fp.omc_doc, k.fp.omc_mult, k.n_omc, *pj, k.s_plan.at(c->in_blob)));
        CU(cudaEventRecord(c->ev[EV_GRP1], c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    std::vector<float> pin_sc;
    std::vector<uint8_t> pin_pr;
    if (k.pin_items && (pj->out_scores || pj->out_present)) {
        pin_sc.resize(pj->doc.size());
        pin_pr.resize(pj->doc.size());
        CU(cudaMemcpyAsync(pin_sc.data(), c->pin_score.p, pin_sc.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(pin_pr.data(), c->pin_present.p, pin_pr.size(), cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    c->timing.d2h_bytes = k.out_bytes;
    if (k.write_hits) {
        memcpy(r.out_doc_ids, h, size_t(B) * limit * 8);
        memcpy(r.out_scores, h + k.o_sc, size_t(B) * limit * 4);
        memcpy(r.out_n, h + k.o_n, size_t(B) * 4);
    }
    memcpy(r.out_count, h + k.o_cnt, size_t(B) * 8);
    if (k.write_hits && r.out_sort_values)
        for (uint32_t q = 0; q < B; q++)
            for (uint32_t i = 0; i < limit; i++) {
                const size_t o = size_t(q) * limit + i;
                r.out_sort_values[o] = i < r.out_n[q] ? value_of(k, q, r.out_doc_ids[o]) : 0.0;
            }
    if (gj && gj->out_values)   // run_groups' copies are complete (synchronised above)
        for (uint32_t q = 0; q < B; q++) {
            if (gj->q_h[q] == GROUP_NONE) continue;
            const uint32_t G = gj->h[gj->q_h[q]]->n_groups;
            for (size_t row = gj->q_row[q]; row < size_t(gj->q_row[q]) + G; row++)
                for (uint32_t i = 0; i < gj->stride; i++) {
                    const size_t o = row * gj->stride + i;
                    gj->out_values[o] = i < gj->out_n[row] ? value_of(k, q, gj->out_doc[o]) : 0.0;
                }
        }
    if (!pin_sc.empty())
        for (uint32_t q = 0; q < B; q++)
            for (uint32_t j = 0; j < pj->cnt[q]; j++) {
                const size_t i = size_t(pj->pins->q_pin_offsets[q]) + j, s = size_t(q) * pj->stride + j;
                if (pj->out_scores) pj->out_scores[i] = pin_sc[s];
                if (pj->out_present) pj->out_present[i] = pin_pr[s];
            }
    OCTRY(finish_timing(c, k.has_v && k.vlimit && k.emb->n_rows > 0, k.has_ft, true, k.did_comm));
    if (gj) {   // the group stage is device work of this call too
        float ms = 0.f;
        CU(cudaEventElapsedTime(&ms, c->ev[EV_GRP0], c->ev[EV_GRP1]));
        c->timing.device_ms += ms;
    }
    return OC_OK;
}

static int where_stage(SearchCall &k);

// The stages of one search under the ctx lock, up to its results in the ctx's output blob (k.dout) and workspaces.
static int search_stages(SearchCall &k) {
    oc_ctx *c = k.c; const SearchReq &r = k.r;
    // facets: the requests resolved to their distinct document slices (the work list goes up with the first upload)
    if (k.facets) OCTRY(facet_plan(*r.fj, k.fpl));
    begin_call(c);
    if (k.p->q_where) OCTRY(where_stage(k));
    OCTRY(vector_first(k));
    OCTRY(ft_descriptors(k));
    OCTRY(ft_stream(k));
    if (k.has_ft && !k.per_q) OCTRY(ft_share_dense(k));
    OCTRY(omc_plan(k));
    sort_group_plan(k);
    OCTRY(main_upload(k));
    if (k.has_ft) OCTRY(bm25_stage(k));
    OCTRY(device_tail(k));
    return rerun_checks(k);
}

static int search_impl(oc_ctx *c, oc_emb *emb, oc_str *str, const SearchReq &r) {
    SearchCall k(c, emb, str, r);
    OCTRY(search_check(k));
    if (k.B == 0) return OC_OK;
    // the published snapshot of the string store: grabbed once, immutable for the whole call (a commit may
    // publish the next version meanwhile); taken before the lock so a last reference dies outside it
    k.snap = str ? str_snapshot(str) : nullptr;
    k.S = k.snap.get();
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    OCTRY(search_stages(k));
    return copy_out(k);
}

extern "C" int oc_search(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, uint64_t *out_doc_ids,
                         float *out_scores, uint32_t *out_n, uint64_t *out_count) {
    SearchReq r(p, out_doc_ids, out_scores, out_n, out_count);
    r.q_filters_ok = r.q_params_ok = true;
    return search_impl(c, emb, str, r);
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
    double *d_values = nullptr;            // device: the values of a number field (read by oc_facets_commit_ex)
    std::vector<uint64_t> offsets;         // host: n_variants + 1
    std::vector<double> values;            // host: ascending (number field)
};
// The pending ops of a filter-field handle (oc_facets, oc_geo_field), applied in call order by its next commit.
// Guarded by `mu`; the fields of the handle itself are replaced only by a commit, under the ctx lock.
struct FcIns { uint64_t doc, seq; double value, lat, lon; uint32_t field, variant; bool unique; };
struct FcPending {
    std::mutex mu;
    bool committing = false;
    uint64_t seq = 0, version = 0;
    std::vector<FcIns> ins;
    std::unordered_map<uint64_t, uint64_t> del;                  // doc -> seq of its last delete (every field)
    std::map<std::pair<uint32_t, uint64_t>, uint64_t> clr;       // (field, doc) -> seq of its last clear
    std::vector<uint8_t> number;                                 // per field, as the pending ops see it
    std::vector<uint32_t> n_var;                                 //   (new string_filter keys count at once)
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};   // fc_merge's two device phases
    ~FcPending() {
        if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    }
};
struct oc_facets {
    oc_ctx *ctx;
    uint64_t nbits;                        // DocumentId space [0, nbits)
    std::vector<FacetField> fields;
    FcPending pend;
};

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
        for (auto &fl : f->fields) { cudaFree(fl.docs); cudaFree(fl.d_values); }
    }
    delete f;
}
static int facets_add(oc_facets *f, FacetField &&fl, const uint64_t *doc_ids, uint32_t *out_field) {
    oc_ctx *c = f->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    std::lock_guard<std::mutex> gp(f->pend.mu);
    if (f->pend.committing) return fail(OC_ERR_INVALID, "a field added while a commit of the store is in flight");
    CU(cudaSetDevice(c->device));
    if (fl.n_docs) {
        cudaError_t e = cudaMalloc(&fl.docs, fl.n_docs * 8);
        if (e == cudaSuccess) e = cudaMemcpy(fl.docs, doc_ids, fl.n_docs * 8, cudaMemcpyHostToDevice);
        if (e == cudaSuccess && fl.number) e = cudaMalloc(&fl.d_values, fl.n_docs * 8);
        if (e == cudaSuccess && fl.number) e = cudaMemcpy(fl.d_values, fl.values.data(), fl.n_docs * 8, cudaMemcpyHostToDevice);
        if (e != cudaSuccess) {
            cudaFree(fl.docs); cudaFree(fl.d_values);
            return fail(e == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "facet field upload: %s", cudaGetErrorString(e));
        }
    }
    f->pend.number.push_back(fl.number);
    f->pend.n_var.push_back(fl.number ? 0u : uint32_t(fl.offsets.size() - 1));
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
    // each variant's documents ascending, the order oc_facets_commit_ex merges into (a slice is read as a set)
    std::vector<uint64_t> sorted;
    for (uint32_t v = 0; v < n_variants && sorted.empty(); v++)
        if (!std::is_sorted(doc_ids + variant_offsets[v], doc_ids + variant_offsets[v + 1])) sorted.assign(doc_ids, doc_ids + fl.n_docs);
    for (uint32_t v = 0; v < n_variants && !sorted.empty(); v++)
        std::sort(sorted.begin() + variant_offsets[v], sorted.begin() + variant_offsets[v + 1]);
    return facets_add(f, std::move(fl), sorted.empty() ? doc_ids : sorted.data(), out_field);
}
extern "C" int oc_facets_add_number_field(oc_facets *f, uint64_t n, const double *values_sorted, const uint64_t *doc_ids,
                                          uint32_t *out_field) {
    if (!f || (n && (!values_sorted || !doc_ids))) return fail(OC_ERR_INVALID, "bad arguments");
    for (uint64_t i = 1; i < n; i++)
        if (!(values_sorted[i] >= values_sorted[i - 1])) return fail(OC_ERR_INVALID, "values must be ascending (no NaN)");
    FacetField fl;
    fl.number = true; fl.n_docs = n;
    // ascending (value order, document): -0.0 before +0.0 and a run of equal values by document, the order
    // oc_facets_commit_ex merges into (a range is read as a set)
    auto key = [&](uint64_t i) { return std::make_pair(oc::fc_order(values_sorted[i]), doc_ids[i]); };
    bool ordered = true;
    for (uint64_t i = 1; i < n && ordered; i++) ordered = !(key(i) < key(i - 1));
    std::vector<uint64_t> docs;
    if (ordered) {
        fl.values.assign(values_sorted, values_sorted + n);
    } else {
        std::vector<uint64_t> o(n);
        for (uint64_t i = 0; i < n; i++) o[i] = i;
        std::sort(o.begin(), o.end(), [&](uint64_t a, uint64_t b) { return key(a) < key(b); });
        fl.values.resize(n); docs.resize(n);
        for (uint64_t i = 0; i < n; i++) { fl.values[i] = values_sorted[o[i]]; docs[i] = doc_ids[o[i]]; }
    }
    return facets_add(f, std::move(fl), ordered ? doc_ids : docs.data(), out_field);
}

// ------------------------------------------------------------------------------------ filter-field commit (facet_commit.cuh)
static void geo_unit(double lat, double lon, double u[3]);
static bool geo_valid(double lat, double lon);

// One field's merge: the committed entries (kind 0: CSR docs + offsets, 1: number values + docs, 2: geopoint blob) and
// the surviving pending entries, sorted by (key, call order), into new device arrays of the exact size.  Runs on `st`.
enum { FC_CSR = 0, FC_NUMBER = 1, FC_GEO = 2 };
struct FcMergeIn {
    int kind = FC_CSR;
    uint64_t n_a = 0;
    const uint64_t *a_docs = nullptr;          // CSR / number: the committed documents
    const double *a_vals = nullptr;            // number: the committed values; geo: the committed blob
    const std::vector<uint64_t> *old_off = nullptr;
    uint32_t n_var = 0;                        // CSR: variants of the next version (>= old_off->size() - 1)
    std::vector<uint64_t> kill;                // ascending documents whose committed entries go
    std::vector<oc::FcKey> kb;                 // pending keys, sorted
    std::vector<uint32_t> b_keep;              // 1, or 2 for a set-semantics insert
    std::vector<double> b_cols;                // number: n_b values; geo: x, y, z, lat, lon columns of n_b each
};
struct FcMergeOut {
    uint64_t n = 0, kept = 0, added = 0, ws = 0;
    float device_ms = 0;                       // the two device phases (keys .. scans, scatter .. copies), by events
    void *dev = nullptr;                       // CSR / number: docs; geo: the blob
    double *d_values = nullptr;                // number
    std::vector<uint64_t> offsets;             // CSR: n_var + 1
    std::vector<double> values;                // number: the host copy
};
static int fc_merge(cudaStream_t st, cudaEvent_t *ev, const FcMergeIn &in, FcMergeOut &o) {
    using oc::FcKey;
    const uint64_t n_a = in.n_a, n_b = in.kb.size(), n_kill = in.kill.size();
    if (n_a + n_b >= uint64_t(INT32_MAX)) return fail(OC_ERR_UNSUPPORTED, "filter-field commit: %llu entries >= 2^31 - 1",
                                                      (unsigned long long)(n_a + n_b));   // cub::DeviceScan counts in int
    const uint64_t n_oo = in.kind == FC_CSR ? in.old_off->size() : 0, n_no = in.kind == FC_CSR ? uint64_t(in.n_var) + 1 : 0;
    size_t scan_a = 0, scan_b = 0;
    if (cub::DeviceScan::ExclusiveSum(nullptr, scan_a, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)(n_a + 1), st) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)(n_b + 1), st) != cudaSuccess)
        return fail(OC_ERR_CUDA, "filter-field commit: scan size");
    // workspace: [uploaded: kb | kill | b_cols | old_off | b_keep] [ka | a_keep | a_rank | b_rank | new_off | scan]
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t o_kb = 0, o_kill = o_kb + al(n_b * 16), o_cols = o_kill + al(n_kill * 8), o_oo = o_cols + al(in.b_cols.size() * 8),
                 o_bk = o_oo + al(n_oo * 8), up = o_bk + al((n_b + 1) * 4);
    const size_t o_ka = up, o_ak = o_ka + al(n_a * 16), o_ar = o_ak + al((n_a + 1) * 4), o_br = o_ar + al((n_a + 1) * 4),
                 o_no = o_br + al((n_b + 1) * 4), o_scan = o_no + al(n_no * 8), total = o_scan + al(std::max(scan_a, scan_b));
    std::vector<uint8_t> h(up, 0);
    if (n_b) memcpy(h.data() + o_kb, in.kb.data(), n_b * 16);
    if (n_kill) memcpy(h.data() + o_kill, in.kill.data(), n_kill * 8);
    if (!in.b_cols.empty()) memcpy(h.data() + o_cols, in.b_cols.data(), in.b_cols.size() * 8);
    if (n_oo) memcpy(h.data() + o_oo, in.old_off->data(), n_oo * 8);
    if (n_b) memcpy(h.data() + o_bk, in.b_keep.data(), n_b * 4);   // b_keep[n_b] = 0
    uint8_t *w = nullptr;
    if (cudaMallocAsync(&w, total, st) != cudaSuccess) return fail(OC_ERR_OOM, "filter-field commit: %zu B of workspace", total);
    o.ws = total;
    int rc = OC_OK;
    auto done = [&](int r) { cudaFreeAsync(w, st); if (r != OC_OK) { cudaFree(o.dev); cudaFree(o.d_values); o.dev = nullptr; o.d_values = nullptr; } return r; };
    const FcKey *kb = reinterpret_cast<const FcKey *>(w + o_kb);
    const uint64_t *kill = reinterpret_cast<const uint64_t *>(w + o_kill);
    const double *cols = reinterpret_cast<const double *>(w + o_cols);
    const uint64_t *oo = reinterpret_cast<const uint64_t *>(w + o_oo);
    uint32_t *bk = reinterpret_cast<uint32_t *>(w + o_bk), *ak = reinterpret_cast<uint32_t *>(w + o_ak);
    uint32_t *ar = reinterpret_cast<uint32_t *>(w + o_ar), *br = reinterpret_cast<uint32_t *>(w + o_br);
    FcKey *ka = reinterpret_cast<FcKey *>(w + o_ka);
    uint64_t *no = reinterpret_cast<uint64_t *>(w + o_no);
    const unsigned ga = (unsigned)((n_a + oc::FC_THREADS) / oc::FC_THREADS), gb = (unsigned)((n_b + oc::FC_THREADS - 1) / oc::FC_THREADS);
    cudaError_t e = cudaMemcpyAsync(w, h.data(), up, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaEventRecord(ev[0], st);
    if (e == cudaSuccess) {
        if (in.kind == FC_CSR)
            oc::fc_keys_csr_kernel<<<ga, oc::FC_THREADS, 0, st>>>(in.a_docs, n_a, oo, uint32_t(n_oo - 1), kill, n_kill, ka, ak);
        else if (in.kind == FC_NUMBER)
            oc::fc_keys_num_kernel<<<ga, oc::FC_THREADS, 0, st>>>(in.a_vals, in.a_docs, n_a, kill, n_kill, ka, ak);
        else
            oc::fc_keys_geo_kernel<<<ga, oc::FC_THREADS, 0, st>>>(reinterpret_cast<const uint64_t *>(in.a_vals + 5 * n_a), n_a, kill, n_kill, ka, ak);
        if (std::find(in.b_keep.begin(), in.b_keep.end(), 2u) != in.b_keep.end())
            oc::fc_unique_kernel<<<gb, oc::FC_THREADS, 0, st>>>(ka, ak, n_a, kb, n_b, bk);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(w + o_scan, scan_a, ak, ar, (int)(n_a + 1), st);
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(w + o_scan, scan_b, bk, br, (int)(n_b + 1), st);
    uint32_t tot[2] = {0, 0};
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tot[0], ar + n_a, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaEventRecord(ev[1], st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tot[1], br + n_b, 4, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&o.device_ms, ev[0], ev[1]);
    if (e != cudaSuccess) return done(fail(OC_ERR_CUDA, "filter-field commit: %s", cudaGetErrorString(e)));
    o.kept = tot[0]; o.added = tot[1]; o.n = o.kept + o.added;
    const size_t row = in.kind == FC_GEO ? 48 : 8;
    if (o.n && (e = cudaMalloc(&o.dev, o.n * row)) == cudaSuccess && in.kind == FC_NUMBER) e = cudaMalloc(&o.d_values, o.n * 8);
    if (e != cudaSuccess) return done(fail(e == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "filter-field commit: %llu entries: %s",
                                          (unsigned long long)o.n, cudaGetErrorString(e)));
    if ((e = cudaEventRecord(ev[2], st)) != cudaSuccess) return done(fail(OC_ERR_CUDA, "filter-field commit: %s", cudaGetErrorString(e)));
    auto scatter = [&](auto wr) {
        if (n_a) oc::fc_scatter_a_kernel<<<(unsigned)((n_a + oc::FC_THREADS - 1) / oc::FC_THREADS), oc::FC_THREADS, 0, st>>>(ka, ak, ar, n_a, kb, br, n_b, wr);
        if (n_b) oc::fc_scatter_b_kernel<<<gb, oc::FC_THREADS, 0, st>>>(ka, ar, n_a, kb, bk, br, n_b, wr);
    };
    if (o.n) {
        if (in.kind == FC_CSR) scatter(oc::FcCsrW{in.a_docs, kb, static_cast<uint64_t *>(o.dev)});
        else if (in.kind == FC_NUMBER) scatter(oc::FcNumW{in.a_vals, in.a_docs, cols, kb, o.d_values, static_cast<uint64_t *>(o.dev)});
        else scatter(oc::FcGeoW{in.a_vals, n_a, cols, n_b, kb, static_cast<double *>(o.dev), o.n});
    }
    if (in.kind == FC_CSR) {
        oc::fc_offsets_kernel<<<(unsigned)((n_no + oc::FC_THREADS - 1) / oc::FC_THREADS), oc::FC_THREADS, 0, st>>>(
            oo, uint32_t(n_oo - 1), ar, kb, br, n_b, in.n_var, no);
        o.offsets.resize(n_no);
    }
    e = cudaGetLastError();
    if (e == cudaSuccess && in.kind == FC_CSR) e = cudaMemcpyAsync(o.offsets.data(), no, n_no * 8, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && in.kind == FC_NUMBER && o.n) {   // the host copy range leaves binary-search, from the merge result
        o.values.resize(o.n);
        e = cudaMemcpyAsync(o.values.data(), o.d_values, o.n * 8, cudaMemcpyDeviceToHost, st);
    }
    if (e == cudaSuccess) e = cudaEventRecord(ev[3], st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    float ms2 = 0;
    if (e == cudaSuccess) e = cudaEventElapsedTime(&ms2, ev[2], ev[3]);
    o.device_ms += ms2;
    if (e != cudaSuccess) rc = fail(OC_ERR_CUDA, "filter-field commit: %s", cudaGetErrorString(e));
    return done(rc);
}

// The pending ops of `P` for field `field`, filtered (an insert survives unless a later delete or clear names its
// document; a set-semantics insert also unless an earlier survivor has its key) and keyed; `kill` = the documents whose
// committed entries go.  O(pending log pending).
static void fc_take(const FcPending &P, const std::vector<FcIns> &ins, const std::unordered_map<uint64_t, uint64_t> &del,
                    const std::map<std::pair<uint32_t, uint64_t>, uint64_t> &clr, uint32_t field, int kind, FcMergeIn &in) {
    auto killed_after = [&](uint64_t doc, uint64_t seq) {
        auto d = del.find(doc);
        if (d != del.end() && d->second > seq) return true;
        auto c = clr.find(std::make_pair(field, doc));
        return c != clr.end() && c->second > seq;
    };
    struct KH { size_t operator()(const std::pair<uint64_t, uint64_t> &k) const { return std::hash<uint64_t>()(k.first * 0x9E3779B97F4A7C15ull ^ k.second); } };
    std::unordered_set<std::pair<uint64_t, uint64_t>, KH> seen;
    std::vector<std::pair<oc::FcKey, size_t>> keyed;   // (key, index into ins): ins is in call order
    for (size_t i = 0; i < ins.size(); i++) {
        const FcIns &x = ins[i];
        if (x.field != field || killed_after(x.doc, x.seq)) continue;
        oc::FcKey k = kind == FC_CSR ? oc::FcKey{x.variant, x.doc} : kind == FC_NUMBER ? oc::FcKey{oc::fc_order(x.value), x.doc} : oc::FcKey{x.doc, 0};
        if (!seen.insert(std::make_pair(k.hi, k.lo)).second && x.unique) continue;
        keyed.emplace_back(k, i);
    }
    std::sort(keyed.begin(), keyed.end(), [](const std::pair<oc::FcKey, size_t> &a, const std::pair<oc::FcKey, size_t> &b) {
        return oc::fc_less(a.first, b.first) || (oc::fc_equal(a.first, b.first) && a.second < b.second);
    });
    const size_t n_b = keyed.size();
    in.kb.resize(n_b); in.b_keep.resize(n_b);
    in.b_cols.assign(kind == FC_NUMBER ? n_b : kind == FC_GEO ? 5 * n_b : 0, 0.0);
    for (size_t j = 0; j < n_b; j++) {
        const FcIns &x = ins[keyed[j].second];
        in.kb[j] = keyed[j].first;
        in.b_keep[j] = x.unique ? 2u : 1u;
        if (kind == FC_NUMBER) in.b_cols[j] = x.value;
        if (kind == FC_GEO) {   // the unit vector as oc_geo_field_create computes it, so both give the same bits
            double u[3];
            geo_unit(x.lat, x.lon, u);
            for (int c = 0; c < 3; c++) in.b_cols[c * n_b + j] = u[c];
            in.b_cols[3 * n_b + j] = x.lat; in.b_cols[4 * n_b + j] = x.lon;
        }
    }
    in.kill.clear();
    for (const auto &kv : del) in.kill.push_back(kv.first);
    for (auto it = clr.lower_bound(std::make_pair(field, uint64_t(0))); it != clr.end() && it->first.first == field; ++it)
        in.kill.push_back(it->first.second);
    std::sort(in.kill.begin(), in.kill.end());
    in.kill.erase(std::unique(in.kill.begin(), in.kill.end()), in.kill.end());
    (void)P;
}

// Starts a commit: refuses a second one and a pending document >= new_nbits, then copies the ops to merge.
static int fc_begin(FcPending &P, uint64_t nbits, uint64_t new_nbits, int device, std::vector<FcIns> &ins,
                    std::unordered_map<uint64_t, uint64_t> &del, std::map<std::pair<uint32_t, uint64_t>, uint64_t> &clr, uint64_t &cut) {
    std::lock_guard<std::mutex> g(P.mu);
    if (P.committing) return fail(OC_ERR_INVALID, "a commit of this handle is already in flight");
    if (new_nbits < nbits) return fail(OC_ERR_INVALID, "new_nbits %llu < nbits %llu: the DocumentId space only grows",
                                       (unsigned long long)new_nbits, (unsigned long long)nbits);
    for (const FcIns &x : P.ins)
        if (x.doc >= new_nbits) return fail(OC_ERR_INVALID, "pending document %llu >= new_nbits %llu", (unsigned long long)x.doc,
                                            (unsigned long long)new_nbits);
    if (cudaSetDevice(device) != cudaSuccess) return fail(OC_ERR_CUDA, "cudaSetDevice failed");
    if (!P.stream) {
        CU(cudaStreamCreateWithFlags(&P.stream, cudaStreamNonBlocking));
        for (cudaEvent_t &e : P.ev) CU(cudaEventCreate(&e));
    }
    P.committing = true;
    ins = P.ins; del = P.del; clr = P.clr; cut = P.seq;
    return OC_OK;
}
// Ends a commit: on success the ops it merged leave the queue (ops that arrived meanwhile stay), and the version moves on.
static uint64_t fc_end(FcPending &P, bool ok, size_t n_ins, uint64_t cut) {
    std::lock_guard<std::mutex> g(P.mu);
    P.committing = false;
    if (!ok) return P.version;
    P.ins.erase(P.ins.begin(), P.ins.begin() + n_ins);
    for (auto it = P.del.begin(); it != P.del.end();) it = it->second <= cut ? P.del.erase(it) : std::next(it);
    for (auto it = P.clr.begin(); it != P.clr.end();) it = it->second <= cut ? P.clr.erase(it) : std::next(it);
    return ++P.version;
}
static int fc_queue_check(const FcPending &P, uint32_t field, bool number, uint64_t n, const uint64_t *doc_ids) {
    if (n && !doc_ids) return fail(OC_ERR_INVALID, "NULL doc_ids");
    if (field >= P.number.size()) return fail(OC_ERR_INVALID, "field %u: the store has %zu fields", field, P.number.size());
    if (bool(P.number[field]) != number) return fail(OC_ERR_INVALID, "field %u is a %s field", field, P.number[field] ? "number" : "bool / string_filter");
    return OC_OK;
}

extern "C" int oc_facets_add_variant(oc_facets *f, uint32_t field, uint32_t *variant_out) {
    if (!f || !variant_out) return fail(OC_ERR_INVALID, "NULL argument");
    FcPending &P = f->pend;
    std::lock_guard<std::mutex> g(P.mu);
    OCTRY(fc_queue_check(P, field, false, 0, nullptr));
    if (P.n_var[field] == UINT32_MAX - 1) return fail(OC_ERR_UNSUPPORTED, "field %u: 2^32 - 2 variants", field);
    *variant_out = P.n_var[field]++;
    return OC_OK;
}
extern "C" int oc_facets_insert_variants(oc_facets *f, uint32_t field, uint64_t n, const uint64_t *doc_ids, const uint32_t *variants,
                                         uint32_t flags) {
    if (!f || (n && !variants)) return fail(OC_ERR_INVALID, "NULL argument");
    if (flags & ~OC_FACET_UNIQUE) return fail(OC_ERR_INVALID, "unknown insert flags 0x%x", flags);
    FcPending &P = f->pend;
    std::lock_guard<std::mutex> g(P.mu);
    OCTRY(fc_queue_check(P, field, false, n, doc_ids));
    for (uint64_t i = 0; i < n; i++)
        if (variants[i] >= P.n_var[field]) return fail(OC_ERR_INVALID, "entry %llu: variant %u: field %u has %u variants",
                                                        (unsigned long long)i, variants[i], field, P.n_var[field]);
    for (uint64_t i = 0; i < n; i++) P.ins.push_back(FcIns{doc_ids[i], ++P.seq, 0.0, 0.0, 0.0, field, variants[i], bool(flags & OC_FACET_UNIQUE)});
    return OC_OK;
}
extern "C" int oc_facets_insert_numbers(oc_facets *f, uint32_t field, uint64_t n, const uint64_t *doc_ids, const double *values) {
    if (!f || (n && !values)) return fail(OC_ERR_INVALID, "NULL argument");
    FcPending &P = f->pend;
    std::lock_guard<std::mutex> g(P.mu);
    OCTRY(fc_queue_check(P, field, true, n, doc_ids));
    for (uint64_t i = 0; i < n; i++)
        if (std::isnan(values[i])) return fail(OC_ERR_INVALID, "entry %llu: NaN value", (unsigned long long)i);
    for (uint64_t i = 0; i < n; i++) P.ins.push_back(FcIns{doc_ids[i], ++P.seq, values[i], 0.0, 0.0, field, 0, false});
    return OC_OK;
}
extern "C" int oc_facets_clear(oc_facets *f, uint32_t field, uint64_t n, const uint64_t *doc_ids) {
    if (!f) return fail(OC_ERR_INVALID, "NULL argument");
    FcPending &P = f->pend;
    std::lock_guard<std::mutex> g(P.mu);
    if (n && !doc_ids) return fail(OC_ERR_INVALID, "NULL doc_ids");
    if (field >= P.number.size()) return fail(OC_ERR_INVALID, "field %u: the store has %zu fields", field, P.number.size());
    for (uint64_t i = 0; i < n; i++) P.clr[std::make_pair(field, doc_ids[i])] = ++P.seq;
    return OC_OK;
}
extern "C" int oc_facets_delete(oc_facets *f, uint64_t n, const uint64_t *doc_ids) {
    if (!f || (n && !doc_ids)) return fail(OC_ERR_INVALID, "NULL argument");
    FcPending &P = f->pend;
    std::lock_guard<std::mutex> g(P.mu);
    for (uint64_t i = 0; i < n; i++) P.del[doc_ids[i]] = ++P.seq;
    return OC_OK;
}

extern "C" int oc_facets_commit_ex(oc_facets *f, uint64_t new_nbits, oc_filter_commit_t *out) {
    if (!f) return fail(OC_ERR_INVALID, "NULL argument");
    const auto wall0 = std::chrono::steady_clock::now();
    oc_ctx *c = f->ctx;
    FcPending &P = f->pend;
    std::vector<FcIns> ins;
    std::unordered_map<uint64_t, uint64_t> del;
    std::map<std::pair<uint32_t, uint64_t>, uint64_t> clr;
    uint64_t cut = 0;
    std::vector<uint32_t> n_var;
    {
        std::lock_guard<std::mutex> g(c->mu);   // nbits and the field list change only under it (and not during a commit)
        OCTRY(fc_begin(P, f->nbits, new_nbits, c->device, ins, del, clr, cut));
        std::lock_guard<std::mutex> gp(P.mu);
        n_var = P.n_var;
    }
    // the published fields are not replaced until this commit publishes, so they are read without the ctx lock
    const size_t nf = f->fields.size();
    std::vector<FcMergeOut> res(nf);
    std::vector<bool> fresh(nf, false);
    oc_filter_commit_t st{};
    int rc = OC_OK;
    for (size_t fi = 0; fi < nf && rc == OC_OK; fi++) {
        const FacetField &fl = f->fields[fi];
        FcMergeIn in;
        in.kind = fl.number ? FC_NUMBER : FC_CSR;
        fc_take(P, ins, del, clr, uint32_t(fi), in.kind, in);
        if (in.kb.empty() && in.kill.empty()) {   // unchanged (a CSR field may still gain empty variants)
            st.rows_kept += fl.n_docs;
            continue;
        }
        in.n_a = fl.n_docs; in.a_docs = fl.docs; in.a_vals = fl.d_values; in.old_off = &fl.offsets; in.n_var = n_var[fi];
        rc = fc_merge(P.stream, P.ev, in, res[fi]);
        fresh[fi] = rc == OC_OK;
        st.device_ms += res[fi].device_ms;
        st.rows_kept += res[fi].kept; st.rows_dropped += fl.n_docs - res[fi].kept; st.rows_added += res[fi].added;
        st.workspace_bytes = std::max(st.workspace_bytes, res[fi].ws);
    }
    if (rc != OC_OK) {
        for (size_t fi = 0; fi < nf; fi++) if (fresh[fi]) { cudaFree(res[fi].dev); cudaFree(res[fi].d_values); }
        fc_end(P, false, 0, 0);
        return rc;
    }
    // publish: every reader of the fields holds the ctx lock and works on the ctx stream, so once the stream has
    // drained nothing refers to the previous arrays
    std::vector<void *> old;
    {
        std::lock_guard<std::mutex> g(c->mu);
        cudaSetDevice(c->device);
        for (size_t fi = 0; fi < nf; fi++) {
            FacetField &fl = f->fields[fi];
            if (!fresh[fi]) {
                if (!fl.number) fl.offsets.resize(size_t(n_var[fi]) + 1, fl.offsets.back());
                continue;
            }
            old.push_back(fl.docs); old.push_back(fl.d_values);
            fl.docs = static_cast<uint64_t *>(res[fi].dev); fl.d_values = res[fi].d_values; fl.n_docs = res[fi].n;
            if (fl.number) fl.values.swap(res[fi].values); else fl.offsets.swap(res[fi].offsets);
        }
        f->nbits = new_nbits;
        cudaStreamSynchronize(c->stream);
        for (void *p : old) cudaFree(p);
        // the version number moves with the arrays, so a reader under the ctx lock sees them together
        st.version = fc_end(P, true, ins.size(), cut);
    }
    st.wall_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    if (out) *out = st;
    return OC_OK;
}

extern "C" int oc_facets_read_field(oc_facets *f, uint32_t field, uint32_t *n_variants, uint64_t *n_entries, uint64_t *offsets,
                                    double *values, uint64_t *doc_ids) {
    if (!f || !n_variants || !n_entries) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = f->ctx;
    std::lock_guard<std::mutex> g(c->mu);
    if (field >= f->fields.size()) return fail(OC_ERR_INVALID, "field %u: the store has %zu fields", field, f->fields.size());
    const FacetField &fl = f->fields[field];
    const uint32_t cap_v = *n_variants;
    const uint64_t cap_n = *n_entries;
    *n_variants = fl.number ? 0 : uint32_t(fl.offsets.size() - 1);
    *n_entries = fl.n_docs;
    if (!doc_ids && !offsets && !values) return OC_OK;
    if (((doc_ids || (fl.number && values)) && cap_n < fl.n_docs) || (!fl.number && offsets && cap_v < *n_variants))
        return fail(OC_ERR_INVALID, "arrays hold %llu entries / %u variants, the field has %llu / %u", (unsigned long long)cap_n, cap_v,
                    (unsigned long long)fl.n_docs, *n_variants);
    CU(cudaSetDevice(c->device));
    if (fl.n_docs && doc_ids) CU(cudaMemcpy(doc_ids, fl.docs, fl.n_docs * 8, cudaMemcpyDeviceToHost));
    if (fl.number && values) std::copy(fl.values.begin(), fl.values.end(), values);
    if (!fl.number && offsets) std::copy(fl.offsets.begin(), fl.offsets.end(), offsets);
    return OC_OK;
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
// The work list of the facet counts: block b counts the 1024 documents [1024 (b - block0), ...) of the slice it falls in
// against the bitmap row of every (row, count) pair of that slice.  The chunk is read once however many counts want it.
// The warps' partial counts of up to 32 pairs are summed in shared memory behind one pair of barriers, then one atomic
// per pair and block: a warp-level atomic per pair was measured 9 % slower (the adds contend on the same counters).
__global__ void __launch_bounds__(256) facet_slice_count_kernel(const FacetSliceDev *slices, uint32_t n_slices, const uint2 *pairs,
                                                                const uint32_t *bits, uint64_t stride_words, uint64_t nbits_cap,
                                                                unsigned long long *out) {
    uint32_t lo = 0, hi = n_slices - 1;   // the last slice with block0 <= blockIdx.x
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (slices[mid].block0 <= blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const FacetSliceDev s = slices[lo];
    const uint64_t base = uint64_t(blockIdx.x - s.block0) * 1024;
    uint64_t d[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const uint64_t i = base + threadIdx.x + u * 256;
        const uint64_t v = i < s.n ? s.docs[i] : ~0ull;
        d[u] = v < nbits_cap ? v : ~0ull;
    }
    __shared__ uint32_t s_c[8][32];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (uint32_t k0 = 0; k0 < s.n_pairs; k0 += 32) {
        const uint32_t kn = min(32u, s.n_pairs - k0);
        for (uint32_t k = 0; k < kn; k++) {
            const uint32_t *bq = bits + size_t(pairs[s.pair0 + k0 + k].x) * stride_words;
            uint32_t c = 0;
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (d[u] != ~0ull) c += (bq[d[u] >> 5] >> (d[u] & 31)) & 1u;
            c = __reduce_add_sync(0xffffffffu, c);
            if (lane == 0) s_c[warp][k] = c;
        }
        __syncthreads();
        if (warp == 0 && lane < kn) {
            uint32_t t = 0;
#pragma unroll
            for (int w = 0; w < 8; w++) t += s_c[w][lane];
            if (t) atomicAdd(out + pairs[s.pair0 + k0 + lane].y, (unsigned long long)t);
        }
        __syncthreads();
    }
}

// The slice [lo, hi) of a field's device documents that a where leaf or a facet count selects: variant `arg` of a bool /
// string_filter field, or the values v of a number field with a <= v <= b, an end open under the OC_RANGE_* flags in
// `arg` (a > b: empty).  False: the field has no variant `arg`.
static bool facet_slice(const FacetField &fl, uint32_t arg, double a, double b, uint64_t &lo, uint64_t &hi) {
    if (!fl.number) {
        if (arg + uint64_t(1) >= fl.offsets.size()) return false;
        lo = fl.offsets[arg]; hi = fl.offsets[arg + 1];
        return true;
    }
    const auto &v = fl.values;   // ascending, no NaN
    lo = (arg & OC_RANGE_LO_OPEN) ? std::upper_bound(v.begin(), v.end(), a) - v.begin()
                                  : std::lower_bound(v.begin(), v.end(), a) - v.begin();
    hi = (arg & OC_RANGE_HI_OPEN) ? std::lower_bound(v.begin(), v.end(), b) - v.begin()
                                  : std::upper_bound(v.begin(), v.end(), b) - v.begin();
    hi = std::max(lo, hi);
    return true;
}

// A request's slice [lo, hi) of its field's device documents.  nan: refuse a NaN bound (oc_search_facets passes it on).
static int facet_resolve(const oc_facets *fc, const oc_facet_req &rq, size_t i, bool nan, uint64_t &lo, uint64_t &hi) {
    if (rq.field >= fc->fields.size()) return fail(OC_ERR_INVALID, "facet request %zu: unknown field %u", i, rq.field);
    const FacetField &fl = fc->fields[rq.field];
    if (fl.number && nan && (std::isnan(rq.from) || std::isnan(rq.to))) return fail(OC_ERR_INVALID, "facet request %zu: NaN range bound", i);
    // flags 0: NumberFilter::Between is inclusive on both ends (number_field.rs:376, 604-631)
    if (!facet_slice(fl, fl.number ? 0 : rq.variant, rq.from, rq.to, lo, hi))
        return fail(OC_ERR_INVALID, "facet request %zu: unknown variant %u", i, rq.variant);
    return OC_OK;
}

// Dedupes the job's requests into distinct (field, lo, hi) slices and lists, per slice, the (bitmap row, count) pairs
// that want it.  Empty slices launch nothing: their counts stay 0.  Called under the ctx lock.
static int facet_plan(const FacetJob &fj, FacetPlan &pl) {
    struct Key {
        uint32_t field; uint64_t lo, hi;
        bool operator==(const Key &o) const { return field == o.field && lo == o.lo && hi == o.hi; }
    };
    struct KeyHash { size_t operator()(const Key &k) const { return std::hash<uint64_t>()(k.lo * 0x9E3779B97F4A7C15ull ^ k.hi ^ (uint64_t(k.field) << 40)); } };
    std::unordered_map<Key, uint32_t, KeyHash> idx;
    std::vector<std::vector<uint2>> want;
    for (size_t k = 0; k < fj.q.size(); k++) {
        const oc_facet_req &rq = fj.reqs[fj.r[k]];
        uint64_t lo = 0, hi = 0;
        OCTRY(facet_resolve(fj.fc, rq, fj.r[k], false, lo, hi));
        if (hi == lo) continue;
        auto it = idx.emplace(Key{rq.field, lo, hi}, (uint32_t)pl.slices.size()).first;
        if (it->second == pl.slices.size()) {
            const FacetField &fl = fj.fc->fields[rq.field];
            pl.slices.push_back(FacetSliceDev{fl.docs + lo, hi - lo, 0, 0, 0});
            want.emplace_back();
        }
        want[it->second].push_back(make_uint2(fj.q[k], fj.d_out ? (uint32_t)fj.o[k] : (uint32_t)k));
    }
    uint64_t blocks = 0;
    for (size_t s = 0; s < pl.slices.size(); s++) {
        FacetSliceDev &sd = pl.slices[s];
        sd.block0 = (uint32_t)blocks;
        sd.pair0 = (uint32_t)pl.pairs.size();
        sd.n_pairs = (uint32_t)want[s].size();
        pl.pairs.insert(pl.pairs.end(), want[s].begin(), want[s].end());
        blocks += (sd.n + 1023) / 1024;
        if (blocks > 0x7fffffffull) return fail(OC_ERR_UNSUPPORTED, "facets: %llu document chunks >= 2^31", (unsigned long long)blocks);
    }
    pl.n_blocks = (uint32_t)blocks;
    return OC_OK;
}

static int run_facets(oc_ctx *c, const FacetJob &fj, const FacetPlan &pl, uint32_t B, bool has_ft, bool has_v, const StrSnap *S,
                      uint32_t n_tiles, uint32_t vlimit) {
    oc_facets *fc = fj.fc;
    const size_t n_out = fj.q.size();
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
        if (has_v && vlimit) {   // (limit 0: no vector hit)
            facet_mark_hits_kernel<<<(B * vlimit + 255) / 256, 256, 0, c->stream>>>(c->v_doc.as<uint64_t>(), c->v_cnt.as<uint32_t>(), vlimit, B,
                                                                                  c->dbits.as<uint32_t>(), doc_words, fc->nbits);
            launched(c);
        }
        bits = c->dbits.as<uint32_t>(); stride = doc_words; cap_bits = fc->nbits;
    }
    if (!fj.d_out) {
        OCTRY(c->facet_out.ensure(n_out * 8));
        CU(cudaMemsetAsync(c->facet_out.p, 0, n_out * 8, c->stream));
    }
    if (pl.n_blocks) {
        facet_slice_count_kernel<<<pl.n_blocks, 256, 0, c->stream>>>(pl.d_slices, (uint32_t)pl.slices.size(), pl.d_pairs, bits, stride,
                                                                     cap_bits, fj.d_out ? fj.d_out : c->facet_out.as<unsigned long long>());
        launched(c);
        CU(cudaGetLastError());
    }
    if (fj.d_out) return OC_OK;
    std::vector<uint64_t> counts(n_out);
    CU(cudaMemcpyAsync(counts.data(), c->facet_out.p, n_out * 8, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    for (size_t k = 0; k < n_out; k++) fj.out_counts[fj.o[k]] = counts[k];
    return OC_OK;
}

// The facet pass the reference runs for a request: the score map re-scored WITHOUT the where-filter (search.rs:361-396:
// only the uncommitted deletes stay excluded, and stores tombstone deletes at once), so that the counts do not collapse
// onto the selected category.  The hits of this pass are dropped.
// q_params_ok: the sub-batch pass of oc_search_q_facets (oc_search_facets takes one set of scalars).
static void drop_filters(oc_search_params &q) {
    q.filter_bits = nullptr; q.filter_nbits = 0; q.filter = nullptr; q.q_filters = nullptr; q.q_where = nullptr;
}
// Query b of p has a filter that drop_filters removes: its facets count on the unfiltered pass.
static bool facet_filtered(const oc_search_params *p, uint32_t b) {
    return p->filter || p->filter_bits || (p->q_filters && p->q_filters[b]) ||
           (p->q_where && p->q_where->q_node_offsets && p->q_where->q_node_offsets[b + 1] > p->q_where->q_node_offsets[b]);
}
static int facets_unfiltered(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, FacetJob &fj, bool q_params_ok) {
    oc_search_params q = *p;
    drop_filters(q);
    const uint32_t B = p->n_queries;
    std::vector<uint64_t> docs(size_t(B) * p->limit), cnt(B);
    std::vector<float> scores(size_t(B) * p->limit);
    std::vector<uint32_t> n(B);
    SearchReq r(&q, docs.data(), scores.data(), n.data(), cnt.data());
    r.fj = &fj;
    r.q_filters_ok = true;
    r.q_params_ok = q_params_ok;
    return search_impl(c, emb, str, r);
}

extern "C" int oc_search_facets(oc_ctx *c, oc_emb *emb, oc_str *str, oc_facets *facets, const oc_search_params *p,
                                const oc_facet_req *reqs, uint32_t n_reqs, uint64_t *out_counts) {
    if (!c || !p || !facets || !out_counts || (n_reqs && !reqs)) return fail(OC_ERR_INVALID, "NULL argument");
    if (facets->ctx != c) return fail(OC_ERR_INVALID, "facets belong to another ctx");
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "facets over a sharded search: count per shard and add the counts");
    if (n_reqs == 0) return OC_OK;
    const uint32_t B = p->n_queries;
    FacetJob fj;
    fj.fc = facets; fj.reqs = reqs; fj.out_counts = out_counts;
    for (uint32_t q = 0; q < B; q++)
        for (uint32_t r = 0; r < n_reqs; r++) { fj.q.push_back(q); fj.r.push_back(r); fj.o.push_back(size_t(q) * n_reqs + r); }
    return facets_unfiltered(c, emb, str, p, fj, false);
}

extern "C" int oc_facets_check(const oc_facets *f, const oc_facet_req *reqs, uint32_t n) {
    if (!f || (n && !reqs)) return fail(OC_ERR_INVALID, "NULL argument");
    std::lock_guard<std::mutex> g(f->ctx->mu);
    uint64_t lo, hi;
    for (uint32_t i = 0; i < n; i++) OCTRY(facet_resolve(f, reqs[i], i, true, lo, hi));
    return OC_OK;
}

// ------------------------------------------------------------------------------------ groups
// GroupContext::execute (read/index/group.rs) + sort_groups (read/sort.rs:129-230): the group CSR is built once on
// the host; per call its documents are mapped to string rows and group_topk_kernel (group.cuh) runs one CTA per
// (query, group) over the score map the search left on the device.  struct oc_group_by is defined with GroupJob.
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

// mode: the batch's (with per-query parameters, q_plan gives each query's own)
static int run_groups(oc_ctx *c, const GroupJob &gj, int mode, const StrSnap *S, uint32_t n_tiles, uint32_t vlimit,
                      const uint64_t *omc_doc, const float *omc_mult, uint32_t n_omc, const PinJob &pj, const QueryPlan *q_plan) {
    const uint32_t R = gj.rows, top = gj.top;
    if (R == 0) return OC_OK;
    const bool has_ft = mode != OC_MODE_VECTOR && n_tiles > 0;
    if (has_ft)   // each handle's documents -> string rows (identity, or a binary search over the ascending row_doc)
        for (oc_group_by *g : gj.h) {
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
    const size_t n_out = size_t(R) * top;
    OCTRY(c->grp_doc.ensure(std::max<size_t>(n_out, 1) * 8));
    OCTRY(c->grp_score.ensure(std::max<size_t>(n_out, 1) * 4));
    OCTRY(c->grp_n.ensure(size_t(R) * 4));
    GroupParams gp{};
    gp.handles = gj.d_hand;
    gp.top = top;
    gp.kp2 = std::max<uint32_t>(32, next_pow2(top));
    gp.vp2 = next_pow2(std::max<uint32_t>(vlimit, 1));
    gp.has_ft = has_ft; gp.hybrid = mode == OC_MODE_HYBRID;
    gp.mbits = c->mbits.as<uint32_t>(); gp.row_words = uint64_t(n_tiles) * (BM25_TILE / 32);
    gp.row_ft = c->row_ft.as<float>();
    gp.gmin = c->grp_gmin.as<float>(); gp.den = c->grp_den.as<float>();
    gp.v_doc = c->grp_vdoc.as<uint64_t>(); gp.v_score = c->grp_vscore.as<float>(); gp.v_n = c->grp_vn.as<uint32_t>();
    gp.v_stride = std::max<uint32_t>(vlimit, 1);
    gp.omc_doc = omc_doc; gp.omc_mult = omc_mult; gp.n_omc = n_omc;
    gp.out_doc = c->grp_doc.as<uint64_t>(); gp.out_score = c->grp_score.as<float>(); gp.out_n = c->grp_n.as<uint32_t>();
    gp.ents = gj.d_ents;
    gp.q_plan = q_plan;
    const size_t smem = (size_t(GROUP_BUF) + gp.kp2 + gp.vp2) * 8 + size_t(gp.vp2) * 4;
    for (int by_field = 0; by_field < 2; by_field++) {   // score order, then field order: one launch per work list
        const uint32_t s0 = by_field ? gj.n_score_spans : 0u, s1 = by_field ? gj.n_spans : gj.n_score_spans;
        const uint32_t i0 = by_field ? gj.n_score_items : 0u, i1 = by_field ? R : gj.n_score_items;
        if (i1 == i0) continue;
        gp.spans = gj.d_spans + s0; gp.n_spans = s1 - s0; gp.item0 = i0;
        const void *kern = by_field ? (const void *)group_sort_topk_kernel : (const void *)group_topk_kernel;
        CU(smem_cfg(c->device, kern, smem));
        if (by_field) group_sort_topk_kernel<<<i1 - i0, GROUP_THREADS, smem, c->stream>>>(gp);
        else group_topk_kernel<<<i1 - i0, GROUP_THREADS, smem, c->stream>>>(gp);
        launched(c);
        CU(cudaGetLastError());
    }
    if (gj.keep_top) return OC_OK;
    const uint64_t *res_doc = gp.out_doc;
    const float *res_score = gp.out_score;
    const uint32_t *res_n = gp.out_n;
    if (!gj.direct) {   // every list at the caller's stride, spliced for the queries with items
        const size_t n_res = size_t(R) * gj.stride;
        OCTRY(c->pin_gdoc.ensure(std::max<size_t>(n_res, 1) * 8));
        OCTRY(c->pin_gscore.ensure(std::max<size_t>(n_res, 1) * 4));
        OCTRY(c->pin_gn.ensure(size_t(R) * 4));
        GroupPinParams xp{};
        xp.handles = gj.d_hand; xp.spans = gj.d_spans; xp.n_spans = gj.n_spans;
        xp.stride = gj.stride; xp.top = top;
        xp.kp2 = std::max<uint32_t>(32, next_pow2(pj.stride));
        xp.doc = pj.d_doc; xp.pos = pj.d_pos; xp.score = c->pin_score.as<float>();
        xp.cnt = pj.splice ? pj.d_cnt : nullptr; xp.item_stride = pj.stride;
        xp.top_doc = gp.out_doc; xp.top_score = gp.out_score; xp.top_n = gp.out_n;
        xp.out_doc = c->pin_gdoc.as<uint64_t>(); xp.out_score = c->pin_gscore.as<float>(); xp.out_n = c->pin_gn.as<uint32_t>();
        const size_t psmem = pin_splice_smem(xp.kp2, top, std::min<uint32_t>(gj.stride, top + pj.stride));
        group_pin_splice_kernel<<<R, PIN_THREADS, psmem, c->stream>>>(xp);
        launched(c);
        CU(cudaGetLastError());
        res_doc = xp.out_doc; res_score = xp.out_score; res_n = xp.out_n;
    }
    const size_t n_res = size_t(R) * gj.stride;
    if (n_res) {
        CU(cudaMemcpyAsync(gj.out_doc, res_doc, n_res * 8, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(gj.out_score, res_score, n_res * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU(cudaMemcpyAsync(gj.out_n, res_n, size_t(R) * 4, cudaMemcpyDeviceToHost, c->stream));
    return OC_OK;
}

static int pins_check_flat(const oc_search_params *p, const PinJob &pj) {
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "pins over a sharded search: scores and the hybrid normalisation are global");
    if (pj.splice && !p->q_params && (uint64_t(p->limit) + p->offset) * 2 > OC_MAX_TOPK)   // (q_params: per query, qparams_plan)
        return fail(OC_ERR_UNSUPPORTED, "pins: 2 x (limit+offset) %llu > %u", (unsigned long long)(uint64_t(p->limit) + p->offset) * 2,
                    OC_MAX_TOPK);
    return OC_OK;
}

// The group list depth of query b at max_results m: 2 x m for an active query (pins apply and it has items, spliced into
// its groups; sort.rs:137-142), else m.  group_stride must also hold an active query's items.
static int group_depth(uint32_t b, uint32_t m, const PinJob &pj, uint32_t group_stride, uint32_t &depth) {
    if (m > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "query %u: max_results %u > %u", b, m, OC_MAX_TOPK);
    const bool active = pj.splice && pj.cnt[b] > 0;
    if (active && 2 * m > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "query %u: pins: 2 x max_results %u > %u", b, 2 * m, OC_MAX_TOPK);
    const uint64_t need = active ? 2ull * m + pj.cnt[b] : m;
    if (group_stride < need) return fail(OC_ERR_INVALID, "query %u: group_stride %u < %llu", b, group_stride, (unsigned long long)need);
    depth = active ? 2 * m : m;
    return OC_OK;
}

// One index's GroupJob for a batch: query b groups by q[b] (groups NULL: none) with pj's items.  skip_empty
// (oc_search_indexes_ex): a handle without groups is left out after its ctx check; its query's depth is checked on the
// collection's keys, which it may not have.
static int group_job_plan(oc_ctx *c, uint32_t B, const oc_group_req *q, const PinJob &pj, uint32_t group_stride, bool skip_empty,
                          GroupJob &gj) {
    gj.q_h.assign(B, GROUP_NONE);
    gj.q_m.assign(B, 0);
    gj.q_row.assign(B, 0);
    uint64_t rows = 0;
    for (uint32_t b = 0; b < B; b++) {
        const oc_group_by *g = q[b].groups;
        if (!g) continue;
        if (g->ctx != c) return fail(OC_ERR_INVALID, "group_by of query %u belongs to another ctx", b);
        if (skip_empty && g->n_groups == 0) continue;
        uint32_t depth;
        OCTRY(group_depth(b, q[b].max_results, pj, group_stride, depth));
        uint32_t h = 0;
        while (h < gj.h.size() && gj.h[h] != g) h++;
        if (h == gj.h.size()) gj.h.push_back(const_cast<oc_group_by *>(g));   // only its per-call row map is refreshed, under the ctx lock
        gj.q_h[b] = h; gj.q_m[b] = q[b].max_results; gj.q_row[b] = (uint32_t)rows;   // refused below past 2^31 rows
        rows += g->n_groups;
    }
    // the work list is a 1-D grid of (query, group) items
    if (rows > 0x7fffffffull) return fail(OC_ERR_UNSUPPORTED, "groups: %llu (query, group) rows >= 2^31", (unsigned long long)rows);
    gj.rows = (uint32_t)rows;
    return OC_OK;
}

// The one path of the grouped calls: query b takes q[b] (groups NULL: no groups) with its items and, per_query
// (oc_search_q_groups), its q_filters entry; the flat hits follow oc_search_q_sorted.  The wrappers below pass one
// request for every query.  Nothing is written on failure.
static int groups_impl(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_group_req *q, const oc_pins *pins,
                       uint32_t group_stride, bool per_query, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                       uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present,
                       uint64_t *out_group_doc_ids, float *out_group_scores, double *out_group_sort_values, uint32_t *out_group_n,
                       const FacetJob *fj = nullptr) {
    if (!c || !p || !q || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    const uint32_t B = p->n_queries;
    SortJob sj{};
    for (uint32_t b = 0; b < B; b++) OCTRY(sort_job_add(c, q[b].sort, sj));
    PinJob pj;
    OCTRY(pin_job_init(pins, B, pj));
    OCTRY(pins_check_flat(p, pj));
    pj.out_scores = out_pin_scores; pj.out_present = out_pin_present;
    GroupJob gj;
    OCTRY(group_job_plan(c, B, q, pj, group_stride, false, gj));
    bool flat_only = false;   // some query has neither groups nor facets: its hits are oc_search_q_sorted's, which needs limit >= 1
    for (uint32_t b = 0; b < B; b++) {
        if (q[b].groups) continue;
        const bool flat = !(fj && fj->q_off[b + 1] > fj->q_off[b]);
        if (flat && p->q_params && p->q_params[b].limit == 0)
            return fail(OC_ERR_INVALID, "q_params[%u]: limit must be >= 1 when the query has no groups%s", b, fj ? " and no facets" : "");
        flat_only = flat_only || flat;
    }
    if (flat_only && p->limit == 0) return fail(OC_ERR_INVALID, "limit must be >= 1 when a query has no groups%s", fj ? " and no facets" : "");
    if (gj.rows && (!out_group_n || (group_stride && (!out_group_doc_ids || !out_group_scores)))) return fail(OC_ERR_INVALID, "NULL group output");
    gj.stride = group_stride;
    gj.out_doc = out_group_doc_ids; gj.out_score = out_group_scores; gj.out_n = out_group_n; gj.out_values = out_group_sort_values;
    SearchReq r(p, out_doc_ids, out_scores, out_n, out_count);
    r.out_sort_values = out_sort_values; r.fj = fj; r.gj = &gj; r.pj = &pj;
    r.sj = sj.f.empty() ? nullptr : &sj;   // every query in score order: the flat hits are oc_search_pinned's
    r.q_filters_ok = r.q_params_ok = per_query;
    return search_impl(c, emb, str, r);
}

// oc_search_pinned, oc_search_sorted and oc_search_q_sorted: the flat hits with the items of pins, in field order where
// sj has a sort (else in score order: oc_search_pinned's hits, sort values NaN).  Nothing is written on failure.
static int sorted_impl(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const SortJob &sj, const oc_pins *pins,
                       bool q_filters_ok, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                       uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present) {
    PinJob pj;
    OCTRY(pin_job_init(pins, p->n_queries, pj));
    OCTRY(pins_check_flat(p, pj));
    pj.out_scores = out_pin_scores; pj.out_present = out_pin_present;
    SearchReq r(p, out_doc_ids, out_scores, out_n, out_count);
    r.out_sort_values = out_sort_values; r.pj = &pj;
    r.sj = sj.f.empty() ? nullptr : &sj;
    r.q_filters_ok = r.q_params_ok = q_filters_ok;
    return search_impl(c, emb, str, r);
}

extern "C" uint64_t oc_group_by_n_groups(const oc_group_by *g) { return g ? g->n_groups : 0; }

extern "C" int oc_search_groups(oc_ctx *c, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                                uint32_t max_results, uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n, uint64_t *out_count,
                                uint64_t *out_group_doc_ids, float *out_group_scores, uint32_t *out_group_n) {
    if (!c || !p || !groups || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (groups->n_groups && (!out_group_n || (max_results && (!out_group_doc_ids || !out_group_scores))))
        return fail(OC_ERR_INVALID, "NULL group output");
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "groups over a sharded search: hybrid normalisation and the vector set are global");
    if (p->n_queries > 65535) return fail(OC_ERR_UNSUPPORTED, "groups: n_queries %u > 65535", p->n_queries);
    const std::vector<oc_group_req> req(p->n_queries, oc_group_req{groups, max_results, oc_sort{nullptr, OC_SORT_ASC}});
    return groups_impl(c, emb, str, p, req.data(), nullptr, max_results, false, out_doc_ids, out_scores, nullptr, out_n, out_count,
                       nullptr, nullptr, out_group_doc_ids, out_group_scores, nullptr, out_group_n);
}

// ------------------------------------------------------------------------------------ pin rules (pins.cuh)

extern "C" int oc_search_pinned(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_pins *pins,
                                uint64_t *out_doc_ids, float *out_scores, uint32_t *out_n, uint64_t *out_count,
                                float *out_pin_scores, uint8_t *out_pin_present) {
    if (!c || !p) return fail(OC_ERR_INVALID, "NULL argument");
    return sorted_impl(c, emb, str, p, SortJob{}, pins, false, out_doc_ids, out_scores, nullptr, out_n, out_count, out_pin_scores,
                       out_pin_present);
}

extern "C" int oc_search_groups_pinned(oc_ctx *c, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                                       uint32_t max_results, const oc_pins *pins, uint32_t group_stride, uint64_t *out_doc_ids,
                                       float *out_scores, uint32_t *out_n, uint64_t *out_count, uint64_t *out_group_doc_ids,
                                       float *out_group_scores, uint32_t *out_group_n) {
    if (!c || !p || !groups || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (groups->n_groups && (!out_group_n || (group_stride && (!out_group_doc_ids || !out_group_scores))))
        return fail(OC_ERR_INVALID, "NULL group output");
    if (p->n_queries > 65535) return fail(OC_ERR_UNSUPPORTED, "groups: n_queries %u > 65535", p->n_queries);
    const std::vector<oc_group_req> req(p->n_queries, oc_group_req{groups, max_results, oc_sort{nullptr, OC_SORT_ASC}});
    return groups_impl(c, emb, str, p, req.data(), pins, group_stride, false, out_doc_ids, out_scores, nullptr, out_n, out_count,
                       nullptr, nullptr, out_group_doc_ids, out_group_scores, nullptr, out_group_n);
}

// ------------------------------------------------------------------------------------ sortBy (sort.cuh, sort_build.cuh)
// The entries of one sort field build: documents and values in device memory, or on the host (uploaded first).
struct SortBuildIn {
    uint64_t n = 0;
    const uint64_t *h_docs = nullptr, *d_docs = nullptr;
    const double *h_vals = nullptr, *d_vals = nullptr;
    const std::vector<uint64_t> *off = nullptr;   // or a variant field: its offsets (host copy) and
    const double *var_vals = nullptr;             //   one value per variant (host)
};
// Builds both orders of `f` on the ctx stream (sort_build.cuh).  Called under the ctx lock; on failure `f` is freed.
static int sort_field_build(oc_ctx *c, const SortBuildIn &in, oc_sort_field *f) {
    const uint64_t n = in.n, nbits = f->nbits;
    const uint32_t n_var = in.off ? uint32_t(in.off->size() - 1) : 0;
    auto bad = [&](int code) { sort_field_free(f); return code; };
    if (n >= uint64_t(INT32_MAX))   // cub counts in int, and a rank is a uint32
        return bad(fail(OC_ERR_UNSUPPORTED, "sort field: %llu entries >= 2^31 - 1", (unsigned long long)n));
    cudaStream_t st = c->stream;
    const int end_bit = 64 - __builtin_clzll(nbits);   // every kept document is below 2^end_bit
    size_t b_doc = 0, b_asc = 0, b_desc = 0, b_scan = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, b_doc, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const unsigned long long *)nullptr,
                                        (unsigned long long *)nullptr, (int)n, 0, end_bit, st) != cudaSuccess ||
        cub::DeviceRadixSort::SortPairs(nullptr, b_asc, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                        (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)n, 0, 64, st) != cudaSuccess ||
        cub::DeviceRadixSort::SortPairsDescending(nullptr, b_desc, (const unsigned long long *)nullptr, (unsigned long long *)nullptr,
                                                  (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)n, 0, 64, st) != cudaSuccess ||
        cub::DeviceScan::ExclusiveSum(nullptr, b_scan, (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)(n + 1), st) != cudaSuccess)
        return bad(fail(OC_ERR_CUDA, "sort field: cub temp size"));
    // workspace: [uploaded: docs | values | offsets | variant values] doc_a | key_a | doc_b | key_b | first | keep | rank | value | cub
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t o_docs = 0, o_vals = o_docs + al(in.h_docs ? n * 8 : 0), o_off = o_vals + al(in.h_vals ? n * 8 : 0),
                 o_vv = o_off + al(in.off ? (n_var + 1) * 8 : 0), o_da = o_vv + al(n_var * 8);
    const size_t o_ka = o_da + al(n * 4), o_db = o_ka + al(n * 8), o_kb = o_db + al(n * 4), o_first = o_kb + al(n * 8),
                 o_keep = o_first + al(nbits * 4), o_rank = o_keep + al((n + 1) * 4), o_val = o_rank + al((n + 1) * 4),
                 o_cub = o_val + al(n * 8), total = o_cub + al(std::max(std::max(b_doc, b_scan), std::max(b_asc, b_desc)));
    struct Release {   // every way out waits for the stream, then gives the workspace back
        oc_ctx *c;
        ~Release() { cudaStreamSynchronize(c->stream); c->sfb_ws.release(); }
    } release{c};
    if (c->sfb_ws.ensure(total) != OC_OK) return bad(OC_ERR_OOM);
    uint8_t *w = c->sfb_ws.as<uint8_t>();
    auto at = [&](size_t o) { return static_cast<void *>(w + o); };
    const uint64_t *docs = in.d_docs ? in.d_docs : static_cast<const uint64_t *>(at(o_docs));
    const oc::SfSource src{in.d_vals ? in.d_vals : in.h_vals ? static_cast<const double *>(at(o_vals)) : nullptr,
                           static_cast<const uint64_t *>(at(o_off)), static_cast<const double *>(at(o_vv)), n_var};
    uint32_t *da = static_cast<uint32_t *>(at(o_da)), *db = static_cast<uint32_t *>(at(o_db));
    unsigned long long *ka = static_cast<unsigned long long *>(at(o_ka)), *kb = static_cast<unsigned long long *>(at(o_kb));
    uint32_t *first = static_cast<uint32_t *>(at(o_first)), *keep = static_cast<uint32_t *>(at(o_keep));
    uint32_t *rank = static_cast<uint32_t *>(at(o_rank));
    double *val = static_cast<double *>(at(o_val));
    const unsigned g = (unsigned)((n + oc::SF_THREADS - 1) / oc::SF_THREADS), g1 = (unsigned)((n + oc::SF_THREADS) / oc::SF_THREADS);
    cudaError_t e = cudaSuccess;
    if (n && in.h_docs) e = cudaMemcpyAsync(at(o_docs), in.h_docs, n * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && n && in.h_vals) e = cudaMemcpyAsync(at(o_vals), in.h_vals, n * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && in.off) e = cudaMemcpyAsync(at(o_off), in.off->data(), (n_var + 1) * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && in.off && n_var) e = cudaMemcpyAsync(at(o_vv), in.var_vals, n_var * 8, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && n) {
        oc::sf_keys_kernel<<<g, oc::SF_THREADS, 0, st>>>(docs, n, nbits, src, da, ka);
        launched(c);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(at(o_cub), b_doc, da, db, ka, kb, (int)n, 0, end_bit, st);   // by document
    }
    if (e != cudaSuccess) return bad(fail(OC_ERR_CUDA, "sort field build: %s", cudaGetErrorString(e)));
    for (int ord = OC_SORT_ASC; ord <= OC_SORT_DESC; ord++) {
        SortOrder &o = f->ord[ord];
        uint32_t cnt = 0;
        if (n) {   // entries in rank order with repeats (doc_a, key_a), then the first position of each document
            e = ord == OC_SORT_ASC ? cub::DeviceRadixSort::SortPairs(at(o_cub), b_asc, kb, ka, db, da, (int)n, 0, 64, st)
                                   : cub::DeviceRadixSort::SortPairsDescending(at(o_cub), b_desc, kb, ka, db, da, (int)n, 0, 64, st);
            if (e == cudaSuccess) e = cudaMemsetAsync(first, 0xff, nbits * 4, st);
            if (e == cudaSuccess) {
                oc::sf_first_kernel<<<g, oc::SF_THREADS, 0, st>>>(da, n, first);
                oc::sf_keep_kernel<<<g1, oc::SF_THREADS, 0, st>>>(da, n, first, keep);
                launched(c); launched(c);
                e = cudaGetLastError();
            }
            if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(at(o_cub), b_scan, keep, rank, (int)(n + 1), st);
            if (e == cudaSuccess) e = cudaMemcpyAsync(&cnt, rank + n, 4, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        }
        o.n = cnt;
        if (e == cudaSuccess) e = cudaMalloc(&o.rank_doc, std::max<size_t>(o.n, 1) * 8);
        if (e == cudaSuccess) e = cudaMalloc(&o.doc_rank, nbits * 4);
        if (e == cudaSuccess) e = cudaMalloc(&o.rank_row, (o.n + 1) * 4);
        if (e == cudaSuccess) e = cudaMemsetAsync(o.doc_rank, 0xff, nbits * 4, st);             // RANK_NONE: no value
        if (e == cudaSuccess) e = cudaMemsetAsync(o.rank_row + o.n, 0xff, 4, st);               // the sentinel
        if (e == cudaSuccess && o.n) {
            oc::sf_scatter_kernel<<<g, oc::SF_THREADS, 0, st>>>(da, ka, rank, n, o.rank_doc, o.doc_rank, val);
            launched(c);
            e = cudaGetLastError();
        }
        o.h_doc_rank.resize(nbits);
        o.h_value.resize(o.n);
        if (e == cudaSuccess) e = cudaMemcpyAsync(o.h_doc_rank.data(), o.doc_rank, nbits * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess && o.n) e = cudaMemcpyAsync(o.h_value.data(), val, o.n * 8, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess)
            return bad(fail(e == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "sort field build: %s", cudaGetErrorString(e)));
    }
    return OC_OK;
}

extern "C" int oc_sort_field_create(oc_ctx *c, uint64_t nbits, uint64_t n, const uint64_t *doc_ids, const double *values,
                                    oc_sort_field **out) {
    if (!c || !out || nbits == 0 || (n && (!doc_ids || !values))) return fail(OC_ERR_INVALID, "bad arguments");
    if (nbits >= RANK_NONE) return fail(OC_ERR_INVALID, "nbits %llu >= 2^32 - 1", (unsigned long long)nbits);
    for (uint64_t i = 0; i < n; i++)
        if (values[i] != values[i]) return fail(OC_ERR_INVALID, "sort value %llu is NaN", (unsigned long long)i);
    std::lock_guard<std::mutex> lk(c->mu);
    if (cudaSetDevice(c->device) != cudaSuccess) return fail(OC_ERR_CUDA, "cudaSetDevice failed");
    oc_sort_field *f = new oc_sort_field();
    f->ctx = c; f->nbits = nbits;
    SortBuildIn in;
    in.n = n; in.h_docs = doc_ids; in.h_vals = values;
    OCTRY(sort_field_build(c, in, f));
    *out = f;
    return OC_OK;
}

extern "C" int oc_sort_field_from_facets(oc_facets *fs, uint32_t field, const double *variant_values, oc_sort_field **out) {
    if (!fs || !out) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = fs->ctx;
    std::lock_guard<std::mutex> lk(c->mu);   // one whole published version: a commit publishes under this lock
    if (field >= fs->fields.size()) return fail(OC_ERR_INVALID, "field %u: the store has %zu fields", field, fs->fields.size());
    const FacetField &fl = fs->fields[field];
    if (fl.number && variant_values) return fail(OC_ERR_INVALID, "field %u is a number field: variant_values must be NULL", field);
    if (!fl.number && !variant_values) return fail(OC_ERR_INVALID, "field %u is a variant field: variant_values is NULL", field);
    const uint32_t n_var = fl.number ? 0 : uint32_t(fl.offsets.size() - 1);
    for (uint32_t v = 0; v < n_var; v++)
        if (variant_values[v] != variant_values[v]) return fail(OC_ERR_INVALID, "variant %u: value is NaN", v);
    if (fs->nbits >= RANK_NONE) return fail(OC_ERR_INVALID, "nbits %llu >= 2^32 - 1", (unsigned long long)fs->nbits);
    if (cudaSetDevice(c->device) != cudaSuccess) return fail(OC_ERR_CUDA, "cudaSetDevice failed");
    oc_sort_field *f = new oc_sort_field();
    f->ctx = c; f->nbits = fs->nbits;
    {
        std::lock_guard<std::mutex> gp(fs->pend.mu);
        f->facets_version = fs->pend.version;
    }
    SortBuildIn in;
    in.n = fl.n_docs; in.d_docs = fl.docs;
    if (fl.number) in.d_vals = fl.d_values;
    else { in.off = &fl.offsets; in.var_vals = variant_values; }
    OCTRY(sort_field_build(c, in, f));
    *out = f;
    return OC_OK;
}

extern "C" int oc_sort_field_read(const oc_sort_field *f, int order, uint64_t *nbits, uint64_t *n, uint64_t *rank_doc, double *rank_value,
                                  uint64_t *facets_version) {
    if (!f || !n) return fail(OC_ERR_INVALID, "NULL argument");
    if (order != OC_SORT_ASC && order != OC_SORT_DESC) return fail(OC_ERR_INVALID, "sort order %d is neither ASC nor DESC", order);
    const SortOrder &o = f->ord[order];
    const uint64_t cap = *n;
    *n = o.n;
    if (nbits) *nbits = f->nbits;
    if (facets_version) *facets_version = f->facets_version;
    if (!rank_doc && !rank_value) return OC_OK;
    if (cap < o.n) return fail(OC_ERR_INVALID, "arrays hold %llu entries, the order has %llu", (unsigned long long)cap, (unsigned long long)o.n);
    if (rank_value) std::copy(o.h_value.begin(), o.h_value.end(), rank_value);
    if (rank_doc && o.n) {
        std::lock_guard<std::mutex> lk(f->ctx->mu);
        CU(cudaSetDevice(f->ctx->device));
        CU(cudaMemcpy(rank_doc, o.rank_doc, o.n * 8, cudaMemcpyDeviceToHost));
    }
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
    OCTRY(sort_job_init(c, sort, p->n_queries, sj));
    return sorted_impl(c, emb, str, p, sj, pins, false, out_doc_ids, out_scores, out_sort_values, out_n, out_count, out_pin_scores,
                       out_pin_present);
}

extern "C" int oc_search_groups_sorted(oc_ctx *c, oc_emb *emb, oc_str *str, oc_group_by *groups, const oc_search_params *p,
                                       uint32_t max_results, const oc_sort *sort, const oc_pins *pins, uint32_t group_stride,
                                       uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                                       uint64_t *out_count, uint64_t *out_group_doc_ids, float *out_group_scores,
                                       double *out_group_sort_values, uint32_t *out_group_n) {
    if (!c || !p || !groups || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (groups->n_groups && (!out_group_n || (group_stride && (!out_group_doc_ids || !out_group_scores))))
        return fail(OC_ERR_INVALID, "NULL group output");
    if (!sort || !sort->field) return fail(OC_ERR_INVALID, "NULL sort");   // (a NULL field is score order in a request)
    if (p->n_queries > 65535) return fail(OC_ERR_UNSUPPORTED, "groups: n_queries %u > 65535", p->n_queries);
    const std::vector<oc_group_req> req(p->n_queries, oc_group_req{groups, max_results, *sort});
    return groups_impl(c, emb, str, p, req.data(), pins, group_stride, false, out_doc_ids, out_scores, out_sort_values, out_n,
                       out_count, nullptr, nullptr, out_group_doc_ids, out_group_scores, out_group_sort_values, out_group_n);
}

// One batch in which every query has its own sort (or score order), its own pins and, with q_filters, its own filter:
// query b gets what it gets alone through oc_search_sorted (a sort) or oc_search_pinned (score order, sort values NaN).
extern "C" int oc_search_q_sorted(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_sort *q_sorts,
                                  const oc_pins *pins, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                                  uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present) {
    if (!c || !p || !q_sorts) return fail(OC_ERR_INVALID, "NULL argument");
    SortJob sj{};
    for (uint32_t b = 0; b < p->n_queries; b++) OCTRY(sort_job_add(c, q_sorts[b], sj));
    return sorted_impl(c, emb, str, p, sj, pins, true, out_doc_ids, out_scores, out_sort_values, out_n, out_count, out_pin_scores,
                       out_pin_present);
}

// The pass that re-scores the sub-batch `sub` of p's filtered queries for their facets (counts fj, rows: places in sub):
// q holds their vectors and token CSR and their q_params entries, without filters, groups, sorts or pins.
struct FacetSubBatch {
    FacetJob fj;
    std::vector<uint32_t> sub;
    oc_search_params q;
    std::vector<float> vecs;
    std::vector<uint32_t> q_tok{0}, tok_term{0}, t_field, t_id;
    std::vector<float> t_weight;
    std::vector<oc_query_params> sub_qp;
};
static void facet_sub_batch(const oc_search_params *p, const oc_emb *emb, const std::vector<uint32_t> &sub, FacetSubBatch &sb) {
    const uint32_t S = (uint32_t)sub.size();
    oc_search_params &q = sb.q;
    q = *p;
    drop_filters(q);
    q.n_queries = S;
    std::vector<float> &vecs = sb.vecs, &t_weight = sb.t_weight;
    std::vector<uint32_t> &q_tok = sb.q_tok, &tok_term = sb.tok_term, &t_field = sb.t_field, &t_id = sb.t_id;
    // per-query parameters: the sub-batch's entries; a vector entry's row and a text entry's tokens are the ones read
    std::vector<oc_query_params> &sub_qp = sb.sub_qp;
    bool sub_v = p->mode != OC_MODE_FULLTEXT, sub_ft = p->mode != OC_MODE_VECTOR;
    if (p->q_params) {
        sub_v = sub_ft = false;
        for (uint32_t b : sub) {
            sub_qp.push_back(p->q_params[b]);
            sub_v = sub_v || p->q_params[b].mode != OC_MODE_FULLTEXT;
            sub_ft = sub_ft || p->q_params[b].mode != OC_MODE_VECTOR;
        }
        q.q_params = sub_qp.data();
    }
    auto text_of = [&](uint32_t b) { return !p->q_params || p->q_params[b].mode != OC_MODE_VECTOR; };
    if (sub_v && emb && p->q_vecs) {
        const size_t dim = emb->dim;
        vecs.resize(size_t(S) * dim);
        for (uint32_t s = 0; s < S; s++)
            if (!p->q_params || p->q_params[sub[s]].mode != OC_MODE_FULLTEXT)
                memcpy(vecs.data() + size_t(s) * dim, p->q_vecs + size_t(sub[s]) * dim, dim * 4);
        q.q_vecs = vecs.data();
    }
    if (sub_ft && p->q_token_offsets) {
        for (uint32_t b : sub) {
            if (!text_of(b)) { q_tok.push_back((uint32_t)tok_term.size() - 1); continue; }
            for (uint32_t t = p->q_token_offsets[b]; t < p->q_token_offsets[b + 1]; t++) {
                for (uint32_t e = p->token_term_offsets[t]; e < p->token_term_offsets[t + 1]; e++) {
                    t_field.push_back(p->term_field[e]);
                    t_id.push_back(p->term_id[e]);
                    t_weight.push_back(p->term_weight ? p->term_weight[e] : 1.0f);
                }
                tok_term.push_back((uint32_t)t_id.size());
            }
            q_tok.push_back((uint32_t)tok_term.size() - 1);
        }
        t_field.push_back(0); t_id.push_back(0); t_weight.push_back(1.0f);   // never read: non-NULL arrays for an empty CSR
        q.q_token_offsets = q_tok.data(); q.token_term_offsets = tok_term.data();
        q.term_field = t_field.data(); q.term_id = t_id.data(); q.term_weight = t_weight.data();
    }
}
// Splits the counts (query, request, output slot) of items: an unfiltered query's go to mj, on the main pass, a filtered
// query's to sb, whose sub-batch takes those queries in the order of their first item.
static void facet_split(const oc_search_params *p, const oc_emb *emb, oc_facets *fc, const oc_facet_req *reqs,
                        const std::vector<uint3> &items, FacetJob &mj, FacetSubBatch &sb) {
    mj.fc = sb.fj.fc = fc; mj.reqs = sb.fj.reqs = reqs;
    sb.fj.hits_optional = true;
    std::vector<uint32_t> sub_of(p->n_queries, 0xffffffffu);
    for (const uint3 &it : items) {
        const bool filtered = facet_filtered(p, it.x);
        if (filtered && sub_of[it.x] == 0xffffffffu) { sub_of[it.x] = (uint32_t)sb.sub.size(); sb.sub.push_back(it.x); }
        FacetJob &j = filtered ? sb.fj : mj;
        j.q.push_back(filtered ? sub_of[it.x] : it.x); j.r.push_back(it.y); j.o.push_back(it.z);
    }
    if (!sb.sub.empty()) facet_sub_batch(p, emb, sb.sub, sb);
}

// ------------------------------------------------------------------------------------ one call over the indexes (index_merge.cuh)
static bool same_f32(float a, float b) { return memcmp(&a, &b, 4) == 0; }
// the request fields of oc_search_indexes, which every index must share
static bool same_request(const oc_search_params *a, const oc_search_params *b) {
    if (a->n_queries != b->n_queries || a->mode != b->mode || a->limit != b->limit || a->offset != b->offset ||
        a->vector_limit != b->vector_limit || !same_f32(a->similarity, b->similarity) || !same_f32(a->threshold, b->threshold) ||
        !same_f32(a->bm25_k, b->bm25_k) || !same_f32(a->bm25_b, b->bm25_b) || !a->q_params != !b->q_params)
        return false;
    for (uint32_t q = 0; a->q_params && q < a->n_queries; q++) {
        const oc_query_params &x = a->q_params[q], &y = b->q_params[q];
        if (x.mode != y.mode || x.limit != y.limit || x.offset != y.offset || !same_f32(x.similarity, y.similarity) ||
            !same_f32(x.threshold, y.threshold) || x.vector_limit != y.vector_limit)
            return false;
    }
    return true;
}
// one index's timing added to the call's
static void timing_add(oc_timing &t, const oc_timing &a) {
    t.h2d_ms += a.h2d_ms; t.device_ms += a.device_ms; t.d2h_ms += a.d2h_ms; t.scan_ms += a.scan_ms; t.bm25_ms += a.bm25_ms;
    t.fuse_ms += a.fuse_ms; t.comm_ms += a.comm_ms; t.kernel_launches += a.kernel_launches; t.scan_launches += a.scan_launches;
    t.scan_bytes += a.scan_bytes; t.bm25_postings += a.bm25_postings; t.h2d_bytes += a.h2d_bytes; t.d2h_bytes += a.d2h_bytes;
    t.scan_tensor_core = std::max(t.scan_tensor_core, a.scan_tensor_core); t.scan_unproven += a.scan_unproven;
    if (a.scan_launches) t.scan_variant = a.scan_variant;
    t.scan_sweep_ms += a.scan_sweep_ms; t.rerun_ms += a.rerun_ms; t.scan_rescored = std::max(t.scan_rescored, a.scan_rescored);
    t.bm25_dense_items += a.bm25_dense_items; t.bm25_dense_skipped += a.bm25_dense_skipped;
}

// The groups of one batch of oc_search_indexes_ex: per index its GroupJob (local rows) and, per distinct combination of
// (handle, key map) over the indexes, the source table of the collection keys (built once per combination).
struct MiGroups {
    uint32_t rows = 0, gtop = 0, sets = 0;   // gtop: the largest depth of a per-index list, also the merge's largest take
    std::vector<GroupJob> gj;              // [n_idx]
    std::vector<uint32_t> src_g;           // source tables, concatenated
    std::vector<GroupHandle> set_h;        // [set][n_idx]
    std::vector<GroupSpan> spans;          // one per query with collection groups
    std::vector<uint32_t> q_lrow;          // [n_idx][B]
};
// Checks the groups of ex and plans them.  Nothing is written on failure.
static int mi_groups_plan(oc_ctx *c, uint32_t ni, uint32_t B, const oc_index_extras *ex, const uint32_t *q_n_keys,
                          const uint32_t *q_max_results, uint32_t group_stride, const std::vector<uint8_t> &q_active,
                          const PinJob &pj_all, MiGroups &mg) {
    bool any = false;
    for (uint32_t i = 0; ex && i < ni; i++) any = any || ex[i].q_groups;
    for (uint32_t b = 0; q_n_keys && b < B; b++) any = any || q_n_keys[b];
    if (!any) return OC_OK;
    if (!q_n_keys || !q_max_results) return fail(OC_ERR_INVALID, "groups: NULL q_n_keys / q_max_results");
    mg.gj.resize(ni);
    mg.q_lrow.assign(size_t(ni) * B, 0);
    uint64_t rows = 0;
    for (uint32_t b = 0; b < B; b++) {
        if (!q_n_keys[b]) continue;
        uint32_t depth = 0;
        OCTRY(group_depth(b, q_max_results[b], pj_all, group_stride, depth));
        rows += q_n_keys[b];
        mg.gtop = std::max(mg.gtop, depth);
    }
    if (rows > 0x7fffffffull) return fail(OC_ERR_UNSUPPORTED, "groups: %llu collection group rows >= 2^31", (unsigned long long)rows);
    mg.rows = (uint32_t)rows;
    // each index's GroupJob, with the depth of an active query although its own pins do not apply
    std::vector<oc_group_req> req(B);
    for (uint32_t i = 0; i < ni; i++) {
        GroupJob &gj = mg.gj[i];
        const oc_index_extras *e = ex ? &ex[i] : nullptr;
        if (e && e->q_groups && !e->q_group_keys) return fail(OC_ERR_INVALID, "index %u: q_groups without q_group_keys", i);
        for (uint32_t b = 0; b < B; b++) req[b] = oc_group_req{e && e->q_groups ? e->q_groups[b] : nullptr, q_max_results[b], oc_sort{}};
        if (const int rc = group_job_plan(c, B, req.data(), pj_all, group_stride, true, gj))
            return fail(rc, "index %u: %s", i, std::string(g_err).c_str());
        gj.keep_top = true;
        gj.q_deep = q_active;
        std::copy(gj.q_row.begin(), gj.q_row.end(), mg.q_lrow.begin() + size_t(i) * B);
    }
    // the source tables: one per distinct (handle, key map) combination; a query's span points at its combination
    std::map<std::vector<uintptr_t>, std::pair<uint32_t, uint32_t>> sets;   // combination -> (table offset, set)
    uint32_t first = 0;
    for (uint32_t b = 0; b < B; b++) {
        const uint32_t nk = q_n_keys[b];
        std::vector<uintptr_t> key(size_t(2) * ni + 1, 0);
        key[0] = nk;
        for (uint32_t i = 0; i < ni; i++) {
            const oc_group_by *g = ex && ex[i].q_groups ? ex[i].q_groups[b] : nullptr;
            if (!g || !g->n_groups) continue;
            if (!ex[i].q_group_keys[b]) return fail(OC_ERR_INVALID, "index %u: query %u has groups and no key map", i, b);
            key[1 + 2 * i] = uintptr_t(g);
            key[2 + 2 * i] = uintptr_t(ex[i].q_group_keys[b]);
        }
        auto it = sets.find(key);
        if (it == sets.end()) {
            const uint32_t off = (uint32_t)mg.src_g.size();
            if (uint64_t(off) + uint64_t(nk) * ni > 0x7fffffffull) return fail(OC_ERR_UNSUPPORTED, "groups: source tables >= 2^31 entries");
            mg.src_g.resize(size_t(off) + size_t(nk) * ni, IM_NO_SRC);
            for (uint32_t i = 0; i < ni; i++) {
                const oc_group_by *g = reinterpret_cast<const oc_group_by *>(key[1 + 2 * i]);
                const uint32_t *km = reinterpret_cast<const uint32_t *>(key[2 + 2 * i]);
                mg.set_h.push_back(g ? GroupHandle{g->off, g->docs, nullptr, g->n_groups} : GroupHandle{nullptr, nullptr, nullptr, 0});
                for (uint32_t l = 0; g && l < g->n_groups; l++) {
                    if (km[l] >= nk) return fail(OC_ERR_INVALID, "index %u, query %u: group %u has key %u >= q_n_keys %u", i, b, l, km[l], nk);
                    uint32_t &e = mg.src_g[off + size_t(km[l]) * ni + i];
                    if (e != IM_NO_SRC) return fail(OC_ERR_INVALID, "index %u, query %u: groups %u and %u have one key %u", i, b, e, l, km[l]);
                    e = l;
                }
            }
            it = sets.emplace(key, std::make_pair(off, mg.sets++)).first;
        }
        if (!nk) continue;
        mg.spans.push_back(GroupSpan{first, b, it->second.first, 0, q_max_results[b], it->second.second, first});
        first += nk;
    }
    return OC_OK;
}

// search_on_indexes: every index through its own stages into a per-index slot of the ctx's workspaces (under one ctx
// lock), then its group lists and facet counts, then index_merge_kernel and index_group_merge_kernel and one copy of
// the merged blob.  Nothing is written on failure.
extern "C" int oc_search_indexes_ex(oc_ctx *c, uint32_t n_indexes, const oc_index_query *ix, const oc_index_extras *ex,
                                    const oc_pins *pins, const uint32_t *q_n_keys, const uint32_t *q_max_results,
                                    uint32_t group_stride, const uint32_t *q_facet_offsets, uint64_t *out_doc_ids, float *out_scores,
                                    double *out_sort_values, uint32_t *out_n, uint64_t *out_count, float *out_pin_scores,
                                    uint8_t *out_pin_present, uint64_t *out_group_doc_ids, float *out_group_scores,
                                    double *out_group_sort_values, uint32_t *out_group_n, uint64_t *out_facet_counts) {
    if (!c || !ix || !out_doc_ids || !out_scores || !out_n || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (n_indexes == 0 || n_indexes > OC_MAX_INDEXES) return fail(OC_ERR_INVALID, "n_indexes %u: expected 1 .. %u", n_indexes, OC_MAX_INDEXES);
    for (uint32_t i = 0; i < n_indexes; i++) {
        if (!ix[i].p) return fail(OC_ERR_INVALID, "index %u: NULL params", i);
        if (ix[i].p->sharded) return fail(OC_ERR_UNSUPPORTED, "index %u: sharded search", i);
        if (!same_request(ix[i].p, ix[0].p)) return fail(OC_ERR_INVALID, "index %u: its request fields differ from index 0's", i);
    }
    const oc_search_params *p0 = ix[0].p;
    const uint32_t B = p0->n_queries, limit = p0->limit;
    if (p0->vector_limit) return fail(OC_ERR_INVALID, "vector_limit must be 0: every index runs at vector_limit = limit");
    if (limit == 0) return fail(OC_ERR_INVALID, "limit must be >= 1");
    // per query: score order, or one order over every index's sort handle
    std::vector<uint8_t> q_sort(B, IM_BY_SCORE);
    bool any_sorted = false;
    for (uint32_t b = 0; b < B; b++) {
        uint32_t n_field = 0;
        int order = -1;
        bool same = true;
        for (uint32_t i = 0; i < n_indexes; i++) {
            if (!ix[i].q_sorts || !ix[i].q_sorts[b].field) continue;
            same = same && (order < 0 || ix[i].q_sorts[b].order == order);
            order = ix[i].q_sorts[b].order;
            n_field++;
        }
        if (n_field == 0) continue;
        if (n_field != n_indexes || !same) return fail(OC_ERR_INVALID, "query %u: a sort on some indexes only, or orders that differ", b);
        if (order != OC_SORT_ASC && order != OC_SORT_DESC) return fail(OC_ERR_INVALID, "query %u: sort order %d is neither ASC nor DESC", b, order);
        q_sort[b] = order == OC_SORT_ASC ? IM_ASC : IM_DESC;
        any_sorted = true;
    }
    // pins: every index looks the items up (apply = 0); the merges splice the active queries
    PinJob pj_all;
    OCTRY(pin_job_init(pins, B, pj_all));
    oc_pins pins0{};
    if (pins) { pins0 = *pins; pins0.apply = 0; }
    std::vector<uint8_t> q_active(B, 0);
    bool any_active = false;
    for (uint32_t b = 0; b < B; b++) { q_active[b] = pj_all.splice && pj_all.cnt[b] > 0; any_active = any_active || q_active[b]; }
    // each query's page and each index's depth: limit + offset, twice that for an active query
    std::vector<uint2> q_page(B, make_uint2(p0->offset, limit));
    std::vector<oc_query_params> qp;
    uint64_t depth = 0;
    if (p0->q_params) {
        qp.assign(p0->q_params, p0->q_params + B);
        for (uint32_t b = 0; b < B; b++) {
            const oc_query_params &e = p0->q_params[b];
            if (e.vector_limit) return fail(OC_ERR_INVALID, "q_params[%u]: vector_limit must be 0", b);
            if (e.limit == 0) return fail(OC_ERR_INVALID, "q_params[%u]: limit must be >= 1", b);
            if (e.limit > limit) return fail(OC_ERR_INVALID, "q_params[%u]: limit %u > p->limit %u (the row stride)", b, e.limit, limit);
            const uint64_t d = (uint64_t(e.limit) + e.offset) * (q_active[b] ? 2 : 1);
            if (d > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "q_params[%u]: per-index depth %llu > %u", b, (unsigned long long)d, OC_MAX_TOPK);
            qp[b].limit = (uint32_t)d; qp[b].offset = 0; qp[b].vector_limit = e.limit;
            q_page[b] = make_uint2(e.offset, e.limit);
            depth = std::max(depth, d);
        }
    } else {
        depth = (uint64_t(limit) + p0->offset) * (any_active ? 2 : 1);
        if (depth > OC_MAX_TOPK) return fail(OC_ERR_UNSUPPORTED, "per-index depth %llu > %u", (unsigned long long)depth, OC_MAX_TOPK);
    }
    const uint32_t stride = (uint32_t)std::max<uint64_t>(depth, 1);
    // groups: each index's local rows and the collection's source tables
    MiGroups mg;
    OCTRY(mi_groups_plan(c, n_indexes, B, ex, q_n_keys, q_max_results, group_stride, q_active, pj_all, mg));
    const bool groups = !mg.gj.empty();
    if (mg.rows && (!out_group_n || (group_stride && (!out_group_doc_ids || !out_group_scores))))
        return fail(OC_ERR_INVALID, "NULL group output");
    // facets: per index, the requests of its unfiltered queries count on its main pass, those of its filtered queries on
    // an unfiltered pass over their sub-batch; every count is added to its collection slot
    bool any_facets = false;
    for (uint32_t i = 0; ex && i < n_indexes; i++) any_facets = any_facets || (ex[i].facets && ex[i].n_facet_reqs);
    const uint32_t *off = q_facet_offsets;
    const uint32_t s0 = off ? off[0] : 0, n_slots = off ? off[B] - off[0] : 0;
    if (off)
        for (uint32_t b = 0; b < B; b++)
            if (off[b + 1] < off[b]) return fail(OC_ERR_INVALID, "q_facet_offsets is not monotone at query %u", b);
    if (any_facets && !off) return fail(OC_ERR_INVALID, "facet requests without q_facet_offsets");
    if (n_slots && !out_facet_counts) return fail(OC_ERR_INVALID, "NULL facet counts");
    std::vector<FacetJob> fjm(n_indexes);
    std::vector<FacetSubBatch> fsb(n_indexes);
    for (uint32_t i = 0; any_facets && i < n_indexes; i++) {
        const oc_index_extras &e = ex[i];
        if (!e.facets || !e.n_facet_reqs) continue;
        if (e.facets->ctx != c) return fail(OC_ERR_INVALID, "index %u: facets belong to another ctx", i);
        if (!e.facet_reqs || !e.facet_slots) return fail(OC_ERR_INVALID, "index %u: NULL facet_reqs / facet_slots", i);
        OCTRY(oc_facets_check(e.facets, e.facet_reqs, e.n_facet_reqs));
        std::vector<uint8_t> seen(n_slots, 0);
        std::vector<uint3> items;
        for (uint32_t r = 0; r < e.n_facet_reqs; r++) {
            const uint32_t s = e.facet_slots[r];
            if (s < s0 || s - s0 >= n_slots) return fail(OC_ERR_INVALID, "index %u: facet request %u: slot %u outside [%u, %u)", i, r, s, s0, s0 + n_slots);
            if (seen[s - s0]) return fail(OC_ERR_INVALID, "index %u: two facet requests on slot %u", i, s);
            seen[s - s0] = 1;
            const uint32_t b = uint32_t(std::upper_bound(off, off + B + 1, s) - off) - 1;   // the query whose range holds s
            items.push_back(make_uint3(b, r, s - s0));
        }
        facet_split(ix[i].p, ix[i].emb, e.facets, e.facet_reqs, items, fjm[i], fsb[i]);
    }
    // every index's calls, checked before anything runs
    std::vector<oc_search_params> ps(n_indexes);
    std::vector<SortJob> sjs(n_indexes);
    std::vector<PinJob> pjs(n_indexes);
    std::vector<std::unique_ptr<SearchReq>> reqs;
    std::vector<std::unique_ptr<SearchCall>> calls, fcalls(n_indexes);
    const bool with_pj = pins || any_sorted || groups;
    for (uint32_t i = 0; i < n_indexes; i++) {
        ps[i] = *ix[i].p;
        ps[i].limit = stride; ps[i].offset = 0; ps[i].vector_limit = limit;
        ps[i].q_params = qp.empty() ? nullptr : qp.data();
        for (uint32_t b = 0; any_sorted && b < B; b++)
            OCTRY(sort_job_add(c, ix[i].q_sorts ? ix[i].q_sorts[b] : oc_sort{nullptr, OC_SORT_ASC}, sjs[i]));
        if (with_pj) OCTRY(pin_job_init(pins ? &pins0 : nullptr, B, pjs[i]));
        reqs.emplace_back(new SearchReq(&ps[i], out_doc_ids, out_scores, out_n, out_count));   // (its tail, copy_out, never runs)
        SearchReq &r = *reqs.back();
        r.pj = with_pj ? &pjs[i] : nullptr;
        r.sj = any_sorted ? &sjs[i] : nullptr;
        r.gj = groups && mg.gj[i].rows ? &mg.gj[i] : nullptr;
        r.fj = fjm[i].q.empty() ? nullptr : &fjm[i];
        r.q_filters_ok = r.q_params_ok = true;
        calls.emplace_back(new SearchCall(c, ix[i].emb, ix[i].str, r));
        OCTRY(search_check(*calls.back()));
        if (!fsb[i].sub.empty()) {   // the unfiltered facet pass of the index's filtered queries
            reqs.emplace_back(new SearchReq(&fsb[i].q, out_doc_ids, out_scores, out_n, out_count));
            SearchReq &fr = *reqs.back();
            fr.fj = &fsb[i].fj;
            fr.q_filters_ok = fr.q_params_ok = true;
            fcalls[i].reset(new SearchCall(c, ix[i].emb, ix[i].str, fr));
            OCTRY(search_check(*fcalls[i]));
        }
    }
    if (B == 0) return OC_OK;
    for (uint32_t i = 0; i < n_indexes; i++) {   // each index's string snapshot, before the lock
        calls[i]->snap = ix[i].str ? str_snapshot(ix[i].str) : nullptr;
        calls[i]->S = calls[i]->snap.get();
        if (fcalls[i]) { fcalls[i]->snap = calls[i]->snap; fcalls[i]->S = calls[i]->S; }
    }
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    const uint32_t pstr = pj_all.stride;
    const size_t per = size_t(B) * stride, nps = size_t(B) * pstr;
    OCTRY(c->mi_doc.ensure(n_indexes * per * 8));
    OCTRY(c->mi_score.ensure(n_indexes * per * 4));
    OCTRY(c->mi_n.ensure(size_t(n_indexes) * B * 4));
    OCTRY(c->mi_cnt.ensure(size_t(n_indexes) * B * 8));
    if (any_sorted) OCTRY(c->mi_val.ensure(n_indexes * per * 8));
    if (pstr) { OCTRY(c->mi_pscore.ensure(n_indexes * nps * 4)); OCTRY(c->mi_ppresent.ensure(n_indexes * nps)); }
    // the group lists of every index: [n_idx][rows][gtop]
    uint32_t grows = 0;
    for (const GroupJob &gj : mg.gj) grows = std::max(grows, gj.rows);
    const size_t gper = size_t(grows) * mg.gtop;
    if (groups) {
        OCTRY(c->mg_doc.ensure(std::max<size_t>(n_indexes * gper, 1) * 8));
        OCTRY(c->mg_score.ensure(std::max<size_t>(n_indexes * gper, 1) * 4));
        OCTRY(c->mg_n.ensure(std::max<size_t>(size_t(n_indexes) * grows, 1) * 4));
        if (any_sorted) OCTRY(c->mg_val.ensure(std::max<size_t>(n_indexes * gper, 1) * 8));
    }
    // the merged blob: the page, counts and pin outputs, then the group rows and the facet counts
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t R = mg.rows, gs = group_stride;
    const size_t o_sc = al(size_t(B) * limit * 8), o_val = o_sc + al(size_t(B) * limit * 4), o_n = o_val + al(size_t(B) * limit * 8),
                 o_cnt = o_n + al(size_t(B) * 4), o_ps = o_cnt + al(size_t(B) * 8), o_pp = o_ps + al(nps * 4), o_gd = o_pp + al(nps),
                 o_gs = o_gd + al(R * gs * 8), o_gv = o_gs + al(R * gs * 4), o_gn = o_gv + al(R * gs * 8), o_fc = o_gn + al(R * 4),
                 out_bytes = o_fc + size_t(n_slots) * 8;
    OCTRY(c->mi_out.ensure(out_bytes));
    uint8_t *dout = c->mi_out.as<uint8_t>();
    unsigned long long *d_fc = reinterpret_cast<unsigned long long *>(dout + o_fc);
    if (n_slots) CU(cudaMemsetAsync(d_fc, 0, size_t(n_slots) * 8, c->stream));
    for (uint32_t i = 0; i < n_indexes; i++) { fjm[i].d_out = d_fc; fsb[i].fj.d_out = d_fc; }
    // where each index's hits find their sort values: the handles' rank values on the device (built once per handle)
    std::vector<ImSortSrc> src(any_sorted ? size_t(n_indexes) * B : 0, ImSortSrc{nullptr, nullptr, 0});
    for (uint32_t i = 0; any_sorted && i < n_indexes; i++) {
        for (uint32_t e = 0; e < sjs[i].f.size(); e++) {
            SortOrder &o = sjs[i].ord(e);
            if (o.rank_value || !o.n) continue;
            CU(cudaMalloc(&o.rank_value, o.n * 8));
            CU(cudaMemcpyAsync(o.rank_value, o.h_value.data(), o.n * 8, cudaMemcpyHostToDevice, c->stream));
        }
        for (uint32_t b = 0; b < B; b++) {
            const uint32_t e = sjs[i].q_ent[b];
            if (e != SORT_BY_SCORE) src[size_t(i) * B + b] = ImSortSrc{sjs[i].ord(e).doc_rank, sjs[i].ord(e).rank_value, sjs[i].f[e]->nbits};
        }
    }
    oc_timing total{};
    // the device time of an index's group and facet stages, read once a later synchronise has passed them
    bool extra_pending = false;
    auto extra_time = [&]() -> int {
        if (!extra_pending) return OC_OK;
        float ms = 0.f;
        CU(cudaEventElapsedTime(&ms, c->ev[EV_GRP0], c->ev[EV_GRP1]));
        total.device_ms += ms;
        extra_pending = false;
        return OC_OK;
    };
    for (uint32_t i = 0; i < n_indexes; i++) {
        SearchCall &k = *calls[i];
        OCTRY(search_stages(k));
        OCTRY(extra_time());
        OCTRY(finish_timing(c, k.has_v && k.vlimit && k.emb->n_rows > 0, k.has_ft, true, k.did_comm));
        c->timing.d2h_bytes = k.out_bytes;
        timing_add(total, c->timing);
        // the index's top list and item lookups into its slot (the next index's stages reuse the ctx's buffers)
        CU(cudaMemcpyAsync(c->mi_doc.as<uint64_t>() + i * per, k.d_doc, per * 8, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(c->mi_score.as<float>() + i * per, k.d_score, per * 4, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(c->mi_n.as<uint32_t>() + size_t(i) * B, k.d_n, size_t(B) * 4, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaMemcpyAsync(c->mi_cnt.as<uint64_t>() + size_t(i) * B, k.dout + k.o_cnt, size_t(B) * 8, cudaMemcpyDeviceToDevice, c->stream));
        if (pstr) {
            CU(cudaMemcpyAsync(c->mi_pscore.as<float>() + i * nps, c->pin_score.p, nps * 4, cudaMemcpyDeviceToDevice, c->stream));
            CU(cudaMemcpyAsync(c->mi_ppresent.as<uint8_t>() + i * nps, c->pin_present.p, nps, cudaMemcpyDeviceToDevice, c->stream));
        }
        // its facet counts, added into the collection slots, and its group lists into its slot
        const GroupJob *gj = k.r.gj;
        const uint32_t l0 = c->call_launches;
        if (k.facets || (gj && gj->rows)) {
            CU(cudaEventRecord(c->ev[EV_GRP0], c->stream));
            if (k.facets) OCTRY(run_facets(c, *k.r.fj, k.fpl, B, k.has_ft, k.has_v, k.S, k.n_tiles, k.vlimit));
            if (gj && gj->rows) {
                OCTRY(run_groups(c, *gj, k.mode, k.S, k.n_tiles, k.vlimit, k.fp.omc_doc, k.fp.omc_mult, k.n_omc, *k.r.pj, k.s_plan.at(c->in_blob)));
                const size_t o = i * gper;
                if (gj->top) {
                    CU(cudaMemcpy2DAsync(c->mg_doc.as<uint64_t>() + o, size_t(mg.gtop) * 8, c->grp_doc.p, size_t(gj->top) * 8,
                                         size_t(gj->top) * 8, gj->rows, cudaMemcpyDeviceToDevice, c->stream));
                    CU(cudaMemcpy2DAsync(c->mg_score.as<float>() + o, size_t(mg.gtop) * 4, c->grp_score.p, size_t(gj->top) * 4,
                                         size_t(gj->top) * 4, gj->rows, cudaMemcpyDeviceToDevice, c->stream));
                }
                CU(cudaMemcpyAsync(c->mg_n.as<uint32_t>() + size_t(i) * grows, c->grp_n.p, size_t(gj->rows) * 4, cudaMemcpyDeviceToDevice, c->stream));
            }
            CU(cudaEventRecord(c->ev[EV_GRP1], c->stream));
            extra_pending = true;
            total.kernel_launches += c->call_launches - l0;
        }
        if (fcalls[i]) {   // the unfiltered facet pass of its filtered queries
            SearchCall &f = *fcalls[i];
            OCTRY(search_stages(f));
            OCTRY(extra_time());
            OCTRY(finish_timing(c, f.has_v && f.vlimit && f.emb->n_rows > 0, f.has_ft, true, f.did_comm));
            c->timing.d2h_bytes = f.out_bytes;
            timing_add(total, c->timing);
            CU(cudaEventRecord(c->ev[EV_GRP0], c->stream));
            const uint32_t l1 = c->call_launches;
            OCTRY(run_facets(c, *f.r.fj, f.fpl, f.B, f.has_ft, f.has_v, f.S, f.n_tiles, f.vlimit));
            CU(cudaEventRecord(c->ev[EV_GRP1], c->stream));
            extra_pending = true;
            total.kernel_launches += c->call_launches - l1;
        }
    }
    // the merges: their tables in one upload, one CTA per query (hits) and per (query, collection group), one copy
    Packer pk;
    const Slot<uint8_t> s_sort = pk.add(q_sort.data(), B), s_act = pk.add(q_active.data(), B);
    const Slot<uint2> s_page = pk.add(q_page.data(), B);
    Slot<ImSortSrc> s_src;
    Slot<uint64_t> s_pdoc;
    Slot<uint32_t> s_ppos, s_pcnt, s_srcg, s_lrow;
    Slot<GroupHandle> s_seth;
    Slot<GroupSpan> s_spans;
    if (any_sorted) s_src = pk.add(src.data(), src.size());
    if (pstr) { s_pdoc = pk.add(pj_all.doc.data(), nps); s_ppos = pk.add(pj_all.pos.data(), nps); s_pcnt = pk.add(pj_all.cnt.data(), B); }
    if (mg.rows) {
        s_srcg = pk.add(mg.src_g.data(), mg.src_g.size());
        s_lrow = pk.add(mg.q_lrow.data(), mg.q_lrow.size());
        s_seth = pk.add(mg.set_h.data(), mg.set_h.size());
        s_spans = pk.add(mg.spans.data(), mg.spans.size());
    }
    OCTRY(c->h_out.ensure(out_bytes));
    CU(cudaEventRecord(c->ev[EV_START], c->stream));
    OCTRY(upload(pk, c->h_in, c->in_blob, c->stream));
    CU(cudaEventRecord(c->ev[EV_H2D], c->stream));
    IndexMergeParams mp{};
    mp.n_idx = n_indexes; mp.B = B; mp.stride = stride;
    mp.doc = c->mi_doc.as<uint64_t>(); mp.score = c->mi_score.as<float>(); mp.n = c->mi_n.as<uint32_t>();
    mp.count = c->mi_cnt.as<unsigned long long>(); mp.value = c->mi_val.as<double>();
    mp.src = s_src.at(c->in_blob); mp.q_sort = s_sort.at(c->in_blob); mp.q_page = s_page.at(c->in_blob); mp.q_active = s_act.at(c->in_blob);
    mp.pin_stride = pstr; mp.kp2 = std::max<uint32_t>(32, next_pow2(pstr));
    mp.pin_doc = s_pdoc.at(c->in_blob); mp.pin_pos = s_ppos.at(c->in_blob); mp.pin_cnt = s_pcnt.at(c->in_blob);
    mp.pin_score = c->mi_pscore.as<float>(); mp.pin_present = c->mi_ppresent.as<uint8_t>();
    mp.take_max = stride; mp.limit = limit;
    mp.out_doc = reinterpret_cast<uint64_t *>(dout); mp.out_score = reinterpret_cast<float *>(dout + o_sc);
    mp.out_value = reinterpret_cast<double *>(dout + o_val); mp.out_n = reinterpret_cast<uint32_t *>(dout + o_n);
    mp.out_count = reinterpret_cast<unsigned long long *>(dout + o_cnt);
    mp.out_pin_score = reinterpret_cast<float *>(dout + o_ps); mp.out_pin_present = dout + o_pp;
    const size_t smem = index_merge_smem(stride, pstr, mp.kp2, limit);
    CU(smem_cfg(c->device, (const void *)index_merge_kernel, smem));
    index_merge_kernel<<<B, IM_THREADS, smem, c->stream>>>(mp);
    launched(c);
    CU(cudaGetLastError());
    if (mg.rows) {
        IndexGroupMergeParams gp{};
        gp.n_idx = n_indexes; gp.B = B;
        gp.spans = s_spans.at(c->in_blob); gp.n_spans = (uint32_t)mg.spans.size();
        gp.src_g = s_srcg.at(c->in_blob); gp.set_h = s_seth.at(c->in_blob); gp.q_lrow = s_lrow.at(c->in_blob);
        gp.rows = grows; gp.gtop = mg.gtop;
        gp.g_doc = c->mg_doc.as<uint64_t>(); gp.g_score = c->mg_score.as<float>(); gp.g_n = c->mg_n.as<uint32_t>();
        gp.g_val = c->mg_val.as<double>();
        gp.src = mp.src; gp.q_sort = mp.q_sort; gp.q_active = mp.q_active;
        gp.pin_stride = pstr; gp.kp2 = mp.kp2; gp.pin_doc = mp.pin_doc; gp.pin_pos = mp.pin_pos; gp.pin_cnt = mp.pin_cnt;
        gp.pin_score = mp.pin_score; gp.pin_present = mp.pin_present;
        gp.take_max = std::max<uint32_t>(mg.gtop, 1);
        gp.n_slots = (uint32_t)std::min<uint64_t>(group_stride, uint64_t(gp.take_max) + pstr);
        gp.stride = group_stride;
        gp.out_doc = reinterpret_cast<uint64_t *>(dout + o_gd); gp.out_score = reinterpret_cast<float *>(dout + o_gs);
        gp.out_value = reinterpret_cast<double *>(dout + o_gv); gp.out_n = reinterpret_cast<uint32_t *>(dout + o_gn);
        const size_t gsmem = index_group_merge_smem(gp.take_max, pstr, gp.kp2, gp.n_slots);
        CU(smem_cfg(c->device, (const void *)index_group_merge_kernel, gsmem));
        index_group_merge_kernel<<<mg.rows, IM_THREADS, gsmem, c->stream>>>(gp);
        launched(c);
        CU(cudaGetLastError());
    }
    CU(cudaEventRecord(c->ev[EV_DEV], c->stream));
    uint8_t *h = c->h_out.as<uint8_t>();
    CU(cudaMemcpyAsync(h, dout, out_bytes, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaEventRecord(c->ev[EV_D2H], c->stream));
    CU(cudaStreamSynchronize(c->stream));
    OCTRY(extra_time());
    memcpy(out_doc_ids, h, size_t(B) * limit * 8);
    memcpy(out_scores, h + o_sc, size_t(B) * limit * 4);
    if (out_sort_values) memcpy(out_sort_values, h + o_val, size_t(B) * limit * 8);
    memcpy(out_n, h + o_n, size_t(B) * 4);
    memcpy(out_count, h + o_cnt, size_t(B) * 8);
    for (uint32_t q = 0; pstr && q < B; q++)
        for (uint32_t j = 0; j < pj_all.cnt[q]; j++) {
            const size_t it = size_t(pins->q_pin_offsets[q]) + j, s = size_t(q) * pstr + j;
            if (out_pin_scores) memcpy(out_pin_scores + it, h + o_ps + s * 4, 4);
            if (out_pin_present) out_pin_present[it] = h[o_pp + s];
        }
    if (R) {
        if (gs) {
            memcpy(out_group_doc_ids, h + o_gd, R * gs * 8);
            memcpy(out_group_scores, h + o_gs, R * gs * 4);
            if (out_group_sort_values) memcpy(out_group_sort_values, h + o_gv, R * gs * 8);
        }
        memcpy(out_group_n, h + o_gn, R * 4);
    }
    if (n_slots) memcpy(out_facet_counts + s0, h + o_fc, size_t(n_slots) * 8);
    auto el = [&](int a, int b) { float ms = 0; cudaEventElapsedTime(&ms, c->ev[a], c->ev[b]); return ms; };
    total.h2d_ms += el(EV_START, EV_H2D);
    total.device_ms += el(EV_H2D, EV_DEV);
    total.fuse_ms += el(EV_H2D, EV_DEV);
    total.d2h_ms += el(EV_DEV, EV_D2H);
    total.kernel_launches += mg.rows ? 2 : 1;
    total.h2d_bytes += pk.total;
    total.d2h_bytes += out_bytes;
    c->timing = total;
    return OC_OK;
}

extern "C" int oc_search_indexes(oc_ctx *c, uint32_t n_indexes, const oc_index_query *ix, const oc_pins *pins,
                                 uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                                 uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present) {
    return oc_search_indexes_ex(c, n_indexes, ix, nullptr, pins, nullptr, nullptr, 0, nullptr, out_doc_ids, out_scores,
                                out_sort_values, out_n, out_count, out_pin_scores, out_pin_present, nullptr, nullptr, nullptr,
                                nullptr, nullptr);
}

// One batch in which every query has its own groups (or none), sort, pins and, with q_filters, filter: query b gets what
// it gets alone through the grouped call or oc_search_q_sorted its request stands for.
extern "C" int oc_search_q_groups(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_group_req *q_groups,
                                  const oc_pins *pins, uint32_t group_stride, uint64_t *out_doc_ids, float *out_scores,
                                  double *out_sort_values, uint32_t *out_n, uint64_t *out_count, float *out_pin_scores,
                                  uint8_t *out_pin_present, uint64_t *out_group_doc_ids, float *out_group_scores,
                                  double *out_group_sort_values, uint32_t *out_group_n) {
    if (!c || !p || !q_groups) return fail(OC_ERR_INVALID, "NULL argument");
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "groups over a sharded search: hybrid normalisation and the vector set are global");
    return groups_impl(c, emb, str, p, q_groups, pins, group_stride, true, out_doc_ids, out_scores, out_sort_values, out_n, out_count,
                       out_pin_scores, out_pin_present, out_group_doc_ids, out_group_scores, out_group_sort_values, out_group_n);
}

// oc_search_q_groups with each query's facets.  A query without a filter counts on the matched-row bitmap of the main
// pass; the queries with a filter and facets are re-scored unfiltered in one more pass over just their sub-batch (adding
// unfiltered copies to the main batch would multiply its row-score workspace).
extern "C" int oc_search_q_facets(oc_ctx *c, oc_emb *emb, oc_str *str, const oc_search_params *p, const oc_group_req *q_groups,
                                  const oc_pins *pins, uint32_t group_stride, oc_facets *facets, const uint32_t *q_facet_offsets,
                                  const oc_facet_req *facet_reqs, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                                  uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present,
                                  uint64_t *out_group_doc_ids, float *out_group_scores, double *out_group_sort_values,
                                  uint32_t *out_group_n, uint64_t *out_facet_counts) {
    if (!c || !p || !facets || !q_facet_offsets) return fail(OC_ERR_INVALID, "NULL argument");
    if (p->sharded) return fail(OC_ERR_UNSUPPORTED, "facets over a sharded search: count per shard and add the counts");
    if (facets->ctx != c) return fail(OC_ERR_INVALID, "facets belong to another ctx");
    const uint32_t B = p->n_queries;
    const uint32_t *off = q_facet_offsets;
    for (uint32_t b = 0; b < B; b++)
        if (off[b + 1] < off[b]) return fail(OC_ERR_INVALID, "q_facet_offsets is not monotone at query %u", b);
    if (off[B] > off[0] && (!facet_reqs || !out_facet_counts)) return fail(OC_ERR_INVALID, "NULL facet requests / counts");
    if (off[B] > off[0]) OCTRY(oc_facets_check(facets, facet_reqs + off[0], off[B] - off[0]));
    std::vector<oc_group_req> none;
    if (!q_groups) {
        none.assign(B, oc_group_req{nullptr, 0, oc_sort{nullptr, OC_SORT_ASC}});
        q_groups = none.data();
    }
    std::vector<uint3> items;
    for (uint32_t b = 0; b < B; b++)
        for (uint32_t i = off[b]; i < off[b + 1]; i++) items.push_back(make_uint3(b, i, i));
    FacetJob mj;
    FacetSubBatch sb;
    facet_split(p, emb, facets, facet_reqs, items, mj, sb);
    mj.out_counts = sb.fj.out_counts = out_facet_counts;
    mj.q_off = off;
    OCTRY(groups_impl(c, emb, str, p, q_groups, pins, group_stride, true, out_doc_ids, out_scores, out_sort_values, out_n, out_count,
                      out_pin_scores, out_pin_present, out_group_doc_ids, out_group_scores, out_group_sort_values, out_group_n, &mj));
    if (sb.sub.empty()) return OC_OK;
    return facets_unfiltered(c, emb, str, &sb.q, sb.fj, true);
}

// ------------------------------------------------------------------------------------ geopoint where-filter leaves (geo.cuh)
static_assert(OC_GEO_MAX_VERTICES == GEO_MAX_VERTICES, "the header's vertex cap is the kernel's staging size");
constexpr double GEO_PI = 3.14159265358979323846;

struct oc_geo_field {
    oc_ctx *ctx;
    uint64_t nbits, n;
    void *blob = nullptr;   // device: x, y, z, lat, lon (f64) then doc (u64), n entries each
    FcPending pend;         // one field (0)
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

extern "C" int oc_geo_field_insert(oc_geo_field *g, uint64_t n, const uint64_t *doc_ids, const double *lat, const double *lon) {
    if (!g || (n && (!doc_ids || !lat || !lon))) return fail(OC_ERR_INVALID, "NULL argument");
    for (uint64_t i = 0; i < n; i++)
        if (!geo_valid(lat[i], lon[i]))
            return fail(OC_ERR_INVALID, "geopoint %llu: invalid coordinates (%g, %g)", (unsigned long long)i, lat[i], lon[i]);
    FcPending &P = g->pend;
    std::lock_guard<std::mutex> lk(P.mu);
    for (uint64_t i = 0; i < n; i++) P.ins.push_back(FcIns{doc_ids[i], ++P.seq, 0.0, lat[i], lon[i], 0, 0, false});
    return OC_OK;
}
extern "C" int oc_geo_field_delete(oc_geo_field *g, uint64_t n, const uint64_t *doc_ids) {
    if (!g || (n && !doc_ids)) return fail(OC_ERR_INVALID, "NULL argument");
    FcPending &P = g->pend;
    std::lock_guard<std::mutex> lk(P.mu);
    for (uint64_t i = 0; i < n; i++) P.del[doc_ids[i]] = ++P.seq;
    return OC_OK;
}
extern "C" int oc_geo_field_commit_ex(oc_geo_field *g, uint64_t new_nbits, oc_filter_commit_t *out) {
    if (!g) return fail(OC_ERR_INVALID, "NULL argument");
    const auto wall0 = std::chrono::steady_clock::now();
    oc_ctx *c = g->ctx;
    FcPending &P = g->pend;
    std::vector<FcIns> ins;
    std::unordered_map<uint64_t, uint64_t> del;
    std::map<std::pair<uint32_t, uint64_t>, uint64_t> clr;
    uint64_t cut = 0;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        OCTRY(fc_begin(P, g->nbits, new_nbits, c->device, ins, del, clr, cut));
    }
    FcMergeIn in;
    in.kind = FC_GEO;
    fc_take(P, ins, del, clr, 0, FC_GEO, in);
    FcMergeOut res;
    oc_filter_commit_t st{};
    const bool changed = !in.kb.empty() || !in.kill.empty();
    if (changed) {
        in.n_a = g->n; in.a_vals = static_cast<const double *>(g->blob);
        const int rc = fc_merge(P.stream, P.ev, in, res);
        if (rc != OC_OK) { fc_end(P, false, 0, 0); return rc; }
        st.rows_kept = res.kept; st.rows_dropped = g->n - res.kept; st.rows_added = res.added; st.workspace_bytes = res.ws;
        st.device_ms = res.device_ms;
    } else {
        st.rows_kept = g->n;
    }
    {   // publish (see oc_facets_commit_ex)
        std::lock_guard<std::mutex> lk(c->mu);
        cudaSetDevice(c->device);
        g->nbits = new_nbits;
        if (changed) {
            void *old = g->blob;
            g->blob = res.dev; g->n = res.n;
            cudaStreamSynchronize(c->stream);
            cudaFree(old);
        }
    }
    st.version = fc_end(P, true, ins.size(), cut);
    st.wall_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - wall0).count();
    if (out) *out = st;
    return OC_OK;
}
extern "C" int oc_geo_field_read(oc_geo_field *g, uint64_t *n, uint64_t *doc_ids, double *lat, double *lon) {
    if (!g || !n) return fail(OC_ERR_INVALID, "NULL argument");
    oc_ctx *c = g->ctx;
    std::lock_guard<std::mutex> lk(c->mu);
    const uint64_t cap = *n;
    *n = g->n;
    if (!doc_ids && !lat && !lon) return OC_OK;
    if (cap < g->n) return fail(OC_ERR_INVALID, "arrays hold %llu points, the field has %llu", (unsigned long long)cap, (unsigned long long)g->n);
    CU(cudaSetDevice(c->device));
    const GeoPoints p = g->pts();
    if (g->n && doc_ids) CU(cudaMemcpy(doc_ids, p.doc, g->n * 8, cudaMemcpyDeviceToHost));
    if (g->n && lat) CU(cudaMemcpy(lat, p.lat, g->n * 8, cudaMemcpyDeviceToHost));
    if (g->n && lon) CU(cudaMemcpy(lon, p.lon, g->n * 8, cudaMemcpyDeviceToHost));
    return OC_OK;
}

// ------------------------------------------------------------------------------------ where programs (where.cuh)
// The where programs of queries [q0, q0 + n), planned on the host: their distinct leaves (keyed on store, field and
// parameters, facet leaves on their resolved slice), their distinct programs of more than one node (keyed on content),
// and the bitmap each query is filtered by.  Workspace slots: the leaves that need a bitmap, then the programs.
struct WherePlan {
    uint64_t nbits = 0, words = 0;
    std::vector<const oc_filter *> leaf_h;   // per distinct leaf: its handle (FILTER), else NULL
    std::vector<uint32_t> leaf_slot;          // per distinct leaf: its workspace slot (not FILTER)
    uint32_t n_leaf_slots = 0;
    std::vector<WhereSlice> slices;           // .bits holds the slot until where_run
    std::vector<WhereGeo> geo;                // .bits holds the slot, .vlon the vertex offset until where_run
    std::vector<double> verts;                // polygon vertices: lon[nv] then lat[nv] per polygon leaf
    uint64_t total = 0;                       // ids of all slices
    std::vector<WhereOp> ops;
    std::vector<WhereProg> progs;             // .out is set by where_run
    // per query: UINT32_MAX unfiltered, else its result: a leaf index (a program of one node) or leaves + program index
    std::vector<uint32_t> q_res;
};
static uint64_t dbits(double x) { uint64_t u; memcpy(&u, &x, 8); return u; }

// Checks queries [q0, q0 + n) of w (c: the ctx they must belong to, NULL: the ctx of the first store or handle, taken
// from *c_out) and, with pl, plans them.  Called with the stores' ctx lock held.
static int where_plan(const oc_where *w, uint32_t q0, uint32_t n, const oc_ctx *c, WherePlan *pl) {
    constexpr uint32_t PROG_BIT = 1u << 31;
    if (!w || !w->q_node_offsets) return fail(OC_ERR_INVALID, "q_where: NULL argument");
    const uint32_t *off = w->q_node_offsets;
    for (uint32_t b = q0; b < q0 + n; b++) {
        if (off[b + 1] < off[b]) return fail(OC_ERR_INVALID, "q_where: q_node_offsets is not monotone at query %u", b);
        if (off[b + 1] > off[b] && !w->nodes) return fail(OC_ERR_INVALID, "q_where: nodes is NULL");
    }
    std::map<std::vector<uint64_t>, uint32_t> leaf_idx, prog_idx;
    if (pl) { pl->nbits = w->nbits; pl->words = (w->nbits + 63) / 64; pl->q_res.assign(n, UINT32_MAX); }
    auto same_ctx = [&](const oc_ctx *x) { if (!c) c = x; return x == c; };
    for (uint32_t b = q0; b < q0 + n; b++) {
        const uint32_t len = off[b + 1] - off[b];
        if (len == 0) continue;
        if (len > OC_WHERE_MAX_NODES) return fail(OC_ERR_INVALID, "q_where[%u]: %u nodes > %u", b, len, OC_WHERE_MAX_NODES);
        std::vector<uint64_t> prog;   // (WHERE_PUSH, leaf) / (op, arity) pairs
        uint32_t sp = 0;
        for (uint32_t i = 0; i < len; i++) {
            const oc_where_node &nd = w->nodes[off[b] + i];
            std::vector<uint64_t> key;
            const oc_filter *h = nullptr;
            const FacetField *ff = nullptr; uint64_t lo = 0, hi = 0;
            const oc_geo_field *g = nullptr;
            double u[3] = {0, 0, 0}, thr = 0; double4 bb{};
            switch (nd.op) {
            case OC_WHERE_NONE: key = {0}; break;
            case OC_WHERE_VARIANT: case OC_WHERE_RANGE: {
                const oc_facets *f = static_cast<const oc_facets *>(nd.src);
                const bool number = nd.op == OC_WHERE_RANGE;
                if (!f) return fail(OC_ERR_INVALID, "q_where[%u] node %u: NULL facet store", b, i);
                if (!same_ctx(f->ctx)) return fail(OC_ERR_INVALID, "q_where[%u] node %u: facet store of another ctx", b, i);
                if (f->nbits != w->nbits)
                    return fail(OC_ERR_INVALID, "q_where[%u] node %u: store nbits %llu != %llu", b, i, (unsigned long long)f->nbits,
                                (unsigned long long)w->nbits);
                if (number && (std::isnan(nd.a) || std::isnan(nd.b))) return fail(OC_ERR_INVALID, "q_where[%u] node %u: NaN range bound", b, i);
                if (number && (nd.arg & ~(OC_RANGE_LO_OPEN | OC_RANGE_HI_OPEN)))
                    return fail(OC_ERR_INVALID, "q_where[%u] node %u: unknown range flags 0x%x", b, i, nd.arg);
                if (nd.field >= f->fields.size())
                    return fail(OC_ERR_INVALID, "q_where[%u] node %u: field %u: the store has %zu fields", b, i, nd.field, f->fields.size());
                ff = &f->fields[nd.field];
                if (ff->number != number)
                    return fail(OC_ERR_INVALID, "q_where[%u] node %u: field %u is a %s field", b, i, nd.field,
                                ff->number ? "number" : "bool / string_filter");
                if (!facet_slice(*ff, nd.arg, nd.a, nd.b, lo, hi))
                    return fail(OC_ERR_INVALID, "q_where[%u] node %u: variant %u: field %u has %zu variants", b, i, nd.arg, nd.field,
                                ff->offsets.size() - 1);
                key = hi > lo ? std::vector<uint64_t>{1, uint64_t(uintptr_t(ff->docs)), lo, hi} : std::vector<uint64_t>{0};
                break;
            }
            case OC_WHERE_GEO_RADIUS: case OC_WHERE_GEO_POLYGON: {
                g = static_cast<const oc_geo_field *>(nd.src);
                if (!g) return fail(OC_ERR_INVALID, "q_where[%u] node %u: NULL geo field", b, i);
                if (!same_ctx(g->ctx)) return fail(OC_ERR_INVALID, "q_where[%u] node %u: geo field of another ctx", b, i);
                if (g->nbits != w->nbits)
                    return fail(OC_ERR_INVALID, "q_where[%u] node %u: geo field nbits %llu != %llu", b, i, (unsigned long long)g->nbits,
                                (unsigned long long)w->nbits);
                const uint64_t inside = nd.arg != 0;
                if (nd.op == OC_WHERE_GEO_RADIUS) {   // the chord threshold of geo_in_radius
                    if (!geo_valid(nd.a, nd.b)) return fail(OC_ERR_INVALID, "q_where[%u] node %u: radius centre: invalid coordinates (%g, %g)", b, i, nd.a, nd.b);
                    if (!(std::isfinite(nd.c) && nd.c >= 0.0)) return fail(OC_ERR_INVALID, "q_where[%u] node %u: radius %g m: not finite and >= 0", b, i, nd.c);
                    geo_unit(nd.a, nd.b, u);
                    const double half = nd.c / (2.0 * OC_GEO_EARTH_RADIUS_M);
                    const double s = std::sin(half);
                    thr = half >= GEO_PI / 2 ? std::numeric_limits<double>::infinity() : 4.0 * s * s;
                    key = {2, uint64_t(uintptr_t(g)), dbits(u[0]), dbits(u[1]), dbits(u[2]), dbits(thr), inside};
                } else {   // the bounding box of geo_in_polygon's pre-test
                    const uint32_t nv = nd.n_vertices;
                    if (nv < 3 || nv > OC_GEO_MAX_VERTICES)
                        return fail(OC_ERR_INVALID, "q_where[%u] node %u: polygon of %u vertices: 3 to %u are supported", b, i, nv, OC_GEO_MAX_VERTICES);
                    if (!w->vertex_lat || !w->vertex_lon) return fail(OC_ERR_INVALID, "q_where[%u] node %u: NULL vertices", b, i);
                    const double *la = w->vertex_lat + nd.first_vertex, *ln = w->vertex_lon + nd.first_vertex;
                    bb = make_double4(ln[0], ln[0], la[0], la[0]);
                    key = {3, uint64_t(uintptr_t(g)), inside, nv};
                    for (uint32_t v = 0; v < nv; v++) {
                        if (!geo_valid(la[v], ln[v]))
                            return fail(OC_ERR_INVALID, "q_where[%u] node %u: polygon vertex %u: invalid coordinates (%g, %g)", b, i, v, la[v], ln[v]);
                        bb.x = std::min(bb.x, ln[v]); bb.y = std::max(bb.y, ln[v]); bb.z = std::min(bb.z, la[v]); bb.w = std::max(bb.w, la[v]);
                        key.push_back(dbits(la[v])); key.push_back(dbits(ln[v]));
                    }
                    bb.x -= GEO_BBOX_MARGIN; bb.y += GEO_BBOX_MARGIN;
                }
                if (g->n == 0) key = {0};   // no point: an empty leaf
                break;
            }
            case OC_WHERE_FILTER:
                h = static_cast<const oc_filter *>(nd.src);
                if (!h) return fail(OC_ERR_INVALID, "q_where[%u] node %u: NULL filter", b, i);
                if (!same_ctx(h->ctx)) return fail(OC_ERR_INVALID, "q_where[%u] node %u: filter of another ctx", b, i);
                if (len > 1 && h->nbits != w->nbits)
                    return fail(OC_ERR_INVALID, "q_where[%u] node %u: filter nbits %llu != %llu", b, i, (unsigned long long)h->nbits,
                                (unsigned long long)w->nbits);
                key = {4, uint64_t(uintptr_t(h))};
                break;
            case OC_WHERE_AND: case OC_WHERE_OR: case OC_WHERE_NOT: {
                const uint32_t ar = nd.op == OC_WHERE_NOT ? 1u : nd.arg;
                if (nd.op != OC_WHERE_NOT && ar < 2) return fail(OC_ERR_INVALID, "q_where[%u] node %u: arity %u < 2", b, i, ar);
                if (sp < ar) return fail(OC_ERR_INVALID, "q_where[%u] node %u: stack underflow", b, i);
                sp -= ar - 1;
                prog.push_back(uint64_t(nd.op) << 32 | ar);
                continue;
            }
            default: return fail(OC_ERR_INVALID, "q_where[%u] node %u: unknown op %u", b, i, nd.op);
            }
            if (++sp > OC_WHERE_MAX_DEPTH) return fail(OC_ERR_INVALID, "q_where[%u]: stack deeper than %u", b, OC_WHERE_MAX_DEPTH);
            if (!pl) continue;
            auto it = leaf_idx.emplace(key, (uint32_t)pl->leaf_h.size()).first;
            if (it->second == pl->leaf_h.size()) {   // a new leaf
                pl->leaf_h.push_back(h);
                pl->leaf_slot.push_back(h ? UINT32_MAX : pl->n_leaf_slots++);
                const uint32_t slot = pl->leaf_slot.back();
                if (key[0] == 1) {
                    pl->slices.push_back(WhereSlice{ff->docs + lo, pl->total, reinterpret_cast<unsigned long long *>(uintptr_t(slot))});
                    pl->total += hi - lo;
                } else if (key[0] == 2 || key[0] == 3) {
                    WhereGeo L{};
                    L.g = g->pts(); L.cx = u[0]; L.cy = u[1]; L.cz = u[2]; L.thr = thr; L.bbox = bb; L.inside = nd.arg != 0;
                    L.bits = reinterpret_cast<unsigned long long *>(uintptr_t(slot));
                    if (key[0] == 3) {
                        L.nv = nd.n_vertices;
                        L.vlon = reinterpret_cast<const double *>(uintptr_t(pl->verts.size()));
                        pl->verts.insert(pl->verts.end(), w->vertex_lon + nd.first_vertex, w->vertex_lon + nd.first_vertex + L.nv);
                        pl->verts.insert(pl->verts.end(), w->vertex_lat + nd.first_vertex, w->vertex_lat + nd.first_vertex + L.nv);
                    }
                    pl->geo.push_back(L);
                }
            }
            prog.push_back(uint64_t(WHERE_PUSH) << 32 | it->second);
        }
        if (sp != 1) return fail(OC_ERR_INVALID, "q_where[%u]: the program leaves %u values, not 1", b, sp);
        if (!pl) continue;
        if (prog.size() == 1) { pl->q_res[b - q0] = uint32_t(prog[0]); continue; }   // one leaf: its bitmap
        auto it = prog_idx.emplace(prog, (uint32_t)pl->progs.size()).first;
        if (it->second == pl->progs.size()) {
            pl->progs.push_back(WhereProg{(uint32_t)pl->ops.size(), (uint32_t)prog.size(), nullptr});
            for (uint64_t o : prog) pl->ops.push_back(WhereOp{uint32_t(o >> 32), uint32_t(o)});
        }
        pl->q_res[b - q0] = PROG_BIT | it->second;   // numbered after the leaves below, once their count is known
    }
    if (pl)
        for (uint32_t &r : pl->q_res)
            if (r != UINT32_MAX && (r & PROG_BIT)) r = (uint32_t)pl->leaf_h.size() + (r & ~PROG_BIT);
    return OC_OK;
}

// Uploads the plan and materialises every leaf and program on c->stream: one zeroing of the leaf bitmaps, then at most
// one launch each of where_scatter_kernel, where_geo_kernel and where_eval_kernel.  bits[r] afterwards: the bitmap of
// result r (a leaf, then the programs) as q_res numbers them.  res_bits (NULL: none) takes the place of result res's
// workspace slot, so a handle's bitmap is written in place; a FILTER leaf keeps its own bitmap.  The result of a plan
// of one query is its last slot, which the workspace then leaves out.
static int where_run(oc_ctx *c, WherePlan &pl, std::vector<const uint64_t *> &bits, uint32_t res = UINT32_MAX,
                     uint64_t *res_bits = nullptr) {
    const uint64_t words = pl.words;
    const uint32_t n_slots = pl.n_leaf_slots + (uint32_t)pl.progs.size();
    const uint32_t n_leaves = (uint32_t)pl.leaf_h.size();
    const uint32_t res_slot = !res_bits || res == UINT32_MAX ? UINT32_MAX
                              : res >= n_leaves              ? pl.n_leaf_slots + (res - n_leaves)
                              : pl.leaf_h[res]               ? UINT32_MAX
                                                             : pl.leaf_slot[res];
    const uint32_t n_ws = res_slot != UINT32_MAX && res_slot + 1 == n_slots ? n_slots - 1 : n_slots;
    OCTRY(c->w_bits.ensure(std::max<size_t>(size_t(n_ws) * words * 8, 8)));
    uint64_t *ws = c->w_bits.as<uint64_t>();
    auto slot_bits = [&](uint32_t s) { return reinterpret_cast<unsigned long long *>(s == res_slot ? res_bits : ws + size_t(s) * words); };
    std::vector<const unsigned long long *> leaf_ptr(pl.leaf_h.size());
    bits.resize(pl.leaf_h.size() + pl.progs.size());
    for (size_t i = 0; i < pl.leaf_h.size(); i++) {
        leaf_ptr[i] = pl.leaf_h[i] ? reinterpret_cast<const unsigned long long *>(pl.leaf_h[i]->bits) : slot_bits(pl.leaf_slot[i]);
        bits[i] = reinterpret_cast<const uint64_t *>(leaf_ptr[i]);
    }
    for (size_t p = 0; p < pl.progs.size(); p++) {
        pl.progs[p].out = slot_bits(pl.n_leaf_slots + (uint32_t)p);
        bits[pl.leaf_h.size() + p] = reinterpret_cast<const uint64_t *>(pl.progs[p].out);
    }
    if (words == 0) return OC_OK;
    Packer pk;
    const Slot<double> s_v = pk.add(pl.verts.data(), pl.verts.size());
    const Slot<WhereSlice> s_s = pk.add(pl.slices.data(), pl.slices.size());
    const Slot<WhereGeo> s_g = pk.add(pl.geo.data(), pl.geo.size());
    const Slot<WhereOp> s_o = pk.add(pl.ops.data(), pl.ops.size());
    const Slot<WhereProg> s_p = pk.add(pl.progs.data(), pl.progs.size());
    const Slot<const unsigned long long *> s_l = pk.add(leaf_ptr.data(), leaf_ptr.size());
    OCTRY(c->w_blob.ensure(pk.total + 256));   // device addresses of the vertices are known from here on
    const double *dv = s_v.at(c->w_blob);
    for (WhereSlice &s : pl.slices) s.bits = slot_bits((uint32_t)uintptr_t(s.bits));
    for (WhereGeo &L : pl.geo) {
        L.bits = slot_bits((uint32_t)uintptr_t(L.bits));
        if (L.nv) { L.vlon = dv + uintptr_t(L.vlon); L.vlat = L.vlon + L.nv; }
    }
    OCTRY(upload(pk, c->h_where, c->w_blob, c->stream));
    const uint32_t n_ws_leaves = std::min(pl.n_leaf_slots, n_ws);
    if (n_ws_leaves) CU(cudaMemsetAsync(ws, 0, size_t(n_ws_leaves) * words * 8, c->stream));
    if (res_slot < pl.n_leaf_slots) CU(cudaMemsetAsync(res_bits, 0, words * 8, c->stream));
    if (pl.total) {
        where_scatter_kernel<<<(unsigned)std::min<uint64_t>((pl.total + 255) / 256, uint64_t(c->prop.multiProcessorCount) * 16), 256, 0,
                               c->stream>>>(s_s.at(c->w_blob), (uint32_t)pl.slices.size(), pl.total, pl.nbits);
        launched(c);
        CU(cudaGetLastError());
    }
    if (!pl.geo.empty()) {
        uint64_t most = 0;
        for (const WhereGeo &L : pl.geo) most = std::max(most, L.g.n);
        // blocks per leaf; the flat grid stays below 2^31 blocks however many leaves there are (a grid-stride loop covers
        // the points)
        const uint64_t n_geo = pl.geo.size();
        const uint32_t gx = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>({(most + GEO_THREADS - 1) / GEO_THREADS,
                                                                                  uint64_t(c->prop.multiProcessorCount) * 8,
                                                                                  uint64_t(INT32_MAX) / n_geo}));
        where_geo_kernel<<<(unsigned)(gx * n_geo), GEO_THREADS, 0, c->stream>>>(s_g.at(c->w_blob), gx);
        launched(c);
        CU(cudaGetLastError());
    }
    if (!pl.progs.empty()) {
        where_eval_kernel<<<dim3((unsigned)((words + 255) / 256), (unsigned)pl.progs.size()), 256, 0, c->stream>>>(
            s_o.at(c->w_blob), s_p.at(c->w_blob), s_l.at(c->w_blob), words, pl.nbits);
        launched(c);
        CU(cudaGetLastError());
    }
    return OC_OK;
}

// The where programs of a search: planned and evaluated on the call's stream, then handed to the q_filters machinery as
// one handle per distinct result bitmap (a FILTER leaf is its own handle).
static int where_stage(SearchCall &k) {
    oc_ctx *c = k.c;
    if (k.B > 65535) return fail(OC_ERR_UNSUPPORTED, "q_where: n_queries %u > 65535", k.B);
    WherePlan pl;
    OCTRY(where_plan(k.p->q_where, 0, k.B, c, &pl));
    std::vector<const uint64_t *> bits;
    OCTRY(where_run(c, pl, bits));
    k.w_handles.resize(bits.size());
    k.w_qf.assign(k.B, nullptr);
    for (uint32_t b = 0; b < k.B; b++) {
        const uint32_t r = pl.q_res[b];
        if (r == UINT32_MAX) continue;
        if (r < pl.leaf_h.size() && pl.leaf_h[r]) { k.w_qf[b] = pl.leaf_h[r]; continue; }
        oc_filter &h = k.w_handles[r];
        h.ctx = c; h.nbits = pl.nbits; h.words = pl.words; h.bits = const_cast<uint64_t *>(bits[r]);
        k.w_qf[b] = &h;
    }
    return qfilter_slots(k, k.w_qf.data());
}

extern "C" int oc_where_check(const oc_where *w, uint32_t n_queries) {
    if (!w || !w->q_node_offsets) return fail(OC_ERR_INVALID, "NULL argument");
    // the stores' fields are read under their ctx lock: the ctx of the program's first store or handle
    const oc_ctx *c = nullptr;
    for (uint32_t i = w->q_node_offsets[0]; w->nodes && i < w->q_node_offsets[n_queries] && !c; i++) {
        const oc_where_node &nd = w->nodes[i];
        if (!nd.src) continue;
        if (nd.op == OC_WHERE_VARIANT || nd.op == OC_WHERE_RANGE) c = static_cast<const oc_facets *>(nd.src)->ctx;
        else if (nd.op == OC_WHERE_GEO_RADIUS || nd.op == OC_WHERE_GEO_POLYGON) c = static_cast<const oc_geo_field *>(nd.src)->ctx;
        else if (nd.op == OC_WHERE_FILTER) c = static_cast<const oc_filter *>(nd.src)->ctx;
    }
    if (!c) return where_plan(w, 0, n_queries, nullptr, nullptr);
    std::lock_guard<std::mutex> g(const_cast<oc_ctx *>(c)->mu);
    return where_plan(w, 0, n_queries, c, nullptr);
}

// Query `query`'s program of w as a new handle, written in place (a lone FILTER node: copied), with one synchronise.
// Called with c's lock held.
static int filter_from_program(oc_ctx *c, const oc_where *w, uint32_t query, oc_filter **out) {
    CU(cudaSetDevice(c->device));
    WherePlan pl;
    OCTRY(where_plan(w, query, 1, c, &pl));
    const uint32_t r = pl.q_res[0];
    const oc_filter *h = r < pl.leaf_h.size() ? pl.leaf_h[r] : nullptr;
    oc_filter *f = nullptr;
    OCTRY(filter_alloc(c, h ? h->nbits : pl.nbits, &f));
    std::vector<const uint64_t *> bits;
    int rc = where_run(c, pl, bits, r, f->bits);
    cudaError_t e = cudaSuccess;
    if (rc == OC_OK && h && f->words) e = cudaMemcpyAsync(f->bits, h->bits, f->words * 8, cudaMemcpyDeviceToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (rc == OC_OK && e != cudaSuccess) rc = fail(OC_ERR_CUDA, "where filter: %s", cudaGetErrorString(e));
    if (rc != OC_OK) {
        cudaFree(f->bits);
        delete f;
        return rc;
    }
    *out = f;
    return OC_OK;
}

extern "C" int oc_filter_from_where(oc_ctx *c, const oc_where *w, uint32_t query, oc_filter **out) {
    if (!c || !w || !w->q_node_offsets || !out) return fail(OC_ERR_INVALID, "NULL argument");
    if (w->q_node_offsets[query + 1] <= w->q_node_offsets[query]) return fail(OC_ERR_INVALID, "q_where[%u]: no program", query);
    std::lock_guard<std::mutex> g(c->mu);
    return filter_from_program(c, w, query, out);
}

// The leaf and combinator calls: each is the one program nodes[0, n) over [0, *nbits).  *nbits is read under the ctx
// lock, as a commit of the store publishes a new one under it.
static int filter_from_nodes(oc_ctx *c, const uint64_t *nbits, const oc_where_node *nodes, uint32_t n, oc_filter **out,
                             const double *vertex_lat = nullptr, const double *vertex_lon = nullptr) {
    std::lock_guard<std::mutex> g(c->mu);
    const uint32_t offsets[2] = {0, n};
    const oc_where w{*nbits, offsets, nodes, vertex_lat, vertex_lon};
    return filter_from_program(c, &w, 0, out);
}
// Nodes below are {op, field, arg, first_vertex, n_vertices, a, b, c, src} (oc_where_node).
extern "C" int oc_filter_facet_variant(const oc_facets *f, uint32_t field, uint32_t variant, oc_filter **out) {
    if (!f || !out) return fail(OC_ERR_INVALID, "NULL argument");
    const oc_where_node nd{OC_WHERE_VARIANT, field, variant, 0, 0, 0, 0, 0, f};
    return filter_from_nodes(f->ctx, &f->nbits, &nd, 1, out);
}
extern "C" int oc_filter_facet_range(const oc_facets *f, uint32_t field, double lo, double hi, uint32_t flags, oc_filter **out) {
    if (!f || !out) return fail(OC_ERR_INVALID, "NULL argument");
    const oc_where_node nd{OC_WHERE_RANGE, field, flags, 0, 0, lo, hi, 0, f};
    return filter_from_nodes(f->ctx, &f->nbits, &nd, 1, out);
}
extern "C" int oc_filter_geo_radius(const oc_geo_field *g, double lat, double lon, double radius_m, int inside, oc_filter **out) {
    if (!g || !out) return fail(OC_ERR_INVALID, "NULL argument");
    const oc_where_node nd{OC_WHERE_GEO_RADIUS, 0, uint32_t(inside != 0), 0, 0, lat, lon, radius_m, g};
    return filter_from_nodes(g->ctx, &g->nbits, &nd, 1, out);
}
extern "C" int oc_filter_geo_polygon(const oc_geo_field *g, const double *lat, const double *lon, uint32_t n_vertices,
                                     int inside, oc_filter **out) {
    if (!g || !out || (n_vertices && (!lat || !lon))) return fail(OC_ERR_INVALID, "NULL argument");
    const oc_where_node nd{OC_WHERE_GEO_POLYGON, 0, uint32_t(inside != 0), 0, n_vertices, 0, 0, 0, g};
    return filter_from_nodes(g->ctx, &g->nbits, &nd, 1, out, lat, lon);
}
// where_plan refuses a handle of another ctx, or of another nbits than a's
static int filter_binary(const oc_filter *a, const oc_filter *b, uint32_t op, oc_filter **out) {
    if (!a || !b || !out) return fail(OC_ERR_INVALID, "NULL argument");
    const oc_where_node nd[3] = {{OC_WHERE_FILTER, 0, 0, 0, 0, 0, 0, 0, a}, {OC_WHERE_FILTER, 0, 0, 0, 0, 0, 0, 0, b}, {op, 0, 2}};
    return filter_from_nodes(a->ctx, &a->nbits, nd, 3, out);
}
extern "C" int oc_filter_and(const oc_filter *a, const oc_filter *b, oc_filter **out) { return filter_binary(a, b, OC_WHERE_AND, out); }
extern "C" int oc_filter_or(const oc_filter *a, const oc_filter *b, oc_filter **out) { return filter_binary(a, b, OC_WHERE_OR, out); }
extern "C" int oc_filter_not(const oc_filter *a, oc_filter **out) {
    if (!a || !out) return fail(OC_ERR_INVALID, "NULL argument");
    const oc_where_node nd[2] = {{OC_WHERE_FILTER, 0, 0, 0, 0, 0, 0, 0, a}, {OC_WHERE_NOT}};
    return filter_from_nodes(a->ctx, &a->nbits, nd, 2, out);
}

// ------------------------------------------------------------------------------------ micro-batching front
struct OcExec {
    oc_ctx *c; oc_emb *e; oc_str *s;
    int operator()(const ocb::Call &k) const {
        switch (k.kind) {
        case ocb::PLAIN: return oc_search(c, e, s, k.p, k.docs, k.scores, k.n, k.count);
        case ocb::SORTED:
            return oc_search_q_sorted(c, e, s, k.p, k.q_sorts, k.pins, k.docs, k.scores, k.sort_values, k.n, k.count, k.pin_scores,
                                      k.pin_present);
        case ocb::GROUPED:
            return oc_search_q_groups(c, e, s, k.p, k.q_groups, k.pins, k.group_stride, k.docs, k.scores, k.sort_values, k.n, k.count,
                                      k.pin_scores, k.pin_present, k.g_docs, k.g_scores, k.g_values, k.g_n);
        case ocb::FACETED:
            return oc_search_q_facets(c, e, s, k.p, k.q_groups, k.pins, k.group_stride, k.facets, k.q_facet_offsets, k.facet_reqs,
                                      k.docs, k.scores, k.sort_values, k.n, k.count, k.pin_scores, k.pin_present, k.g_docs,
                                      k.g_scores, k.g_values, k.g_n, k.f_counts);
        }
        return fail(OC_ERR_INVALID, "unknown call kind %d", (int)k.kind);
    }
    int check(const oc_facets *f, const oc_facet_req *reqs, uint32_t n) const { return oc_facets_check(f, reqs, n); }
};
struct oc_batcher {
    ocb::Batcher<OcExec> q;
    oc_ctx *ctx;
    oc_batcher(OcExec x, uint32_t dim, uint32_t mb, uint32_t mw, bool mixed)
        : q(x, dim, mb, mw, x.e != nullptr, x.s != nullptr, mixed), ctx(x.c) {}
};
extern "C" int oc_batcher_create2(oc_ctx *c, oc_emb *emb, oc_str *str, uint32_t max_batch, uint32_t max_wait_us, uint32_t flags,
                                  oc_batcher **out) {
    if (!c || !out || (!emb && !str)) return fail(OC_ERR_INVALID, "bad arguments");
    if ((emb && emb->ctx != c) || (str && str->ctx != c)) return fail(OC_ERR_INVALID, "store belongs to another ctx");
    if (max_batch == 0 || max_batch > 4096) return fail(OC_ERR_INVALID, "max_batch %u outside 1..4096", max_batch);
    if (flags & ~uint32_t(OC_BATCHER_MIXED)) return fail(OC_ERR_INVALID, "unknown batcher flags 0x%x", flags);
    *out = new oc_batcher(OcExec{c, emb, str}, emb ? emb->dim : 0, max_batch, max_wait_us, (flags & OC_BATCHER_MIXED) != 0);
    return OC_OK;
}
extern "C" int oc_batcher_create(oc_ctx *c, oc_emb *emb, oc_str *str, uint32_t max_batch, uint32_t max_wait_us, oc_batcher **out) {
    return oc_batcher_create2(c, emb, str, max_batch, max_wait_us, 0, out);
}
extern "C" void oc_batcher_destroy(oc_batcher *b) { delete b; }
// The rest of every oc_batcher_search* call once its NULL arguments are checked.  What would fail a whole batch is
// refused here, before the request joins one: a handle of another ctx (a device filter joins as that query's q_filters
// entry), a where program the library would refuse (where_plan's checks against the batcher's ctx, so also a store or
// handle of another ctx), a NULL group output, and what submit refuses.
static int batcher_submit(oc_batcher *b, ocb::Request &r, const char *name) {
    const ocb::Call &k = r.call;
    if (k.p->n_queries != 1) return fail(OC_ERR_INVALID, "%s takes one query per call (n_queries = %u)", name, k.p->n_queries);
    const oc_sort *sort = ocb::sort_of(k);
    if (k.facets && k.facets->ctx != b->ctx) return fail(OC_ERR_INVALID, "facets belong to another ctx");
    if (k.p->filter && k.p->filter->ctx != b->ctx) return fail(OC_ERR_INVALID, "filter belongs to another ctx");
    if (k.p->q_where) {   // a program with a store or handle of another ctx (or any other refusal) fails here, alone
        std::lock_guard<std::mutex> g(b->ctx->mu);
        OCTRY(where_plan(k.p->q_where, 0, 1, b->ctx, nullptr));
    }
    if (sort && sort->field && sort->field->ctx != b->ctx) return fail(OC_ERR_INVALID, "sort field belongs to another ctx");
    if (k.q_groups) {
        if (k.q_groups->groups && k.q_groups->groups->ctx != b->ctx) return fail(OC_ERR_INVALID, "group_by belongs to another ctx");
        r.n_groups = oc_group_by_n_groups(k.q_groups->groups);
        if (r.n_groups && (!k.g_n || (k.group_stride && (!k.g_docs || !k.g_scores)))) return fail(OC_ERR_INVALID, "NULL group output");
    }
    g_err[0] = 0;
    const char *why = nullptr;
    const int rc = b->q.submit(r, &why);
    if (rc != OC_OK && why) return fail(rc, "%s", why);
    // the batch ran on its leader's thread: that is where oc_last_error() holds the detail
    if (rc != OC_OK && g_err[0] == 0) return fail(rc, "the coalesced search of this query's batch failed (detail on the leading caller's thread)");
    return rc;
}
extern "C" int oc_batcher_search(oc_batcher *b, const oc_search_params *p, uint64_t *out_doc_ids, float *out_scores,
                                 uint32_t *out_n, uint64_t *out_count) {
    if (!b || !p || !out_doc_ids || !out_scores || !out_n || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    ocb::Request r{{ocb::PLAIN, p, out_doc_ids, out_scores, out_n, out_count}};
    return batcher_submit(b, r, "oc_batcher_search");
}
extern "C" int oc_batcher_search_sorted(oc_batcher *b, const oc_search_params *p, const oc_sort *sort, const oc_pins *pins,
                                        uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                                        uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present) {
    if (!b || !p || !out_doc_ids || !out_scores || !out_n || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    ocb::Request r{{ocb::SORTED, p, out_doc_ids, out_scores, out_n, out_count, out_sort_values, out_pin_scores, out_pin_present, pins,
                    sort ? sort : ocb::score_order()}};
    return batcher_submit(b, r, "oc_batcher_search_sorted");
}
extern "C" int oc_batcher_search_groups(oc_batcher *b, const oc_search_params *p, const oc_group_req *req, const oc_pins *pins,
                                        uint32_t group_stride, uint64_t *out_doc_ids, float *out_scores, double *out_sort_values,
                                        uint32_t *out_n, uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present,
                                        uint64_t *out_group_doc_ids, float *out_group_scores, double *out_group_sort_values,
                                        uint32_t *out_group_n) {
    if (!b || !p || !req || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (p->limit && (!out_doc_ids || !out_scores || !out_n)) return fail(OC_ERR_INVALID, "NULL argument");
    ocb::Request r{{ocb::GROUPED, p, out_doc_ids, out_scores, out_n, out_count, out_sort_values, out_pin_scores, out_pin_present, pins,
                    nullptr, req, group_stride, out_group_doc_ids, out_group_scores, out_group_sort_values, out_group_n}};
    return batcher_submit(b, r, "oc_batcher_search_groups");
}
extern "C" int oc_batcher_search_faceted(oc_batcher *b, const oc_search_params *p, oc_facets *facets, const oc_facet_req *facet_reqs,
                                         uint32_t n_facet_reqs, const oc_group_req *req, const oc_pins *pins, uint32_t group_stride,
                                         uint64_t *out_doc_ids, float *out_scores, double *out_sort_values, uint32_t *out_n,
                                         uint64_t *out_count, float *out_pin_scores, uint8_t *out_pin_present,
                                         uint64_t *out_group_doc_ids, float *out_group_scores, double *out_group_sort_values,
                                         uint32_t *out_group_n, uint64_t *out_facet_counts) {
    if (!b || !p || !facets || !out_count) return fail(OC_ERR_INVALID, "NULL argument");
    if (p->limit && (!out_doc_ids || !out_scores || !out_n)) return fail(OC_ERR_INVALID, "NULL argument");
    if (n_facet_reqs && (!facet_reqs || !out_facet_counts)) return fail(OC_ERR_INVALID, "NULL facet requests / counts");
    ocb::Request r{{ocb::FACETED, p, out_doc_ids, out_scores, out_n, out_count, out_sort_values, out_pin_scores, out_pin_present, pins,
                    nullptr, req ? req : ocb::no_groups(), group_stride, out_group_doc_ids, out_group_scores, out_group_sort_values,
                    out_group_n, facets, nullptr, facet_reqs, out_facet_counts}, 0, {0, n_facet_reqs}};
    r.call.q_facet_offsets = r.f_off;
    return batcher_submit(b, r, "oc_batcher_search_faceted");
}
extern "C" int oc_batcher_stats(oc_batcher *b, uint64_t *n_queries, uint64_t *n_batches, uint64_t *n_direct) {
    if (!b) return fail(OC_ERR_INVALID, "NULL argument");
    b->q.stats(n_queries, n_batches, n_direct);
    return OC_OK;
}

// ------------------------------------------------------------------------------------ term dictionary / query resolution
// The step the reference performs before the posting walk — tokenize_and_stem (token_score.rs:196-209) and the FST term
// expansion inside StringStorage (string_field.rs:208-225).  On the host, except the tolerance >= 1 expansions of
// oc_dict_resolve_q with a ctx, which run on the device (dict_dev.cuh).
static std::atomic<uint64_t> g_dict_serial{0};
struct oc_dict {
    ocd::Dict d;
    std::shared_ptr<const uint64_t> token;   // the dictionary's serial; the ctx mirrors of it watch this (dict_dev.cuh)
    explicit oc_dict(uint32_t n) : d(n), token(std::make_shared<const uint64_t>(++g_dict_serial)) {}
};
struct oc_resolved { ocd::Resolved r; };

static void dict_mirror_sweep(oc_ctx *c) {
    for (auto it = c->dict_mirrors.begin(); it != c->dict_mirrors.end();)
        it = it->second->owner.expired() ? c->dict_mirrors.erase(it) : std::next(it);
}

// ocd::FuzzyRun on ctx c: refresh d's mirror, count, scan, emit.  One synchronise for the output size, one for the
// output.  Runs under the ctx lock on the ctx stream.
static int dict_fuzzy_device(oc_ctx *c, const oc_dict *d, const std::vector<ocd::FieldDict> &fields, uint64_t gen,
                             const std::vector<ocd::FuzzyPair> &pairs, ocd::FuzzyLists *out) {
    using namespace ocdd;
    std::lock_guard<std::mutex> g(c->mu);
    CU(cudaSetDevice(c->device));
    dict_mirror_sweep(c);
    std::unique_ptr<DictMirror> &mp = c->dict_mirrors[*d->token];
    if (!mp) { mp.reset(new DictMirror(fields.size())); mp->owner = d->token; }
    const cudaError_t se = mp->sync(fields, gen, c->stream);
    if (se != cudaSuccess) {   // a half-refreshed mirror is dropped; the next call builds it again
        c->dict_mirrors.erase(*d->token);
        cudaGetLastError();
        return fail(se == cudaErrorMemoryAllocation ? OC_ERR_OOM : OC_ERR_CUDA, "dictionary mirror upload: %s", cudaGetErrorString(se));
    }
    const DictMirror &M = *mp;
    const uint32_t nf = (uint32_t)fields.size(), np = (uint32_t)pairs.size();
    std::vector<uint32_t> order(np);   // device pair k = pairs[order[k]]: ordered by field
    for (uint32_t i = 0; i < np; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return pairs[a].field < pairs[b].field; });
    std::vector<FzPair> fp(np);
    uint32_t staged = 8;
    for (uint32_t k = 0; k < np; k++) {
        const ocd::FuzzyPair &q = pairs[order[k]];
        FzPair &P = fp[k];
        memset(&P, 0, sizeof(P));
        P.m = (uint32_t)q.tok->size(); P.t = q.t; P.field = q.field;
        memcpy(P.tok, q.tok->data(), P.m);
        staged = std::max(staged, P.m + P.t);
    }
    const uint32_t stride = ((staged + 7) & ~7u) + 4;   // an odd number of words: the threads of a warp hit distinct banks
    std::vector<FzField> ff(nf);
    uint32_t chunks = 0;
    uint64_t slots = 0;
    for (uint32_t fi = 0, k = 0; fi < nf; fi++) {
        FzField &F = ff[fi];
        const DictMirror::Field &m = M.f[fi];
        F.bytes = m.bytes.as<uint8_t>(); F.off = m.off.as<uint64_t>(); F.sorted = m.sorted.as<uint32_t>();
        F.n = (uint32_t)m.n_sorted;
        F.p0 = k;
        while (k < np && fp[k].field == fi) k++;
        F.p1 = k;
        F.chunk0 = chunks;
        F.n_chunks = F.p1 > F.p0 ? (F.n + FZ_CHUNK - 1) / FZ_CHUNK : 0;
        chunks += F.n_chunks;
        for (uint32_t j = F.p0; j < F.p1; j++) { fp[j].slot = (uint32_t)slots; slots += F.n_chunks + 1; }
    }
    if (slots + np > 0xffffffffu) return fail(OC_ERR_UNSUPPORTED, "%u fuzzy pairs over %u chunks", np, chunks);
    const size_t off_p = (nf * sizeof(FzField) + 255) & ~size_t(255), off_o = off_p + ((np * sizeof(FzPair) + 255) & ~size_t(255));
    OCTRY(c->fz_in.ensure(off_o + size_t(np) * 4));
    OCTRY(c->fz_cnt.ensure((slots + np) * 4));
    std::vector<uint8_t> blob(off_o);
    memcpy(blob.data(), ff.data(), nf * sizeof(FzField));
    memcpy(blob.data() + off_p, fp.data(), np * sizeof(FzPair));
    CU(cudaMemcpyAsync(c->fz_in.p, blob.data(), off_o, cudaMemcpyHostToDevice, c->stream));
    const FzField *dF = c->fz_in.as<const FzField>();
    const FzPair *dP = reinterpret_cast<const FzPair *>(c->fz_in.as<uint8_t>() + off_p);
    uint32_t *dO = reinterpret_cast<uint32_t *>(c->fz_in.as<uint8_t>() + off_o);
    uint32_t *cnt = c->fz_cnt.as<uint32_t>(), *tot = cnt + slots;
    const size_t smem = fuzzy_smem(stride);
    // about four CTAs per SM, without slicing a field's pairs finer than a count-pass group
    uint32_t max_pairs = 0;
    for (const FzField &F : ff) max_pairs = std::max(max_pairs, F.p1 - F.p0);
    const uint32_t want = 4u * (uint32_t)c->prop.multiProcessorCount;
    const uint32_t split = chunks ? std::max(1u, std::min((want + chunks - 1) / chunks, (max_pairs + FZ_GROUP - 1) / FZ_GROUP)) : 1;
    if (chunks) {
        CU(smem_cfg(c->device, (const void *)dict_fuzzy_kernel<false>, smem));
        CU(smem_cfg(c->device, (const void *)dict_fuzzy_kernel<true>, smem));
        dict_fuzzy_kernel<false><<<chunks * split, FZ_THREADS, smem, c->stream>>>(dF, nf, dP, stride, split, cnt, nullptr, nullptr, nullptr);
        CU(cudaGetLastError());
        launched(c);
    }
    dict_fuzzy_scan_kernel<<<np, FZ_THREADS, 0, c->stream>>>(dF, dP, cnt, tot);
    CU(cudaGetLastError());
    launched(c);
    std::vector<uint32_t> total(np), out0(np);
    CU(cudaMemcpyAsync(total.data(), tot, size_t(np) * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    uint64_t T = 0;
    for (uint32_t k = 0; k < np; k++) { out0[k] = (uint32_t)T; T += total[k]; }
    if (T > 0xffffffffu) return fail(OC_ERR_UNSUPPORTED, "%llu expanded terms", (unsigned long long)T);
    std::vector<uint32_t> ids(T);
    std::vector<uint8_t> ex(T);
    if (T) {
        OCTRY(c->fz_out.ensure(T * 5));
        uint32_t *d_id = c->fz_out.as<uint32_t>();
        uint8_t *d_ex = reinterpret_cast<uint8_t *>(d_id + T);
        CU(cudaMemcpyAsync(dO, out0.data(), size_t(np) * 4, cudaMemcpyHostToDevice, c->stream));
        dict_fuzzy_kernel<true><<<chunks * split, FZ_THREADS, smem, c->stream>>>(dF, nf, dP, stride, split, cnt, dO, d_id, d_ex);
        CU(cudaGetLastError());
        launched(c);
        CU(cudaMemcpyAsync(ids.data(), d_id, T * 4, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaMemcpyAsync(ex.data(), d_ex, T, cudaMemcpyDeviceToHost, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    std::vector<uint32_t> at(np);
    for (uint32_t k = 0; k < np; k++) at[order[k]] = k;
    out->off.assign(1, 0u);
    out->id.clear(); out->exact.clear();
    out->id.reserve(T); out->exact.reserve(T);
    for (uint32_t i = 0; i < np; i++) {
        const uint32_t k = at[i];
        out->id.insert(out->id.end(), ids.begin() + out0[k], ids.begin() + out0[k] + total[k]);
        out->exact.insert(out->exact.end(), ex.begin() + out0[k], ex.begin() + out0[k] + total[k]);
        out->off.push_back((uint32_t)out->id.size());
    }
    return OC_OK;
}

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
extern "C" int oc_dict_resolve_q(oc_dict *d, oc_ctx *ctx, const oc_resolve_params *p, const oc_resolve_query *q,
                                 oc_resolved **out) {
    if (!d || !p || !out || (p->n_queries && !p->texts)) return fail(OC_ERR_INVALID, "bad arguments");
    for (uint32_t i = 0; i < p->n_queries; i++) if (!p->texts[i]) return fail(OC_ERR_INVALID, "text %u is NULL", i);
    if (!q && p->tolerance > 8) return fail(OC_ERR_UNSUPPORTED, "tolerance %d > 8", p->tolerance);
    if (q) for (uint32_t i = 0; i < p->n_queries; i++)
        if (q[i].tolerance > 8) return fail(OC_ERR_UNSUPPORTED, "query %u: tolerance %d > 8", i, q[i].tolerance);
    std::vector<ocd::ResolveOpts> opts(p->n_queries);
    for (uint32_t i = 0; i < p->n_queries; i++) {
        ocd::ResolveOpts &o = opts[i];
        if (q) { o.exact = q[i].exact != 0; o.tolerance = q[i].tolerance; o.field_boost = q[i].field_boost; o.field_mask = q[i].field_mask; }
        else { o.exact = p->exact != 0; o.tolerance = p->tolerance; o.field_boost = p->field_boost; o.field_mask = p->field_mask; }
        o.exact_match_boost = p->exact_match_boost > 0.f ? p->exact_match_boost : 2.0f;
    }
    const ocd::FuzzyRun run = [&](const std::vector<ocd::FieldDict> &fields, uint64_t gen, const std::vector<ocd::FuzzyPair> &pairs,
                                  ocd::FuzzyLists *lists) { return dict_fuzzy_device(ctx, d, fields, gen, pairs, lists); };
    std::unique_ptr<oc_resolved> r(new oc_resolved());
    OCTRY(d->d.resolve_q(p->texts, p->n_queries, opts, ctx ? &run : nullptr, &r->r));
    *out = r.release();
    return OC_OK;
}
extern "C" uint64_t oc_dict_device_bytes(oc_dict *d, oc_ctx *ctx) {
    if (!d || !ctx) return 0;
    std::lock_guard<std::mutex> g(ctx->mu);
    auto it = ctx->dict_mirrors.find(*d->token);
    return it == ctx->dict_mirrors.end() ? 0 : it->second->device_bytes();
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
