// shard.cuh — K5: document-sharded search across the GPUs of one box (SURVEY.md §8e).
//
// The reference is single-node (readers are full replicas fed by an op-log,
// sides/operation/); there is no reference analogue of this exchange.  Each rank holds a
// contiguous doc-row range of the embedding matrix AND the postings of those rows, with
// GLOBAL N / avg_field_len / per-term df replicated at load time, so BM25 needs no
// per-query collective.  Per query batch there is exactly ONE collective: an NCCL
// all-gather (NVLink/NVSwitch) of a fixed-size record per (rank, query):
//     header  : local match count, local pre-OMC max/min of the fulltext scores, row counts
//     ft list : the rank's best n_keep fulltext candidates by rank proxy (doc, raw score, row)
//     v list  : the rank's <= limit vector hits (doc, -distance, rescaled score, and the
//               LOCAL fulltext score of that doc — both live on the same shard)
// after which every rank runs the same merge kernel: global vector top-`limit` by distance,
// global max/min, fused scores (token_score.rs:393-422), OMC (search.rs:39-48), global
// top-n, count = sum(local counts) + |V \ FT| — bit-identical to the single-GPU kernel.
// Payload at B=256, limit=10: 256 * (40 + 10*16 + 10*32) B = 133 KB per rank: latency-bound.
#pragma once

namespace oc {

struct ShardHdr {          // 40 B
    unsigned long long count_ft;
    float max_ft, min_ft;
    uint32_t n_ft, n_v;
    uint32_t n_rows_str, n_rows_emb;
    uint32_t unproven, pad;   // this rank's tensor-core scan overflowed for the query: every rank re-runs the batch tail
};
struct ShardFt {           // 16 B
    uint64_t doc;
    float ft;
    uint32_t row;
};
struct ShardV {            // 32 B
    uint64_t doc;
    float rawkey, score, ft;
    uint32_t present, srow, erow;
};
__host__ __device__ inline size_t shard_rec_bytes(uint32_t n_keep, uint32_t vlimit) {
    return sizeof(ShardHdr) + size_t(n_keep) * sizeof(ShardFt) + size_t(vlimit) * sizeof(ShardV);
}

struct ShardPackParams {
    FuseParams f;              // local stage products (same fields the single-GPU fuse reads)
    const float *v_raw;        // [q][v_stride] -distance of each local vector hit
    const uint32_t *v_erow;    // [q][v_stride] embedding row of each hit
    uint32_t n_rows_str, n_rows_emb;
    const uint8_t *unproven;   // [q] local overflow flags of the tensor-core scan, or NULL
    uint8_t *out;              // [q] records
    // direct NVLink exchange (oc_comm_p2p_*): after packing, the CTA stores its query's record into the receive
    // window of EVERY rank (peer memory mapped through CUDA IPC) and bumps that rank's arrival counter of the query
    uint32_t p2p_world;        // 0 = off (the records travel by ncclAllGather)
    uint32_t p2p_rank;
    uint8_t *p2p_win[16];      // base of each rank's window for this batch's parity
    uint32_t *p2p_flag[16];    // [q] arrival counters of each rank for this parity
    uint64_t p2p_rank_stride;  // bytes between the slots of two source ranks inside a window
};

__global__ void __launch_bounds__(256) shard_pack_kernel(const ShardPackParams pp) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *buf = reinterpret_cast<uint64_t *>(smem);
    const FuseParams &p = pp.f;
    const uint32_t q = blockIdx.x, tid = threadIdx.x;
    const bool has_ft = p.mode != OC_MODE_VECTOR, has_v = p.mode != OC_MODE_FULLTEXT;
    const size_t rb = shard_rec_bytes(p.n_keep, p.v_stride);
    ShardHdr *hdr = reinterpret_cast<ShardHdr *>(pp.out + size_t(q) * rb);
    ShardFt *fts = reinterpret_cast<ShardFt *>(hdr + 1);
    ShardV *vs = reinterpret_cast<ShardV *>(fts + p.n_keep);
    __shared__ unsigned int s_maxo, s_mino;
    __shared__ unsigned long long s_count;
    if (tid == 0) { s_maxo = f32_ordered(0.f); s_mino = f32_ordered(0.f); s_count = 0; }
    __syncthreads();
    unsigned long long cnt = 0;
    float lmax = 0.f, lmin = 0.f;
    if (has_ft)
        for (uint32_t t = tid; t < p.n_tiles; t += blockDim.x) {
            const size_t s = size_t(q) * p.n_tiles + t;
            cnt += p.tile_count[s];
            lmax = fmaxf(lmax, p.tile_max[s]);
            lmin = fminf(lmin, p.tile_min[s]);
        }
    for (int o = 16; o > 0; o >>= 1) {
        lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((tid & 31) == 0) {
        atomicMax(&s_maxo, f32_ordered(lmax));
        atomicMin(&s_mino, f32_ordered(lmin));
        if (cnt) atomicAdd(&s_count, cnt);
    }
    __syncthreads();
    // local best n_keep fulltext candidates by the tile rank proxy
    uint32_t got = 0;
    if (has_ft) {
        const uint64_t total = uint64_t(p.n_tiles) * p.n_keep;
        // compact the (mostly empty) per-tile candidate lists, sort only the valid keys
        __shared__ uint32_t s_nvalid;
        uint32_t mine = 0;
        for (uint32_t t = tid; t < p.n_tiles; t += blockDim.x) mine += min(p.cand_cnt[size_t(q) * p.n_tiles + t], p.n_keep);
        uint32_t n_valid;
        const uint32_t my_pos = block_exclusive_scan(mine, &n_valid);
        if (tid == 0) s_nvalid = n_valid;
        __syncthreads();
        if (s_nvalid <= p.capb) {
            uint32_t pos = my_pos;
            for (uint32_t t = tid; t < p.n_tiles; t += blockDim.x) {
                const size_t s2 = size_t(q) * p.n_tiles + t;
                const uint32_t c = min(p.cand_cnt[s2], p.n_keep);
                for (uint32_t k = 0; k < c; k++) buf[pos++] = p.cand_key[s2 * p.n_keep + k];
            }
            const uint32_t nv = s_nvalid, np2 = max(32u, next_pow2(nv));
            const uint32_t kp2 = max(32u, next_pow2(p.n_keep));
            if (np2 > 2 * kp2) {   // radix-select the n_keep best, sort only those (same as fuse_topk_kernel)
                uint64_t *sel = buf + p.capb;
                for (uint32_t i = tid; i < kp2; i += blockDim.x) sel[i] = KEY_NONE;
                __syncthreads();
                block_select_largest(buf, nv, p.n_keep, sel);
                group_bitonic_desc(sel, kp2, tid, blockDim.x, 0);
                for (uint32_t i = tid; i < kp2; i += blockDim.x) buf[i] = sel[i];
                __syncthreads();
            } else {
                for (uint32_t i = nv + tid; i < np2; i += blockDim.x) buf[i] = KEY_NONE;
                group_bitonic_desc(buf, np2, tid, blockDim.x, 0);
            }
            got = min(nv, p.n_keep);
        } else {
            got = block_topn_stream(buf, p.capb, p.n_keep, total, [&](uint64_t i) -> uint64_t {
                const uint32_t t = uint32_t(i / p.n_keep), k = uint32_t(i % p.n_keep);
                const size_t s = size_t(q) * p.n_tiles + t;
                return k < p.cand_cnt[s] ? p.cand_key[s * p.n_keep + k] : KEY_NONE;
            });
        }
        for (uint32_t i = tid; i < p.n_keep; i += blockDim.x) {
            ShardFt e{0, 0.f, 0xffffffffu};
            if (i < got) {
                const uint64_t key = buf[i];
                const uint32_t row = key_idx(key);
                const size_t s = size_t(q) * p.n_tiles + row / BM25_TILE;
                float ft = 0.f;
                for (uint32_t k = 0; k < p.cand_cnt[s]; k++)
                    if (p.cand_key[s * p.n_keep + k] == key) { ft = p.cand_ft[s * p.n_keep + k]; break; }
                e.doc = p.str_row_doc_ids ? p.str_row_doc_ids[row] : uint64_t(row);
                e.ft = ft; e.row = row;
            }
            fts[i] = e;
        }
    }
    const uint32_t vc = has_v ? p.v_count[q] : 0;
    for (uint32_t j = tid; j < p.v_stride; j += blockDim.x) {
        ShardV e{0, 0.f, 0.f, 0.f, 0u, 0xffffffffu, 0xffffffffu};
        if (j < vc) {
            const size_t vsi = size_t(q) * p.v_stride + j;
            e.doc = p.v_doc[vsi]; e.rawkey = pp.v_raw[vsi]; e.score = p.v_score[vsi];
            e.erow = pp.v_erow[vsi];
            if (has_ft) { e.ft = p.v_ft[vsi]; e.present = p.v_present[vsi]; e.srow = p.v_row[vsi]; }
        }
        vs[j] = e;
    }
    if (tid == 0) {
        hdr->count_ft = s_count; hdr->max_ft = f32_unordered(s_maxo); hdr->min_ft = f32_unordered(s_mino);
        hdr->n_ft = got; hdr->n_v = vc; hdr->n_rows_str = pp.n_rows_str; hdr->n_rows_emb = pp.n_rows_emb;
        hdr->unproven = pp.unproven ? pp.unproven[q] : 0u; hdr->pad = 0u;
    }
    if (pp.p2p_world) {
        // the record is complete in local memory: push it to every rank's window over NVLink (8-byte stores,
        // coalesced), make it visible system-wide, then signal one arrival per destination
        __threadfence();
        __syncthreads();
        const uint64_t *src = reinterpret_cast<const uint64_t *>(pp.out + size_t(q) * rb);
        const uint32_t n8 = uint32_t(rb / 8);
        for (uint32_t r = 0; r < pp.p2p_world; r++) {
            uint64_t *dst = reinterpret_cast<uint64_t *>(pp.p2p_win[r] + size_t(pp.p2p_rank) * pp.p2p_rank_stride + size_t(q) * rb);
            for (uint32_t i = tid; i < n8; i += blockDim.x) dst[i] = src[i];
        }
        __threadfence_system();
        __syncthreads();
        if (tid < pp.p2p_world) atomicAdd_system(pp.p2p_flag[tid] + q, 1u);
    }
}

struct ShardFuseParams {
    const uint8_t *recv;      // [world][B] records
    uint64_t rank_stride;     // bytes between two source ranks' blocks (n_queries * record bytes after an all-gather)
    const uint32_t *p2p_flag; // NULL, or [B] arrival counters of this rank's window: wait until p2p_expected arrivals
    uint32_t p2p_expected;
    uint32_t world, n_queries;
    int mode;
    uint32_t n_keep, limit, offset, v_stride, capb;
    const uint64_t *omc_doc; const float *omc_mult; uint32_t n_omc;
    uint64_t *out_doc; float *out_score; uint32_t *out_n; unsigned long long *out_count; float *out_min;
    uint8_t *out_flag;        // [q] 1 if any rank flagged the query (identical on every rank)
};

constexpr uint32_t SHARD_MAX_WORLD = 16;

__global__ void __launch_bounds__(256) shard_fuse_kernel(const ShardFuseParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint64_t *buf = reinterpret_cast<uint64_t *>(smem);                       // [capb]
    uint64_t *gv_doc = buf + p.capb;                                           // [v_stride]
    float *gv_score = reinterpret_cast<float *>(gv_doc + p.v_stride);          // merged (vsum)
    float *gv_ft = gv_score + p.v_stride;
    uint32_t *gv_present = reinterpret_cast<uint32_t *>(gv_ft + p.v_stride);
    uint32_t *gv_idx = gv_present + p.v_stride;                                // global string-row index or fallback
    uint32_t *gv_first = gv_idx + p.v_stride;
    float *gv_raw = reinterpret_cast<float *>(gv_first + p.v_stride);          // per-hit rescaled score before merging
    __shared__ uint32_t base_str[SHARD_MAX_WORLD + 1], base_emb[SHARD_MAX_WORLD + 1];
    __shared__ unsigned int s_maxo, s_mino;
    __shared__ unsigned long long s_count;
    __shared__ uint32_t s_gvc;
    const uint32_t q = blockIdx.x, tid = threadIdx.x, W = p.world;
    const bool has_ft = p.mode != OC_MODE_VECTOR, has_v = p.mode != OC_MODE_FULLTEXT;
    const bool hybrid = has_ft && has_v;
    const size_t rb = shard_rec_bytes(p.n_keep, p.v_stride);
    auto hdr_of = [&](uint32_t s) { return reinterpret_cast<const ShardHdr *>(p.recv + size_t(s) * p.rank_stride + size_t(q) * rb); };
    auto ft_of = [&](uint32_t s) { return reinterpret_cast<const ShardFt *>(hdr_of(s) + 1); };
    auto v_of = [&](uint32_t s) { return reinterpret_cast<const ShardV *>(ft_of(s) + p.n_keep); };
    if (p.p2p_flag) {
        // direct exchange: every rank's pack kernel stored this query's record into our window and bumped the counter
        if (tid == 0) {
            unsigned int seen;
            do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(seen) : "l"(p.p2p_flag + q) : "memory"); } while (seen < p.p2p_expected);
        }
        __syncthreads();
        asm volatile("fence.acq_rel.sys;" ::: "memory");
    }
    if (tid == 0) {
        base_str[0] = 0; base_emb[0] = 0;
        for (uint32_t s = 0; s < W; s++) {
            base_str[s + 1] = base_str[s] + hdr_of(s)->n_rows_str;
            base_emb[s + 1] = base_emb[s] + hdr_of(s)->n_rows_emb;
        }
        s_maxo = f32_ordered(0.f); s_mino = f32_ordered(0.f); s_count = 0; s_gvc = 0;
    }
    __syncthreads();

    // ---- 1. global vector top-`limit` by distance (== storage.search(target, limit) over the whole corpus)
    uint32_t gvc = 0;
    if (has_v) {
        const uint64_t total = uint64_t(W) * p.v_stride;
        gvc = block_topn_stream(buf, p.capb, p.v_stride, total, [&](uint64_t i) -> uint64_t {
            const uint32_t s = uint32_t(i / p.v_stride), j = uint32_t(i % p.v_stride);
            if (j >= hdr_of(s)->n_v) return KEY_NONE;
            const ShardV &e = v_of(s)[j];
            return make_key(e.rawkey, base_emb[s] + e.erow);
        });
        for (uint32_t i = tid; i < gvc; i += blockDim.x) {
            const uint32_t gidx = key_idx(buf[i]);
            uint32_t s = 0;
            while (s + 1 < W && gidx >= base_emb[s + 1]) s++;
            const uint32_t erow = gidx - base_emb[s];
            const ShardV *vl = v_of(s);
            for (uint32_t j = 0; j < hdr_of(s)->n_v; j++)
                if (vl[j].erow == erow) {
                    gv_doc[i] = vl[j].doc; gv_raw[i] = vl[j].score; gv_ft[i] = vl[j].ft; gv_present[i] = vl[j].present;
                    gv_idx[i] = (has_ft && vl[j].srow != 0xffffffffu) ? base_str[s] + vl[j].srow : 0xffffffffu;
                    break;
                }
        }
        __syncthreads();
        // output[doc] += score for chunks of one document (embedding_field.rs:273-274)
        for (uint32_t j = tid; j < gvc; j += blockDim.x) {
            bool head = true;
            for (uint32_t i = 0; i < j; i++) if (gv_doc[i] == gv_doc[j]) { head = false; break; }
            float sum = 0.f;
            if (head) for (uint32_t i = j; i < gvc; i++) if (gv_doc[i] == gv_doc[j]) sum = __fadd_rn(sum, gv_raw[i]);
            gv_score[j] = sum; gv_first[j] = head ? 1u : 0u;
        }
        __syncthreads();
        // K4's tie rule (fuse.cuh): the key index of a unique hit is its doc id's rank among the unique hits, so equal
        // scores come out in doc id order; in hybrid mode only a hit without a string row takes it, after FUSE_VONLY
        for (uint32_t j = tid; j < gvc; j += blockDim.x)
            if (gv_first[j] && !(hybrid && gv_idx[j] != 0xffffffffu)) {
                uint32_t r = 0;
                for (uint32_t i = 0; i < gvc; i++) r += (gv_first[i] && gv_doc[i] < gv_doc[j]) ? 1u : 0u;
                gv_idx[j] = hybrid ? FUSE_VONLY + r : r;
            }
        __syncthreads();
    }

    // ---- 2. count and extrema
    unsigned long long cnt = 0;
    float lmax = 0.f, lmin = 0.f;
    if (has_ft)
        for (uint32_t s = tid; s < W; s += blockDim.x) {
            cnt += hdr_of(s)->count_ft;
            lmax = fmaxf(lmax, hdr_of(s)->max_ft);
            lmin = fminf(lmin, hdr_of(s)->min_ft);
        }
    for (uint32_t j = tid; j < gvc; j += blockDim.x)
        if (gv_first[j]) {
            lmax = fmaxf(lmax, gv_score[j]);
            lmin = fminf(lmin, gv_score[j]);
            if (!(has_ft && gv_present[j])) cnt++;
        }
    for (int o = 16; o > 0; o >>= 1) {
        lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
        lmin = fminf(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((tid & 31) == 0) {
        atomicMax(&s_maxo, f32_ordered(lmax));
        atomicMin(&s_mino, f32_ordered(lmin));
        if (cnt) atomicAdd(&s_count, cnt);
    }
    __syncthreads();
    const float gmax = f32_unordered(s_maxo), gmin = f32_unordered(s_mino);
    const float den = __fsub_rn(gmax, gmin);

    auto omc_of = [&](uint64_t doc, bool *found) -> float {
        uint32_t lo = 0, hi = p.n_omc;
        while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (p.omc_doc[m] < doc) lo = m + 1; else hi = m; }
        *found = lo < p.n_omc && p.omc_doc[lo] == doc;
        return *found ? p.omc_mult[lo] : 1.0f;
    };

    // ---- 3. candidates: every shard's fulltext list (minus global vector hits), then the vector hits
    const uint64_t n_ft_slots = has_ft ? uint64_t(W) * p.n_keep : 0;
    const uint64_t total = n_ft_slots + gvc;
    auto load = [&](uint64_t i) -> uint64_t {
        if (i < n_ft_slots) {
            const uint32_t s = uint32_t(i / p.n_keep), k = uint32_t(i % p.n_keep);
            if (k >= hdr_of(s)->n_ft) return KEY_NONE;
            const ShardFt &e = ft_of(s)[k];
            if (hybrid)
                for (uint32_t j = 0; j < gvc; j++) if (gv_doc[j] == e.doc) return KEY_NONE;
            float f = e.ft;
            if (hybrid) f = __fdiv_rn(__fsub_rn(f, gmin), den);
            if (p.n_omc) { bool fd; const float m = omc_of(e.doc, &fd); if (fd) f = __fmul_rn(f, m); }
            return f == f ? make_key(f, base_str[s] + e.row) : KEY_NONE;
        }
        const uint32_t j = uint32_t(i - n_ft_slots);
        if (!gv_first[j]) return KEY_NONE;
        float f;
        uint32_t idx;
        if (hybrid) {
            const float vn = __fdiv_rn(__fsub_rn(gv_score[j], gmin), den);
            const float fn = gv_present[j] ? __fdiv_rn(__fsub_rn(gv_ft[j], gmin), den) : 0.0f;
            f = __fadd_rn(fn, vn);
            idx = gv_idx[j];
        } else {
            f = gv_score[j];
            idx = gv_idx[j];
        }
        if (p.n_omc) { bool fd; const float m = omc_of(gv_doc[j], &fd); if (fd) f = __fmul_rn(f, m); }
        return f == f ? make_key(f, idx) : KEY_NONE;
    };
    __syncthreads();
    const uint32_t got = block_topn_stream(buf, p.capb, p.n_keep, total, load);

    // ---- 4. skip(offset).take(limit); resolve idx -> doc
    const uint32_t n_out = got > p.offset ? min(p.limit, got - p.offset) : 0;
    for (uint32_t i = tid; i < p.limit; i += blockDim.x) {
        uint64_t doc = 0; float sc = 0.f;
        if (i < n_out) {
            const uint64_t k = buf[p.offset + i];
            const uint32_t idx = key_idx(k);
            sc = key_score(k);
            bool found = false;
            if (has_v)
                for (uint32_t j = 0; j < gvc; j++) if (gv_first[j] && gv_idx[j] == idx) { doc = gv_doc[j]; found = true; break; }
            if (!found) {
                uint32_t s = 0;
                while (s + 1 < W && idx >= base_str[s + 1]) s++;
                const uint32_t row = idx - base_str[s];
                const ShardFt *fl = ft_of(s);
                for (uint32_t k2 = 0; k2 < hdr_of(s)->n_ft; k2++) if (fl[k2].row == row) { doc = fl[k2].doc; break; }
            }
        }
        p.out_doc[size_t(q) * p.limit + i] = doc;
        p.out_score[size_t(q) * p.limit + i] = sc;
    }
    if (tid == 0) {
        p.out_n[q] = n_out;
        p.out_count[q] = s_count;
        if (p.out_min) p.out_min[q] = gmin;
        uint32_t fl = 0;
        for (uint32_t s = 0; s < W; s++) fl |= hdr_of(s)->unproven;
        if (p.out_flag) p.out_flag[q] = fl ? 1 : 0;
    }
}

}  // namespace oc

static int run_sharded_merge(oc_ctx *c, const oc_search_params *p, const oc::FuseParams &fp, uint32_t n_rows_str,
                             uint32_t n_rows_emb, uint32_t B, const uint8_t *unproven_dev, uint8_t *out_flag_dev) {
    using namespace oc;
    const uint32_t W = (uint32_t)c->comm.world;
    if (W > SHARD_MAX_WORLD) return fail(OC_ERR_UNSUPPORTED, "world size %u > %u", W, SHARD_MAX_WORLD);
    const size_t rb = shard_rec_bytes(fp.n_keep, fp.v_stride);
    OCTRY(c->shard_send.ensure(rb * B));
    OCTRY(c->shard_recv.ensure(rb * B * W));
    ShardPackParams pp{};
    pp.f = fp;
    pp.v_raw = c->v_raw.as<float>();
    pp.v_erow = c->v_row.as<uint32_t>();
    pp.n_rows_str = n_rows_str; pp.n_rows_emb = n_rows_emb;
    pp.unproven = unproven_dev;
    pp.out = c->shard_send.as<uint8_t>();
    // direct NVLink exchange when the runtime imported the peers' windows and the batch fits them (every rank takes the
    // same decision: it depends on the batch shape only); OC_SHARD_P2P=0: A/B switch back to ncclAllGather
    const char *p2env = getenv("OC_SHARD_P2P");
    const bool p2p = c->p2p.ready && !(p2env && p2env[0] == '0') && rb * B <= P2P_WIN_BYTES && B <= P2P_MAX_Q;
    uint32_t par = 0;
    if (p2p) {
        par = uint32_t(c->p2p.seq & 1u);
        pp.p2p_world = W; pp.p2p_rank = (uint32_t)c->comm.rank; pp.p2p_rank_stride = P2P_WIN_BYTES;
        for (uint32_t r = 0; r < W; r++) {
            pp.p2p_win[r] = c->p2p.peer[r] + P2P_FLAG_BYTES + size_t(par) * W * P2P_WIN_BYTES;
            pp.p2p_flag[r] = reinterpret_cast<uint32_t *>(c->p2p.peer[r]) + size_t(par) * P2P_MAX_Q;
        }
    }
    const size_t pack_smem = size_t(fp.capb) * 8 + size_t(std::max<uint32_t>(32, next_pow2(fp.n_keep))) * 8 + 64;
    CU(smem_cfg(c->device, (const void *)shard_pack_kernel, pack_smem));
    shard_pack_kernel<<<B, 256, pack_smem, c->stream>>>(pp);
    launched(c);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->ev[EV_COMM0], c->stream));
    ShardFuseParams sp{};
    if (p2p) {
        sp.recv = c->p2p.peer[c->comm.rank] + P2P_FLAG_BYTES + size_t(par) * W * P2P_WIN_BYTES;
        sp.rank_stride = P2P_WIN_BYTES;
        sp.p2p_flag = reinterpret_cast<const uint32_t *>(c->p2p.peer[c->comm.rank]) + size_t(par) * P2P_MAX_Q;
        sp.p2p_expected = W * uint32_t((c->p2p.seq >> 1) + 1);
        c->p2p.seq++;
    } else {
        std::string err;
        if (!c->comm.all_gather(c->shard_send.p, c->shard_recv.p, rb * B, c->stream, &err)) return fail(OC_ERR_COMM, "%s", err.c_str());
        sp.recv = c->shard_recv.as<uint8_t>();
        sp.rank_stride = rb * B;
    }
    sp.world = W; sp.n_queries = B; sp.mode = p->mode;
    sp.n_keep = fp.n_keep; sp.limit = fp.limit; sp.offset = fp.offset; sp.v_stride = fp.v_stride;
    sp.capb = std::min<uint32_t>(2048, std::max<uint32_t>(64, next_pow2(std::max<uint32_t>(W * fp.n_keep + fp.v_stride, W * fp.v_stride))));
    sp.capb = std::max<uint32_t>(sp.capb, next_pow2(2 * std::max(fp.n_keep, fp.v_stride)));
    sp.omc_doc = fp.omc_doc; sp.omc_mult = fp.omc_mult; sp.n_omc = fp.n_omc;
    sp.out_doc = fp.out_doc; sp.out_score = fp.out_score; sp.out_n = fp.out_n; sp.out_count = fp.out_count; sp.out_min = fp.out_min;
    sp.out_flag = out_flag_dev;
    const size_t fsmem = size_t(sp.capb) * 8 + size_t(fp.v_stride) * 36 + 64;
    CU(smem_cfg(c->device, (const void *)shard_fuse_kernel, fsmem));
    shard_fuse_kernel<<<B, 256, fsmem, c->stream>>>(sp);
    launched(c);
    CU(cudaGetLastError());
    CU(cudaEventRecord(c->ev[EV_COMM1], c->stream));
    return OC_OK;
}
