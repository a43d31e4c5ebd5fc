// where.cuh — where-clause programs, the one evaluator of where filters on the device: inside a search call
// (oc_search_params.q_where), and for every handle oc_filter_from_where, the leaf calls and And / Or / Not build.
//
// The host plan (capi.cu where_plan) deduplicates the leaves and the programs of a batch and lays every bitmap out in one
// ctx workspace.  Three launches then build every result, however many leaves and queries the batch has:
//   where_scatter_kernel  the facet leaves: one work list of (document slice, leaf bitmap) items over all leaves, one
//                         thread per document id.
//   where_geo_kernel      the geo leaves, a fixed number of blocks each: the per-point tests of geo.cuh, a polygon's
//                         vertices staged in shared memory.
//   where_eval_kernel     every distinct program of more than one node, one per blockIdx.y, one 64-bit word per thread:
//                         the postfix program runs over that word of its leaves, and the padding bits of the last word
//                         are cleared in the value it writes, also over a FILTER handle with a dirty tail.  Clearing
//                         once at the end gives what clearing after every And / Or / Not would.
#pragma once
#include <cstdint>

#include "geo.cuh"
#include "oramacore_b200.h"

namespace oc {

constexpr uint32_t WHERE_PUSH = 0xffffffffu;   // a WhereOp that pushes leaf `arg`; else op is OC_WHERE_AND / OR / NOT

struct WhereOp { uint32_t op, arg; };
struct WhereProg { uint32_t first, n; unsigned long long *out; };
// facet leaves: item i covers the ids [start_i, start_{i+1}) of the concatenated slices
struct WhereSlice { const uint64_t *docs; uint64_t start; unsigned long long *bits; };
struct WhereGeo {
    GeoPoints g;
    double cx, cy, cz, thr;   // radius
    double4 bbox;             // polygon: {lon_min, lon_max, lat_min, lat_max}, widened by GEO_BBOX_MARGIN
    const double *vlon, *vlat;
    uint32_t nv;              // 0: radius
    int inside;
    unsigned long long *bits;
};

__global__ void where_scatter_kernel(const WhereSlice *items, uint32_t n_items, uint64_t total, uint64_t nbits) {
    for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += uint64_t(gridDim.x) * blockDim.x) {
        uint32_t lo = 0, hi = n_items - 1;   // the last item with start <= i
        while (lo < hi) {
            const uint32_t mid = (lo + hi + 1) / 2;
            if (items[mid].start <= i) lo = mid; else hi = mid - 1;
        }
        const WhereSlice s = items[lo];
        const uint64_t d = s.docs[i - s.start];
        if (d < nbits) geo_set(s.bits, d);   // a store may list ids >= nbits: they pass no leaf
    }
}

// gx blocks per leaf in one flat grid: leaf blockIdx.x / gx (gridDim.y would bound the leaves at 65535)
__global__ void __launch_bounds__(GEO_THREADS) where_geo_kernel(const WhereGeo *leaves, uint32_t gx) {
    __shared__ double sx[GEO_MAX_VERTICES], sy[GEO_MAX_VERTICES];
    const WhereGeo &L = leaves[blockIdx.x / gx];
    const uint32_t bx = blockIdx.x % gx;
    const GeoPoints g = L.g;
    const uint32_t nv = L.nv;
    const bool inside = L.inside != 0;
    if (nv) {
        for (uint32_t k = threadIdx.x; k < nv; k += blockDim.x) { sx[k] = L.vlon[k]; sy[k] = L.vlat[k]; }
        __syncthreads();
    }
    for (uint64_t i = uint64_t(bx) * blockDim.x + threadIdx.x; i < g.n; i += uint64_t(gx) * blockDim.x) {
        const bool in = nv ? geo_in_polygon(g.lon[i], g.lat[i], sx, sy, nv, L.bbox)
                           : geo_in_radius(g.x[i], g.y[i], g.z[i], L.cx, L.cy, L.cz, L.thr);
        if (in == inside) geo_set(L.bits, g.doc[i]);
    }
}

__global__ void where_eval_kernel(const WhereOp *ops, const WhereProg *progs, const unsigned long long *const *leaf,
                                  uint64_t words, uint64_t nbits) {
    const uint64_t w = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (w >= words) return;
    const WhereProg pg = progs[blockIdx.y];
    const uint64_t tail = (w == words - 1 && (nbits & 63)) ? (1ull << (nbits & 63)) - 1 : ~0ull;
    uint64_t st[OC_WHERE_MAX_DEPTH];
    uint32_t sp = 0;
    for (uint32_t i = 0; i < pg.n; i++) {
        const WhereOp o = ops[pg.first + i];
        if (o.op == WHERE_PUSH) {
            st[sp++] = leaf[o.arg][w];
        } else if (o.op == OC_WHERE_NOT) {
            st[sp - 1] = ~st[sp - 1];
        } else {
            uint64_t v = st[--sp];
            for (uint32_t k = 1; k < o.arg; k++) {
                const uint64_t u = st[--sp];
                v = o.op == OC_WHERE_AND ? (u & v) : (u | v);
            }
            st[sp++] = v;
        }
    }
    pg.out[w] = st[0] & tail;
}

}  // namespace oc
