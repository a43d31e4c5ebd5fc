// geo.cuh — the per-point tests of a where-filter leaf on a geopoint field, used by where_geo_kernel (where.cuh).
//
// Replaces GeoPointFieldStorage::filter (read/index/geopoint_field.rs:179-229): a full scan of the field's points per
// leaf.  A field holds its points sorted by document id, structure of arrays: the unit vector (x, y, z) of each point
// (computed on the host), its latitude / longitude in degrees and its document id.  A document is in the leaf when at
// least one of its points satisfies the leaf's predicate; geo_set sets its bit.
//
//   geo_in_radius   great-circle distance d <= r as a chord test: |u_p - u_c|^2 <= thr, thr = 4 sin^2(r / 2R) from the
//                   host (+inf when r >= pi R).  Three subtractions and three multiply-adds per point.
//   geo_in_polygon  even-odd ray crossing (PNPOLY) in planar (lon, lat) degrees against vertices staged in shared memory,
//                   after a bounding-box pre-test.  The crossing test is evaluated with explicitly rounded f64
//                   operations in the order (xj - xi) * (y - yi) / (yj - yi) + xi, so no FMA contraction can change a
//                   result.
#pragma once
#include <cstdint>

namespace oc {

constexpr uint32_t GEO_THREADS = 256;
constexpr uint32_t GEO_MAX_VERTICES = 2048;   // OC_GEO_MAX_VERTICES: 2 x 2048 x 8 B = 32 KB of static shared memory
// Widening of the polygon's lon bounds for the pre-test, in degrees.  A crossing abscissa over |lon| <= 180 carries an
// error of a few ulp of 360 (~1e-13): any margin far above that and far below a meaningful distance is exact.
constexpr double GEO_BBOX_MARGIN = 1e-9;

struct GeoPoints {
    const double *x, *y, *z;        // unit vector of each point
    const double *lat, *lon;        // degrees
    const uint64_t *doc;            // ascending; every id < the filter's nbits
    uint64_t n;
};

__device__ __forceinline__ void geo_set(unsigned long long *bits, uint64_t d) {
    atomicOr(bits + (d >> 6), 1ull << (d & 63));
}

__device__ __forceinline__ bool geo_in_radius(double x, double y, double z, double cx, double cy, double cz, double thr) {
    const double dx = x - cx, dy = y - cy, dz = z - cz;
    return dx * dx + dy * dy + dz * dz <= thr;
}

// bbox = {lon_min, lon_max, lat_min, lat_max}.  A point below, above or left of the box crosses an even number of edges
// and one right of it none, so the pre-test only skips points whose test is false.  The lon bounds are widened by the
// host (GEO_BBOX_MARGIN) because a computed crossing abscissa may lie a few ulp outside [min(xi, xj), max(xi, xj)].
__device__ __forceinline__ bool geo_in_polygon(double x, double y, const double *sx, const double *sy, uint32_t nv, double4 bbox) {
    bool in = false;
    if (x >= bbox.x && x <= bbox.y && y >= bbox.z && y <= bbox.w) {
        for (uint32_t k = 0, j = nv - 1; k < nv; j = k++) {
            const double xi = sx[k], yi = sy[k], xj = sx[j], yj = sy[j];
            if ((yi > y) != (yj > y) &&
                x < __dadd_rn(__ddiv_rn(__dmul_rn(__dadd_rn(xj, -xi), __dadd_rn(y, -yi)), __dadd_rn(yj, -yi)), xi))
                in = !in;
        }
    }
    return in;
}

}  // namespace oc
