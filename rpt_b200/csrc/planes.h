// planes.h -- the per-pixel planes of the device Buffer (rptb_buffer), for the scatter / compact kernels (film.cu), the
// feature pass (features.cuh), the feature resolve (denoise.cu) and the C ABI (api.cu).
//
// A buffer's state is a fixed list of planes, each with a number of values per pixel and a value size, in the order
// of the exchange block (rptb_buffer_export_shard).  The colour planes are separate allocations; the four feature
// planes share one allocation of FEATURE_SUMS doubles per element, laid out by feature_planes.
#pragma once
#include "vec.cuh"

namespace rptb {

// HALF (rptb_buffer_create_halves): the sums of a pixel's odd entries (entry k, counted from 0, for odd k), 3 per
// pixel.  Only a buffer with halves holds it.  It is in PlaneSet, so the scatter and compact kernels (film.cu) move it
// like any other plane, but never in the exchange block, whose planes are COLOUR | FEATURES.
enum Plane { SUMS, M2, NORMAL, ALBEDO, HITS, DEPTH, COUNTS, HALF, NPLANES };
constexpr uint32_t COLOUR = 1u << SUMS | 1u << M2 | 1u << COUNTS;
constexpr uint32_t FEATURES = 1u << NORMAL | 1u << ALBEDO | 1u << HITS | 1u << DEPTH;

struct PlaneShape {
    uint32_t values, bytes;  // per pixel, per value
};
RPTB_HD constexpr PlaneShape plane_shape(int k) {
    constexpr PlaneShape t[NPLANES] = {{3, 8}, {1, 8}, {3, 8}, {3, 8}, {1, 8}, {1, 8}, {1, 4}, {3, 8}};
    return t[k];
}

// One pointer per plane; null: the plane is not in the set.
struct PlaneSet {
    void* p[NPLANES];
};

// The feature sums of nelem elements, one plane after the other: normal (3 per pixel), albedo (3), hits, depth.
constexpr uint32_t FEATURE_SUMS = 8;
struct FeaturePlanes {
    double *n, *a, *h, *z;
};
RPTB_HD FeaturePlanes feature_planes(double* base, size_t nelem) { return {base, base + 3 * nelem, base + 6 * nelem, base + 7 * nelem}; }

// The resolved features of a row-major image (rptb_buffer_features): normal (3 per pixel), albedo (3), depth, hit fraction.
struct Aov {
    double *normal, *albedo, *depth, *frac;
};

}  // namespace rptb
