// hostemu_reproject_halves.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by
// rpt_b200/*: `make hostemu` links it into tests/hostemu/_build/libhostemu_reproject.so next to hostemu_reproject.cu,
// and only tests/test_reproject_halves.py calls it.
//
// The history halves of a reprojection and a merge (reproject_pixel_halves, reproject_slot_halves,
// reproject_merge_halves, reproject_merge_slot_halves; reproject.h) compiled for the host, with the same switches as
// hostemu.cu.  Its own translation unit: it needs reproject.h alone.
#include <cstdint>

#include "../../rpt_b200/csrc/reproject.h"

using namespace rptb;

extern "C" {

// reproject_pixel_halves at every pixel of a dw x dh view through dcam (resolved features dnrm, ddepth, dfrac, row-major)
// from the source planes ssums, sm2, scounts, shalf, snrm, sdepth, sfrac (row-major, sw x sh).  Writes out_sums,
// out_m2, out_counts and out_half row-major.
void hostemu_reproject_halves(const rptb_camera* dcam, uint32_t dw, uint32_t dh, const double* dnrm, const double* ddepth,
                              const double* dfrac, const rptb_camera* scam, uint32_t sw, uint32_t sh, const double* ssums, const double* sm2,
                              const uint32_t* scounts, const double* shalf, const double* snrm, const double* sdepth, const double* sfrac,
                              const rptb_reproject* prm, double* out_sums, double* out_m2, uint32_t* out_counts, double* out_half) {
    const ReprojectView dv = reproject_view(*dcam, dw, dh), sv = reproject_view(*scam, sw, sh);
    const ReprojectSource s = {ssums, sm2, scounts, snrm, sdepth, sfrac};
#pragma omp parallel for schedule(static)
    for (int64_t y = 0; y < (int64_t)dh; y++)
        for (uint32_t x = 0; x < dw; x++) {
            const size_t p = (size_t)y * dw + x;
            out_counts[p] = reproject_pixel_halves(dv, sv, s, shalf, x, (uint32_t)y, dnrm + 3 * p, ddepth[p], dfrac[p], *prm,
                                                   out_sums + 3 * p, out_m2 + p, out_half + 3 * p);
        }
}

// reproject_halves_part_kernel on the host: reproject_slot_halves at every element of the compact tiles of shard
// `index` of `count` (nelem elements, feature sums dfeat laid out as feature_planes(dfeat, nelem) over `rays` camera
// rays).  Writes out_sums, out_m2, out_counts, out_half in element order, and *out_reused, the elements with a count > 0.
void hostemu_reproject_halves_part(const rptb_camera* dcam, uint32_t dw, uint32_t dh, uint32_t index, uint32_t count, double* dfeat,
                                   uint64_t nelem, double rays, const rptb_camera* scam, uint32_t sw, uint32_t sh, const double* ssums,
                                   const double* sm2, const uint32_t* scounts, const double* shalf, const double* snrm,
                                   const double* sdepth, const double* sfrac, const rptb_reproject* prm, double* out_sums, double* out_m2,
                                   uint32_t* out_counts, double* out_half, uint64_t* out_reused) {
    const ReprojectView dv = reproject_view(*dcam, dw, dh), sv = reproject_view(*scam, sw, sh);
    const ReprojectSource s = {ssums, sm2, scounts, snrm, sdepth, sfrac};
    const FeaturePlanes f = feature_planes(dfeat, nelem);
    uint64_t reused = 0;
#pragma omp parallel for schedule(static) reduction(+ : reused)
    for (int64_t e = 0; e < (int64_t)nelem; e++) {
        out_counts[e] = reproject_slot_halves(dv, sv, s, shalf, f, rays, index, count, (uint64_t)e, *prm, out_sums + 3 * e, out_m2 + e,
                                              out_half + 3 * e);
        reused += out_counts[e] > 0u;
    }
    *out_reused = reused;
}

// reproject_merge_halves on n synthetic pixels: history hsums (3 per pixel), hm2, hcounts, hhalf (3) merged into the
// fresh sums, m2, counts, half in place.  Writes each pixel's verdict (0 no test, 1 reused, 2 rejected).
void hostemu_merge_halves_pixels(const double* hsums, const double* hm2, const uint32_t* hcounts, const double* hhalf, uint64_t n,
                                 double gamma, double* sums, double* m2, uint32_t* counts, double* half, int32_t* verdict) {
#pragma omp parallel for schedule(static)
    for (int64_t p = 0; p < (int64_t)n; p++)
        verdict[p] = reproject_merge_halves(hsums + 3 * p, hm2[p], hcounts[p], hhalf + 3 * p, gamma, sums + 3 * p, m2 + p, counts + p,
                                            half + 3 * p);
}

// reproject_merge_halves_part_kernel on the host: reproject_merge_slot_halves at every element of the compact tiles of
// shard `index` of `count`, merging into the element-order sums, m2, counts, half in place.  The source as
// hostemu_reproject_halves_part's; *out_reused / *out_rejected: the elements of each verdict.
void hostemu_reproject_merge_halves_part(const rptb_camera* dcam, uint32_t dw, uint32_t dh, uint32_t index, uint32_t count,
                                         double* dfeat, uint64_t nelem, double rays, const rptb_camera* scam, uint32_t sw, uint32_t sh,
                                         const double* ssums, const double* sm2, const uint32_t* scounts, const double* shalf,
                                         const double* snrm, const double* sdepth, const double* sfrac, const rptb_reproject* prm,
                                         double gamma, double* sums, double* m2, uint32_t* counts, double* half, uint64_t* out_reused,
                                         uint64_t* out_rejected) {
    const ReprojectView dv = reproject_view(*dcam, dw, dh), sv = reproject_view(*scam, sw, sh);
    const ReprojectSource s = {ssums, sm2, scounts, snrm, sdepth, sfrac};
    const FeaturePlanes f = feature_planes(dfeat, nelem);
    uint64_t reused = 0, rejected = 0;
#pragma omp parallel for schedule(static) reduction(+ : reused, rejected)
    for (int64_t e = 0; e < (int64_t)nelem; e++) {
        const int v = reproject_merge_slot_halves(dv, sv, s, shalf, f, rays, index, count, (uint64_t)e, *prm, gamma, sums + 3 * e, m2 + e,
                                                  counts + e, half + 3 * e);
        reused += v == 1;
        rejected += v == 2;
    }
    *out_reused = reused;
    *out_rejected = rejected;
}

}  // extern "C"
