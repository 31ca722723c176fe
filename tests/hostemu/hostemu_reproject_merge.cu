// hostemu_reproject_merge.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by
// rpt_b200/*: `make hostemu` links it into tests/hostemu/_build/libhostemu_reproject.so next to hostemu_reproject.cu,
// and only tests/test_reproject_merge.py calls it.
//
// The history test of rptb_buffer_reproject_merge (reproject_merge, reproject_merge_slot; reproject.h) compiled for the
// host, with the same switches as hostemu.cu.  Its own translation unit: it needs reproject.h alone.
#include <cstdint>

#include "../../rpt_b200/csrc/reproject.h"

using namespace rptb;

extern "C" {

// reproject_merge on n synthetic pixels: history hsums (3 per pixel), hm2, hcounts merged into the fresh sums, m2,
// counts in place.  Writes each pixel's verdict (0 no test, 1 reused, 2 rejected).
void hostemu_merge_pixels(const double* hsums, const double* hm2, const uint32_t* hcounts, uint64_t n, double gamma, double* sums,
                          double* m2, uint32_t* counts, int32_t* verdict) {
#pragma omp parallel for schedule(static)
    for (int64_t p = 0; p < (int64_t)n; p++)
        verdict[p] = reproject_merge(hsums + 3 * p, hm2[p], hcounts[p], gamma, sums + 3 * p, m2 + p, counts + p);
}

// reproject_merge_kernel on the host: at every pixel of a dw x dh view through dcam (resolved features dnrm, ddepth,
// dfrac), the history reproject_pixel takes from the source (as hostemu_reproject's) merged into the fresh row-major
// sums, m2, counts in place.  *out_reused / *out_rejected: the pixels of each verdict.
void hostemu_reproject_merge(const rptb_camera* dcam, uint32_t dw, uint32_t dh, const double* dnrm, const double* ddepth,
                             const double* dfrac, const rptb_camera* scam, uint32_t sw, uint32_t sh, const double* ssums, const double* sm2,
                             const uint32_t* scounts, const double* snrm, const double* sdepth, const double* sfrac,
                             const rptb_reproject* prm, double gamma, double* sums, double* m2, uint32_t* counts, uint64_t* out_reused,
                             uint64_t* out_rejected) {
    const ReprojectView dv = reproject_view(*dcam, dw, dh), sv = reproject_view(*scam, sw, sh);
    const ReprojectSource s = {ssums, sm2, scounts, snrm, sdepth, sfrac};
    uint64_t reused = 0, rejected = 0;
#pragma omp parallel for schedule(static) reduction(+ : reused, rejected)
    for (int64_t y = 0; y < (int64_t)dh; y++)
        for (uint32_t x = 0; x < dw; x++) {
            const size_t p = (size_t)y * dw + x;
            double sh3[3], m2h;
            const uint32_t nh = reproject_pixel(dv, sv, s, x, (uint32_t)y, dnrm + 3 * p, ddepth[p], dfrac[p], *prm, sh3, &m2h);
            const int v = reproject_merge(sh3, m2h, nh, gamma, sums + 3 * p, m2 + p, counts + p);
            reused += v == 1;
            rejected += v == 2;
        }
    *out_reused = reused;
    *out_rejected = rejected;
}

// reproject_merge_part_kernel on the host: reproject_merge_slot at every element of the compact tiles of shard `index`
// of `count` (nelem elements, feature sums dfeat laid out as feature_planes(dfeat, nelem) over `rays` camera rays),
// merging into the element-order sums, m2, counts in place.  The source and the tallies as hostemu_reproject_merge's.
void hostemu_reproject_merge_part(const rptb_camera* dcam, uint32_t dw, uint32_t dh, uint32_t index, uint32_t count, double* dfeat,
                                  uint64_t nelem, double rays, const rptb_camera* scam, uint32_t sw, uint32_t sh, const double* ssums,
                                  const double* sm2, const uint32_t* scounts, const double* snrm, const double* sdepth,
                                  const double* sfrac, const rptb_reproject* prm, double gamma, double* sums, double* m2,
                                  uint32_t* counts, uint64_t* out_reused, uint64_t* out_rejected) {
    const ReprojectView dv = reproject_view(*dcam, dw, dh), sv = reproject_view(*scam, sw, sh);
    const ReprojectSource s = {ssums, sm2, scounts, snrm, sdepth, sfrac};
    const FeaturePlanes f = feature_planes(dfeat, nelem);
    uint64_t reused = 0, rejected = 0;
#pragma omp parallel for schedule(static) reduction(+ : reused, rejected)
    for (int64_t e = 0; e < (int64_t)nelem; e++) {
        const int v = reproject_merge_slot(dv, sv, s, f, rays, index, count, (uint64_t)e, *prm, gamma, sums + 3 * e, m2 + e, counts + e);
        reused += v == 1;
        rejected += v == 2;
    }
    *out_reused = reused;
    *out_rejected = rejected;
}

}  // extern "C"
