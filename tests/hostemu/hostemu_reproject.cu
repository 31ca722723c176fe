// hostemu_reproject.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_reproject.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_reproject.so).
//
// The reprojection's per-pixel function (reproject.h) compiled for the host, on top of the denoiser's emulation
// (hostemu_denoise.cu, included whole: its first-hit feature pass gives the features the reprojection reads).  Same
// switches as hostemu.cu.
#include "../../rpt_b200/csrc/reproject.h"
#include "hostemu_denoise.cu"

extern "C" {

// reproject_pixel at every pixel of a dw x dh view through camera dcam (resolved features dnrm (3 per pixel), ddepth,
// dfrac) from the state of a sw x sh view through scam: sums (3 per pixel), m2, counts and its resolved features.
// Writes out_sums (3 per pixel), out_m2, out_counts, row-major.
void hostemu_reproject(const rptb_camera* dcam, uint32_t dw, uint32_t dh, const double* dnrm, const double* ddepth, const double* dfrac,
                       const rptb_camera* scam, uint32_t sw, uint32_t sh, const double* ssums, const double* sm2, const uint32_t* scounts,
                       const double* snrm, const double* sdepth, const double* sfrac, const rptb_reproject* prm, double* out_sums,
                       double* out_m2, uint32_t* out_counts) {
    const ReprojectView dv = reproject_view(*dcam, dw, dh), sv = reproject_view(*scam, sw, sh);
    const ReprojectSource s = {ssums, sm2, scounts, snrm, sdepth, sfrac};
#pragma omp parallel for schedule(static)
    for (int64_t y = 0; y < (int64_t)dh; y++)
        for (uint32_t x = 0; x < dw; x++) {
            const size_t p = (size_t)y * dw + x;
            out_counts[p] = reproject_pixel(dv, sv, s, x, (uint32_t)y, dnrm + 3 * p, ddepth[p], dfrac[p], *prm, out_sums + 3 * p, out_m2 + p);
        }
}

}  // extern "C"
