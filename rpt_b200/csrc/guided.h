// guided.h -- the convergence test of adaptive sampling guided by the denoiser (rptb_sample_into_guided), one set of
// functions for the device (guided.cu, compiled with -fmad=false) and the host emulation (tests/hostemu, -ffp-contract=off).
// tests/guided_ref.py restates it in numpy float64.
//
// After the filter's `iterations` passes over the gathered buffer (denoise.h), a pixel with n entries has the
// demodulated colour i'_p (3), the albedo a_p (3) of its features and the filtered variance v'_p of the last pass.  It
// takes the next entry iff
//     n < min_entries   or   NOT( v'_p <= t * t ),
// where, each operation rounded on its own in exactly this order:
//     c'_k = i'_k * (a_k + eps_a)              the remodulated denoised colour: rptb_buffer_denoise's output, bit for bit
//     m'   = ((c'_0 + c'_1) + c'_2) / 3
//     t    = rel_tol * m' + abs_tol           (a product, then a sum: never fused)
// What follows from this definition:
//   - Non-finite values.  A pixel whose own colour or variance is not finite keeps them through every pass (denoise.h):
//     one with 0 entries has colour 0/0 and one with 1 entry variance 0/0, so v' is NaN, the test compares false and
//     the pixel stays active.  As a neighbour such a pixel has weight 0, so it does not spoil the pixels around it.
//     This covers the pixels a reprojection leaves empty or with one entry.
//   - Units.  v' is in the radiance units the filter propagates: v_p is the variance of the mean before it is divided
//     by the albedo, and the pass forms v' = sum w^2 v_q / (sum w)^2 from the neighbours' radiance variances.  That is
//     the variance of the remodulated c'_p exactly where p's neighbours share its albedo; across an albedo edge it mixes
//     the neighbours' radiance scale into p's.
//   - Correlation between passes.  Each pass treats its inputs as independent, but after the first pass neighbouring
//     outputs share samples, so v' underestimates the true variance of c'.  That is SVGF's approximation, and no factor
//     corrects it here: DESIGN.md section 6e gives the measured ratio.
//   - The plain criterion (adaptive.h) is the guided one with no filter; rptb_sample_into_guided with iterations == 0
//     is rptb_sample_into_adaptive.
#pragma once
#include "../../include/rpt_b200.h"
#include "tile.h"

namespace rptb {

// The test above on one pixel: n, its filtered demodulated colour i (3), albedo (3) and filtered variance v.
RPTB_HD bool guided_active(uint32_t n, const double* i, const double* albedo, double eps_a, double v, const rptb_adaptive& c) {
    if (n < c.min_entries) return true;
    const double c0 = i[0] * (albedo[0] + eps_a), c1 = i[1] * (albedo[1] + eps_a), c2 = i[2] * (albedo[2] + eps_a);
    const double m = ((c0 + c1) + c2) / 3.0;
    const double t = c.rel_tol * m + c.abs_tol;
    return !(v <= t * t);
}

// The test at slot j of owned tile k of part (index, count), over the row-major planes of the whole image: col (3 per
// pixel) and var the last pass's output, albedo (3 per pixel) the resolved features, counts the entries.  A slot past a
// ragged edge is never active.
RPTB_HD bool guided_slot(const double* __restrict__ col, const double* __restrict__ var, const double* __restrict__ albedo,
                         const uint32_t* __restrict__ counts, uint32_t width, uint32_t height, uint32_t index, uint32_t count,
                         uint32_t k, uint32_t j, double eps_a, const rptb_adaptive& c) {
    const int64_t p = tile_pixel(width, height, index + k * count, j);
    if (p < 0) return false;
    return guided_active(counts[p], col + 3 * p, albedo + 3 * p, eps_a, var[p], c);
}

}  // namespace rptb
