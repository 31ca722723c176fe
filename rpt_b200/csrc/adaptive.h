// adaptive.h -- the convergence test of adaptive sampling (rptb_sample_into_adaptive), one function for the device
// (adaptive.cu, compiled with -fmad=false) and the host emulation (tests/hostemu, -ffp-contract=off).
//
// A pixel with n entries, per-channel sums S_c and Welford M2 (summed over the channels) takes the next entry iff
//     n < min_entries   or   NOT( err2 <= t * t ),
// where, each operation rounded on its own in exactly this order:
//     dn   = (double)n
//     err2 = M2 / (((dn - 1) * dn) * 3)          the channel-mean variance of the pixel's mean
//     m    = ((S_0 + S_1) + S_2) / (3 * dn)      the pixel's mean, averaged over the channels
//     t    = rel_tol * m + abs_tol               (a product, then a sum: never fused)
// The test is written as NOT(<=) so that a NaN statistic -- which compares false -- keeps the pixel rendering.  The
// same expressions in numpy float64 make the same decision on the same (n, S, M2).
#pragma once
#include "../../include/rpt_b200.h"
#include "vec.cuh"

namespace rptb {

// err2 above: the channel-mean variance of the mean of a pixel with n entries and M2 (also the denoiser's, denoise.h)
RPTB_HD double mean_variance(uint32_t n, double m2) {
    const double dn = (double)n;
    return m2 / (((dn - 1.0) * dn) * 3.0);
}

RPTB_HD bool adaptive_active(uint32_t n, double s0, double s1, double s2, double m2, const rptb_adaptive& c) {
    if (n < c.min_entries) return true;
    const double dn = (double)n;
    const double err2 = mean_variance(n, m2);
    const double m = ((s0 + s1) + s2) / (3.0 * dn);
    const double t = c.rel_tol * m + c.abs_tol;
    return !(err2 <= t * t);
}

}  // namespace rptb
