// select.h -- the per-pixel choice of the filter's pass count from a half-buffer estimate of each level's error
// (rptb_buffer_denoise_select), one set of functions for the device (select.cu, compiled with -fmad=false) and the host
// emulation (tests/hostemu, -ffp-contract=off).  Every operation is a double rounded on its own, in the order written
// here, so tests/select_ref.py (numpy float64) restates it; only exp (in the filter's weights) may differ from numpy's.
//
// Level k of a pixel is rptb_buffer_denoise's output with iterations = k: level 0 is the raw mean S / n, level k >= 1
// the remodulated colour after pass k.  halves.h gives, per pixel q and channel c, i_0 and u_0 (the demodulation) and
// i_k and U_k (after pass k with the buffer's parameters; i_k is the plain filter's bit for bit).  With A_c = a_c + eps_a:
//     D_c = i_k,c - i_0,c
//     t_c = (D_c * D_c + 2 * (U_k,c * u_0,c)) - u_0,c * u_0,c
//     m_k = (((t_0 * A_0) * A_0 + (t_1 * A_1) * A_1) + (t_2 * A_2) * A_2) / 3
// m_k is unbiased for the mean squared error of level k (bias included) when the weights do not depend on the entries
// and the pixels are independent: E[D^2] = bias^2 + Var(c'_k) - 2 Cov(c'_k, c_0) + Var(c_0), E[U_k u_0] =
// W_pp Var(c_0) = Cov(c'_k, c_0) and E[u_0^2] = Var(c_0), so E[m_k] = bias^2 + Var(c'_k).  At level 0, D = 0 and
// 2x - x is exact: m_0 = u_0^2, the raw mean's variance.
//     M_k(p) = (sum K m_k(q)) / (sum K) over the 5x5 taps q in the image with a finite m_k(q),
//              K = k_u * k_v, k = (1/16, 1/4, 3/8, 1/4, 1/16) (the filter's own kernel), rows outer; NaN with no such tap
// One m_k is a difference of squares and may be negative; the smoothing makes it usable.  Level 0 starts as the best;
// level k replaces the best iff M_k < best M, strictly (NaN never wins, a tie keeps the weaker filter).  The output is
// the best level's value, computed by denoise_finish_kernel's expressions, so every pixel is rptb_buffer_denoise(
// iterations = level) at that pixel, bit for bit.
#pragma once
#include "halves.h"

namespace rptb {

// m_k of one pixel from its level-k i (3) and U (3), its level-0 i (3) and u (3), and its albedo (3).
RPTB_HD double select_m(const double* ik, const double* Uk, const double* i0, const double* u0, const double* albedo, double eps_a) {
    double t[3];
    for (int c = 0; c < 3; c++) {
        const double D = ik[c] - i0[c];
        t[c] = (D * D + 2.0 * (Uk[c] * u0[c])) - u0[c] * u0[c];
    }
    const double A0 = albedo[0] + eps_a, A1 = albedo[1] + eps_a, A2 = albedo[2] + eps_a;
    return (((t[0] * A0) * A0 + (t[1] * A1) * A1) + (t[2] * A2) * A2) / 3.0;
}

// M_k at pixel (x, y) from the m_k plane (1 per pixel).
RPTB_HD double select_smooth(const double* __restrict__ m, uint32_t width, uint32_t height, uint32_t x, uint32_t y) {
    const double k5[5] = {1.0 / 16.0, 1.0 / 4.0, 3.0 / 8.0, 1.0 / 4.0, 1.0 / 16.0};
    double ms = 0.0, mw = 0.0;
    for (int v = -2; v <= 2; v++)
        for (int u = -2; u <= 2; u++) {
            const int64_t qx = (int64_t)x + u, qy = (int64_t)y + v;
            if (qx < 0 || qy < 0 || qx >= (int64_t)width || qy >= (int64_t)height) continue;
            const double mq = m[(size_t)qy * width + (size_t)qx];
            if (!denoise_finite(mq)) continue;
            const double k = k5[u + 2] * k5[v + 2];
            ms = ms + k * mq;
            mw = mw + k;
        }
    return ms / mw;
}

// One level's step at pixel p = (x, y): M_k from m, and with k == 0 the start (level 0, M_0, the raw mean S / n), with
// k >= 1 the replacement of the best iff M_k < best M (the colour c' = i_k * (a + eps_a)).  best (3), *best_M, *level:
// the pixel's running choice.
RPTB_HD void select_level(const double* __restrict__ m, const double* __restrict__ ik, const double* __restrict__ albedo,
                          const double* __restrict__ sums, const uint32_t* __restrict__ counts, uint32_t width, uint32_t height,
                          uint32_t x, uint32_t y, uint32_t k, double eps_a, double* best, double* best_M, uint8_t* level) {
    const size_t p = (size_t)y * width + x;
    const double M = select_smooth(m, width, height, x, y);
    if (k == 0) {
        for (int c = 0; c < 3; c++) best[c] = sums[3 * p + c] / (double)counts[p];
        *best_M = M;
        *level = 0;
        return;
    }
    if (!(M < *best_M)) return;
    for (int c = 0; c < 3; c++) best[c] = ik[3 * p + c] * (albedo[3 * p + c] + eps_a);
    *best_M = M;
    *level = (uint8_t)k;
}

}  // namespace rptb
