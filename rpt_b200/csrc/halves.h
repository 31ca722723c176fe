// halves.h -- the error estimate of the denoised image from two half buffers (rptb_buffer_denoise_error,
// rptb_sample_into_guided_error), one set of functions for the device (halves.cu, compiled with -fmad=false) and the host
// emulation (tests/hostemu, -ffp-contract=off).  Every operation is a double rounded on its own, in the order written
// here, so tests/halves_ref.py (numpy float64) restates it; only exp (in the filter's weights) may differ from numpy's.
//
// A buffer with halves (rptb_buffer_create_halves) keeps, beside a pixel's sums S (3), the sums HALF (3) of its odd
// entries: entry k, k the pixel's count before the add, goes into HALF iff k is odd.  So with n entries
//     S_B = HALF, S_A = S - S_B, n_B = floor(n / 2), n_A = n - n_B.
// Per pixel q and channel c:
//     u_q = ((S_A / n_A - S_B / n_B) * f) / (a_q + eps_a),   f = sqrt(n_A * n_B) / n
// NaN in every channel when n_B = 0.  For i.i.d. entries E[u^2] = Var(S / n) (before the albedo), whatever n: the
// difference of the halves' means has variance sigma^2 (1/n_A + 1/n_B) = sigma^2 n / (n_A n_B).
// Each a-trous pass (denoise.h) filters u with the weights w_pq it computes from the full buffer's colour and variance
// (denoise_taps, shared with denoise_pixel, so c' and v' stay bit for bit rptb_buffer_denoise's):
//     U'_p = (sum w u_q) / (sum of w over the taps whose u (all three channels) is finite),  sums in tap order,
// and a pixel whose own i or v is not finite keeps its u, as it keeps its colour.  The square of the filtered difference
// is then an unbiased estimate of the variance of c' under those weights, correlations between the passes included.
// After the last pass:
//     r_c = U'_c * (a_c + eps_a)                          remodulated, as c' is
//     e_p = ((r_0 * r_0 + r_1 * r_1) + r_2 * r_2) / 3     the channel mean of the square, in the units of v'
//     E_p = (sum k e_q) / (sum k) over the 3x3 taps q in the image with a finite e_q, k = (1/4, 1/2, 1/4) x (1/4, 1/2, 1/4)
// (the variance prefilter's kernel and tap rule, denoise.h): e_p alone is a 3-dof chi^2 sample.
#pragma once
#include "denoise.h"

namespace rptb {

// u of one pixel from its sums S (3), odd-entry sums half (3), count n and albedo (3).
RPTB_HD void halves_u(const double* S, const double* half, uint32_t n, const double* albedo, double eps_a, double* u) {
    const uint32_t nb = n >> 1, na = n - nb;
    if (nb == 0) {
        u[0] = u[1] = u[2] = (double)NAN;
        return;
    }
    const double dA = (double)na, dB = (double)nb;
    const double f = ::sqrt(dA * dB) / (double)n;
    for (int k = 0; k < 3; k++) {
        const double sb = half[k], sa = S[k] - sb;
        u[k] = ((sa / dA - sb / dB) * f) / (albedo[k] + eps_a);
    }
}

// denoise_pixel's sums and outputs, plus the filtered u over the taps whose u is finite and its output out_u[3] (p's own
// u when p keeps its colour).
struct HalvesSums : DenoiseSums {
    const double* __restrict__ u;
    double* out_u;
    double swu = 0.0, su0 = 0.0, su1 = 0.0, su2 = 0.0;
    RPTB_HD HalvesSums(double* c, double* v, const double* u_, double* ou) : DenoiseSums(c, v), u(u_), out_u(ou) {}
    RPTB_HD void operator()(size_t q, double w, double iq0, double iq1, double iq2, double vq) {
        DenoiseSums::operator()(q, w, iq0, iq1, iq2, vq);
        const double u0 = u[3 * q], u1 = u[3 * q + 1], u2 = u[3 * q + 2];
        if (!(denoise_finite(u0) && denoise_finite(u1) && denoise_finite(u2))) return;
        swu = swu + w;
        su0 = su0 + w * u0;
        su1 = su1 + w * u1;
        su2 = su2 + w * u2;
    }
    RPTB_HD void keep(size_t p, double ip0, double ip1, double ip2, double vp) {
        DenoiseSums::keep(p, ip0, ip1, ip2, vp);
        for (int k = 0; k < 3; k++) out_u[k] = u[3 * p + k];
    }
    RPTB_HD void finish(size_t p) {
        DenoiseSums::finish(p);
        out_u[0] = su0 / swu;
        out_u[1] = su1 / swu;
        out_u[2] = su2 / swu;
    }
};

// One a-trous pass at pixel (x, y) with step h: denoise_pixel's out_col[3] and *out_var, bit for bit, and out_u[3]
// from u (3 per pixel).
RPTB_HD void halves_pixel(const double* __restrict__ col, const double* __restrict__ var, const double* __restrict__ u,
                          const double* __restrict__ nrm, const double* __restrict__ depth, const double* __restrict__ albedo,
                          uint32_t width, uint32_t height, uint32_t x, uint32_t y, uint32_t h, const rptb_denoise& d, double* out_col,
                          double* out_var, double* out_u) {
    HalvesSums s(out_col, out_var, u, out_u);
    denoise_taps(col, var, nrm, depth, albedo, width, height, x, y, h, d, s);
}

// e of one pixel from its filtered U (3) and albedo (3).
RPTB_HD double halves_e(const double* U, const double* albedo, double eps_a) {
    const double r0 = U[0] * (albedo[0] + eps_a), r1 = U[1] * (albedo[1] + eps_a), r2 = U[2] * (albedo[2] + eps_a);
    return ((r0 * r0 + r1 * r1) + r2 * r2) / 3.0;
}

// E at pixel (x, y) from the last pass's U (3 per pixel) and the albedo (3 per pixel).
RPTB_HD double halves_error(const double* __restrict__ U, const double* __restrict__ albedo, uint32_t width, uint32_t height, uint32_t x,
                            uint32_t y, double eps_a) {
    const double k3[3] = {0.25, 0.5, 0.25};
    double es = 0.0, ew = 0.0;
    for (int v = -1; v <= 1; v++)
        for (int u = -1; u <= 1; u++) {
            const int64_t qx = (int64_t)x + u, qy = (int64_t)y + v;
            if (qx < 0 || qy < 0 || qx >= (int64_t)width || qy >= (int64_t)height) continue;
            const size_t q = (size_t)qy * width + (size_t)qx;
            const double eq = halves_e(U + 3 * q, albedo + 3 * q, eps_a);
            if (!denoise_finite(eq)) continue;
            const double k = k3[u + 1] * k3[v + 1];
            es = es + k * eq;
            ew = ew + k;
        }
    return es / ew;
}

}  // namespace rptb
