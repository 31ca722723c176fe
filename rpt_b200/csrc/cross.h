// cross.h -- the cross-filtered denoiser with a smoothed selection map (rptb_buffer_denoise_cross), one set of functions
// for the device (cross.cu, compiled with -fmad=false) and the host emulation (tests/hostemu, -ffp-contract=off).  Every
// operation is a double rounded on its own, in the order written here, so tests/cross_ref.py (numpy float64) restates
// it; only exp (in the filter's weights) may differ from numpy's.
//
// Each half of a buffer with halves (halves.h) is filtered with weights computed from the other half alone (cross-
// filtering: Rousselle, Manzi & Zwicker 2013; Bitterli et al. 2016), and the candidate levels are blended through smoothed
// selection maps rather than a hard per-pixel argmin (Rousselle, Knaus & Zwicker 2012).  Per pixel, half A is the even
// entries and half B the odd ones: S_B = HALF, S_A = S - S_B, n_B = floor(n / 2), n_A = n - n_B; A_c = a_c + eps_a and
// v = mean_variance(n, M2), the plain demodulation's variance.
//
// Demodulate (NaN in all of i_A, i_B, v_A, v_B when n_B = 0, as halves_u):
//     i_H = (S_H / n_H) / A,   v_H = (v * n) / n_H      (an unbiased estimate of the variance of half H's mean)
// Two guide chains, k = 1 .. iterations.  Chain H's guide G_H,k = (colour, variance) is one denoise_taps pass over
// G_H,k-1 with the buffer's features and parameters, G_H,0 = (i_H, v_H); with the same weights w^H it filters the other
// half's payload, X_H^,k = (sum w^H X_H^,k-1,q) / (sum of w^H over the taps whose X (all three channels) is finite),
// X_H^,0 = i_H^, and a pixel whose own guide is not finite keeps its X.  That is halves.h's HalvesSums with X in u's
// place, so each chain runs as halves_pass_kernel.  So X_A,k = W^B_k i_A, with W^B_k the composite weights of B's own
// chain: they do not depend on A's entries.  Two dependences remain: v_H comes from the full buffer's M2, and the
// features share camera rays with the first entries (sample_features), so the weights are not independent of the colour
// in principle.  Both are weaker than the luminance edge-stop on the colour being filtered, which this removes.
// Candidate levels, per channel:
//     O_0 = S / n                                             (denoise_finish_kernel's expression)
//     O_k = (((n_A * X_A,k) + (n_B * X_B,k)) / n) * A           k >= 1
// Risk per level, on remodulated values, with mean_c(x) = ((x_0 + x_1) + x_2) / 3:
//     d^A = A * (X_A,k - i_B,0),  d^B = A * (X_B,k - i_A,0),  e = A * (X_A,k - X_B,k)
//     m^A = mean_c(d^A * d^A) - v_B,  m^B = mean_c(d^B * d^B) - v_A,  D = mean_c(e * e)
//     m_k = 0.5 * ((m^A - (D * n_B) / n) + (m^B - (D * n_A) / n)) + ((D * n_A) * n_B) / (n * n)
// Derivation.  With weights W that do not depend on the entries, the same for both halves, and i.i.d. entries of
// per-entry variance behind W (V_1 = the remodulated variance of one entry filtered by W, b = W mu - mu the bias): X_A =
// W i_A is independent of i_B,0, so E[mean_c (d^A)^2] = b^2 + V_1 / n_A + Var(A i_B,0), and E[v_B] = Var(A i_B,0): E[m^A]
// = b^2 + V_1 / n_A; likewise E[m^B] = b^2 + V_1 / n_B; E[D] = V_1 (1 / n_A + 1 / n_B) = V_1 n / (n_A n_B).  So each
// bracket is b^2 in expectation, and O_k = W (n_A i_A + n_B i_B)
// / n = W i has Var(O_k) = V_1 / n = E[D] n_A n_B / n^2: E[m_k] = b^2 + Var(O_k), the level's mean squared error, for every
// count, odd ones included.  At level 0 (X_H,0 = i_H, b = 0) the brackets vanish in expectation and m_0 estimates
// Var(S / n).  One m_k is a difference of squares and may be negative; the smoothing below makes it usable.
// Selection map:
//     M_k    = select_smooth(m_k)   (5x5, the filter's binomial kernel, taps in the image with a finite m_k; select.h)
//     k*     = argmin_k M_k: level 0 starts, a strictly smaller M_k replaces the best, NaN never wins (select_level's rule)
//     beta_k = (sum K [k*(q) = k]) / (sum K) over the 5x5 taps q in the image, K the same binomial kernel, rows outer
//     out    = sum_k beta_k O_k, M^ = sum_k beta_k M_k, in level order over the levels with beta_k != 0; the first such
//              level sets the sums (out = beta_k O_k), so a pixel whose whole 5x5 neighbourhood chose k gets O_k, bit for
//              bit (beta_k = 1 exactly: the two sums add the same weights in the same order).
// M^ is NaN where a blended level's M_k had no finite tap.
#pragma once
#include "select.h"

namespace rptb {

// The row-major planes of one level of both chains (cross.cu, api.cu): chain A's guide colour (3 per pixel) and variance
// and its payload X_B (3), chain B's guide and its payload X_A.
struct CrossSet {
    double *colA, *varA, *XB, *colB, *varB, *XA;
};

// The demodulated halves of one pixel from its sums S (3), odd-entry sums half (3), M2, count n and albedo (3):
// i_A (3), *v_A, i_B (3), *v_B.
RPTB_HD void cross_demodulate(const double* S, const double* half, double m2, uint32_t n, const double* albedo, double eps_a,
                              double* iA, double* vA, double* iB, double* vB) {
    const uint32_t nb = n >> 1, na = n - nb;
    if (nb == 0) {
        iA[0] = iA[1] = iA[2] = iB[0] = iB[1] = iB[2] = *vA = *vB = (double)NAN;
        return;
    }
    const double dA = (double)na, dB = (double)nb;
    const double vn = mean_variance(n, m2) * (double)n;
    *vA = vn / dA;
    *vB = vn / dB;
    for (int c = 0; c < 3; c++) {
        const double A = albedo[c] + eps_a;
        const double sb = half[c], sa = S[c] - sb;
        iA[c] = (sa / dA) / A;
        iB[c] = (sb / dB) / A;
    }
}

// m_k of one pixel from its level-k payloads X_A (3), X_B (3), its level-0 i_A (3), i_B (3), v_A, v_B, count and albedo (3).
RPTB_HD double cross_m(const double* XA, const double* XB, const double* iA0, const double* iB0, double vA, double vB, uint32_t n,
                       const double* albedo, double eps_a) {
    const uint32_t nb = n >> 1, na = n - nb;
    const double dA = (double)na, dB = (double)nb, dn = (double)n;
    double a[3], b[3], e[3];
    for (int c = 0; c < 3; c++) {
        const double A = albedo[c] + eps_a;
        const double da = A * (XA[c] - iB0[c]), db = A * (XB[c] - iA0[c]), de = A * (XA[c] - XB[c]);
        a[c] = da * da;
        b[c] = db * db;
        e[c] = de * de;
    }
    const double mA = ((a[0] + a[1]) + a[2]) / 3.0 - vB;
    const double mB = ((b[0] + b[1]) + b[2]) / 3.0 - vA;
    const double D = ((e[0] + e[1]) + e[2]) / 3.0;
    return 0.5 * ((mA - (D * dB) / dn) + (mB - (D * dA) / dn)) + ((D * dA) * dB) / (dn * dn);
}

// O_k (k >= 1) of one pixel from its payloads X_A (3), X_B (3), count and albedo (3).
RPTB_HD void cross_output(const double* XA, const double* XB, uint32_t n, const double* albedo, double eps_a, double* O) {
    const uint32_t nb = n >> 1, na = n - nb;
    const double dA = (double)na, dB = (double)nb, dn = (double)n;
    for (int c = 0; c < 3; c++) O[c] = ((dA * XA[c] + dB * XB[c]) / dn) * (albedo[c] + eps_a);
}

// One level's step of the argmin at pixel (x, y): M_k from m, and with k == 0 the start, with k >= 1 the replacement iff
// M_k < best M.  *best_M, *level: the pixel's running choice.
RPTB_HD void cross_level(const double* __restrict__ m, uint32_t width, uint32_t height, uint32_t x, uint32_t y, uint32_t k,
                         double* best_M, uint8_t* level) {
    const double M = select_smooth(m, width, height, x, y);
    if (k == 0) {
        *best_M = M;
        *level = 0;
        return;
    }
    if (!(M < *best_M)) return;
    *best_M = M;
    *level = (uint8_t)k;
}

// beta_k at pixel (x, y) from the chosen levels (1 byte per pixel); *first: no tap chose a level below k, so k is the
// first level this pixel blends.
RPTB_HD double cross_beta(const uint8_t* __restrict__ level, uint32_t width, uint32_t height, uint32_t x, uint32_t y, uint32_t k,
                          bool* first) {
    const double k5[5] = {1.0 / 16.0, 1.0 / 4.0, 3.0 / 8.0, 1.0 / 4.0, 1.0 / 16.0};
    double bs = 0.0, bw = 0.0;
    bool below = false;
    for (int v = -2; v <= 2; v++)
        for (int u = -2; u <= 2; u++) {
            const int64_t qx = (int64_t)x + u, qy = (int64_t)y + v;
            if (qx < 0 || qy < 0 || qx >= (int64_t)width || qy >= (int64_t)height) continue;
            const uint32_t lq = level[(size_t)qy * width + (size_t)qx];
            const double K = k5[u + 2] * k5[v + 2];
            if (lq == k) bs = bs + K;
            below = below || lq < k;
            bw = bw + K;
        }
    *first = !below;
    return bs / bw;
}

// One level's step of the blend at pixel p = (x, y): with beta_k != 0, O_k (k == 0: S / n; else from X_A, X_B) and M_k
// (from m) enter out (3) and *M_hat, the first blended level setting them.
RPTB_HD void cross_blend(const uint8_t* __restrict__ level, const double* __restrict__ m, const double* __restrict__ XA,
                         const double* __restrict__ XB, const double* __restrict__ sums, const uint32_t* __restrict__ counts,
                         const double* __restrict__ albedo, uint32_t width, uint32_t height, uint32_t x, uint32_t y, uint32_t k,
                         double eps_a, double* out, double* M_hat) {
    bool first;
    const double b = cross_beta(level, width, height, x, y, k, &first);
    if (b == 0.0) return;
    const size_t p = (size_t)y * width + x;
    double O[3];
    if (k == 0) {
        for (int c = 0; c < 3; c++) O[c] = sums[3 * p + c] / (double)counts[p];
    } else {
        cross_output(XA + 3 * p, XB + 3 * p, counts[p], albedo + 3 * p, eps_a, O);
    }
    const double M = select_smooth(m, width, height, x, y);
    if (first) {
        for (int c = 0; c < 3; c++) out[c] = b * O[c];
        *M_hat = b * M;
    } else {
        for (int c = 0; c < 3; c++) out[c] = out[c] + b * O[c];
        *M_hat = *M_hat + b * M;
    }
}

}  // namespace rptb
