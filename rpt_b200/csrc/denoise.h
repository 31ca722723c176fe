// denoise.h -- the per-pixel arithmetic of rptb_buffer_denoise and rptb_buffer_features, one set of functions for the
// device (denoise.cu, compiled with -fmad=false) and the host emulation (tests/hostemu, -ffp-contract=off).  Every
// operation is a double rounded on its own, in the order written here, so tests/denoise_ref.py (numpy float64) restates
// it; only exp may differ from numpy's in the last bit.
//
// Features (what a pixel's primary rays saw at their first hit).  Per pixel the buffer keeps, over `rays` camera rays,
// the double sums H (hits), Sn (flipped shading normals), Sz (hit distances) and Sa (material colours of the hits):
//     N = Sn / sqrt((Sn.x*Sn.x + Sn.y*Sn.y) + Sn.z*Sn.z), or 0 when that length is 0
//     z = Sz / H, or +inf when H = 0
//     a = (Sa + (rays - H)) / rays       per channel: a miss sees the environment, whose albedo is 1
//     f = H / rays                       the hit fraction
//
// The filter (SVGF's spatial part: Schied et al. 2017 on the edge-avoiding a-trous wavelet of Dammertz et al. 2010).
//   Demodulate:  i_p = c_p / (a_p + eps_a) per channel;  v_p = var_p, the variance of the mean in radiance units
//                lum(r, g, b) = (0.2126 r + 0.7152 g) + 0.0722 b
//   Pass k (h = 2^k), taps q = p + h (u, v), u, v in -2..2, row by row (v outer, u inner), taps outside the image skipped:
//     K   = k_u * k_v,  k = (1/16, 1/4, 3/8, 1/4, 1/16)
//     w_n = powu(max(0, N_p . N_q), sigma_n)  (binary exponentiation, below); 1 when N_p and N_q are both 0
//     w_z = exp(-|z_p - z_q| / (sigma_z * D + eps_z)),  eps_z = 1e-3 * z_p,
//           D = min(|gx_p (x_p - x_q) + gy_p (y_p - y_q)|, |gx_q (x_p - x_q) + gy_q (y_p - y_q)|):  the depth change
//           both pixels' planes allow (a pixel straddling a silhouette has a steep gradient; its flat neighbour's
//           gradient stops it); 0 when exactly one of z_p, z_q is inf, 1 when both are
//     w_l = exp(-|l_p - l_q| / (sigma_l * sqrt(g_p) + eps_l)),  eps_l = 1e-10,  l_p = lum(i_p (.) A_p),
//           l_q = lum(i_q (.) A_p), A_p = a_p + eps_a:  both colours seen through p's albedo, in the radiance units of
//           the variance (a saturated albedo would otherwise scale the two apart)
//     w   = ((K * w_n) * w_z) * w_l;  the centre tap's w is K(0, 0) = 9/64 whatever the features say
//     a neighbour whose i (any channel) or v is not finite has w = 0
//     i'_p = (sum w i_q) / (sum w),   v'_p = (sum (w * w) v_q) / ((sum w) * (sum w))   (sums in tap order)
//   g_p is v prefiltered by (1/4, 1/2, 1/4) x (1/4, 1/2, 1/4) over the in-image taps with a finite v, divided by the sum
//   of their kernel weights, and then at most v_p: a pixel does not borrow a wider tolerance from a noisier neighbour
//   (the pixels that straddle an edge are the noisy ones).  (gx, gy) is the depth gradient at p: in x, of the forward (z(x+1) - z_p) and backward
//   (z_p - z(x-1)) differences that exist and are finite, the one of smaller magnitude (the backward one on a tie, 0 when
//   neither exists); in y the same.  A pixel whose own i or v is not finite keeps them.
//   Remodulate:  c'_p = i_p * (a_p + eps_a).
#pragma once
#include "../../include/rpt_b200.h"
#include "adaptive.h"

namespace rptb {

constexpr uint32_t kDenoiseMaxIterations = 12;
constexpr double kDenoiseEpsZ = 1e-3;   // eps_z relative to z_p: curved surfaces leave the gradient's plane
constexpr double kDenoiseEpsL = 1e-10;  // eps_l: keeps 0/0 out of w_l where the variance is 0

RPTB_HD double denoise_lum(double r, double g, double b) { return (0.2126 * r + 0.7152 * g) + 0.0722 * b; }

// x^e by binary exponentiation, multiplications in this order: r *= b for a set bit, then b *= b while bits remain.
RPTB_HD double denoise_powu(double x, uint32_t e) {
    double r = 1.0, b = x;
    while (e) {
        if (e & 1u) r = r * b;
        e >>= 1;
        if (e) b = b * b;
    }
    return r;
}

RPTB_HD bool denoise_finite(double x) { return x - x == 0.0; }

// The resolved features of one pixel from its sums H, Sn (3), Sz, Sa (3) over `rays`: N (3), z, a (3), hit fraction f.
RPTB_HD void features_resolve(double H, const double* sn, double sz, const double* sa, double rays, double* N, double* z,
                              double* a, double* f) {
    const double len = ::sqrt((sn[0] * sn[0] + sn[1] * sn[1]) + sn[2] * sn[2]);
    for (int k = 0; k < 3; k++) N[k] = len > 0.0 ? sn[k] / len : 0.0;
    *z = H > 0.0 ? sz / H : (double)INFINITY;
    const double miss = rays - H;
    for (int k = 0; k < 3; k++) a[k] = (sa[k] + miss) / rays;
    *f = H / rays;
}

// Demodulated colour and variance of one pixel: c = S / n divided by the albedo as above, var = M2 / ((n-1) n 3)
// (adaptive.h's statistic).  out_i: 3 values, *out_v: 1.
RPTB_HD void denoise_demodulate(const double* S, double m2, uint32_t n, const double* albedo, double eps_a, double* out_i,
                                double* out_v) {
    const double dn = (double)n;
    const double a0 = albedo[0] + eps_a, a1 = albedo[1] + eps_a, a2 = albedo[2] + eps_a;
    out_i[0] = (S[0] / dn) / a0;
    out_i[1] = (S[1] / dn) / a1;
    out_i[2] = (S[2] / dn) / a2;
    *out_v = mean_variance(n, m2);
}

// One-sided depth difference choice at p along one axis (see the header comment).
RPTB_HD double denoise_grad1(double zm, bool has_m, double z, double zp, bool has_p) {
    const double b = z - zm, f = zp - z;
    const bool ok_b = has_m && denoise_finite(b), ok_f = has_p && denoise_finite(f);
    if (ok_b && ok_f) return ::fabs(f) < ::fabs(b) ? f : b;
    if (ok_b) return b;
    if (ok_f) return f;
    return 0.0;
}

// The depth gradient (gx, gy) at pixel (x, y).
RPTB_HD void denoise_grad(const double* __restrict__ depth, uint32_t width, uint32_t height, uint32_t x, uint32_t y, double& gx,
                          double& gy) {
    const size_t p = (size_t)y * width + x;
    const double z = depth[p];
    gx = denoise_grad1(x > 0 ? depth[p - 1] : 0.0, x > 0, z, x + 1 < width ? depth[p + 1] : 0.0, x + 1 < width);
    gy = denoise_grad1(y > 0 ? depth[p - width] : 0.0, y > 0, z, y + 1 < height ? depth[p + width] : 0.0, y + 1 < height);
}

// The taps of one a-trous pass at pixel (x, y) with step h over row-major planes: col (3 per pixel) and var the current
// demodulated colour and variance, nrm (3 per pixel), depth and albedo (3 per pixel) the resolved features.  Calls
// tap(q, w, i_q (3), v_q) for every tap with its weight w, in tap order (a neighbour with w = 0 because its i or v is not
// finite is not called), then tap.finish(p).  When p's own i or v is not finite it calls tap.keep(p, i_p (3), v_p) alone.
// denoise_pixel and halves_pixel (halves.h) share it, so the error estimate runs over exactly the filter's weights.
template <class Tap>
RPTB_HD void denoise_taps(const double* __restrict__ col, const double* __restrict__ var, const double* __restrict__ nrm,
                          const double* __restrict__ depth, const double* __restrict__ albedo, uint32_t width, uint32_t height,
                          uint32_t x, uint32_t y, uint32_t h, const rptb_denoise& d, Tap& tap) {
    const size_t p = (size_t)y * width + x;
    const double ip0 = col[3 * p], ip1 = col[3 * p + 1], ip2 = col[3 * p + 2], vp = var[p];
    if (!(denoise_finite(ip0) && denoise_finite(ip1) && denoise_finite(ip2) && denoise_finite(vp))) {
        tap.keep(p, ip0, ip1, ip2, vp);
        return;
    }
    const double k5[5] = {1.0 / 16.0, 1.0 / 4.0, 3.0 / 8.0, 1.0 / 4.0, 1.0 / 16.0};
    const double k3[3] = {0.25, 0.5, 0.25};
    // g_p: the variance prefiltered over 3x3
    double gs = 0.0, gw = 0.0;
    for (int v = -1; v <= 1; v++)
        for (int u = -1; u <= 1; u++) {
            const int64_t qx = (int64_t)x + u, qy = (int64_t)y + v;
            if (qx < 0 || qy < 0 || qx >= (int64_t)width || qy >= (int64_t)height) continue;
            const double vq = var[(size_t)qy * width + (size_t)qx];
            if (!denoise_finite(vq)) continue;
            const double k = k3[u + 1] * k3[v + 1];
            gs = gs + k * vq;
            gw = gw + k;
        }
    const double gf = gs / gw;
    const double g = vp < gf ? vp : gf;
    const double np0 = nrm[3 * p], np1 = nrm[3 * p + 1], np2 = nrm[3 * p + 2];
    const bool np_zero = np0 == 0.0 && np1 == 0.0 && np2 == 0.0;
    const double zp = depth[p];
    const bool zp_inf = !denoise_finite(zp);
    double gx, gy;
    denoise_grad(depth, width, height, x, y, gx, gy);
    const double eps_z = kDenoiseEpsZ * zp;
    const double A0 = albedo[3 * p] + d.albedo_eps, A1 = albedo[3 * p + 1] + d.albedo_eps, A2 = albedo[3 * p + 2] + d.albedo_eps;
    const double lp = denoise_lum(ip0 * A0, ip1 * A1, ip2 * A2);
    const double lden = d.sigma_luminance * ::sqrt(g) + kDenoiseEpsL;
    for (int v = -2; v <= 2; v++)
        for (int u = -2; u <= 2; u++) {
            const int64_t dx = (int64_t)u * h, dy = (int64_t)v * h;
            const int64_t qx = (int64_t)x + dx, qy = (int64_t)y + dy;
            if (qx < 0 || qy < 0 || qx >= (int64_t)width || qy >= (int64_t)height) continue;
            const size_t q = (size_t)qy * width + (size_t)qx;
            const double iq0 = col[3 * q], iq1 = col[3 * q + 1], iq2 = col[3 * q + 2], vq = var[q];
            const double K = k5[u + 2] * k5[v + 2];
            double w;
            if (u == 0 && v == 0) {
                w = K;
            } else {
                if (!(denoise_finite(iq0) && denoise_finite(iq1) && denoise_finite(iq2) && denoise_finite(vq))) continue;
                const double nq0 = nrm[3 * q], nq1 = nrm[3 * q + 1], nq2 = nrm[3 * q + 2];
                double wn;
                if (np_zero && nq0 == 0.0 && nq1 == 0.0 && nq2 == 0.0) {
                    wn = 1.0;
                } else {
                    const double c = (np0 * nq0 + np1 * nq1) + np2 * nq2;
                    wn = denoise_powu(c > 0.0 ? c : 0.0, d.sigma_normal);
                }
                const double zq = depth[q];
                const bool zq_inf = !denoise_finite(zq);
                double wz;
                if (zp_inf || zq_inf) {
                    wz = zp_inf && zq_inf ? 1.0 : 0.0;
                } else {
                    double gqx, gqy;
                    denoise_grad(depth, width, height, (uint32_t)qx, (uint32_t)qy, gqx, gqy);
                    const double dp_ = ::fabs(gx * (double)(-dx) + gy * (double)(-dy));
                    const double dq_ = ::fabs(gqx * (double)(-dx) + gqy * (double)(-dy));
                    const double plane = dq_ < dp_ ? dq_ : dp_;
                    wz = ::exp(-(::fabs(zp - zq) / (d.sigma_depth * plane + eps_z)));
                }
                const double lq = denoise_lum(iq0 * A0, iq1 * A1, iq2 * A2);
                const double wl = ::exp(-(::fabs(lp - lq) / lden));
                w = ((K * wn) * wz) * wl;
            }
            tap(q, w, iq0, iq1, iq2, vq);
        }
    tap.finish(p);
}

// The filter's sums over the taps -- sum w, sum (w * w) v_q and sum w i_q, in tap order -- and its outputs out_col[3],
// *out_var: i'_p = (sum w i_q) / (sum w), v'_p = (sum (w * w) v_q) / ((sum w) * (sum w)), or p's own i and v (keep).
struct DenoiseSums {
    double* out_col;
    double* out_var;
    double sw = 0.0, sww = 0.0, s0 = 0.0, s1 = 0.0, s2 = 0.0;
    RPTB_HD DenoiseSums(double* c, double* v) : out_col(c), out_var(v) {}
    RPTB_HD void operator()(size_t, double w, double iq0, double iq1, double iq2, double vq) {
        sw = sw + w;
        sww = sww + (w * w) * vq;
        s0 = s0 + w * iq0;
        s1 = s1 + w * iq1;
        s2 = s2 + w * iq2;
    }
    RPTB_HD void keep(size_t, double ip0, double ip1, double ip2, double vp) {
        out_col[0] = ip0;
        out_col[1] = ip1;
        out_col[2] = ip2;
        *out_var = vp;
    }
    RPTB_HD void finish(size_t) {
        out_col[0] = s0 / sw;
        out_col[1] = s1 / sw;
        out_col[2] = s2 / sw;
        *out_var = sww / (sw * sw);
    }
};

// One a-trous pass at pixel (x, y) with step h (planes as denoise_taps).  Writes out_col[3], *out_var.
RPTB_HD void denoise_pixel(const double* __restrict__ col, const double* __restrict__ var, const double* __restrict__ nrm,
                           const double* __restrict__ depth, const double* __restrict__ albedo, uint32_t width, uint32_t height,
                           uint32_t x, uint32_t y, uint32_t h, const rptb_denoise& d, double* out_col, double* out_var) {
    DenoiseSums s(out_col, out_var);
    denoise_taps(col, var, nrm, depth, albedo, width, height, x, y, h, d, s);
}

}  // namespace rptb
