// reproject.h -- the per-pixel arithmetic of rptb_buffer_reproject, one set of functions for the device (reproject.cu,
// compiled with -fmad=false) and the host emulation (tests/hostemu, -ffp-contract=off).  Every operation is a double
// rounded on its own, in the order written here, so tests/reproject_ref.py (numpy float64) restates it bit for bit.
//
// The temporal half of SVGF (Schied et al., HPG 2017) for a camera move over an immutable scene: a pixel of the new
// view finds the world point its first hits saw, projects it into the old view and takes the history of the old
// pixels around it that saw the same surface.
//
// Cameras.  D = direction, U = up, R = normalize(D x U), dc = 1 / tan(fov / 2), as fill_args (flatten.h) derives them.
// In a W x H view, dim = max(W, H), the centre ray of pixel (x, y) is r = (dc D + xn R) + yn U (per component), with
//     xn = ((2x + 1) - W) / dim,   yn = ((2(H - y) - 1) - H) / dim.
// dot(a, b) = (a0 b0 + a1 b1) + a2 b2;  cross(a, b) = (a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0);  |a| = sqrt(dot(a, a)).
//
// Per destination pixel p with resolved features N_p, z_p and hit fraction f_p:
//     f_p > 0:  X = eye_dst + z_p (r / |r|),  v = X - eye_src,  l = |v|     (a surface: reprojected by position)
//     f_p = 0:  v = r / |r|,  l = +inf                                      (the environment: reprojected by direction)
// Projection into the source view, by Cramer's rule (up need not be orthogonal to direction):
//     a = dc_s D_s,  b = R_s,  c = U_s,  det = dot(a, cross(b, c))
//     alpha = dot(v, cross(b, c)) / det,  beta = dot(a, cross(v, c)) / det,  gamma = dot(a, cross(b, v)) / det
//     only alpha > 0 has history;  xs = beta / alpha,  ys = gamma / alpha
//     px = (xs dim_s + (W_s - 1)) / 2,  py = ((H_s - 1) - ys dim_s) / 2     (continuous source pixel; integers are centres)
// Taps: x0 = floor(px), y0 = floor(py), fx = px - x0, fy = py - y0; the four taps (x0, y0), (x0 + 1, y0), (x0, y0 + 1),
// (x0 + 1, y0 + 1) in that order, with weights wx * wy from wx = (1 - fx, fx), wy = (1 - fy, fy).  A tap q is valid iff
// its weight is > 0, it lies in the source image, n_q >= 2, its three sums and its M2 are finite, and
//     surface (f_p > 0):      f_q > 0,  |z_q - l| <= depth_tol * l,  dot(N_p, N_q) >= normal_cos
//     environment (f_p = 0):  f_q = 0.
// History: W = sum of the valid taps' weights (in tap order).  W < kReprojectMinWeight: no history (sums 0, M2 0, count
// 0).  Otherwise, with w^_q = w_q / W, in tap order:
//     mu_c = sum w^_q * (S_qc / n_q),   s2 = sum w^_q * (M2_q / (n_q - 1)),   n_h = min(max_history, min over valid q of n_q)
// and the pixel gets sums mu_c * n_h, M2 s2 * (n_h - 1) and count n_h: the mean and the per-entry variance of its
// neighbourhood, carried as if n_h entries had made them.
//
// The device runs the function per element of each destination part's compact tiles (reproject_slot), for a whole
// buffer and a shard buffer (rptb_buffer_reproject_shard) alike: the element's pixel is tile_pixel's, its features
// resolve from the element's own feature sums (features_resolve, denoise.h), and the source is whole and row-major as
// above.  So every pixel gets the bits reproject_pixel gives it over row-major features.
//
// Testing history against fresh entries (rptb_buffer_reproject_merge): dst already holds fresh entries S_f (3), M2_f, n_f
// of its own view, and the history S_h, M2_h, n_h that reproject_pixel gives the pixel is merged in only where the two
// agree.  Nothing happens (and the pixel is not counted) when n_h = 0 or n_f < 2.  Otherwise
//     delta_c = S_hc / n_h - S_fc / n_f,   d2 = (delta_0 delta_0 + delta_1 delta_1) + delta_2 delta_2,
//     v = M2_f / ((n_f - 1) n_f) + M2_h / ((n_h - 1) n_h)      (the channel-summed variance of the difference of the means)
// and the history is rejected -- the pixel keeps its bits -- iff d2 > gamma^2 v (gamma^2 = gamma * gamma).  gamma = +inf
// accepts every history (inf * 0 is NaN, and a comparison with NaN is false); gamma = 0 rejects any history whose mean
// differs.  Accepted, the pixel becomes the parallel (Chan et al.) combination of the two groups:
//     n = n_f + n_h,   S_c = S_fc + S_hc,   M2 = (M2_f + M2_h) + d2 ((double)n_f (double)n_h / (double)n)
// whose between-means term carries the disagreement into the variance the adaptive criterion and the denoiser read.  The
// test reads the pixel's own fresh state only, no neighbourhood: a 3x3 window would cross tile borders into other shards,
// and per pixel the shards' merges stay the whole buffer's bits with no exchange.  reproject_merge_slot is the per-element
// form for a shard's compact tiles, as reproject_slot is reproject_pixel's.
//
// History halves (a dst with halves from a src with halves, rptb_buffer_create_halves).  Each src pixel q also keeps
// H_q, the sums of its odd entries (halves.h).  Per valid tap q of a pixel with history, in tap order, with
// n_Bq = floor(n_q / 2) and n_Aq = n_q - n_Bq:
//     g_q = sqrt((n_Aq n_Bq) / n_q),   delta_qc = ((S_qc - H_qc) / n_Aq - H_qc / n_Bq) * g_q
// the tap's half-mean difference in per-entry units (Var delta_q = sigma_q^2); then, in tap order,
//     t_c = sum w^_q * delta_qc,   w2 = sum w^_q * w^_q,   d_c = t_c / sqrt(w2)
// (for independent taps Var d is a weighted mean of the sigma_q^2), and with n_hB = floor(n_h / 2), n_hA = n_h - n_hB:
//     H_hc = n_hB * mu_c - d_c * sqrt((n_hA n_hB) / n_h)
// is the history's HALF.  halves_u of (mu n_h, H_h, n_h) is then u = d / sqrt(n_h) before the albedo, E[u^2] =
// sigma^2 / n_h: the variance of the mean that the history claims through its capped count.  The taps' own half-means
// would show the noise of up to n_q >> max_history entries, and the error estimate would call stale history converged.
// A pixel with no history, and an element past a ragged edge, gets HALF 0.  The sums, M2 and count are reproject_pixel's.
//
// Merged (reproject_merge_halves): no test and a rejection leave HALF untouched; an accepted history adds H_hc to
// HALF_c when n_f is even and (S_hc - H_hc), the history's A half, when n_f is odd.  So n_B = floor((n_f + n_h) / 2), as
// halves_u assumes, and every later entry k still goes into HALF iff k is odd.
#pragma once
#include <cmath>

#include "../../include/rpt_b200.h"
#include "denoise.h"
#include "planes.h"
#include "tile.h"
#include "vec.cuh"

namespace rptb {

constexpr double kReprojectMinWeight = 1e-2;  // SVGF's threshold on the summed weight of the consistent taps

// One view: a camera and the image size it renders.
struct ReprojectView {
    double eye[3], D[3], U[3], R[3];
    double dc, dim;
    uint32_t width, height;
};

// The source planes, row-major: sums (3 per pixel), M2, counts, and the resolved features normal (3), depth, hit fraction.
struct ReprojectSource {
    const double* sums;
    const double* m2;
    const uint32_t* counts;
    const double* nrm;
    const double* depth;
    const double* frac;
};

inline ReprojectView reproject_view(const rptb_camera& c, uint32_t width, uint32_t height) {
    ReprojectView v;
    const double* di = c.direction;
    const double* up = c.up;
    const double right[3] = {di[1] * up[2] - di[2] * up[1], di[2] * up[0] - di[0] * up[2], di[0] * up[1] - di[1] * up[0]};
    const double len = std::sqrt((right[0] * right[0] + right[1] * right[1]) + right[2] * right[2]);
    for (int k = 0; k < 3; k++) {
        v.eye[k] = c.eye[k];
        v.D[k] = di[k];
        v.U[k] = up[k];
        v.R[k] = right[k] / len;
    }
    v.dc = 1.0 / std::tan(c.fov / 2.0);
    v.width = width;
    v.height = height;
    v.dim = (double)(width > height ? width : height);
    return v;
}

RPTB_HD double reproject_dot(const double* a, const double* b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

RPTB_HD void reproject_cross(const double* a, const double* b, double* o) {
    o[0] = a[1] * b[2] - a[2] * b[1];
    o[1] = a[2] * b[0] - a[0] * b[2];
    o[2] = a[0] * b[1] - a[1] * b[0];
}

RPTB_HD bool reproject_finite(double x) { return x - x == 0.0; }

// The history of destination pixel (x, y) of view dv from the source state s seen through view sv.  Np (3), zp, fp: the
// pixel's resolved features.  Writes out_sums[3] and *out_m2, returns the count.  HALVES: also the history's HALF
// out_half[3] from the source's row-major HALF shalf (3 per pixel).
template <bool HALVES>
RPTB_HD uint32_t reproject_history(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const double* shalf,
                                   uint32_t x, uint32_t y, const double* Np, double zp, double fp, const rptb_reproject& prm,
                                   double* out_sums, double* out_m2, double* out_half) {
    out_sums[0] = 0.0;
    out_sums[1] = 0.0;
    out_sums[2] = 0.0;
    *out_m2 = 0.0;
    if constexpr (HALVES) out_half[0] = out_half[1] = out_half[2] = 0.0;
    const double xn = ((double)(2u * x + 1u) - (double)dv.width) / dv.dim;
    const double yn = ((double)(2u * (dv.height - y) - 1u) - (double)dv.height) / dv.dim;
    double r[3];
    for (int k = 0; k < 3; k++) r[k] = (dv.dc * dv.D[k] + xn * dv.R[k]) + yn * dv.U[k];
    const double rl = ::sqrt(reproject_dot(r, r));
    const bool surface = fp > 0.0;
    double v[3], ell;
    if (surface) {
        for (int k = 0; k < 3; k++) v[k] = (dv.eye[k] + zp * (r[k] / rl)) - sv.eye[k];
        ell = ::sqrt(reproject_dot(v, v));
    } else {
        for (int k = 0; k < 3; k++) v[k] = r[k] / rl;
        ell = (double)INFINITY;
    }
    const double a[3] = {sv.dc * sv.D[0], sv.dc * sv.D[1], sv.dc * sv.D[2]};
    double bc[3], vc[3], bv[3];
    reproject_cross(sv.R, sv.U, bc);
    reproject_cross(v, sv.U, vc);
    reproject_cross(sv.R, v, bv);
    const double det = reproject_dot(a, bc);
    const double alpha = reproject_dot(v, bc) / det;
    const double beta = reproject_dot(a, vc) / det;
    const double gamma = reproject_dot(a, bv) / det;
    if (!(alpha > 0.0)) return 0u;
    const double xs = beta / alpha, ys = gamma / alpha;
    const double px = (xs * sv.dim + (double)(sv.width - 1u)) / 2.0;
    const double py = ((double)(sv.height - 1u) - ys * sv.dim) / 2.0;
    // every tap lies outside (or has weight 0) past these bounds; they also keep a huge or NaN position off the casts
    if (!(px > -1.0 && px < (double)sv.width && py > -1.0 && py < (double)sv.height)) return 0u;
    const double x0 = ::floor(px), y0 = ::floor(py);
    const double fx = px - x0, fy = py - y0;
    const double wx[2] = {1.0 - fx, fx}, wy[2] = {1.0 - fy, fy};
    double w[4];
    int64_t q[4];
    double W = 0.0;
    uint32_t nmin = 0xFFFFFFFFu;
    for (int t = 0; t < 4; t++) {
        w[t] = 0.0;
        q[t] = -1;
        const double wt = wx[t & 1] * wy[t >> 1];
        const int64_t qx = (int64_t)x0 + (t & 1), qy = (int64_t)y0 + (t >> 1);
        if (!(wt > 0.0) || qx < 0 || qy < 0 || qx >= (int64_t)sv.width || qy >= (int64_t)sv.height) continue;
        const int64_t i = qy * (int64_t)sv.width + qx;
        const uint32_t n = s.counts[i];
        if (n < 2u) continue;
        if (!(reproject_finite(s.sums[3 * i]) && reproject_finite(s.sums[3 * i + 1]) && reproject_finite(s.sums[3 * i + 2]) &&
              reproject_finite(s.m2[i])))
            continue;
        const double fq = s.frac[i];
        if (surface) {
            if (!(fq > 0.0)) continue;
            if (!(::fabs(s.depth[i] - ell) <= prm.depth_tol * ell)) continue;
            if (!(reproject_dot(Np, s.nrm + 3 * i) >= prm.normal_cos)) continue;
        } else if (fq != 0.0) {
            continue;
        }
        w[t] = wt;
        q[t] = i;
        W = W + wt;
        nmin = n < nmin ? n : nmin;
    }
    if (!(W >= kReprojectMinWeight)) return 0u;
    double mu0 = 0.0, mu1 = 0.0, mu2 = 0.0, s2 = 0.0;
    double t0 = 0.0, t1 = 0.0, t2 = 0.0, w2 = 0.0;  // HALVES: the weighted half-mean differences, the squared weights
    for (int t = 0; t < 4; t++) {
        if (q[t] < 0) continue;
        const int64_t i = q[t];
        const double wh = w[t] / W;
        const double dn = (double)s.counts[i];
        mu0 = mu0 + wh * (s.sums[3 * i] / dn);
        mu1 = mu1 + wh * (s.sums[3 * i + 1] / dn);
        mu2 = mu2 + wh * (s.sums[3 * i + 2] / dn);
        s2 = s2 + wh * (s.m2[i] / (double)(s.counts[i] - 1u));
        if constexpr (HALVES) {
            const uint32_t nb = s.counts[i] >> 1;
            const double dB = (double)nb, dA = (double)(s.counts[i] - nb);
            const double g = ::sqrt((dA * dB) / dn);
            const double* hq = shalf + 3 * i;
            t0 = t0 + wh * (((s.sums[3 * i] - hq[0]) / dA - hq[0] / dB) * g);
            t1 = t1 + wh * (((s.sums[3 * i + 1] - hq[1]) / dA - hq[1] / dB) * g);
            t2 = t2 + wh * (((s.sums[3 * i + 2] - hq[2]) / dA - hq[2] / dB) * g);
            w2 = w2 + wh * wh;
        }
    }
    const uint32_t nh = prm.max_history < nmin ? prm.max_history : nmin;
    const double dh = (double)nh;
    out_sums[0] = mu0 * dh;
    out_sums[1] = mu1 * dh;
    out_sums[2] = mu2 * dh;
    *out_m2 = s2 * (double)(nh - 1u);
    if constexpr (HALVES) {
        const uint32_t nb = nh >> 1;
        const double dB = (double)nb, dA = (double)(nh - nb);
        const double sw = ::sqrt(w2), k = ::sqrt((dA * dB) / dh);
        out_half[0] = dB * mu0 - (t0 / sw) * k;
        out_half[1] = dB * mu1 - (t1 / sw) * k;
        out_half[2] = dB * mu2 - (t2 / sw) * k;
    }
    return nh;
}

RPTB_HD uint32_t reproject_pixel(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, uint32_t x, uint32_t y,
                                 const double* Np, double zp, double fp, const rptb_reproject& prm, double* out_sums, double* out_m2) {
    return reproject_history<false>(dv, sv, s, nullptr, x, y, Np, zp, fp, prm, out_sums, out_m2, nullptr);
}

// reproject_pixel with the history's HALF out_half[3] from the source's row-major HALF shalf (see History halves above).
RPTB_HD uint32_t reproject_pixel_halves(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const double* shalf,
                                        uint32_t x, uint32_t y, const double* Np, double zp, double fp, const rptb_reproject& prm,
                                        double* out_sums, double* out_m2, double* out_half) {
    return reproject_history<true>(dv, sv, s, shalf, x, y, Np, zp, fp, prm, out_sums, out_m2, out_half);
}

// The history of element `slot` of the compact tiles of shard `index` of `count` of view dv: its pixel is
// tile_pixel(dv.width, dv.height, index + (slot / 128) * count, slot % 128), and its features resolve from the element's
// sums in f (the part's feature planes) over `rays` camera rays.  Writes out_sums[3] and *out_m2, returns the count; an
// element past a ragged edge gets sums 0, M2 0 and count 0.
template <bool HALVES>
RPTB_HD uint32_t reproject_slot_history(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const double* shalf,
                                        const FeaturePlanes& f, double rays, uint32_t index, uint32_t count, uint64_t slot,
                                        const rptb_reproject& prm, double* out_sums, double* out_m2, double* out_half) {
    const int64_t p = tile_pixel(dv.width, dv.height, index + (uint32_t)(slot >> 7) * count, (uint32_t)(slot & 127u));
    if (p < 0) {
        out_sums[0] = 0.0;
        out_sums[1] = 0.0;
        out_sums[2] = 0.0;
        *out_m2 = 0.0;
        if constexpr (HALVES) out_half[0] = out_half[1] = out_half[2] = 0.0;
        return 0u;
    }
    double N[3], z, a[3], fp;
    features_resolve(f.h[slot], f.n + 3 * slot, f.z[slot], f.a + 3 * slot, rays, N, &z, a, &fp);
    return reproject_history<HALVES>(dv, sv, s, shalf, (uint32_t)(p % dv.width), (uint32_t)(p / dv.width), N, z, fp, prm, out_sums,
                                     out_m2, out_half);
}

RPTB_HD uint32_t reproject_slot(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const FeaturePlanes& f,
                                double rays, uint32_t index, uint32_t count, uint64_t slot, const rptb_reproject& prm,
                                double* out_sums, double* out_m2) {
    return reproject_slot_history<false>(dv, sv, s, nullptr, f, rays, index, count, slot, prm, out_sums, out_m2, nullptr);
}

// reproject_slot with the history's HALF out_half[3] (0 past a ragged edge) from the source's row-major HALF shalf.
RPTB_HD uint32_t reproject_slot_halves(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const double* shalf,
                                       const FeaturePlanes& f, double rays, uint32_t index, uint32_t count, uint64_t slot,
                                       const rptb_reproject& prm, double* out_sums, double* out_m2, double* out_half) {
    return reproject_slot_history<true>(dv, sv, s, shalf, f, rays, index, count, slot, prm, out_sums, out_m2, out_half);
}

// Merges the history sh[3], m2h, nh into the fresh state sums[3], *m2, *count in place when the test above accepts it.
// Returns 0 for no test (nh = 0 or n_f < 2), 1 for reused, 2 for rejected.
RPTB_HD int reproject_merge(const double* sh, double m2h, uint32_t nh, double gamma, double* sums, double* m2, uint32_t* count) {
    const uint32_t nf = *count;
    if (nh == 0u || nf < 2u) return 0;
    const double dnf = (double)nf, dnh = (double)nh;
    const double d0 = sh[0] / dnh - sums[0] / dnf;
    const double d1 = sh[1] / dnh - sums[1] / dnf;
    const double d2c = sh[2] / dnh - sums[2] / dnf;
    const double d2 = (d0 * d0 + d1 * d1) + d2c * d2c;
    const double v = *m2 / ((double)(nf - 1u) * dnf) + m2h / ((double)(nh - 1u) * dnh);
    if (d2 > (gamma * gamma) * v) return 2;
    const uint32_t n = nf + nh;
    sums[0] = sums[0] + sh[0];
    sums[1] = sums[1] + sh[1];
    sums[2] = sums[2] + sh[2];
    *m2 = (*m2 + m2h) + d2 * ((dnf * dnh) / (double)n);
    *count = n;
    return 1;
}

// reproject_merge at element `slot` of shard `index` of `count`'s compact tiles: the history reproject_slot gives it,
// merged into the element's fresh sums[3], *m2, *n.  An element past a ragged edge is left untouched (and returns 0).
RPTB_HD int reproject_merge_slot(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const FeaturePlanes& f,
                                 double rays, uint32_t index, uint32_t count, uint64_t slot, const rptb_reproject& prm, double gamma,
                                 double* sums, double* m2, uint32_t* n) {
    double sh[3], m2h;
    const uint32_t nh = reproject_slot(dv, sv, s, f, rays, index, count, slot, prm, sh, &m2h);
    return reproject_merge(sh, m2h, nh, gamma, sums, m2, n);
}

// reproject_merge with the history's HALF hh[3] and the fresh HALF half[3]: an accepted history adds its B half (n_f
// even) or its A half (n_f odd) to half.  Same verdict, sums, M2 and count.
RPTB_HD int reproject_merge_halves(const double* sh, double m2h, uint32_t nh, const double* hh, double gamma, double* sums, double* m2,
                                   uint32_t* count, double* half) {
    const uint32_t nf = *count;
    const int verdict = reproject_merge(sh, m2h, nh, gamma, sums, m2, count);
    if (verdict == 1) {
        const bool odd = (nf & 1u) != 0u;
        for (int k = 0; k < 3; k++) half[k] = half[k] + (odd ? sh[k] - hh[k] : hh[k]);
    }
    return verdict;
}

// reproject_merge_slot with the source's row-major HALF shalf and the element's fresh HALF half[3].
RPTB_HD int reproject_merge_slot_halves(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const double* shalf,
                                        const FeaturePlanes& f, double rays, uint32_t index, uint32_t count, uint64_t slot,
                                        const rptb_reproject& prm, double gamma, double* sums, double* m2, uint32_t* n, double* half) {
    double sh[3], m2h, hh[3];
    const uint32_t nh = reproject_slot_halves(dv, sv, s, shalf, f, rays, index, count, slot, prm, sh, &m2h, hh);
    return reproject_merge_halves(sh, m2h, nh, hh, gamma, sums, m2, n, half);
}

}  // namespace rptb
