// hostemu_denoise.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by rpt_b200/*:
// only tests/test_denoise.py builds and loads it (`make hostemu`, tests/hostemu/_build/libhostemu_denoise.so).
//
// The denoiser's device code compiled for the host, on top of the host emulation of hostemu.cu (included whole, so its
// scenes and dispatch are the ones used here): the first-hit feature pass (features.cuh, through pick_closest_hit over
// the HitVariants lists, as launch_features_impl dispatches) and the per-pixel functions of denoise.h.  Same switches
// as hostemu.cu.
#include "../../rpt_b200/csrc/denoise.h"
#include "../../rpt_b200/csrc/features.cuh"
#include "hostemu.cu"

namespace {

template <class R>
int run_features(const SceneView<R>& sv, const RenderArgs<R>& a, int features, double* acc) {
    using List = std::conditional_t<M<R>::literal, HitVariantsF64, HitVariantsF32>;
    const Variant v = pick_closest_hit(features, 0, M<R>::literal);
    const bool found = visit(List{}, v, [&](auto t) {
        using T = decltype(t);
#pragma omp parallel for schedule(dynamic, 1)
        for (int64_t bx = 0; bx < (int64_t)a.ntiles_mine; bx++)
            for (uint32_t th = 0; th < (uint32_t)RENDER_THREADS; th++) feature_thread<R, T::feat>(sv, a, (uint32_t)bx, th, acc);
    });
    return found ? v.feat : -1;
}

}  // namespace

extern "C" {

// The feature pass of one rptb_buffer_add_features call on a fresh buffer (one replica), gathered row-major: out holds
// width*height*8 doubles, the planes normal sums (3 per pixel), albedo sums (3), hits, depth sums.  Returns the FEAT bits
// of the closest-hit variant that ran, or -1.
int hostemu_features(const hostemu_scene* s, const rptb_camera* cam, const rptb_render_params* p, double* out) {
    if (!s || !cam || !p || !out || p->width == 0 || p->height == 0) return -1;
    auto run = [&](auto tag, const auto& sv) -> int {
        using R = decltype(tag);
        RenderArgs<R> a;
        fill_args(cam, p, a);
        const size_t nelem = (size_t)a.ntiles_mine * RENDER_THREADS, npix = (size_t)p->width * p->height;
        std::vector<double> acc(nelem * FEATURE_SUMS, 0.0);
        const int feat = run_features<R>(sv, a, s->features, acc.data());
        const FeaturePlanes f = feature_planes(acc.data(), nelem);
        const FeaturePlanes o = feature_planes(out, npix);
        for (size_t e = 0; e < nelem; e++) {
            const uint32_t tile = (uint32_t)(e / RENDER_THREADS), j = (uint32_t)(e % RENDER_THREADS);
            const uint32_t x = (tile % a.tiles_x) * TILE_W + ((j >> 5) & 1u) * 8u + (j & 7u);
            const uint32_t y = (tile / a.tiles_x) * TILE_H + (j >> 6) * 4u + ((j >> 3) & 3u);
            if (x >= p->width || y >= p->height) continue;
            const size_t q = (size_t)y * p->width + x;
            for (int k = 0; k < 3; k++) {
                o.n[3 * q + k] = f.n[3 * e + k];
                o.a[3 * q + k] = f.a[3 * e + k];
            }
            o.h[q] = f.h[e];
            o.z[q] = f.z[e];
        }
        return feat;
    };
    if (p->precision == RPTB_PRECISION_F64) return run(0.0, s->v64);
    return run(0.0f, s->v32);
}

// features_resolve on n pixels (planes as hostemu_features writes them): N (3n), z (n), a (3n), f (n).
void hostemu_features_resolve(const double* sums, uint64_t n, double rays, double* nrm, double* z, double* albedo, double* frac) {
    for (uint64_t p = 0; p < n; p++)
        features_resolve(sums[6 * n + p], sums + 3 * p, sums[7 * n + p], sums + 3 * n + 3 * p, rays, nrm + 3 * p, z + p, albedo + 3 * p,
                         frac + p);
}

// denoise_demodulate on n pixels.
void hostemu_demodulate(const double* sums, const double* m2, const uint32_t* counts, uint64_t n, const double* albedo, double eps_a,
                        double* col, double* var) {
    for (uint64_t p = 0; p < n; p++) denoise_demodulate(sums + 3 * p, m2[p], counts[p], albedo + 3 * p, eps_a, col + 3 * p, var + p);
}

// One a-trous pass (denoise_pixel at every pixel) with step h.
void hostemu_denoise_pass(const double* col, const double* var, const double* nrm, const double* depth, const double* albedo, uint32_t width,
                          uint32_t height,
                          uint32_t h, const rptb_denoise* d, double* out_col, double* out_var) {
#pragma omp parallel for schedule(static)
    for (int64_t y = 0; y < (int64_t)height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const size_t p = (size_t)y * width + x;
            denoise_pixel(col, var, nrm, depth, albedo, width, height, x, (uint32_t)y, h, *d, out_col + 3 * p, out_var + p);
        }
}

}  // extern "C"
