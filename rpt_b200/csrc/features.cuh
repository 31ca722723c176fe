// features.cuh -- the first-hit feature pass of the device Buffer (rptb_buffer_add_features): for every pixel and sample,
// the render's camera ray (camera.cuh, same Philox key and draws) through Renderer::get_closest_hit, and the per-pixel
// sums the denoiser is guided by.  Instantiated in kernels_f32.cu and kernels_f64.cu, so each precision is compiled with
// the switches its render kernels use; tests/hostemu runs the same body on the host.
#pragma once
#include <type_traits>

#include "camera.cuh"
#include "integrator.cuh"
#include "launch.h"
#include "planes.h"

namespace rptb {

// Element e = block_x * 128 + thread_x of the replica's compact tile-major layout (RenderArgs::compact): pixel thread_x
// of owned tile block_x.  Adds samples [first_sample, first_sample + iterations) to element e of the feature planes at
// `acc` (planes.h, ntiles_mine * 128 elements), in sample order.
template <class R, int FEAT>
RPTB_D void feature_thread(const SceneView<R>& sv, const RenderArgs<R>& a, const uint32_t block_x, const uint32_t thread_x,
                           double* __restrict__ acc) {
    const uint32_t tile = a.shard_index + block_x * a.shard_count;
    const uint32_t tx = tile % a.tiles_x, ty = tile / a.tiles_x;
    const uint32_t warp = thread_x >> 5, lane = thread_x & 31u;
    const uint32_t x = tx * TILE_W + (warp & 1u) * 8u + (lane & 7u);
    const uint32_t y = ty * TILE_H + (warp >> 1) * 4u + (lane >> 3);
    if (x >= a.width || y >= a.height) return;
    const uint32_t pix = y * a.width + x;
    const R tmin = (R)1e-12;  // EPSILON, renderer.rs:14
    const R dim = (R)max(a.width, a.height);
    const R xn = ((R)(2u * x + 1u) - (R)a.width) / dim;
    const R yn = ((R)(2u * (a.height - y) - 1u) - (R)a.height) / dim;
    const size_t e = (size_t)block_x * RENDER_THREADS + thread_x;
    const FeaturePlanes f = feature_planes(acc, (size_t)a.ntiles_mine * RENDER_THREADS);
    double hits = f.h[e], n0 = f.n[3 * e], n1 = f.n[3 * e + 1], n2 = f.n[3 * e + 2], z = f.z[e];
    double a0 = f.a[3 * e], a1 = f.a[3 * e + 1], a2 = f.a[3 * e + 2];
    for (uint32_t i = 0; i < a.iterations; i++) {
        Rng<R> rng;
        rng.init(a.seed, pix, a.first_sample + i);
        Vec3<R> ro, rd;
        camera_ray(a.cam, xn, yn, dim, rng, ro, rd);
        Hit<R> h;
        h.t = M<R>::inf();
        h.obj = -1;
        TravStats ts = {0, 0, 0, 0, 0};
        closest_hit<R, false, FEAT>(sv, ro, rd, tmin, false, h, ts);
        if (h.obj < 0) continue;
        const ObjectRec<R>& ob = sv.objects[h.obj];
        Vec3<R> n = finalize_hit<R, FEAT>(sv, ob, ro, rd, h).n;
        if (dot(n, rd) > (R)0) n = -n;  // facing the ray
        const MaterialRec<R>& m = sv.materials[ob.material];
        hits = hits + 1.0;
        n0 = n0 + (double)n.x;
        n1 = n1 + (double)n.y;
        n2 = n2 + (double)n.z;
        z = z + (double)h.t;
        a0 = a0 + (double)m.color[0];
        a1 = a1 + (double)m.color[1];
        a2 = a2 + (double)m.color[2];
    }
    f.h[e] = hits;
    f.n[3 * e] = n0; f.n[3 * e + 1] = n1; f.n[3 * e + 2] = n2;
    f.z[e] = z;
    f.a[3 * e] = a0; f.a[3 * e + 1] = a1; f.a[3 * e + 2] = a2;
}

#ifdef __CUDACC__
template <class R, int FEAT>
__global__ void __launch_bounds__(RENDER_THREADS) features_kernel(const __grid_constant__ SceneView<R> sv,
                                                                  const __grid_constant__ RenderArgs<R> a, double* __restrict__ acc) {
    feature_thread<R, FEAT>(sv, a, blockIdx.x, threadIdx.x, acc);
}
#endif

// The closest-hit variant (pick_closest_hit without counters) over the replica's owned tiles.
template <class R>
cudaError_t launch_features_impl(const SceneView<R>& sv, const RenderArgs<R>& a, int features, double* acc, cudaStream_t stream) {
    if (a.ntiles_mine == 0) return cudaSuccess;
    using List = std::conditional_t<M<R>::literal, HitVariantsF64, HitVariantsF32>;
    const bool found = visit(List{}, pick_closest_hit(features, 0, M<R>::literal), [&](auto v) {
        using T = decltype(v);
        features_kernel<R, T::feat><<<a.ntiles_mine, RENDER_THREADS, 0, stream>>>(sv, a, acc);
    });
    if (!found) return cudaErrorInvalidValue;
    return cudaGetLastError();
}

}  // namespace rptb
