// launch_impl.cuh -- templated bodies of the launchers declared in launch.h.
#pragma once
#include <type_traits>

#include "integrator.cuh"
#include "launch.h"

namespace rptb {

template <class R>
cudaError_t launch_render_impl(const SceneView<R>& sv, const RenderArgs<R>& args, int stats, int features,
                               cudaStream_t stream, uint32_t* launches) {
    uint32_t nl = 0;
    const size_t nvals = (size_t)args.width * args.height * 3;
    if (args.shard_count > 1 && !args.compact) {  // other shards' pixels must read as zero
        clear_kernel<R><<<(unsigned)((nvals + 255) / 256), 256, 0, stream>>>(args.out, nvals);
        nl++;
    }
    if (args.ntiles_mine > 0) {
        const dim3 grid(args.ntiles_mine, args.ngroups), block(RENDER_THREADS);
        using List = std::conditional_t<M<R>::literal, RenderVariantsF64, RenderVariantsF32>;
        const bool found = visit(List{}, pick_render(features, stats, M<R>::literal, args.max_bounces), [&](auto v) {
            using T = decltype(v);
            render_kernel<R, T::maxd, T::stats, T::feat><<<grid, block, 0, stream>>>(sv, args);
        });
        if (!found) return cudaErrorInvalidValue;
        nl++;
        if (args.nchunks > 1) {
            resolve_chunks_kernel<R><<<args.ntiles_mine, RENDER_THREADS, 0, stream>>>(args);
            nl++;
        }
    }
    if (launches) *launches = nl;
    return cudaGetLastError();
}

template <class R>
cudaError_t launch_closest_hit_impl(const SceneView<R>& sv, const double* rays, uint64_t n, double tmin, double* out_t,
                                    int32_t* out_obj, double* out_n, DeviceCounters* counters, int stats, int features,
                                    cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    const unsigned grid = (unsigned)((n + 127) / 128);
    using List = std::conditional_t<M<R>::literal, HitVariantsF64, HitVariantsF32>;
    const bool found = visit(List{}, pick_closest_hit(features, stats, M<R>::literal), [&](auto v) {
        using T = decltype(v);
        // with the lane-group traversal compiled in, a scene with a BVH is queried the way it is rendered
        if constexpr (!M<R>::literal && RPTB_COOP_MAX > 0 && (T::feat & F_BVH) != 0)
            closest_hit_coop_kernel<T::stats, T::feat><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
        else
            closest_hit_kernel<R, T::stats, T::feat><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
    });
    if (!found) return cudaErrorInvalidValue;
    return cudaGetLastError();
}

template <class R>
cudaError_t launch_bsdf_impl(const MaterialRec<R>& m, const double* dirs, uint64_t n, double* out, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    bsdf_kernel<R><<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(m, dirs, n, out);
    return cudaGetLastError();
}

template <class R>
cudaError_t launch_sample_f_impl(const MaterialRec<R>& m, const double* dirs, uint64_t n, uint64_t seed, double* out_wi,
                                 double* out_pdf, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    sample_f_kernel<R><<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(m, dirs, n, seed, out_wi, out_pdf);
    return cudaGetLastError();
}

template <class R>
cudaError_t launch_illuminate_impl(const SceneView<R>& sv, uint32_t light, const double* pos, uint64_t n, uint64_t seed,
                                   double* out_i, double* out_wi, double* out_dist, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    illuminate_kernel<R, F_EVERY><<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(sv, light, pos, n, seed, out_i, out_wi, out_dist);
    return cudaGetLastError();
}

#define RPTB_DEFINE_LAUNCHERS(SUFFIX, R)                                                                            \
    cudaError_t launch_render_##SUFFIX(const SceneView<R>& sv, const RenderArgs<R>& args, int stats,                \
                                       int features, cudaStream_t stream, uint32_t* launches) {                     \
        return launch_render_impl<R>(sv, args, stats, features, stream, launches);                                  \
    }                                                                                                               \
    cudaError_t launch_closest_hit_##SUFFIX(const SceneView<R>& sv, const double* rays, uint64_t n, double tmin,    \
                                            double* out_t, int32_t* out_obj, double* out_n,                         \
                                            DeviceCounters* counters, int stats, int features,                      \
                                            cudaStream_t stream) {                                                  \
        return launch_closest_hit_impl<R>(sv, rays, n, tmin, out_t, out_obj, out_n, counters, stats, features,      \
                                          stream);                                                                  \
    }                                                                                                               \
    cudaError_t launch_bsdf_##SUFFIX(const MaterialRec<R>& m, const double* dirs, uint64_t n, double* out,          \
                                     cudaStream_t stream) {                                                         \
        return launch_bsdf_impl<R>(m, dirs, n, out, stream);                                                        \
    }                                                                                                               \
    cudaError_t launch_sample_f_##SUFFIX(const MaterialRec<R>& m, const double* dirs, uint64_t n, uint64_t seed,    \
                                         double* out_wi, double* out_pdf, cudaStream_t stream) {                    \
        return launch_sample_f_impl<R>(m, dirs, n, seed, out_wi, out_pdf, stream);                                  \
    }                                                                                                               \
    cudaError_t launch_illuminate_##SUFFIX(const SceneView<R>& sv, uint32_t light, const double* pos, uint64_t n,   \
                                           uint64_t seed, double* out_i, double* out_wi, double* out_dist,          \
                                           cudaStream_t stream) {                                                   \
        return launch_illuminate_impl<R>(sv, light, pos, n, seed, out_i, out_wi, out_dist, stream);                 \
    }

}  // namespace rptb
