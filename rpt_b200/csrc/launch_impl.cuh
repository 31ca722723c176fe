// launch_impl.cuh -- templated bodies of the launchers declared in launch.h.
#pragma once
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
        // (MAXD sizes the f64 gate's level stack; the f32 path composes the clamps forward and has no depth limit of its own)
        if (args.max_bounces <= 16 || !M<R>::literal) {
            // pick the instantiation compiled for exactly the features this scene has (tree scenes do not
            // take the parameter-space tables: measured slower with them)
            const int base = features & F_ALL;
            const bool small = (features & F_SMALL) != 0;
            // kd-trees over whole shapes and MonomialSurface live in one extra instantiation (F_EVERY), so
            // the variants tuned for the BASELINE scenes carry none of that code
            const bool ext = (features & F_EXT) != 0;
            // counting passes: stats == 1 counts what the product path traverses (the BVH when the scene has one),
            // stats == 2 walks the reference-shaped kd-trees (the algorithmic work of SURVEY 8d)
            const bool count_bvh = !M<R>::literal && stats == 1 && (features & F_BVH);
            if (count_bvh) render_kernel<R, 16, true, F_EVERY | F_BVH><<<grid, block, 0, stream>>>(sv, args);
            else if (stats) render_kernel<R, 16, true, F_EVERY><<<grid, block, 0, stream>>>(sv, args);
            else if (!M<R>::literal && ext && (features & F_BVH)) render_kernel<R, 16, false, F_EVERY | F_BVH><<<grid, block, 0, stream>>>(sv, args);
            else if (ext) render_kernel<R, 16, false, F_EVERY><<<grid, block, 0, stream>>>(sv, args);
            else if constexpr (M<R>::literal) render_kernel<R, 16, false><<<grid, block, 0, stream>>>(sv, args);  // the f64 gate is not specialised
            else if ((features & F_BVH) && base == F_TREE) render_kernel<R, 16, false, F_TREE | F_BVH><<<grid, block, 0, stream>>>(sv, args);
            else if (features & F_BVH) render_kernel<R, 16, false, F_ALL | F_BVH><<<grid, block, 0, stream>>>(sv, args);
            else if (base == 0 && small) render_kernel<R, 16, false, F_SMALL><<<grid, block, 0, stream>>>(sv, args);
            else if (base == 0) render_kernel<R, 16, false, 0><<<grid, block, 0, stream>>>(sv, args);
            else if (base == F_TREE) render_kernel<R, 16, false, F_TREE><<<grid, block, 0, stream>>>(sv, args);
            else if (base == (F_TRANSP | F_HDRI) && small) render_kernel<R, 16, false, F_TRANSP | F_HDRI | F_SMALL><<<grid, block, 0, stream>>>(sv, args);
            else if (base == (F_TRANSP | F_HDRI)) render_kernel<R, 16, false, F_TRANSP | F_HDRI><<<grid, block, 0, stream>>>(sv, args);
            else render_kernel<R, 16, false><<<grid, block, 0, stream>>>(sv, args);
        } else {
            // f64 gate, deep paths (max_bounces > 16): the level stack sized for MAX_BOUNCES_SUPPORTED
            if constexpr (M<R>::literal) {
                if (stats) render_kernel<R, (int)MAX_BOUNCES_SUPPORTED, true, F_EVERY><<<grid, block, 0, stream>>>(sv, args);
                else render_kernel<R, (int)MAX_BOUNCES_SUPPORTED, false, F_EVERY><<<grid, block, 0, stream>>>(sv, args);
            }
        }
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
    // stats == 1: counters of the structure the product path traverses; stats == 2: the reference-shaped kd-trees
    // (with the lane-group traversal compiled in, a scene with a BVH is queried the way it is rendered)
    if constexpr (!M<R>::literal && RPTB_COOP_MAX > 0) {
        if (stats != 2 && (features & F_BVH)) {
            if (stats) closest_hit_coop_kernel<true, F_EVERY | F_BVH><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
            else closest_hit_coop_kernel<false, F_EVERY | F_BVH><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
            return cudaGetLastError();
        }
    }
    if (!M<R>::literal && stats == 1 && (features & F_BVH)) closest_hit_kernel<R, true, F_EVERY | F_BVH><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
    else if (stats) closest_hit_kernel<R, true, F_EVERY><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
    else if (!M<R>::literal && (features & F_BVH)) closest_hit_kernel<R, false, F_EVERY | F_BVH><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
    else closest_hit_kernel<R, false, F_EVERY><<<grid, 128, 0, stream>>>(sv, rays, n, tmin, out_t, out_obj, out_n, counters);
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
