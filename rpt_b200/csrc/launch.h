// launch.h -- host-callable launchers, one set per precision (each set lives in its
// own translation unit so the f64 parity gate can be compiled with -fmad=false).
#pragma once
#include "scene_dev.cuh"

namespace rptb {

#define RPTB_DECLARE_LAUNCHERS(SUFFIX, R)                                                                          \
    cudaError_t launch_render_##SUFFIX(const SceneView<R>& sv, const RenderArgs<R>& args, int stats,               \
                                       int features, cudaStream_t stream, uint32_t* launches);                     \
    cudaError_t launch_closest_hit_##SUFFIX(const SceneView<R>& sv, const double* rays, uint64_t n, double tmin,   \
                                            double* out_t, int32_t* out_obj, double* out_n,                        \
                                            DeviceCounters* counters, int stats, int features,                     \
                                            cudaStream_t stream);                                                  \
    cudaError_t launch_bsdf_##SUFFIX(const MaterialRec<R>& m, const double* dirs, uint64_t n, double* out,         \
                                     cudaStream_t stream);                                                         \
    cudaError_t launch_sample_f_##SUFFIX(const MaterialRec<R>& m, const double* dirs, uint64_t n, uint64_t seed,   \
                                         double* out_wi, double* out_pdf, cudaStream_t stream);                    \
    cudaError_t launch_illuminate_##SUFFIX(const SceneView<R>& sv, uint32_t light, const double* pos, uint64_t n,  \
                                           uint64_t seed, double* out_i, double* out_wi, double* out_dist,         \
                                           cudaStream_t stream);

RPTB_DECLARE_LAUNCHERS(f32, float)
RPTB_DECLARE_LAUNCHERS(f64, double)

// ---- wavefront engine (f32 only; wavefront.cuh) -------------------------------------------
struct WfBuffers;
// bytes of device memory the engine needs for (npaths, Ks sampled lights, maxd levels)
size_t wavefront_bytes(uint32_t npaths, uint32_t Ks, uint32_t maxd);
// carve `mem` (wavefront_bytes big, 256-byte aligned) into the engine's arrays
void wavefront_carve(void* mem, uint32_t npix, uint32_t G, uint32_t Ks, uint32_t maxd, WfBuffers* out);
uint32_t wavefront_groups(uint32_t npix, uint32_t nchunks);
size_t wavefront_struct_size();
// run Renderer::sample with the wavefront schedule: everything is enqueued on `stream` (the step loop is a CUDA graph
// WHILE node re-armed on the device); the call does not wait
cudaError_t run_wavefront_f32(const SceneView<float>& sv, const RenderArgs<float>& args, const WfBuffers* bufs,
                              bool stats, bool use_bvh, cudaStream_t stream, uint32_t* launches);

// ---- the vertex-at-once f32 megakernel (integrator_vx.cuh; its own translation unit, kernels_vx.cu) -----------------
// stats as in launch_render_f32.  args.ks must be <= VX_MAX_SHADOW (vx_supported).
cudaError_t launch_render_vx_f32(const SceneView<float>& sv, const RenderArgs<float>& args, int stats, int features,
                                 cudaStream_t stream, uint32_t* launches);
bool vx_supported(uint32_t sampled_lights);

// max_bounces the render kernels are instantiated for
constexpr uint32_t MAX_BOUNCES_SUPPORTED = 64;

// ---- which instantiation serves a scene ------------------------------------------------------------------------------
// The kernels are instantiated per scene feature set (FEAT), counting pass (STATS) and, for the f64 gate's level stack,
// depth (MAXD).  The pick_* functions choose the variant from the features the kernels see (kernel_features, flatten.h);
// the lists below are every variant that is compiled.  launch_impl.cuh, kernels_vx.cu and the host emulation
// (tests/hostemu) all dispatch through both, so a variant a scene is sent to always exists and is the same everywhere.
struct Variant {
    bool stats;
    int feat;
    int maxd;  // render_kernel's level stack; 0 where there is none (vertex-at-once, closest hit)
};

// render_kernel<R, MAXD, STATS, FEAT> (the slot engine).  stats: rptb_render_params::collect_stats -- 1 counts what the
// product path traverses (the BVH when the scene has one), 2 walks the reference-shaped kd-trees.
constexpr Variant pick_render(int features, int stats, bool f64, uint32_t max_bounces) {
    const int base = features & F_ALL;
    const bool small = (features & F_SMALL) != 0, ext = (features & F_EXT) != 0;
    const bool bvh = !f64 && (features & F_BVH) != 0;  // F_BVH and F_FLAT are f32 only
    const bool flat = !f64 && (features & F_FLAT) != 0;
    // (the f32 path composes the clamps forward and has no depth limit of its own)
    if (f64 && max_bounces > 16) return {stats != 0, F_EVERY, (int)MAX_BOUNCES_SUPPORTED};
    // kd-trees over whole shapes and MonomialSurface live in one extra instantiation (F_EVERY), so the variants tuned
    // for the BASELINE scenes carry none of that code
    if (stats == 1 && bvh) return {true, F_EVERY | F_BVH, 16};
    if (stats) return {true, F_EVERY, 16};
    if (ext && bvh) return {false, F_EVERY | F_BVH, 16};
    if (ext) return {false, F_EVERY, 16};
    if (f64) return {false, F_ALL, 16};  // the f64 gate is not specialised
    // tree scenes do not take the parameter-space tables: measured slower with them
    if (bvh && base == F_TREE) return {false, F_TREE | F_BVH, 16};
    if (bvh) return {false, F_ALL | F_BVH, 16};
    // (the glass variant keeps the scan: its two transformed spheres are cheaper from parameter space than the table
    // is through L1 -- 43.7 against 44.0 ms at 256 spp on one H100 80GB HBM3 at a 400 W power limit)
    if (base == 0 && flat && small) return {false, F_FLAT | F_SMALL, 16};
    if (base == 0 && flat) return {false, F_FLAT, 16};
    if (base == 0 && small) return {false, F_SMALL, 16};
    if (base == 0) return {false, 0, 16};
    if (base == F_TREE) return {false, F_TREE, 16};
    if (base == (F_TRANSP | F_HDRI) && small) return {false, F_TRANSP | F_HDRI | F_SMALL, 16};
    if (base == (F_TRANSP | F_HDRI)) return {false, F_TRANSP | F_HDRI, 16};
    return {false, F_ALL, 16};
}

// render_kernel_vx<STATS, FEAT> (f32 only): the slot engine's variants without the packed table
constexpr Variant pick_render_vx(int features, int stats) {
    const int base = features & F_ALL;
    const bool small = (features & F_SMALL) != 0, ext = (features & F_EXT) != 0, bvh = (features & F_BVH) != 0;
    if (stats == 1 && bvh) return {true, F_EVERY | F_BVH, 0};
    if (stats) return {true, F_EVERY, 0};
    if (ext && bvh) return {false, F_EVERY | F_BVH, 0};
    if (ext) return {false, F_EVERY, 0};
    if (bvh && base == F_TREE) return {false, F_TREE | F_BVH, 0};
    if (bvh) return {false, F_ALL | F_BVH, 0};
    if (base == 0 && small) return {false, F_SMALL, 0};
    if (base == 0) return {false, 0, 0};
    if (base == F_TREE) return {false, F_TREE, 0};
    if (base == (F_TRANSP | F_HDRI) && small) return {false, F_TRANSP | F_HDRI | F_SMALL, 0};
    if (base == (F_TRANSP | F_HDRI)) return {false, F_TRANSP | F_HDRI, 0};
    return {false, F_ALL, 0};
}

// closest_hit_kernel<R, STATS, FEAT> (rptb_closest_hit).  stats == 1: counters of the structure the product path
// traverses; stats == 2: the reference-shaped kd-trees.  Without counters a flat scene is walked through the table the
// megakernel walks.
constexpr Variant pick_closest_hit(int features, int stats, bool f64) {
    const bool bvh = !f64 && (features & F_BVH) != 0;
    if (bvh && stats != 2) return {stats != 0, F_EVERY | F_BVH, 0};
    if (!f64 && !stats && (features & F_FLAT)) return {false, F_FLAT, 0};
    return {stats != 0, F_EVERY, 0};
}

// The compiled variants, one type per entry of a list.
template <bool STATS, int FEAT, int MAXD = 0>
struct V {
    static constexpr bool stats = STATS;
    static constexpr int feat = FEAT;
    static constexpr int maxd = MAXD;
};
template <class... Vs>
struct VariantList {
    static constexpr bool has(Variant v) { return ((Vs::stats == v.stats && Vs::feat == v.feat && Vs::maxd == v.maxd) || ...); }
};

// visit(List{}, v, fn) calls fn(V<...>{}) for the entry equal to v (instantiating fn for every entry); false if there is
// none -- a scene sent to a variant that is not compiled is an error, never a quiet fall-back
template <class Fn>
bool visit(VariantList<>, Variant, Fn&&) { return false; }
template <class First, class... Rest, class Fn>
bool visit(VariantList<First, Rest...>, Variant v, Fn&& fn) {
    if (First::stats == v.stats && First::feat == v.feat && First::maxd == v.maxd) {
        fn(First{});
        return true;
    }
    return visit(VariantList<Rest...>{}, v, fn);
}

using RenderVariantsF32 = VariantList<
    V<true, F_EVERY | F_BVH, 16>, V<true, F_EVERY, 16>, V<false, F_EVERY | F_BVH, 16>, V<false, F_EVERY, 16>,
    V<false, F_TREE | F_BVH, 16>, V<false, F_ALL | F_BVH, 16>, V<false, F_FLAT | F_SMALL, 16>, V<false, F_FLAT, 16>,
    V<false, F_SMALL, 16>, V<false, 0, 16>, V<false, F_TREE, 16>, V<false, F_TRANSP | F_HDRI | F_SMALL, 16>,
    V<false, F_TRANSP | F_HDRI, 16>, V<false, F_ALL, 16>>;
// (the F_BVH entries of the f64 lists are compiled but never picked: F_BVH is f32 only)
using RenderVariantsF64 = VariantList<
    V<true, F_EVERY | F_BVH, 16>, V<true, F_EVERY, 16>, V<false, F_EVERY | F_BVH, 16>, V<false, F_EVERY, 16>,
    V<false, F_ALL, 16>, V<true, F_EVERY, (int)MAX_BOUNCES_SUPPORTED>, V<false, F_EVERY, (int)MAX_BOUNCES_SUPPORTED>>;
using RenderVariantsVx = VariantList<
    V<true, F_EVERY | F_BVH>, V<true, F_EVERY>, V<false, F_EVERY | F_BVH>, V<false, F_EVERY>, V<false, F_TREE | F_BVH>,
    V<false, F_ALL | F_BVH>, V<false, F_SMALL>, V<false, 0>, V<false, F_TREE>, V<false, F_TRANSP | F_HDRI | F_SMALL>,
    V<false, F_TRANSP | F_HDRI>, V<false, F_ALL>>;
using HitVariantsF32 = VariantList<V<false, F_FLAT>, V<true, F_EVERY | F_BVH>, V<true, F_EVERY>, V<false, F_EVERY | F_BVH>,
                                   V<false, F_EVERY>>;
using HitVariantsF64 = VariantList<V<true, F_EVERY | F_BVH>, V<true, F_EVERY>, V<false, F_EVERY | F_BVH>, V<false, F_EVERY>>;

}  // namespace rptb
