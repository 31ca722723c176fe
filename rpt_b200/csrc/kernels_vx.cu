// kernels_vx.cu -- the vertex-at-once f32 megakernel (integrator_vx.cuh), instantiated per scene feature set.
#include "integrator_vx.cuh"
#include "launch.h"

namespace rptb {

bool vx_supported(uint32_t sampled_lights) { return sampled_lights <= VX_MAX_SHADOW; }

cudaError_t launch_render_vx_f32(const SceneView<float>& sv, const RenderArgs<float>& args, int stats, int features,
                                 cudaStream_t stream, uint32_t* launches) {
    uint32_t nl = 0;
    const size_t nvals = (size_t)args.width * args.height * 3;
    if (args.shard_count > 1 && !args.compact) {  // other shards' pixels must read as zero
        clear_kernel<float><<<(unsigned)((nvals + 255) / 256), 256, 0, stream>>>(args.out, nvals);
        nl++;
    }
    if (args.ntiles_mine > 0) {
        const dim3 grid(args.ntiles_mine, args.ngroups);
        const size_t smem = sizeof(uint32_t) * vx_shared_words(args.ks + 1u);
        // the same feature-specialised variants as the slot engine (launch.h); no MAXD: there is no level stack
        const bool found = visit(RenderVariantsVx{}, pick_render_vx(features, stats), [&](auto v) {
            using T = decltype(v);
            render_kernel_vx<T::stats, T::feat><<<grid, RENDER_THREADS, smem, stream>>>(sv, args);
        });
        if (!found) return cudaErrorInvalidValue;
        nl++;
        if (args.nchunks > 1) {
            resolve_chunks_kernel<float><<<args.ntiles_mine, RENDER_THREADS, 0, stream>>>(args);
            nl++;
        }
    }
    if (launches) *launches = nl;
    return cudaGetLastError();
}

}  // namespace rptb
