// kernels_f32.cu -- the product path: every kernel instantiated for Real = float.
#include <cstdlib>

#include <cstring>

#include "features.cuh"
#include "launch_impl.cuh"
#include "wavefront.cuh"

namespace rptb {
RPTB_DEFINE_LAUNCHERS(f32, float)
cudaError_t launch_features_f32(const SceneView<float>& sv, const RenderArgs<float>& args, int features, double* acc, cudaStream_t stream) {
    return launch_features_impl<float>(sv, args, features, acc, stream);
}

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

size_t wavefront_struct_size() { return sizeof(WfBuffers); }

// paths in flight per owned pixel slot: enough to keep ~2M paths alive, never more than there are chunks
uint32_t wavefront_groups(uint32_t npix, uint32_t nchunks) {
    if (npix == 0) return 1;
    uint32_t g = (2000000u + npix - 1u) / npix;
    if (g > nchunks) g = nchunks;
    return g < 1u ? 1u : g;
}

size_t wavefront_bytes(uint32_t npaths, uint32_t Ks, uint32_t maxd) {
    const size_t n = npaths, slots = n * (Ks + 1);
    return align256(n * sizeof(WfPath)) + align256(n * Ks * 3 * sizeof(float) + 16) + align256(n * maxd * 6 * sizeof(float) + 16) +
           align256(slots * sizeof(WfRay)) + align256(slots * sizeof(WfHit)) + align256(slots * sizeof(uint32_t)) + 256;
}

void wavefront_carve(void* mem, uint32_t npix, uint32_t G, uint32_t Ks, uint32_t maxd, WfBuffers* out) {
    const uint32_t npaths = npix * G;
    out->npix = npix;
    out->G = G;
    char* p = (char*)mem;
    const size_t n = npaths, slots = n * (Ks + 1);
    out->paths = (WfPath*)p; p += align256(n * sizeof(WfPath));
    out->contrib = (float*)p; p += align256(n * Ks * 3 * sizeof(float) + 16);
    out->levels = (float*)p; p += align256(n * maxd * 6 * sizeof(float) + 16);
    out->rays = (WfRay*)p; p += align256(slots * sizeof(WfRay));
    out->hits = (WfHit*)p; p += align256(slots * sizeof(WfHit));
    out->list = (uint32_t*)p; p += align256(slots * sizeof(uint32_t));
    out->count = (uint32_t*)p;  // [0] rays emitted this step, [1] fetch cursor of the trace kernel, [2] a path is pending, [3] steps left
    out->npaths = npaths;
    out->Ks = Ks;
    out->maxd = maxd;
}

// Closes one step of the loop ON THE DEVICE: the body of the graph's WHILE node runs again iff a path is still not done
// after this step (wf_shade_kernel sets count[2]; a path that emitted a ray is one of them) and the step budget is not
// spent.
__global__ void wf_continue_kernel(const WfBuffers b, cudaGraphConditionalHandle handle) {
    uint32_t left = b.count[3];
    if (left) left--;
    b.count[3] = left;
    cudaGraphSetConditional(handle, (b.count[2] != 0u && left != 0u) ? 1u : 0u);
}
__global__ void wf_set_kernel(uint32_t* p, uint32_t v) { *p = v; }

#define WF_CU(call)                  \
    do {                             \
        cudaError_t e_ = (call);     \
        if (e_ != cudaSuccess) {     \
            if (exec) cudaGraphExecDestroy(exec); \
            if (graph) cudaGraphDestroy(graph);   \
            if (cap) cudaStreamDestroy(cap);      \
            return e_;               \
        }                            \
    } while (0)

// Renderer::sample with the wavefront schedule.  Everything is enqueued on `stream` and the call returns without
// waiting: the shade / trace step loop is a CUDA graph whose WHILE node is re-armed by wf_continue_kernel on the device
// (no host round trip per step, no host-side termination poll), so rptb_render_samples_device keeps its stream contract.
cudaError_t run_wavefront_f32(const SceneView<float>& sv, const RenderArgs<float>& args, const WfBuffers* bufs,
                              bool stats, bool use_bvh, cudaStream_t stream, uint32_t* launches) {
    const WfBuffers b = *bufs;
    uint32_t nl = 0;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaStream_t cap = nullptr;
    const size_t nvals = (size_t)args.width * args.height * 3;
    if (args.shard_count > 1 && !args.compact) {
        clear_kernel<float><<<(unsigned)((nvals + 255) / 256), 256, 0, stream>>>(args.out, nvals);
        nl++;
    }
    if (b.npaths == 0) {
        if (launches) *launches = nl;
        return cudaGetLastError();
    }
    const unsigned pgrid = (b.npaths + WF_THREADS - 1) / WF_THREADS;
    wf_init_kernel<<<pgrid, WF_THREADS, 0, stream>>>(args, b);
    nl++;
    // persistent trace grid: as many CTAs as are resident at once
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // with counters the trace kernel always walks the reference-shaped kd-trees (their counts are the algorithmic work)
    const bool bvh = !stats && sv.nmeshes > 0 && use_bvh;
    if (stats) WF_CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wf_trace_kernel<true, false>, WF_THREADS, 0));
    else if (bvh) WF_CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wf_trace_kernel<false, true>, WF_THREADS, 0));
    else WF_CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, wf_trace_kernel<false, false>, WF_THREADS, 0));
    const unsigned tgrid = (unsigned)(sms * (per_sm > 0 ? per_sm : 1));
    // The step budget.  A sample with n <= max_bounces + 1 segments takes at most n + 1 steps after the step that emitted
    // its camera ray: one per segment, and the step that finishes it (it consumes the last vertex's shadow rays, or the
    // miss of its last segment) emits the next sample's camera ray or marks the path done.  The first step emits the
    // first camera ray, so a path of S samples needs at most S (max_bounces + 2) + 1 steps, within the budget of
    // S (max_bounces + 2) + 2.  A path runs ceil(nchunks / G) chunks of `chunk` samples.  The loop ends earlier, after
    // the first step that leaves every path done.
    const unsigned long long per_path = (unsigned long long)((args.nchunks + b.G - 1) / b.G) * args.chunk;
    unsigned long long max_steps = (per_path < args.iterations ? per_path : args.iterations) * (args.max_bounces + 2ull) + 2ull;
    if (max_steps > 0xFFFFFFFFull) max_steps = 0xFFFFFFFFull;
    wf_set_kernel<<<1, 1, 0, stream>>>(b.count + 3, (uint32_t)max_steps);

    // graph = one WHILE node; its body = one step (reset the ray list, shade, trace, decide whether to go on)
    WF_CU(cudaGraphCreate(&graph, 0));
    cudaGraphConditionalHandle handle;
    WF_CU(cudaGraphConditionalHandleCreate(&handle, graph, 1, cudaGraphCondAssignDefault));
    cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
    np.type = cudaGraphNodeTypeConditional;
    np.conditional.handle = handle;
    np.conditional.type = cudaGraphCondTypeWhile;
    np.conditional.size = 1;
    cudaGraphNode_t node;
    WF_CU(cudaGraphAddNode(&node, graph, nullptr, 0, &np));
    cudaGraph_t body = np.conditional.phGraph_out[0];
    WF_CU(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
    WF_CU(cudaStreamBeginCaptureToGraph(cap, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
    cudaMemsetAsync(b.count, 0, 3 * sizeof(uint32_t), cap);
    if (stats) wf_shade_kernel<true><<<pgrid, WF_THREADS, 0, cap>>>(sv, args, b);
    else wf_shade_kernel<false><<<pgrid, WF_THREADS, 0, cap>>>(sv, args, b);
    if (stats) wf_trace_kernel<true, false><<<tgrid, WF_THREADS, 0, cap>>>(sv, b, b.list, args.counters);
    else if (bvh) wf_trace_kernel<false, true><<<tgrid, WF_THREADS, 0, cap>>>(sv, b, b.list, nullptr);
    else wf_trace_kernel<false, false><<<tgrid, WF_THREADS, 0, cap>>>(sv, b, b.list, nullptr);
    wf_continue_kernel<<<1, 1, 0, cap>>>(b, handle);
    WF_CU(cudaStreamEndCapture(cap, nullptr));
    WF_CU(cudaGraphInstantiate(&exec, graph, 0));
    WF_CU(cudaGraphLaunch(exec, stream));
    nl += 3;  // the kernels of ONE step (how often the WHILE body ran is decided on the device)

    if (args.nchunks > 1) resolve_chunks_kernel<float><<<args.ntiles_mine, RENDER_THREADS, 0, stream>>>(args);
    else wf_finish_kernel<<<pgrid, WF_THREADS, 0, stream>>>(args, b);
    nl++;
    if (launches) *launches = nl;
    const cudaError_t e = cudaGetLastError();
    // the executable graph may be destroyed while a launch of it is in flight: the runtime defers the release
    cudaGraphExecDestroy(exec);
    cudaGraphDestroy(graph);
    cudaStreamDestroy(cap);
    return e;
}
}  // namespace rptb
