// api.cu -- the extern "C" boundary of include/rpt_b200.h: flattens a
// rptb_scene_desc into the device layout of scene_dev.cuh and drives the kernels.
//
// What it stands in for on the reference side (ekzhang/rpt @815b21c):
//   rptb_scene_create          the borrowed &Scene of Renderer (src/renderer.rs:20) +
//                              Transformed::new precomputation (src/shape.rs:111-124)
//   rptb_render_samples[_device] Renderer::sample (src/renderer.rs:117-129)
//   rptb_closest_hit           Renderer::get_closest_hit (src/renderer.rs:211-220)
//   rptb_bsdf_eval / sample_f  Material::bsdf / sample_f (src/material.rs:125-313)
//   rptb_build_kdtree          KdTree::new (src/kdtree.rs:108-119,235-355)
//   rptb_film_resolve          Buffer::image (src/buffer.rs:43-56,75-93)
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "../../include/rpt_b200.h"
#include "flatten.h"
#include "launch.h"

namespace rptb {
cudaError_t launch_film_resolve(const double* sums, uint32_t nbatches, uint32_t width, uint32_t height,
                                uint32_t radius, uint8_t* out, cudaStream_t stream);
cudaError_t launch_convert_f64_to_f32(const double* in, float* out, size_t n, cudaStream_t stream);
cudaError_t launch_film_variance(const double* batches, uint32_t nbatches, uint64_t npixels, double* out_sum, cudaStream_t stream);
int parse_obj_text(const char* text, size_t len, std::vector<double>& tris, std::string& err);
struct ObjGroup {
    rptb_material material;
    uint64_t first_tri, ntris;
};
int parse_obj_mtl_text(const char* obj, size_t obj_len, const char* mtl, size_t mtl_len, std::vector<double>& tris,
                       std::vector<ObjGroup>& groups, std::string& err);
int parse_stl_bytes(const void* data, size_t len, std::vector<double>& tris, std::string& err);
}  // namespace rptb

using namespace rptb;

// What RPTB_ACCEL_AUTO means when the environment does not say (tools/gpu_accel.py compares the two): the BVH
// renders the same images several times faster on the teapot and the dragon proxy.
#ifndef RPTB_ACCEL_DEFAULT
#define RPTB_ACCEL_DEFAULT RPTB_ACCEL_BVH
#endif

namespace {

thread_local std::string g_error;

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_error = buf;
    return code;
}

#define CU(call)                                                                                       \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess)                                                                         \
            return fail(e_ == cudaErrorMemoryAllocation ? RPTB_ERR_OOM : RPTB_ERR_CUDA, "%s: %s (%s:%d)", #call, \
                        cudaGetErrorString(e_), __FILE__, __LINE__);                                   \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    bool ok = false;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        ok = cudaSetDevice(dev) == cudaSuccess;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// Stream-ordered allocations from a memory pool of the library's OWN (one per device, created on first use):
// creating and destroying a scene per call (what the reference's `Renderer::render` on a host `Scene`
// amounts to) costs microseconds instead of the 1-400 ms cudaMalloc/cudaFree took, because the pool keeps
// what is freed while scenes are alive.  The device's default pool -- which torch, NCCL and the host
// application share -- is left alone; when the last scene on a device is destroyed the pool is trimmed to
// nothing, so the memory goes back to the driver.
struct DevicePool {
    cudaMemPool_t pool = nullptr;
    int scenes = 0;
};
std::mutex g_pool_mutex;
DevicePool g_pools[64];

cudaError_t pool_alloc(void** p, size_t bytes, cudaStream_t stream) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) return cudaMallocAsync(p, bytes, stream);
    cudaMemPool_t pool;
    {
        std::lock_guard<std::mutex> lk(g_pool_mutex);
        DevicePool& dp = g_pools[dev];
        if (!dp.pool) {
            cudaMemPoolProps props;
            std::memset(&props, 0, sizeof(props));
            props.allocType = cudaMemAllocationTypePinned;
            props.handleTypes = cudaMemHandleTypeNone;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = dev;
            const cudaError_t e = cudaMemPoolCreate(&dp.pool, &props);
            if (e != cudaSuccess) return e;
            uint64_t keep = UINT64_MAX;
            cudaMemPoolSetAttribute(dp.pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        pool = dp.pool;
    }
    return cudaMallocFromPoolAsync(p, bytes, pool, stream);
}
// Page-locked staging for the device -> host copy of rptb_render_samples: one buffer per device, kept for the life of the
// process (it is at most one image large).  cudaHostAlloc / cudaFreeHost cost milliseconds each -- with a scene created and
// destroyed per Renderer::render() call they were a quarter of the end-to-end overhead (tools/gpu_e2e_multi.py).
struct StageCache {
    void* p = nullptr;
    size_t bytes = 0;
    bool in_use = false;
};
StageCache g_stage[64];

// Returns a page-locked buffer of at least `bytes`; *cached = it must go back with stage_release (else cudaFreeHost).
cudaError_t stage_acquire(int dev, size_t bytes, void** out, size_t* out_bytes, bool* cached) {
    *cached = false;
    if (dev >= 0 && dev < 64) {
        std::lock_guard<std::mutex> lk(g_pool_mutex);
        StageCache& c = g_stage[dev];
        if (!c.in_use) {
            if (c.bytes < bytes) {
                if (c.p) cudaFreeHost(c.p);
                c.p = nullptr;
                c.bytes = 0;
                const cudaError_t e = cudaHostAlloc(&c.p, bytes, cudaHostAllocDefault);
                if (e != cudaSuccess) return e;
                c.bytes = bytes;
            }
            c.in_use = true;
            *out = c.p;
            *out_bytes = c.bytes;
            *cached = true;
            return cudaSuccess;
        }
    }
    *out_bytes = bytes;
    return cudaHostAlloc(out, bytes, cudaHostAllocDefault);  // a second scene rendering on the same device at the same time
}
void stage_release(int dev, void* p, bool cached) {
    if (!p) return;
    if (!cached) {
        cudaFreeHost(p);
        return;
    }
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    if (dev >= 0 && dev < 64 && g_stage[dev].p == p) g_stage[dev].in_use = false;
}

void pool_scene_born(int dev) {
    if (dev < 0 || dev >= 64) return;
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    g_pools[dev].scenes++;
}
void pool_scene_gone(int dev) {  // call after the scene's frees have completed
    if (dev < 0 || dev >= 64) return;
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    DevicePool& dp = g_pools[dev];
    if (dp.scenes > 0 && --dp.scenes == 0 && dp.pool) cudaMemPoolTrimTo(dp.pool, 0);
}

// All device allocations of a scene, freed together.
struct Arena {
    std::vector<void*> ptrs;
    uint64_t bytes = 0;
    cudaStream_t stream = nullptr;
    template <class T>
    cudaError_t upload(const std::vector<T>& host, const T** dev) {
        *dev = nullptr;
        if (host.empty()) return cudaSuccess;
        void* p = nullptr;
        cudaError_t e = pool_alloc(&p, host.size() * sizeof(T), stream);
        if (e != cudaSuccess) return e;
        ptrs.push_back(p);
        bytes += host.size() * sizeof(T);
        // pageable source: the call returns once the bytes are staged, `host` may die afterwards
        e = cudaMemcpyAsync(p, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice, stream);
        *dev = (const T*)p;
        return e;
    }
    void release() {
        for (void* p : ptrs) cudaFreeAsync(p, stream);
        ptrs.clear();
    }
};

}  // namespace

struct rptb_scene {
    int device = 0;
    cudaStream_t stream = nullptr;
    Arena arena;
    SceneView<float> view32;
    SceneView<double> view64;
    DeviceCounters* counters = nullptr;
    // cached output buffers of rptb_render_samples
    float* out32 = nullptr;
    double* out64 = nullptr;
    size_t out_vals = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::mutex lock;
    uint64_t f32_bytes = 0;
    // wavefront engine: scratch memory (path state, rays, hits) cached between calls
    int features = 0;               // F_TREE | F_TRANSP | F_HDRI actually present in the scene
    bool has_tree = false;          // some mesh's kd-tree is more than one leaf
    uint64_t tree_nodes = 0;        // kd nodes over all meshes
    double wlo[3] = {INFINITY, INFINITY, INFINITY}, whi[3] = {-INFINITY, -INFINITY, -INFINITY};  // world bounds of the meshes
    uint32_t sampled_lights = 0;    // non-ambient lights
    void* wf_mem = nullptr;
    size_t wf_bytes = 0;
    double* partial = nullptr;      // per-chunk pixel sums of the megakernel (nchunks > 1)
    size_t partial_bytes = 0;
    // A render enqueued on a caller's stream returns before it has run, while it still uses the scratch above
    // (partial, counters, out64, wf_mem).  `busy` is recorded behind it; the next call on ANY stream -- and every
    // stream-ordered free or reallocation of scratch on `stream` -- first waits for it.
    cudaEvent_t busy = nullptr;
    bool busy_pending = false;
    // page-locked staging for the device -> host copy of rptb_render_samples
    void* stage = nullptr;
    size_t stage_bytes = 0;
    bool stage_cached = false;
    // rptb_scene_create_multi: the replicas on the other devices (this handle is replica 0)
    std::vector<rptb_scene*> peers;
};

namespace {

// rptb_scene_desc::accel: AUTO -> RPTB_ACCEL env (kdtree | bvh) -> the library default
uint32_t resolve_accel(uint32_t accel) {
    if (accel == RPTB_ACCEL_KDTREE || accel == RPTB_ACCEL_BVH) return accel;
    if (const char* e = getenv("RPTB_ACCEL")) {
        if (std::strcmp(e, "bvh") == 0) return RPTB_ACCEL_BVH;
        if (std::strcmp(e, "kdtree") == 0) return RPTB_ACCEL_KDTREE;
    }
    return RPTB_ACCEL_DEFAULT;
}

// bind_scene's uploader: every array goes to the device through the scene's arena
struct ArenaPut {
    Arena& arena;
    cudaError_t error = cudaSuccess;
    template <class T>
    bool operator()(std::vector<T>& host, const T** where) {
        error = arena.upload(host, where);
        return error == cudaSuccess;
    }
    uint64_t bytes() const { return arena.bytes; }
};

// Uploads the flattened scene to s->device (the current device).  `release` = drop the host copies of the big
// arrays as they are handed over (the last -- or only -- replica).
int scene_bind_device(HostScene& hs, rptb_scene* s, bool release) {
    CU(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
    pool_scene_born(s->device);  // (paired with pool_scene_gone in destroy_replica, which keys on the stream's existence)
    s->arena.stream = s->stream;
    ArenaPut put{s->arena};
    if (!bind_scene(hs, put, release, s->view32, s->view64, s->f32_bytes)) CU(put.error);
    s->features = kernel_features(hs);
    s->has_tree = hs.has_tree;
    s->tree_nodes = hs.tree_nodes;
    s->sampled_lights = hs.sampled_lights;
    for (int k = 0; k < 3; k++) {
        s->wlo[k] = hs.wlo[k];
        s->whi[k] = hs.whi[k];
    }
    CU(pool_alloc((void**)&s->counters, sizeof(DeviceCounters), s->stream));
    CU(cudaMemsetAsync(s->counters, 0, sizeof(DeviceCounters), s->stream));
    CU(cudaEventCreate(&s->ev0));
    CU(cudaEventCreate(&s->ev1));
    CU(cudaEventCreateWithFlags(&s->busy, cudaEventDisableTiming));
    CU(cudaStreamSynchronize(s->stream));  // the scene is resident when create returns
    return RPTB_OK;
}

int flatten_desc(const rptb_scene_desc* d, HostScene& hs) {
    std::string err;
    const int rc = flatten_scene(d, hs, err, resolve_accel(d->accel) == RPTB_ACCEL_BVH);
    if (rc != RPTB_OK) return fail(rc, "%s", err.c_str());
    return RPTB_OK;
}

// Orders `target` (and the library's own stream, on which scratch is freed and reallocated) behind a render
// that an earlier call left running on a caller's stream.
int wait_busy(rptb_scene* s, cudaStream_t target) {
    if (!s->busy_pending) return RPTB_OK;
    CU(cudaStreamWaitEvent(s->stream, s->busy, 0));
    if (target != s->stream) CU(cudaStreamWaitEvent(target, s->busy, 0));
    return RPTB_OK;
}

int check_params(const rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p) {
    if (!s || !cam || !p) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (p->width == 0 || p->height == 0) return fail(RPTB_ERR_BAD_ARG, "empty image %ux%u", p->width, p->height);
    if ((uint64_t)p->width * p->height > 0x7FFFFFFFull / 4) return fail(RPTB_ERR_UNSUPPORTED, "image too large");
    if (p->iterations == 0) return fail(RPTB_ERR_BAD_ARG, "iterations must be > 0 (the reference divides by it)");
    if (p->max_bounces > MAX_BOUNCES_SUPPORTED) return fail(RPTB_ERR_UNSUPPORTED, "max_bounces %u > %u", p->max_bounces, MAX_BOUNCES_SUPPORTED);
    const uint32_t sc = p->shard_count ? p->shard_count : 1;
    if (p->shard_index >= sc) return fail(RPTB_ERR_BAD_ARG, "shard_index %u >= shard_count %u", p->shard_index, sc);
    if (p->precision > RPTB_PRECISION_F64) return fail(RPTB_ERR_BAD_ARG, "bad precision %u", p->precision);
    if (p->engine > RPTB_ENGINE_WAVEFRONT) return fail(RPTB_ERR_BAD_ARG, "bad engine %u", p->engine);
    if (p->collect_stats > 2) return fail(RPTB_ERR_BAD_ARG, "bad collect_stats %u", p->collect_stats);
    if (p->engine == RPTB_ENGINE_WAVEFRONT && p->precision != RPTB_PRECISION_F32)
        return fail(RPTB_ERR_UNSUPPORTED, "the wavefront engine is f32 only (the f64 parity gate is the megakernel)");
    if (p->engine == RPTB_ENGINE_WAVEFRONT && s->sampled_lights > 8)
        return fail(RPTB_ERR_UNSUPPORTED, "the wavefront engine handles at most 8 sampled lights (scene has %u)", s->sampled_lights);
    return RPTB_OK;
}

// Which schedule renders this call (include/rpt_b200.h, rptb_engine).
bool use_wavefront(const rptb_scene* s, const rptb_render_params* p) {
    if (p->precision != RPTB_PRECISION_F32) return false;
    if (s->features & F_EXT) return false;  // kd-trees over shapes / MonomialSurface: megakernel only
    if (p->engine == RPTB_ENGINE_WAVEFRONT) return true;
    if (p->engine == RPTB_ENGINE_MEGAKERNEL) return false;
    // measured with the reference-shaped kd-trees: the megakernel wins while traversal is cheap (teapot:
    // 2 487 nodes), the wavefront wins once it dominates (dragon proxy: 823 k nodes).  Through the BVH a ray
    // costs ~25 node visits and ~3 triangle tests on either mesh and the megakernel wins on both.
    if (s->features & F_BVH) return false;
    return s->has_tree && s->tree_nodes >= 50000 && s->sampled_lights <= 8;
}

void read_stats(const DeviceCounters& c, rptb_stats* st) {
    st->segments = c.segments;
    st->rays = c.rays;
    st->node_visits = c.node_visits;
    st->tri_tests = c.tri_tests;
    st->mesh_hits = c.mesh_hits;
    st->env_lookups = c.env_lookups;
    st->object_tests = c.object_tests;
    st->bvh_node_visits = c.bvh_node_visits;
    st->bvh_tri_tests = c.bvh_tri_tests;
}

// Chunk-sum scratch of the megakernel: nchunks * ntiles_mine * 128 * 3 doubles.
template <class R>
int ensure_partial(rptb_scene* s, RenderArgs<R>& a) {
    if (a.nchunks <= 1) return RPTB_OK;
    const size_t need = (size_t)a.nchunks * a.ntiles_mine * 128u * 3u * sizeof(double);
    if (need > s->partial_bytes) {
        if (s->partial) cudaFreeAsync(s->partial, s->stream);
        s->partial = nullptr;
        s->partial_bytes = 0;
        CU(pool_alloc((void**)&s->partial, need, s->stream));
        CU(cudaStreamSynchronize(s->stream));
        s->partial_bytes = need;
    }
    a.partial = s->partial;
    return RPTB_OK;
}

// Launch the render on `stream` into a device buffer of the precision's type.  `compact`: see RenderArgs::compact.
int render_launch(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, float* out32, double* out64,
                  cudaStream_t stream, bool want_counters, bool compact, uint32_t* launches) {
    if (want_counters) CU(cudaMemsetAsync(s->counters, 0, sizeof(DeviceCounters), stream));
    if (p->precision == RPTB_PRECISION_F32) {
        RenderArgs<float> a;
        fill_args(cam, p, a);
        a.out = out32;
        a.compact = compact ? 1u : 0u;
        a.counters = want_counters ? s->counters : nullptr;
        if (use_wavefront(s, p)) {
            const uint32_t npix = a.ntiles_mine * 128u;
            const uint32_t G = wavefront_groups(npix, a.nchunks);
            const uint32_t npaths = npix * G;
            const uint32_t maxd = p->max_bounces > 0 ? p->max_bounces : 1;
            const size_t need = wavefront_bytes(npaths, s->sampled_lights, maxd);
            {
                const int rc = ensure_partial(s, a);
                if (rc != RPTB_OK) return rc;
            }
            if (need > s->wf_bytes) {
                if (s->wf_mem) cudaFreeAsync(s->wf_mem, s->stream);
                s->wf_mem = nullptr;
                s->wf_bytes = 0;
                CU(pool_alloc(&s->wf_mem, need, s->stream));
                CU(cudaStreamSynchronize(s->stream));  // the render may run on a caller's stream
                s->wf_bytes = need;
            }
            std::vector<char> bufs(wavefront_struct_size());
            wavefront_carve(s->wf_mem, npix, G, s->sampled_lights, maxd, (WfBuffers*)bufs.data());
            CU(run_wavefront_f32(s->view32, a, (const WfBuffers*)bufs.data(), p->collect_stats != 0, (s->features & F_BVH) != 0, stream, launches));
        } else {
            const int rc = ensure_partial(s, a);
            if (rc != RPTB_OK) return rc;
            a.ks = s->sampled_lights;
            // RPTB_VX=1 selects the vertex-at-once schedule (integrator_vx.cuh) where it has ray slots for the scene's lights.
            // Measured before the port to the H100: it lost to the slot schedule on every BASELINE config but glass, so the
            // slot schedule stays the default.  A counting pass over the reference-shaped kd-trees
            // (collect_stats = 2) is always the slot engine's.
            static const bool vx_on = getenv("RPTB_VX") != nullptr && std::strcmp(getenv("RPTB_VX"), "1") == 0;
            if (vx_on && vx_supported(a.ks) && p->collect_stats != 2) CU(launch_render_vx_f32(s->view32, a, (int)p->collect_stats, s->features, stream, launches));
            else CU(launch_render_f32(s->view32, a, (int)p->collect_stats, s->features, stream, launches));
        }
    } else {
        RenderArgs<double> a;
        fill_args(cam, p, a);
        a.out = out64;
        a.compact = compact ? 1u : 0u;
        a.counters = want_counters ? s->counters : nullptr;
        const int rc = ensure_partial(s, a);
        if (rc != RPTB_OK) return rc;
        CU(launch_render_f64(s->view64, a, (int)p->collect_stats, s->features, stream, launches));
    }
    return RPTB_OK;
}

int ensure_out(rptb_scene* s, size_t nvals) {
    if (s->out_vals >= nvals) return RPTB_OK;
    if (s->out32) cudaFreeAsync(s->out32, s->stream);
    if (s->out64) cudaFreeAsync(s->out64, s->stream);
    s->out32 = nullptr;
    s->out64 = nullptr;
    s->out_vals = 0;
    CU(pool_alloc((void**)&s->out32, nvals * sizeof(float), s->stream));
    CU(pool_alloc((void**)&s->out64, nvals * sizeof(double), s->stream));
    CU(cudaStreamSynchronize(s->stream));
    s->out_vals = nvals;
    return RPTB_OK;
}

int ensure_stage(rptb_scene* s, size_t bytes) {
    if (s->stage_bytes >= bytes) return RPTB_OK;
    stage_release(s->device, s->stage, s->stage_cached);
    s->stage = nullptr;
    s->stage_bytes = 0;
    CU(stage_acquire(s->device, bytes, &s->stage, &s->stage_bytes, &s->stage_cached));
    return RPTB_OK;
}

// One replica's share of Renderer::sample, straight into the caller's host image: render the pixel tiles t with
// t % shard_count == shard_index into a compact tile-major device buffer, copy exactly those pixels back
// through page-locked staging and scatter them into out_rgb (row-major doubles).  Pixels of other shards are not
// touched.  Runs on the library's own stream and returns when out_rgb holds this shard.
int render_shard_to_host(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, double* out_rgb, rptb_stats* stats) {
    std::lock_guard<std::mutex> lk(s->lock);
    DeviceGuard g(s->device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", s->device);
    int rc = wait_busy(s, s->stream);
    if (rc != RPTB_OK) return rc;
    const uint32_t sc = p->shard_count ? p->shard_count : 1u;
    const uint32_t tiles_x = (p->width + 15u) / 16u, tiles_y = (p->height + 7u) / 8u, ntiles = tiles_x * tiles_y;
    const uint32_t mine = ntiles > p->shard_index ? (ntiles - p->shard_index + sc - 1u) / sc : 0u;
    const size_t nvals = (size_t)mine * 128u * 3u;
    const bool f32 = p->precision == RPTB_PRECISION_F32;
    rc = ensure_out(s, nvals ? nvals : 1);
    if (rc != RPTB_OK) return rc;
    rc = ensure_stage(s, (nvals ? nvals : 1) * sizeof(double));
    if (rc != RPTB_OK) return rc;
    uint32_t launches = 0;
    CU(cudaEventRecord(s->ev0, s->stream));
    rc = render_launch(s, cam, p, s->out32, s->out64, s->stream, true, true, &launches);
    if (rc != RPTB_OK) return rc;
    CU(cudaEventRecord(s->ev1, s->stream));
    DeviceCounters c;
    CU(cudaMemcpyAsync(&c, s->counters, sizeof(c), cudaMemcpyDeviceToHost, s->stream));
    if (nvals) {
        if (f32) CU(cudaMemcpyAsync(s->stage, s->out32, nvals * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
        else CU(cudaMemcpyAsync(s->stage, s->out64, nvals * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    }
    CU(cudaStreamSynchronize(s->stream));
    s->busy_pending = false;
    const float* h32 = (const float*)s->stage;
    const double* h64 = (const double*)s->stage;
    const uint32_t W = p->width, H = p->height;
#pragma omp parallel for schedule(static) if (mine > 64)
    for (int64_t k = 0; k < (int64_t)mine; k++) {
        const uint32_t tile = p->shard_index + (uint32_t)k * sc;
        const uint32_t tx = tile % tiles_x, ty = tile / tiles_x;
        for (uint32_t j = 0; j < 128u; j++) {  // thread j of the CTA: warp (j >> 5) covers an 8 x 4 block of the 16 x 8 tile
            const uint32_t warp = j >> 5, lane = j & 31u;
            const uint32_t x = tx * 16u + (warp & 1u) * 8u + (lane & 7u), y = ty * 8u + (warp >> 1) * 4u + (lane >> 3);
            if (x >= W || y >= H) continue;
            const size_t src = ((size_t)k * 128u + j) * 3u;
            double* dst = out_rgb + 3 * ((size_t)y * W + x);
            if (f32) { dst[0] = (double)h32[src]; dst[1] = (double)h32[src + 1]; dst[2] = (double)h32[src + 2]; }
            else { dst[0] = h64[src]; dst[1] = h64[src + 1]; dst[2] = h64[src + 2]; }
        }
    }
    if (stats) {
        std::memset(stats, 0, sizeof(*stats));
        read_stats(c, stats);
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
        stats->gpu_ms = ms;
        stats->launches = launches;
        stats->engine = use_wavefront(s, p) ? RPTB_ENGINE_WAVEFRONT : RPTB_ENGINE_MEGAKERNEL;
    }
    return RPTB_OK;
}

void destroy_replica(rptb_scene* s) {
    DeviceGuard g(s->device);
    if (s->busy_pending && s->busy) cudaEventSynchronize(s->busy);  // a render may still run on a caller's stream
    if (s->stream) cudaStreamSynchronize(s->stream);
    s->arena.release();
    if (s->counters) cudaFreeAsync(s->counters, s->stream);
    if (s->wf_mem) cudaFreeAsync(s->wf_mem, s->stream);
    if (s->partial) cudaFreeAsync(s->partial, s->stream);
    stage_release(s->device, s->stage, s->stage_cached);
    if (s->out32) cudaFreeAsync(s->out32, s->stream);
    if (s->out64) cudaFreeAsync(s->out64, s->stream);
    if (s->stream) cudaStreamSynchronize(s->stream);
    if (s->ev0) cudaEventDestroy(s->ev0);
    if (s->ev1) cudaEventDestroy(s->ev1);
    if (s->busy) cudaEventDestroy(s->busy);
    if (s->stream) {
        cudaStreamDestroy(s->stream);
        pool_scene_gone(s->device);  // counted by scene_bind_device right before the stream was made
    }
    delete s;
}

}  // namespace

// ================================================================== C ABI ======
extern "C" {

const char* rptb_last_error(void) { return g_error.c_str(); }

int rptb_device_count(void) {
    int n = 0;
    const cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) return fail(RPTB_ERR_NO_DEVICE, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
    return n;
}

int rptb_scene_create_multi(const rptb_scene_desc* desc, const int* devices, int ndevices, rptb_scene** out) {
    if (!desc || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    if ((desc->nmaterials && !desc->materials) || (desc->nobjects && !desc->objects) || (desc->nlights && !desc->lights) ||
        (desc->nmeshes && !desc->meshes))
        return fail(RPTB_ERR_BAD_ARG, "null table with non-zero count");
    if (desc->ngroups && !desc->groups) return fail(RPTB_ERR_BAD_ARG, "null table with non-zero count");
    for (uint32_t i = 0; i < desc->nlights; i++)
        if (desc->lights[i].kind == RPTB_LIGHT_OBJECT && desc->lights[i].object.kind == RPTB_SHAPE_PLANE)
            return fail(RPTB_ERR_UNSUPPORTED, "light %u: a plane cannot be sampled (Plane::sample is unimplemented!() in the reference)", i);
    {
        std::string err;
        const int vrc = validate_scene(desc, err);
        if (vrc != RPTB_OK) return fail(vrc, "%s", err.c_str());
    }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(RPTB_ERR_NO_DEVICE, "no CUDA device");
    if (ndevices <= 0 || ndevices > 64) return fail(RPTB_ERR_BAD_ARG, "ndevices %d", ndevices);
    std::vector<int> devs(ndevices);
    for (int i = 0; i < ndevices; i++) {
        devs[i] = devices ? devices[i] : i;
        if (devs[i] < 0 || devs[i] >= ndev) return fail(RPTB_ERR_BAD_ARG, "device %d of %d", devs[i], ndev);
        for (int j = 0; j < i; j++)
            if (devs[j] == devs[i]) return fail(RPTB_ERR_BAD_ARG, "device %d listed twice", devs[i]);
    }
    std::vector<rptb_scene*> reps;
    int rc = RPTB_OK;
    try {
        HostScene hs;  // flattened once (kd-tree folding, BVH build), uploaded once per device
        rc = flatten_desc(desc, hs);
        for (int i = 0; rc == RPTB_OK && i < ndevices; i++) {
            DeviceGuard g(devs[i]);
            if (!g.ok) {
                rc = fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", devs[i]);
                break;
            }
            rptb_scene* s = new (std::nothrow) rptb_scene();
            if (!s) {
                rc = fail(RPTB_ERR_OOM, "host allocation failed");
                break;
            }
            s->device = devs[i];
            std::memset(&s->view32, 0, sizeof(s->view32));
            std::memset(&s->view64, 0, sizeof(s->view64));
            reps.push_back(s);
            rc = scene_bind_device(hs, s, i + 1 == ndevices);
            s->features = kernel_features(hs);
            s->has_tree = hs.has_tree;
            s->tree_nodes = hs.tree_nodes;
            s->sampled_lights = hs.sampled_lights;
            for (int k = 0; k < 3; k++) {
                s->wlo[k] = hs.wlo[k];
                s->whi[k] = hs.whi[k];
            }
        }
    } catch (const std::bad_alloc&) {
        rc = fail(RPTB_ERR_OOM, "host allocation failed while flattening the scene");
    }
    if (rc != RPTB_OK) {
        const std::string keep = g_error;
        for (rptb_scene* r : reps) destroy_replica(r);
        g_error = keep;
        return rc;
    }
    reps[0]->peers.assign(reps.begin() + 1, reps.end());
    *out = reps[0];
    return RPTB_OK;
}

int rptb_scene_create(const rptb_scene_desc* desc, int device, rptb_scene** out) {
    return rptb_scene_create_multi(desc, &device, 1, out);
}

void rptb_scene_destroy(rptb_scene* s) {
    if (!s) return;
    for (rptb_scene* r : s->peers) destroy_replica(r);
    destroy_replica(s);
}

uint64_t rptb_scene_device_bytes(const rptb_scene* s) { return s ? s->f32_bytes : 0; }

int rptb_scene_device_count(const rptb_scene* s) { return s ? 1 + (int)s->peers.size() : 0; }

int rptb_render_samples_device(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, float* out_dev,
                               void* stream_v, rptb_stats* stats) {
    int rc = check_params(s, cam, p);
    if (rc != RPTB_OK) return rc;
    if (!out_dev) return fail(RPTB_ERR_BAD_ARG, "null output");
    if (!s->peers.empty())
        return fail(RPTB_ERR_UNSUPPORTED, "a multi-device handle renders into host memory (rptb_render_samples); device-resident "
                                          "output is per device: create one handle per GPU and shard with shard_index / shard_count");
    std::lock_guard<std::mutex> lk(s->lock);
    DeviceGuard g(s->device);
    cudaStream_t stream = stream_v ? (cudaStream_t)stream_v : s->stream;
    rc = wait_busy(s, stream);
    if (rc != RPTB_OK) return rc;
    const bool compact = p->compact_out != 0;
    size_t nvals = (size_t)p->width * p->height * 3;
    if (compact) {
        const uint32_t sc = p->shard_count ? p->shard_count : 1u;
        const uint32_t ntiles = ((p->width + 15u) / 16u) * ((p->height + 7u) / 8u);
        nvals = (size_t)(ntiles > p->shard_index ? (ntiles - p->shard_index + sc - 1u) / sc : 0u) * 384u;
    }
    uint32_t launches = 0;
    if (stats) CU(cudaEventRecord(s->ev0, stream));
    if (p->precision == RPTB_PRECISION_F32) {
        rc = render_launch(s, cam, p, out_dev, nullptr, stream, stats != nullptr, compact, &launches);
        if (rc != RPTB_OK) return rc;
    } else {
        rc = ensure_out(s, nvals);
        if (rc != RPTB_OK) return rc;
        rc = render_launch(s, cam, p, nullptr, s->out64, stream, stats != nullptr, compact, &launches);
        if (rc != RPTB_OK) return rc;
        CU(launch_convert_f64_to_f32(s->out64, out_dev, nvals, stream));
        launches++;
    }
    if (stats) {
        CU(cudaEventRecord(s->ev1, stream));
        DeviceCounters c;
        CU(cudaMemcpyAsync(&c, s->counters, sizeof(c), cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
        s->busy_pending = false;
        std::memset(stats, 0, sizeof(*stats));
        read_stats(c, stats);
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, s->ev0, s->ev1));
        stats->gpu_ms = ms;
        stats->launches = launches;
        stats->engine = use_wavefront(s, p) ? RPTB_ENGINE_WAVEFRONT : RPTB_ENGINE_MEGAKERNEL;
    } else if (!stream_v) {
        CU(cudaStreamSynchronize(stream));
        s->busy_pending = false;
    } else {
        // still running on the caller's stream when we return: later calls order themselves behind this point
        CU(cudaEventRecord(s->busy, stream));
        s->busy_pending = true;
    }
    return RPTB_OK;
}

int rptb_render_samples(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, double* out_rgb,
                        rptb_stats* stats) {
    int rc = check_params(s, cam, p);
    if (rc != RPTB_OK) return rc;
    if (!out_rgb) return fail(RPTB_ERR_BAD_ARG, "null output");
    const uint32_t outer = p->shard_count ? p->shard_count : 1u;
    const uint32_t nrep = 1u + (uint32_t)s->peers.size();
    const size_t nvals = (size_t)p->width * p->height * 3;
    // pixels of the caller's OTHER shards read as zero (as rptb_render_samples_device leaves them)
    if (outer > 1) std::memset(out_rgb, 0, nvals * sizeof(double));
    if (nrep == 1) return render_shard_to_host(s, cam, p, out_rgb, stats);
    // Renderer::sample's fan-out (src/renderer.rs:117-129: rayon over rows) across the replicas: one host thread
    // per GPU, replica i renders the pixel tiles t with t % (outer * nrep) == shard_index * nrep + i and copies
    // exactly those pixels into out_rgb.  Every pixel has one owner and the RNG is keyed by pixel, so the image
    // is bit-identical for any number of devices; there is nothing to reduce, hence no collective.
    std::vector<int> rcs(nrep, RPTB_OK);
    std::vector<std::string> errs(nrep);
    std::vector<rptb_stats> sts(nrep);
    std::vector<std::thread> workers;
    for (uint32_t i = 0; i < nrep; i++) {
        workers.emplace_back([&, i]() {
            rptb_render_params q = *p;
            q.shard_count = outer * nrep;
            q.shard_index = p->shard_index * nrep + i;
            rptb_scene* rep = i == 0 ? s : s->peers[i - 1];
            rcs[i] = render_shard_to_host(rep, cam, &q, out_rgb, &sts[i]);
            if (rcs[i] != RPTB_OK) errs[i] = g_error;  // g_error is thread-local
        });
    }
    for (std::thread& t : workers) t.join();
    for (uint32_t i = 0; i < nrep; i++)
        if (rcs[i] != RPTB_OK) return fail(rcs[i], "device %d: %s", i == 0 ? s->device : s->peers[i - 1]->device, errs[i].c_str());
    if (stats) {
        std::memset(stats, 0, sizeof(*stats));
        for (uint32_t i = 0; i < nrep; i++) {
            stats->segments += sts[i].segments; stats->rays += sts[i].rays;
            stats->node_visits += sts[i].node_visits; stats->tri_tests += sts[i].tri_tests;
            stats->mesh_hits += sts[i].mesh_hits; stats->env_lookups += sts[i].env_lookups;
            stats->object_tests += sts[i].object_tests;
            stats->bvh_node_visits += sts[i].bvh_node_visits; stats->bvh_tri_tests += sts[i].bvh_tri_tests;
            stats->gpu_ms = std::max(stats->gpu_ms, sts[i].gpu_ms);  // the devices run concurrently
            stats->launches += sts[i].launches;
        }
        stats->engine = sts[0].engine;
    }
    return RPTB_OK;
}

int rptb_closest_hit(rptb_scene* s, const double* rays, uint64_t n, double t_min, uint32_t precision, double* out_t,
                     int32_t* out_object, double* out_normal, rptb_stats* stats) {
    if (!s || (n && (!rays || !out_t || !out_object))) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (precision > RPTB_PRECISION_F64) return fail(RPTB_ERR_BAD_ARG, "bad precision %u", precision);
    if (stats) std::memset(stats, 0, sizeof(*stats));
    if (n == 0) return RPTB_OK;
    std::lock_guard<std::mutex> lk(s->lock);
    DeviceGuard g(s->device);
    double *d_rays = nullptr, *d_t = nullptr, *d_n = nullptr;
    int32_t* d_obj = nullptr;
    auto cleanup = [&]() {
        cudaFree(d_rays);
        cudaFree(d_t);
        cudaFree(d_n);
        cudaFree(d_obj);
    };
#define CUC(call)                                                                                            \
    do {                                                                                                     \
        cudaError_t e_ = (call);                                                                             \
        if (e_ != cudaSuccess) {                                                                             \
            cleanup();                                                                                       \
            return fail(e_ == cudaErrorMemoryAllocation ? RPTB_ERR_OOM : RPTB_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
        }                                                                                                    \
    } while (0)
    CUC(cudaMalloc(&d_rays, n * 6 * sizeof(double)));
    CUC(cudaMalloc(&d_t, n * sizeof(double)));
    CUC(cudaMalloc(&d_obj, n * sizeof(int32_t)));
    if (out_normal) CUC(cudaMalloc(&d_n, n * 3 * sizeof(double)));
    CUC(cudaMemcpyAsync(d_rays, rays, n * 6 * sizeof(double), cudaMemcpyHostToDevice, s->stream));
    CUC(cudaMemsetAsync(s->counters, 0, sizeof(DeviceCounters), s->stream));
    CUC(cudaEventRecord(s->ev0, s->stream));
    if (precision == RPTB_PRECISION_F32)
        CUC(launch_closest_hit_f32(s->view32, d_rays, n, t_min, d_t, d_obj, d_n, stats ? s->counters : nullptr, stats ? 1 : 0, s->features, s->stream));
    else
        CUC(launch_closest_hit_f64(s->view64, d_rays, n, t_min, d_t, d_obj, d_n, stats ? s->counters : nullptr, stats ? 1 : 0, s->features, s->stream));
    CUC(cudaEventRecord(s->ev1, s->stream));
    CUC(cudaMemcpyAsync(out_t, d_t, n * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    CUC(cudaMemcpyAsync(out_object, d_obj, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s->stream));
    if (out_normal) CUC(cudaMemcpyAsync(out_normal, d_n, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    DeviceCounters c;
    CUC(cudaMemcpyAsync(&c, s->counters, sizeof(c), cudaMemcpyDeviceToHost, s->stream));
    CUC(cudaStreamSynchronize(s->stream));
    if (stats) {
        read_stats(c, stats);
        float ms = 0;
        cudaEventElapsedTime(&ms, s->ev0, s->ev1);
        stats->gpu_ms = ms;
        stats->launches = 1;
    }
    cleanup();
    return RPTB_OK;
}

int64_t rptb_tile_pixel(uint32_t width, uint32_t height, uint32_t shard_index, uint32_t shard_count, uint32_t k, uint32_t j) {
    const uint32_t sc = shard_count ? shard_count : 1u;
    const uint32_t tiles_x = (width + 15u) / 16u, tiles_y = (height + 7u) / 8u;
    const uint64_t tile = (uint64_t)shard_index + (uint64_t)k * sc;
    if (width == 0 || height == 0 || j >= 128u || shard_index >= sc || tile >= (uint64_t)tiles_x * tiles_y) return -1;
    const uint32_t tx = (uint32_t)(tile % tiles_x), ty = (uint32_t)(tile / tiles_x);
    const uint32_t warp = j >> 5, lane = j & 31u;
    const uint32_t x = tx * 16u + (warp & 1u) * 8u + (lane & 7u), y = ty * 8u + (warp >> 1) * 4u + (lane >> 3);
    if (x >= width || y >= height) return -1;
    return (int64_t)y * width + x;
}

int rptb_illuminate(rptb_scene* s, uint32_t light, const double* pos, uint64_t n, uint64_t seed, uint32_t precision,
                    double* out_intensity, double* out_wi, double* out_dist) {
    if (!s || (n && (!pos || !out_intensity || !out_wi || !out_dist))) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (precision > RPTB_PRECISION_F64) return fail(RPTB_ERR_BAD_ARG, "bad precision %u", precision);
    if (light >= s->view32.nlights) return fail(RPTB_ERR_BAD_ARG, "light %u of %u", light, s->view32.nlights);
    if (n == 0) return RPTB_OK;
    std::lock_guard<std::mutex> lk(s->lock);
    DeviceGuard g(s->device);
    double *d_pos = nullptr, *d_i = nullptr, *d_wi = nullptr, *d_dist = nullptr;
    auto cleanup = [&]() {
        cudaFree(d_pos);
        cudaFree(d_i);
        cudaFree(d_wi);
        cudaFree(d_dist);
    };
    CUC(cudaMalloc(&d_pos, n * 3 * sizeof(double)));
    CUC(cudaMalloc(&d_i, n * 3 * sizeof(double)));
    CUC(cudaMalloc(&d_wi, n * 3 * sizeof(double)));
    CUC(cudaMalloc(&d_dist, n * sizeof(double)));
    CUC(cudaMemcpyAsync(d_pos, pos, n * 3 * sizeof(double), cudaMemcpyHostToDevice, s->stream));
    if (precision == RPTB_PRECISION_F32) CUC(launch_illuminate_f32(s->view32, light, d_pos, n, seed, d_i, d_wi, d_dist, s->stream));
    else CUC(launch_illuminate_f64(s->view64, light, d_pos, n, seed, d_i, d_wi, d_dist, s->stream));
    CUC(cudaMemcpyAsync(out_intensity, d_i, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    CUC(cudaMemcpyAsync(out_wi, d_wi, n * 3 * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    CUC(cudaMemcpyAsync(out_dist, d_dist, n * sizeof(double), cudaMemcpyDeviceToHost, s->stream));
    CUC(cudaStreamSynchronize(s->stream));
    cleanup();
    return RPTB_OK;
}

static int point_eval(const rptb_material* m, const double* dirs, uint64_t n, uint32_t in_stride, uint64_t seed,
                      uint32_t precision, int device, double* out_a, uint32_t a_stride, double* out_b, bool sample) {
    if (!m || (n && (!dirs || !out_a))) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (precision > RPTB_PRECISION_F64) return fail(RPTB_ERR_BAD_ARG, "bad precision %u", precision);
    if (n == 0) return RPTB_OK;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(RPTB_ERR_NO_DEVICE, "no CUDA device");
    if (device < 0 || device >= ndev) return fail(RPTB_ERR_BAD_ARG, "device %d of %d", device, ndev);
    DeviceGuard g(device);
    double *d_in = nullptr, *d_a = nullptr, *d_b = nullptr;
    auto cleanup = [&]() {
        cudaFree(d_in);
        cudaFree(d_a);
        cudaFree(d_b);
    };
    CUC(cudaMalloc(&d_in, n * in_stride * sizeof(double)));
    CUC(cudaMalloc(&d_a, n * a_stride * sizeof(double)));
    if (sample) CUC(cudaMalloc(&d_b, n * sizeof(double)));
    CUC(cudaMemcpy(d_in, dirs, n * in_stride * sizeof(double), cudaMemcpyHostToDevice));
    if (precision == RPTB_PRECISION_F32) {
        MaterialRec<float> r;
        fill_material(*m, r);
        if (sample) CUC(launch_sample_f_f32(r, d_in, n, seed, d_a, d_b, 0));
        else CUC(launch_bsdf_f32(r, d_in, n, d_a, 0));
    } else {
        MaterialRec<double> r;
        fill_material(*m, r);
        if (sample) CUC(launch_sample_f_f64(r, d_in, n, seed, d_a, d_b, 0));
        else CUC(launch_bsdf_f64(r, d_in, n, d_a, 0));
    }
    CUC(cudaMemcpy(out_a, d_a, n * a_stride * sizeof(double), cudaMemcpyDeviceToHost));
    if (sample) CUC(cudaMemcpy(out_b, d_b, n * sizeof(double), cudaMemcpyDeviceToHost));
    cleanup();
    return RPTB_OK;
}

int rptb_bsdf_eval(const rptb_material* m, const double* dirs, uint64_t n, uint32_t precision, int device, double* out) {
    return point_eval(m, dirs, n, 9, 0, precision, device, out, 3, nullptr, false);
}

int rptb_sample_f(const rptb_material* m, const double* dirs, uint64_t n, uint64_t seed, uint32_t precision, int device,
                  double* out_wi, double* out_pdf) {
    if (n && !out_pdf) return fail(RPTB_ERR_BAD_ARG, "null argument");
    return point_eval(m, dirs, n, 6, seed, precision, device, out_wi, 3, out_pdf, true);
}

static int build_kdtree_common(const double* data, uint64_t n, bool boxes, rptb_kdtree_out* out) {
    if (!out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    std::memset(out, 0, sizeof(*out));
    if (n == 0 || !data) return fail(RPTB_ERR_BAD_ARG, boxes ? "no boxes" : "no triangles");
    if (n >= (1ull << 31)) return fail(RPTB_ERR_UNSUPPORTED, "too many objects for one kd-tree");
    try {
        std::vector<rptb_kdnode> nodes;
        std::vector<uint32_t> refs;
        uint32_t depth = 0, max_leaf = 0;
        if (boxes) build_kdtree_boxes_host(data, n, nodes, refs, depth, max_leaf);
        else build_kdtree_host(data, n, nodes, refs, depth, max_leaf);
        out->nodes = (rptb_kdnode*)std::malloc(sizeof(rptb_kdnode) * nodes.size());
        out->refs = (uint32_t*)std::malloc(sizeof(uint32_t) * std::max<size_t>(refs.size(), 1));
        if (!out->nodes || !out->refs) {
            std::free(out->nodes);
            std::free(out->refs);
            std::memset(out, 0, sizeof(*out));
            return fail(RPTB_ERR_OOM, "host allocation failed");
        }
        std::memcpy(out->nodes, nodes.data(), sizeof(rptb_kdnode) * nodes.size());
        std::memcpy(out->refs, refs.data(), sizeof(uint32_t) * refs.size());
        out->nnodes = nodes.size();
        out->nrefs = refs.size();
        out->depth = depth;
        out->max_leaf = max_leaf;
    } catch (const std::bad_alloc&) {
        return fail(RPTB_ERR_OOM, "host allocation failed");
    }
    return RPTB_OK;
}

int rptb_build_kdtree(const double* tris, uint64_t ntris, rptb_kdtree_out* out) {
    return build_kdtree_common(tris, ntris, false, out);
}

int rptb_build_kdtree_boxes(const double* boxes, uint64_t nboxes, rptb_kdtree_out* out) {
    return build_kdtree_common(boxes, nboxes, true, out);
}

void rptb_free_kdtree(rptb_kdtree_out* out) {
    if (!out) return;
    std::free(out->nodes);
    std::free(out->refs);
    std::memset(out, 0, sizeof(*out));
}

int rptb_parse_obj(const char* text, uint64_t len, double** out_tris, uint64_t* out_ntris) {
    if (!text || !out_tris || !out_ntris) return fail(RPTB_ERR_BAD_ARG, "null argument");
    *out_tris = nullptr;
    *out_ntris = 0;
    try {
        std::vector<double> tris;
        std::string err;
        if (parse_obj_text(text, (size_t)len, tris, err) != 0) return fail(RPTB_ERR_BAD_ARG, "%s", err.c_str());
        const size_t n = tris.size();
        double* p = (double*)std::malloc(sizeof(double) * (n ? n : 1));
        if (!p) return fail(RPTB_ERR_OOM, "host allocation failed");
        std::memcpy(p, tris.data(), sizeof(double) * n);
        *out_tris = p;
        *out_ntris = n / 18;
    } catch (const std::bad_alloc&) {
        return fail(RPTB_ERR_OOM, "host allocation failed");
    }
    return RPTB_OK;
}

void rptb_free_triangles(double* tris) { std::free(tris); }

// Copies a triangle vector into a malloc'd block the caller frees with rptb_free_triangles.
static double* export_triangles(const std::vector<double>& tris) {
    const size_t n = tris.size();
    double* p = (double*)std::malloc(sizeof(double) * (n ? n : 1));
    if (p && n) std::memcpy(p, tris.data(), sizeof(double) * n);
    return p;
}

int rptb_parse_obj_mtl(const char* obj_text, uint64_t obj_len, const char* mtl_text, uint64_t mtl_len,
                       rptb_obj_groups_out* out) {
    if (!obj_text || !mtl_text || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    std::memset(out, 0, sizeof(*out));
    try {
        std::vector<double> tris;
        std::vector<ObjGroup> groups;
        std::string err;
        if (parse_obj_mtl_text(obj_text, (size_t)obj_len, mtl_text, (size_t)mtl_len, tris, groups, err) != 0)
            return fail(RPTB_ERR_BAD_ARG, "%s", err.c_str());
        double* t = export_triangles(tris);
        rptb_obj_group* g = (rptb_obj_group*)std::malloc(sizeof(rptb_obj_group) * (groups.empty() ? 1 : groups.size()));
        if (!t || !g) {
            std::free(t);
            std::free(g);
            return fail(RPTB_ERR_OOM, "host allocation failed");
        }
        for (size_t i = 0; i < groups.size(); i++) {
            g[i].material = groups[i].material;
            g[i].first_tri = groups[i].first_tri;
            g[i].ntris = groups[i].ntris;
        }
        out->tris = t;
        out->ntris = tris.size() / 18;
        out->groups = g;
        out->ngroups = groups.size();
    } catch (const std::bad_alloc&) {
        return fail(RPTB_ERR_OOM, "host allocation failed");
    }
    return RPTB_OK;
}

void rptb_free_obj_groups(rptb_obj_groups_out* out) {
    if (!out) return;
    std::free(out->tris);
    std::free(out->groups);
    std::memset(out, 0, sizeof(*out));
}

int rptb_parse_stl(const void* data, uint64_t len, double** out_tris, uint64_t* out_ntris) {
    if (!data || !out_tris || !out_ntris) return fail(RPTB_ERR_BAD_ARG, "null argument");
    *out_tris = nullptr;
    *out_ntris = 0;
    try {
        std::vector<double> tris;
        std::string err;
        if (parse_stl_bytes(data, (size_t)len, tris, err) != 0) return fail(RPTB_ERR_BAD_ARG, "%s", err.c_str());
        double* p = export_triangles(tris);
        if (!p) return fail(RPTB_ERR_OOM, "host allocation failed");
        *out_tris = p;
        *out_ntris = tris.size() / 18;
    } catch (const std::bad_alloc&) {
        return fail(RPTB_ERR_OOM, "host allocation failed");
    }
    return RPTB_OK;
}

int rptb_film_variance(const double* batches, uint32_t nbatches, uint64_t npixels, int device, double* out) {
    if (!batches || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (nbatches < 2) return fail(RPTB_ERR_BAD_ARG, "variance needs at least two entries per pixel");
    if (npixels == 0) return fail(RPTB_ERR_BAD_ARG, "empty image");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(RPTB_ERR_NO_DEVICE, "no CUDA device");
    if (device < 0 || device >= ndev) return fail(RPTB_ERR_BAD_ARG, "device %d of %d", device, ndev);
    DeviceGuard g(device);
    const size_t n = (size_t)nbatches * npixels * 3;
    double *d_in = nullptr, *d_out = nullptr;
    auto cleanup = [&]() {
        cudaFree(d_in);
        cudaFree(d_out);
    };
    CUC(cudaMalloc(&d_in, n * sizeof(double)));
    CUC(cudaMalloc(&d_out, sizeof(double)));
    CUC(cudaMemcpy(d_in, batches, n * sizeof(double), cudaMemcpyHostToDevice));
    CUC(cudaMemset(d_out, 0, sizeof(double)));
    CUC(launch_film_variance(d_in, nbatches, npixels, d_out, 0));
    double sum = 0.0;
    CUC(cudaMemcpy(&sum, d_out, sizeof(double), cudaMemcpyDeviceToHost));
    cleanup();
    *out = sum / (double)npixels;
    return RPTB_OK;
}

int rptb_film_resolve(const double* sums, uint32_t nbatches, uint32_t width, uint32_t height, uint32_t box_radius,
                      int device, uint8_t* out_rgb8) {
    if (!sums || !out_rgb8) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (nbatches == 0) return fail(RPTB_ERR_BAD_ARG, "Pixel found with no samples");  // buffer.rs:89
    if (width == 0 || height == 0) return fail(RPTB_ERR_BAD_ARG, "empty image");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(RPTB_ERR_NO_DEVICE, "no CUDA device");
    if (device < 0 || device >= ndev) return fail(RPTB_ERR_BAD_ARG, "device %d of %d", device, ndev);
    DeviceGuard g(device);
    const size_t nvals = (size_t)width * height * 3;
    double* d_in = nullptr;
    uint8_t* d_out = nullptr;
    auto cleanup = [&]() {
        cudaFree(d_in);
        cudaFree(d_out);
    };
    CUC(cudaMalloc(&d_in, nvals * sizeof(double)));
    CUC(cudaMalloc(&d_out, nvals));
    CUC(cudaMemcpy(d_in, sums, nvals * sizeof(double), cudaMemcpyHostToDevice));
    CUC(launch_film_resolve(d_in, nbatches, width, height, box_radius, d_out, 0));
    CUC(cudaMemcpy(out_rgb8, d_out, nvals, cudaMemcpyDeviceToHost));
    cleanup();
    return RPTB_OK;
}

}  // extern "C"
