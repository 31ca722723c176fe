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

#include <algorithm>
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
#include "delta.h"
#include "denoise.h"
#include "flatten.h"
#include "launch.h"
#include "planes.h"
#include "reproject.h"
#include "tile.h"

namespace rptb {
cudaError_t launch_film_resolve(const double* sums, uint32_t nbatches, uint32_t width, uint32_t height,
                                uint32_t radius, uint8_t* out, cudaStream_t stream);
cudaError_t launch_convert_f64_to_f32(const double* in, float* out, size_t n, cudaStream_t stream);
cudaError_t launch_film_variance(const double* batches, uint32_t nbatches, uint64_t npixels, double* out_sum, cudaStream_t stream);
// the device Buffer: film.cu
cudaError_t launch_buffer_accumulate(const float* in32, const double* in64, bool rowmajor, const uint8_t* mask, uint64_t nelem,
                                     uint32_t width, uint32_t height, uint32_t shard_index, uint32_t shard_count, double* sums,
                                     double* m2, uint32_t* counts, double* half, cudaStream_t stream);
cudaError_t launch_buffer_half_scatter(const double* src, double* dst, uint64_t nelem, uint32_t width, uint32_t height, uint32_t shard_index,
                                       uint32_t shard_count, cudaStream_t stream);
cudaError_t launch_buffer_move(bool compact, const PlaneSet& src, const PlaneSet& dst, uint64_t nelem, uint32_t width, uint32_t height,
                               uint32_t shard_index, uint32_t shard_count, cudaStream_t stream);
uint32_t buffer_variance_blocks(uint64_t npixels);
cudaError_t launch_buffer_variance_sum(const double* m2, const uint32_t* counts, uint64_t npixels, double* partial,
                                       double* out_sum, cudaStream_t stream);
cudaError_t launch_film_resolve_counted(const double* sums, const uint32_t* counts, uint32_t width, uint32_t height,
                                        uint32_t radius, uint8_t* out, cudaStream_t stream);
// the active pixels and warp blocks of an adaptive call: adaptive.cu
size_t adaptive_temp_bytes(uint32_t tiles);
cudaError_t launch_adaptive_select(const double* sums, const double* m2, const uint32_t* counts, uint32_t tiles, uint32_t width,
                                   uint32_t height, uint32_t shard_index, uint32_t shard_count, const rptb_adaptive& crit,
                                   uint8_t* mask, uint8_t* flags, uint32_t* ids, uint32_t* len, unsigned long long* active_pixels,
                                   void* temp, size_t temp_bytes, cudaStream_t stream);
cudaError_t launch_adaptive_list(const uint8_t* flags, uint32_t tiles, uint32_t* ids, uint32_t* len, void* temp, size_t temp_bytes,
                                 cudaStream_t stream);
// the mask of a guided adaptive call: guided.cu
cudaError_t launch_guided_mark(const double* col, const double* var, const double* albedo, const uint32_t* counts, uint32_t width,
                               uint32_t height, uint32_t index, uint32_t count, uint32_t tiles, double eps_a, const rptb_adaptive& crit,
                               uint8_t* mask, uint8_t* flags, unsigned long long* active_pixels, cudaStream_t stream);
// the delta exchange of a shard buffer: delta.cu
size_t delta_temp_bytes(uint64_t nelem);
cudaError_t launch_delta_export(const uint8_t* mask, uint64_t nelem, const double* sums, const double* m2, const uint32_t* counts,
                                void* block, uint32_t capacity, uint32_t pixels, uint32_t* selected, void* temp, size_t temp_bytes,
                                cudaStream_t stream);
cudaError_t launch_delta_import(const void* blocks, uint32_t shard_count, uint32_t capacity, double* sums, double* m2, uint32_t* counts,
                                cudaStream_t stream);
// the feature planes and the denoiser: denoise.cu
cudaError_t launch_features_resolve(const FeaturePlanes& f, uint64_t npix, double rays, const Aov& out, cudaStream_t stream);
cudaError_t launch_denoise(const double* sums, const double* m2, const uint32_t* counts, const double* nrm,
                           const double* depth, const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d,
                           double* const col[2], double* const var[2], double* out, cudaStream_t stream, uint32_t* launches);
cudaError_t launch_denoise_passes(const double* sums, const double* m2, const uint32_t* counts, const double* nrm, const double* depth,
                                  const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d, double* const col[2],
                                  double* const var[2], const double** out_col, const double** out_var, cudaStream_t stream,
                                  uint32_t* launches);
// the error estimate from two half buffers: halves.cu
cudaError_t launch_halves_error(const double* sums, const double* m2, const double* half, const uint32_t* counts, const double* nrm,
                                const double* depth, const double* albedo, uint32_t width, uint32_t height, const rptb_denoise& d,
                                double* const col[2], double* const var[2], double* const u[2], double* E, const double** out_col,
                                cudaStream_t stream, uint32_t* launches);
// the reprojection and the least count: reproject.cu
cudaError_t launch_reproject_part(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s, const FeaturePlanes& f,
                                  double rays, uint32_t index, uint32_t count, uint64_t nelem, const rptb_reproject& prm, double* sums,
                                  double* m2, uint32_t* counts, unsigned long long* reused, cudaStream_t stream);
cudaError_t launch_reproject_merge_part(const ReprojectView& dv, const ReprojectView& sv, const ReprojectSource& s,
                                        const FeaturePlanes& f, double rays, uint32_t index, uint32_t count, uint64_t nelem,
                                        const rptb_reproject& prm, double gamma, double* sums, double* m2, uint32_t* counts,
                                        unsigned long long* tally, cudaStream_t stream);
cudaError_t launch_buffer_min_count(const uint32_t* counts, uint64_t npix, uint32_t* out, cudaStream_t stream);
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

// Replica i of a scene: the handle itself, then its peers.
rptb_scene* replica(rptb_scene* s, uint32_t i) { return i == 0 ? s : s->peers[i - 1]; }

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

// ---- the device-resident Buffer (src/buffer.rs:6-93) ------------------------------------------------------------
// One part per replica of the scene it was created on, each holding that replica's own 16x8 tiles in the compact
// tile-major layout (film.cu): 3 running sums and one Welford M2 per pixel, in double, and its entry count.  The buffer owns its memory
// (cudaMalloc, so destroy hands it back to the driver), its streams and its events, so it and its scene may be
// destroyed in either order.  `done` is recorded behind every accumulate -- on the scene's stream (rptb_sample_into)
// or on the part's own (rptb_buffer_add_samples) -- and every later operation on the part waits for it.

// One copy of a buffer's per-pixel planes (planes.h), n elements a plane.  Each group is null until allocated: the
// colour planes, one allocation each, the feature sums, one allocation of FEATURE_SUMS doubles an element, and the HALF
// plane of a buffer with halves (not in a PlaneSet: it moves by its own kernel).
struct Planes {
    size_t n = 0;
    double* sums = nullptr;
    double* m2 = nullptr;
    uint32_t* counts = nullptr;
    double* feat = nullptr;
    double* half = nullptr;
    // the allocated planes of `mask`
    PlaneSet set(uint32_t mask) const {
        const FeaturePlanes f = feat ? feature_planes(feat, n) : FeaturePlanes{};
        PlaneSet s = {{sums, m2, f.n, f.a, f.h, f.z, counts}};
        for (int k = 0; k < NPLANES; k++)
            if (!(mask >> k & 1u)) s.p[k] = nullptr;
        return s;
    }
};

struct BufferPart {
    int device = 0;
    // this part's place in the tile deal: it holds the tiles t with t % count == index.  Part i of a whole buffer of n
    // parts is (i, n); the one part of a shard buffer (rptb_buffer_create_shard) is the shard's own pair.
    uint32_t index = 0, count = 1;
    uint32_t tiles = 0;          // tiles t with t % count == index
    // tiles * 128 elements: the colour planes from creation on, the feature sums from the buffer's first
    // rptb_buffer_add_features on
    Planes planes;
    double* upload = nullptr;    // a host entry, row-major width*height*3 (first add_samples allocates it)
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    // from the buffer's first adaptive call on, that call's scratch: the pixel mask (tiles*128), the flag and the id
    // list of the active 8x4 warp blocks (tiles*4), the list's length, the number of active pixels, and the select's
    // temporary storage
    uint8_t* mask = nullptr;
    uint8_t* flags = nullptr;
    uint32_t* ids = nullptr;
    uint32_t* len = nullptr;
    unsigned long long* active = nullptr;
    void* temp = nullptr;
    size_t temp_bytes = 0;
    // from a shard's first rptb_buffer_export_delta on: the select's count of listed slots and its temporary storage
    uint32_t* delta_len = nullptr;
    void* delta_temp = nullptr;
    size_t delta_temp_bytes = 0;
    std::vector<void*> mem;      // everything above that cudaMalloc gave, on the part's device
};

// The camera one side of a buffer (its entries or its features) was made with, for rptb_buffer_reproject: none yet, one
// camera (bitwise), several, or unknown (a host entry).
struct CameraRecord {
    enum State { NONE, ONE, MIXED, UNKNOWN } state = NONE;
    rptb_camera cam;
    void note(const rptb_camera& c) {
        if (state == NONE) {
            state = ONE;
            cam = c;
        } else if (state == ONE && std::memcmp(&cam, &c, sizeof(c)) != 0) {
            state = MIXED;
        }
    }
};

struct rptb_buffer {
    uint32_t width = 0, height = 0, radius = 0;
    // accumulate calls.  No pixel holds more entries, and -- unless the buffer was reprojected -- every pixel holds at
    // least min(entries, 2): see rptb_buffer_denoise
    uint32_t entries = 0;
    // rptb_buffer_reproject wrote its entries: pixels may hold 0 or 1 entries, and image / variance / denoise look at the
    // least count on the device.  `entries` is then max_history plus the calls since, a bound.
    bool reprojected = false;
    // rptb_buffer_create_shard: the buffer holds one shard of the image (parts[0]'s index and count), and its whole-image
    // reads are refused until the shards are gathered into a whole buffer (rptb_buffer_import_shards)
    bool shard = false;
    // rptb_buffer_create_halves: every part holds the HALF plane, and every accumulate adds a pixel's odd entries to it
    bool halves = false;
    CameraRecord entry_cam, feat_cam;
    // The delta exchange (rptb_buffer_export_delta, rptb_buffer_import_deltas) checks against `state`, which every call
    // that changes the buffer bumps: an entry, a feature pass, a host entry, a reprojection or merge, an import.
    // exported: a shard's state at its last export (full or delta).  masked: a shard's state right after its last
    // adaptive or guided call, whose mask (parts[0].mask) is then exactly the pixels that call changed.  imported /
    // imported_shards: a whole buffer's state right after an import (full or delta), and of how many shards.
    uint64_t state = 0, exported = UINT64_MAX, masked = UINT64_MAX, imported = UINT64_MAX;
    uint32_t imported_shards = 0;
    std::vector<BufferPart> parts;
    // on parts[0]'s device, each group allocated by its first gather: the image's planes row-major (width*height
    // elements), and the staging another part's planes are copied into (as many elements as the largest such part)
    Planes rows, staging;
    // with the colour rows: the variance block partials, then the total; the image
    double* partial = nullptr;
    uint8_t* rgb8 = nullptr;
    uint64_t feature_rays = 0;       // camera rays per pixel in the feature sums
    double* aov = nullptr;           // with the feature rows, width*height*8: the resolved features (buffer_aov)
    double* dn = nullptr;            // the denoiser's, width*height*11: colour (3) and variance ping-pong planes, then c' (3)
    double* hv = nullptr;            // the error estimate's (halves.cu), width*height*7: u (3) ping-pong planes, then E
    // allocated by the first guided adaptive call on a buffer of several parts: the mask and flags of parts[1..] (as many
    // tiles as the largest holds, *132 bytes) marked here before they go to the part, and their active pixel count
    uint8_t* guide_mask = nullptr;
    unsigned long long* guide_active = nullptr;
    // allocated by the first reprojection into the buffer: the reused-pixel counter and the least count
    unsigned long long* reused = nullptr;
    uint32_t* min_count = nullptr;
    std::vector<void*> mem;          // everything above that cudaMalloc gave, on parts[0]'s device
    std::mutex lock;
};

namespace {

uint32_t buffer_tiles(uint32_t width, uint32_t height, uint32_t index, uint32_t nparts) {
    const uint32_t ntiles = ((width + 15u) / 16u) * ((height + 7u) / 8u);
    return ntiles > index ? (ntiles - index + nparts - 1u) / nparts : 0u;
}

size_t plane_bytes(int k, size_t n) { return n * plane_shape(k).values * plane_shape(k).bytes; }

// cudaMalloc on the current device, recorded in `mem` for buffer_free.
template <class T>
cudaError_t own(std::vector<void*>& mem, T** p, size_t bytes) {
    const cudaError_t e = cudaMalloc((void**)p, bytes);
    if (e == cudaSuccess) mem.push_back(*p);
    return e;
}

void buffer_free(rptb_buffer* b) {
    for (size_t i = 0; i < b->parts.size(); i++) {
        BufferPart& q = b->parts[i];
        DeviceGuard g(q.device);
        if (q.done) cudaEventSynchronize(q.done);  // an accumulate may still run on the scene's stream
        if (q.stream) cudaStreamSynchronize(q.stream);
        for (void* p : q.mem) cudaFree(p);
        if (i == 0)
            for (void* p : b->mem) cudaFree(p);
        if (q.done) cudaEventDestroy(q.done);
        if (q.stream) cudaStreamDestroy(q.stream);
    }
    delete b;
}

// Allocates the groups of `mask` that `s` does not hold yet, n elements a plane, on the current device.
int planes_alloc(std::vector<void*>& mem, Planes& s, size_t n, uint32_t mask) {
    s.n = n;
    if ((mask & COLOUR) && !s.sums) {
        CU(own(mem, &s.sums, plane_bytes(SUMS, n)));
        CU(own(mem, &s.m2, plane_bytes(M2, n)));
        CU(own(mem, &s.counts, plane_bytes(COUNTS, n)));
    }
    if ((mask & FEATURES) && !s.feat) CU(own(mem, &s.feat, n * FEATURE_SUMS * sizeof(double)));
    if ((mask >> HALF & 1u) && !s.half) CU(own(mem, &s.half, plane_bytes(HALF, n)));
    return RPTB_OK;
}

// halves: the part also holds the HALF plane (rptb_buffer_create_halves).
int buffer_part_alloc(BufferPart& q, bool halves) {
    CU(cudaStreamCreateWithFlags(&q.stream, cudaStreamNonBlocking));
    CU(cudaEventCreateWithFlags(&q.done, cudaEventDisableTiming));
    if (q.tiles) {
        const int rc = planes_alloc(q.mem, q.planes, (size_t)q.tiles * 128u, COLOUR | (halves ? 1u << HALF : 0u));
        if (rc != RPTB_OK) return rc;
        const PlaneSet s = q.planes.set(COLOUR);  // sums() of an empty buffer reads zero
        for (int k = 0; k < NPLANES; k++)
            if (s.p[k]) CU(cudaMemsetAsync(s.p[k], 0, plane_bytes(k, q.planes.n), q.stream));
        if (halves) CU(cudaMemsetAsync(q.planes.half, 0, plane_bytes(HALF, q.planes.n), q.stream));
    }
    CU(cudaEventRecord(q.done, q.stream));
    return RPTB_OK;
}

// The row-major planes of `mask` on parts[0]'s device (its device current), each group allocated on first use together
// with its staging (when the buffer has other parts) and its other scratch.
int buffer_rows_alloc(rptb_buffer* b, uint32_t mask) {
    const size_t npix = (size_t)b->width * b->height;
    size_t most = 0;
    for (size_t i = 1; i < b->parts.size(); i++) most = std::max(most, (size_t)b->parts[i].tiles * 128u);
    if ((mask & COLOUR) && !b->rows.sums) {
        CU(own(b->mem, &b->partial, (buffer_variance_blocks(npix) + 1) * sizeof(double)));
        CU(own(b->mem, &b->rgb8, npix * 3));
    }
    if ((mask & FEATURES) && !b->rows.feat) CU(own(b->mem, &b->aov, npix * FEATURE_SUMS * sizeof(double)));
    const int rc = planes_alloc(b->mem, b->rows, npix, mask);
    if (rc != RPTB_OK || !most) return rc;
    return planes_alloc(b->mem, b->staging, most, mask);
}

// b->aov's planes
Aov buffer_aov(const rptb_buffer* b) {
    const size_t npix = (size_t)b->width * b->height;
    return {b->aov, b->aov + 3 * npix, b->aov + 6 * npix, b->aov + 7 * npix};
}

// Copies n elements of every plane present in both sets from device `from` to device `to`, on `stream`: between a part
// on another device and the staging on parts[0]'s.  cudaMemcpyPeerAsync needs no peer access.
int copy_planes(const PlaneSet& dst, int to, const PlaneSet& src, int from, size_t n, cudaStream_t stream) {
    for (int k = 0; k < NPLANES; k++)
        if (dst.p[k] && src.p[k]) CU(cudaMemcpyPeerAsync(dst.p[k], to, src.p[k], from, plane_bytes(k, n), stream));
    return RPTB_OK;
}

// Scatters the compact planes `src` of shard `index` of `count` (one part of b, or one block of
// rptb_buffer_import_shards) into b's row-major planes of `mask`, on parts[0]'s stream.
int buffer_scatter(rptb_buffer* b, const PlaneSet& src, uint32_t mask, uint32_t index, uint32_t count) {
    const uint64_t nelem = (uint64_t)buffer_tiles(b->width, b->height, index, count) * 128u;
    CU(launch_buffer_move(false, src, b->rows.set(mask), nelem, b->width, b->height, index, count, b->parts[0].stream));
    return RPTB_OK;
}

// Brings the planes of `mask` from every part to parts[0]'s device in row-major order, on parts[0]'s stream (the caller
// has made that device current): part 0 straight from its own planes, the others through the staging.  HALF in `mask`:
// a buffer with halves only.
int buffer_gather(rptb_buffer* b, uint32_t mask) {
    const BufferPart& q0 = b->parts[0];
    int rc = buffer_rows_alloc(b, mask);
    for (size_t i = 0; rc == RPTB_OK && i < b->parts.size(); i++) {
        const BufferPart& q = b->parts[i];
        if (!q.tiles) continue;
        CU(cudaStreamWaitEvent(q0.stream, q.done, 0));
        const PlaneSet src = i == 0 ? q.planes.set(mask) : b->staging.set(mask);
        if (i > 0) rc = copy_planes(src, q0.device, q.planes.set(mask), q.device, q.planes.n, q0.stream);
        if (rc == RPTB_OK) rc = buffer_scatter(b, src, mask, q.index, q.count);
        if (rc != RPTB_OK || !(mask >> HALF & 1u)) continue;
        const double* half = i == 0 ? q.planes.half : b->staging.half;
        if (i > 0) CU(cudaMemcpyPeerAsync(b->staging.half, q0.device, q.planes.half, q.device, plane_bytes(HALF, q.planes.n), q0.stream));
        CU(launch_buffer_half_scatter(half, b->rows.half, q.planes.n, b->width, b->height, q.index, q.count, q0.stream));
    }
    return rc;
}

// The mirror of buffer_gather: writes the row-major planes of `mask` back into every part's compact tiles, on parts[0]'s
// stream (its device current).  Every part must hold those planes.
int buffer_write_back(rptb_buffer* b, uint32_t mask) {
    const BufferPart& q0 = b->parts[0];
    int rc = RPTB_OK;
    for (size_t i = 0; rc == RPTB_OK && i < b->parts.size(); i++) {
        const BufferPart& q = b->parts[i];
        if (!q.tiles) continue;
        const PlaneSet dst = i == 0 ? q.planes.set(mask) : b->staging.set(mask);
        CU(launch_buffer_move(true, b->rows.set(mask), dst, q.planes.n, b->width, b->height, q.index, q.count, q0.stream));
        if (i > 0) rc = copy_planes(q.planes.set(mask), q.device, dst, q0.device, q.planes.n, q0.stream);
    }
    return rc;
}

// The least entry count of any pixel, once buffer_gather has brought the counts (parts[0]'s device current).  A buffer
// that was never reprojected holds at least min(entries, 2) in every pixel (see rptb_buffer_denoise): that, without
// device work.  A reprojected one: the minimum of its counts, waited for.
int buffer_least_count(rptb_buffer* b, uint32_t* least) {
    if (!b->reprojected) {
        *least = std::min(b->entries, 2u);
        return RPTB_OK;
    }
    BufferPart& q0 = b->parts[0];
    CU(launch_buffer_min_count(b->rows.counts, (uint64_t)b->width * b->height, b->min_count, q0.stream));
    CU(cudaMemcpyAsync(least, b->min_count, sizeof(uint32_t), cudaMemcpyDeviceToHost, q0.stream));
    CU(cudaStreamSynchronize(q0.stream));
    return RPTB_OK;
}

// Orders every later call on b behind the work enqueued so far on `stream`, which is on parts[0]'s device (current).
int buffer_order_behind(rptb_buffer* b, cudaStream_t stream) {
    BufferPart& q0 = b->parts[0];
    CU(cudaEventRecord(q0.done, stream));
    for (size_t i = 1; i < b->parts.size(); i++) {
        BufferPart& q = b->parts[i];
        DeviceGuard g(q.device);
        CU(cudaStreamWaitEvent(q.stream, q0.done, 0));
        CU(cudaEventRecord(q.done, q.stream));
    }
    return RPTB_OK;
}

// Gives part q the scratch of the select (its first adaptive call).
int buffer_part_select_alloc(BufferPart& q) {
    if (q.len) return RPTB_OK;
    const size_t nelem = (size_t)q.tiles * 128u, nblocks = (size_t)q.tiles * 4u;
    CU(own(q.mem, &q.len, sizeof(uint32_t)));
    CU(own(q.mem, &q.active, sizeof(unsigned long long)));
    if (q.tiles) {
        CU(own(q.mem, &q.mask, nelem));
        CU(own(q.mem, &q.flags, nblocks));
        CU(own(q.mem, &q.ids, nblocks * sizeof(uint32_t)));
        q.temp_bytes = adaptive_temp_bytes(q.tiles);
        CU(own(q.mem, &q.temp, q.temp_bytes ? q.temp_bytes : 1));
    }
    return RPTB_OK;
}

// The slot megakernel over the warp blocks of `list` only, into the compact out32/out64 scratch (adaptive sampling).
int render_list_launch(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, const RenderList& list,
                       cudaStream_t stream, bool want_counters, uint32_t* launches) {
    if (want_counters) CU(cudaMemsetAsync(s->counters, 0, sizeof(DeviceCounters), stream));
    if (p->precision == RPTB_PRECISION_F32) {
        RenderArgs<float> a;
        fill_args(cam, p, a);
        a.out = s->out32;
        a.compact = 1u;
        a.counters = want_counters ? s->counters : nullptr;
        a.ks = s->sampled_lights;
        const int rc = ensure_partial(s, a);
        if (rc != RPTB_OK) return rc;
        CU(launch_render_list_f32(s->view32, a, list, (int)p->collect_stats, s->features, stream, launches));
    } else {
        RenderArgs<double> a;
        fill_args(cam, p, a);
        a.out = s->out64;
        a.compact = 1u;
        a.counters = want_counters ? s->counters : nullptr;
        const int rc = ensure_partial(s, a);
        if (rc != RPTB_OK) return rc;
        CU(launch_render_list_f64(s->view64, a, list, (int)p->collect_stats, s->features, stream, launches));
    }
    return RPTB_OK;
}

// Enqueues one buffer part's share of one rptb_sample_into on replica r's own stream: render the part's tiles (its
// index of its count) into the compact out32/out64 scratch, then add them to the part as one more entry of every
// pixel.  No host synchronise.  `crit` (rptb_sample_into_adaptive): first decide which pixels and warp blocks are
// active, render those through the list schedule and add the entry to them alone.  `marked` (a guided call): the
// part's mask, flags and active count are already written (guide_mark), and only the list is selected from the flags.
int sample_part(rptb_scene* r, const rptb_camera* cam, const rptb_render_params* p, BufferPart& q, bool want_stats,
                uint32_t* launches, const rptb_adaptive* crit = nullptr, bool marked = false) {
    DeviceGuard g(r->device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", r->device);
    int rc = wait_busy(r, r->stream);
    if (rc != RPTB_OK) return rc;
    const uint32_t index = q.index, nparts = q.count;
    rptb_render_params qp = *p;
    qp.shard_index = index;
    qp.shard_count = nparts;
    const uint64_t nelem = (uint64_t)q.tiles * 128u;
    rc = ensure_out(r, nelem ? nelem * 3 : 1);
    if (rc != RPTB_OK) return rc;
    CU(cudaStreamWaitEvent(r->stream, q.done, 0));  // an add_samples on the part's own stream
    if (crit) {
        rc = buffer_part_select_alloc(q);
        if (rc != RPTB_OK) return rc;
    }
    if (want_stats) CU(cudaEventRecord(r->ev0, r->stream));
    if (crit) {
        if (marked)
            CU(launch_adaptive_list(q.flags, q.tiles, q.ids, q.len, q.temp, q.temp_bytes, r->stream));
        else
            CU(launch_adaptive_select(q.planes.sums, q.planes.m2, q.planes.counts, q.tiles, p->width, p->height, index, nparts, *crit, q.mask,
                                      q.flags, q.ids, q.len, q.active, q.temp, q.temp_bytes, r->stream));
        const RenderList list = {q.ids, q.len, q.mask};
        rc = render_list_launch(r, cam, &qp, list, r->stream, want_stats, launches);
        *launches += q.tiles ? (marked ? 2u : 3u) : 0u;  // the mark kernel (unless marked) and the select's two
    } else {
        rc = render_launch(r, cam, &qp, r->out32, r->out64, r->stream, want_stats, true, launches);
    }
    if (rc != RPTB_OK) return rc;
    if (want_stats && !crit) CU(cudaEventRecord(r->ev1, r->stream));
    const bool f32 = p->precision == RPTB_PRECISION_F32;
    CU(launch_buffer_accumulate(f32 ? r->out32 : nullptr, f32 ? nullptr : r->out64, false, crit ? q.mask : nullptr, nelem, p->width,
                                p->height, index, nparts, q.planes.sums, q.planes.m2, q.planes.counts, q.planes.half, r->stream));
    // (an adaptive call times the whole entry: select, render and accumulate; a plain one its render)
    if (want_stats && crit) CU(cudaEventRecord(r->ev1, r->stream));
    (*launches)++;
    CU(cudaEventRecord(q.done, r->stream));
    // the scratch is read until the accumulate has run: later calls on any stream order themselves behind it
    CU(cudaEventRecord(r->busy, r->stream));
    r->busy_pending = true;
    return RPTB_OK;
}

// ---- the exchange block of a shard buffer (rptb_buffer_export_shard / rptb_buffer_import_shards) ----
// A header of kShardHeaderBytes, then the shard's compact planes in Plane order (planes.h), the feature planes only
// with features, each padded to shard 0's slots (the most any shard holds, as distributed.gather_tiles pads).  Slots past
// the shard's own are not written.
constexpr uint32_t kShardMagic = 0x44524853u;  // "SHRD"
constexpr size_t kShardHeaderBytes = 256;
// ShardHeader::flags: the shard was reprojected (rptb_buffer_reproject_shard), so its pixels may hold 0 or 1 entries
constexpr uint32_t kShardReprojected = 1u;
struct ShardHeader {
    uint32_t magic, with_features, width, height, shard_index, shard_count, entries, flags;
    uint64_t feature_rays;
    ShardCamera entry_cam, feat_cam;
};
static_assert(sizeof(ShardHeader) <= kShardHeaderBytes, "the shard header outgrew its slot");

struct ShardLayout {
    size_t slots;         // pixel slots of every plane: shard 0's tiles * 128
    uint32_t mask;        // the planes in the block
    size_t at[NPLANES];   // their byte offsets in the block
    size_t bytes;         // the block's size
};
ShardLayout shard_layout(uint32_t width, uint32_t height, uint32_t count, bool with_features) {
    ShardLayout l = {};
    l.slots = (size_t)buffer_tiles(width, height, 0, count) * 128u;
    l.mask = COLOUR | (with_features ? FEATURES : 0u);
    l.bytes = kShardHeaderBytes;
    for (int k = 0; k < NPLANES; k++)
        if (l.mask >> k & 1u) {
            l.at[k] = l.bytes;
            l.bytes += plane_bytes(k, l.slots);
        }
    return l;
}

// The planes of the block at `block`.
PlaneSet shard_planes(const ShardLayout& l, const void* block) {
    PlaneSet s = {};
    for (int k = 0; k < NPLANES; k++)
        if (l.mask >> k & 1u) s.p[k] = (char*)block + l.at[k];
    return s;
}

ShardCamera shard_camera(const CameraRecord& r) {
    ShardCamera c;
    std::memset(&c, 0, sizeof(c));
    c.state = (uint32_t)r.state;
    if (r.state == CameraRecord::ONE) c.cam = r.cam;
    return c;
}

CameraRecord camera_record(const ShardCamera& c) {
    CameraRecord r;
    r.state = (CameraRecord::State)c.state;
    r.cam = c.cam;
    return r;
}

// Whole-image reads need every tile: a shard buffer holds only its own.
int refuse_shard(const char* what) {
    return fail(RPTB_ERR_UNSUPPORTED,
                "%s of a shard buffer: it holds only its own tiles; gather the shards into a whole buffer first "
                "(rptb_buffer_export_shard, rptb_buffer_import_shards)",
                what);
}

// What a render into b checks: its parameters; the shard it names, which for a whole buffer is shard_count 0 or 1 only
// and for a shard buffer exactly its own (shard_index, shard_count); its size; and the scene's device list.
int check_render_into(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, const rptb_buffer* b) {
    if (!b) return fail(RPTB_ERR_BAD_ARG, "null argument");
    const int rc = check_params(s, cam, p);
    if (rc != RPTB_OK) return rc;
    const uint32_t sc = p->shard_count ? p->shard_count : 1u;
    const BufferPart& q = b->parts[0];
    if (!b->shard && sc > 1)
        return fail(RPTB_ERR_UNSUPPORTED, "shard_count %u: a buffer holds the whole image (shard with rptb_buffer_create_shard)", sc);
    if (b->shard && (p->shard_index != q.index || sc != q.count))
        return fail(RPTB_ERR_BAD_ARG, "the render is shard %u of %u but the buffer holds shard %u of %u", p->shard_index, sc, q.index,
                    q.count);
    if (p->width != b->width || p->height != b->height)
        return fail(RPTB_ERR_BAD_ARG, "render is %ux%u but the buffer is %ux%u", p->width, p->height, b->width, b->height);
    const uint32_t nparts = 1u + (uint32_t)s->peers.size();
    bool same = nparts == b->parts.size();
    for (uint32_t i = 0; same && i < nparts; i++) same = replica(s, i)->device == b->parts[i].device;
    if (!same) return fail(RPTB_ERR_BAD_ARG, "the buffer was created on a scene with another device list");
    return RPTB_OK;
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
    // RPTB_ALLOW_REPEATED_DEVICES=1 (a testing switch, read on every call): a device may be listed more than once, and
    // each listing is a replica of its own -- its own stream, scratch and tiles, as on a distinct GPU -- so the
    // multi-replica paths run on a single GPU.  It is not faster: the replicas share that GPU.
    const char* rep = getenv("RPTB_ALLOW_REPEATED_DEVICES");
    const bool repeats = rep && std::strcmp(rep, "1") == 0;
    std::vector<int> devs(ndevices);
    for (int i = 0; i < ndevices; i++) {
        devs[i] = devices ? devices[i] : i;
        if (devs[i] < 0 || devs[i] >= ndev) return fail(RPTB_ERR_BAD_ARG, "device %d of %d", devs[i], ndev);
        for (int j = 0; j < i && !repeats; j++)
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
            rcs[i] = render_shard_to_host(replica(s, i), cam, &q, out_rgb, &sts[i]);
            if (rcs[i] != RPTB_OK) errs[i] = g_error;  // g_error is thread-local
        });
    }
    for (std::thread& t : workers) t.join();
    for (uint32_t i = 0; i < nrep; i++)
        if (rcs[i] != RPTB_OK) return fail(rcs[i], "device %d: %s", replica(s, i)->device, errs[i].c_str());
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
    // (a tile index past 32 bits needs an image of 2^39 pixels or more; a render takes at most 2^29)
    if (width == 0 || height == 0 || j >= 128u || shard_index >= sc || tile >= (uint64_t)tiles_x * tiles_y || tile > UINT32_MAX)
        return -1;
    return tile_pixel(width, height, (uint32_t)tile, j);
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

// A whole buffer (shard_count == 0: one part per replica of s, part i dealt (i, nparts)) or the one-part shard buffer of
// (shard_index, shard_count) on s's device; `halves`: a whole buffer with the HALF plane.  The arguments are checked by
// the callers.
static int buffer_create_impl(rptb_scene* s, uint32_t width, uint32_t height, uint32_t box_radius, uint32_t shard_index,
                              uint32_t shard_count, rptb_buffer** out, bool halves = false) {
    rptb_buffer* b = new (std::nothrow) rptb_buffer();
    if (!b) return fail(RPTB_ERR_OOM, "host allocation failed");
    b->width = width;
    b->height = height;
    b->radius = box_radius;
    b->shard = shard_count > 0;
    b->halves = halves;
    const uint32_t nparts = b->shard ? 1u : 1u + (uint32_t)s->peers.size();
    b->parts.resize(nparts);
    int rc = RPTB_OK;
    for (uint32_t i = 0; rc == RPTB_OK && i < nparts; i++) {
        BufferPart& q = b->parts[i];
        q.device = replica(s, i)->device;
        q.index = b->shard ? shard_index : i;
        q.count = b->shard ? shard_count : nparts;
        q.tiles = buffer_tiles(width, height, q.index, q.count);
        DeviceGuard g(q.device);
        rc = g.ok ? buffer_part_alloc(q, halves) : fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", q.device);
    }
    if (rc != RPTB_OK) {
        const std::string keep = g_error;
        buffer_free(b);
        g_error = keep;
        return rc;
    }
    *out = b;
    return RPTB_OK;
}

int rptb_buffer_create(rptb_scene* s, uint32_t width, uint32_t height, uint32_t box_radius, rptb_buffer** out) {
    if (!s || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    if (width == 0 || height == 0) return fail(RPTB_ERR_BAD_ARG, "empty image %ux%u", width, height);
    if ((uint64_t)width * height > 0x7FFFFFFFull / 4) return fail(RPTB_ERR_UNSUPPORTED, "image too large");
    return buffer_create_impl(s, width, height, box_radius, 0, 0, out);
}

int rptb_buffer_create_halves(rptb_scene* s, uint32_t width, uint32_t height, uint32_t box_radius, rptb_buffer** out) {
    if (!s || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    if (width == 0 || height == 0) return fail(RPTB_ERR_BAD_ARG, "empty image %ux%u", width, height);
    if ((uint64_t)width * height > 0x7FFFFFFFull / 4) return fail(RPTB_ERR_UNSUPPORTED, "image too large");
    return buffer_create_impl(s, width, height, box_radius, 0, 0, out, true);
}

int rptb_buffer_create_shard(rptb_scene* s, uint32_t width, uint32_t height, uint32_t box_radius, uint32_t shard_index,
                             uint32_t shard_count, rptb_buffer** out) {
    if (!s || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    if (width == 0 || height == 0) return fail(RPTB_ERR_BAD_ARG, "empty image %ux%u", width, height);
    if ((uint64_t)width * height > 0x7FFFFFFFull / 4) return fail(RPTB_ERR_UNSUPPORTED, "image too large");
    if (shard_index >= shard_count) return fail(RPTB_ERR_BAD_ARG, "shard_index %u >= shard_count %u", shard_index, shard_count);
    if (!s->peers.empty())
        return fail(RPTB_ERR_UNSUPPORTED, "a shard buffer lives on one device, but the scene has %u replicas", 1u + (uint32_t)s->peers.size());
    return buffer_create_impl(s, width, height, box_radius, shard_index, shard_count, out);
}

void rptb_buffer_destroy(rptb_buffer* b) {
    if (b) buffer_free(b);
}

// What a guided call checks of the buffer (locked) when its filter runs: features, and entries and features made
// through `cam` alone, so that the filter's features describe what the entries saw.
static int check_guide_buffer(const rptb_buffer* b, const rptb_camera* cam) {
    if (b->feature_rays == 0) return fail(RPTB_ERR_BAD_ARG, "the buffer holds no features (rptb_buffer_add_features)");
    const char* why[] = {"none", "one", "mixed (several cameras)", "unknown (a host entry)"};
    if (b->feat_cam.state != CameraRecord::ONE) return fail(RPTB_ERR_BAD_ARG, "the buffer's features have no single camera: %s", why[b->feat_cam.state]);
    if (std::memcmp(&b->feat_cam.cam, cam, sizeof(rptb_camera)) != 0)
        return fail(RPTB_ERR_BAD_ARG, "the buffer's features were made through another camera");
    if (b->entry_cam.state != CameraRecord::NONE && b->entry_cam.state != CameraRecord::ONE)
        return fail(RPTB_ERR_BAD_ARG, "the buffer's entries have no single camera: %s", why[b->entry_cam.state]);
    if (b->entry_cam.state == CameraRecord::ONE && std::memcmp(&b->entry_cam.cam, cam, sizeof(rptb_camera)) != 0)
        return fail(RPTB_ERR_BAD_ARG, "the buffer's entries were made through another camera");
    return RPTB_OK;
}

// The denoiser's planes: the resolved features, the colour and variance ping-pong planes and c' in b->dn, and the error
// estimate's u ping-pong planes and E in b->hv.
struct FilterPlanes {
    Aov a;
    double* col[2];
    double* var[2];
    double* out;
    double* u[2];
    double* E;
};

// What every run of the filter over b (locked, parts[0]'s device current) starts with, enqueued on parts[0]'s stream:
// b's colour and features (and with `error` its HALF plane) gathered row-major and the features resolved; b->dn (and
// b->hv) allocated on first use and carved into *f.
static int filter_planes(rptb_buffer* b, bool error, FilterPlanes* f) {
    const size_t npix = (size_t)b->width * b->height;
    const int rc = buffer_gather(b, COLOUR | FEATURES | (error ? 1u << HALF : 0u));
    if (rc != RPTB_OK) return rc;
    const Aov a = buffer_aov(b);
    CU(launch_features_resolve(feature_planes(b->rows.feat, npix), npix, (double)b->feature_rays, a, b->parts[0].stream));
    if (!b->dn) CU(own(b->mem, &b->dn, npix * 11 * sizeof(double)));
    *f = {a, {b->dn, b->dn + 3 * npix}, {b->dn + 6 * npix, b->dn + 7 * npix}, b->dn + 8 * npix, {nullptr, nullptr}, nullptr};
    if (!error) return RPTB_OK;
    if (!b->hv) CU(own(b->mem, &b->hv, npix * 7 * sizeof(double)));
    f->u[0] = b->hv;
    f->u[1] = b->hv + 3 * npix;
    f->E = b->hv + 6 * npix;
    return RPTB_OK;
}

// filter_planes, then the filter's passes (launch_denoise_passes), or with `error` the passes with the error estimate
// (launch_halves_error, a buffer with halves).  *col: the plane holding the last pass's i'; *var: v', or with `error`
// E; *launches: the filter's kernels.
static int buffer_filter(rptb_buffer* b, const rptb_denoise& d, bool error, Aov* a, const double** col, const double** var,
                         uint32_t* launches) {
    FilterPlanes f;
    const int rc = filter_planes(b, error, &f);
    if (rc != RPTB_OK) return rc;
    *a = f.a;
    if (error) {
        *var = f.E;
        CU(launch_halves_error(b->rows.sums, b->rows.m2, b->rows.half, b->rows.counts, f.a.normal, f.a.depth, f.a.albedo, b->width,
                               b->height, d, f.col, f.var, f.u, f.E, col, b->parts[0].stream, launches));
    } else {
        CU(launch_denoise_passes(b->rows.sums, b->rows.m2, b->rows.counts, f.a.normal, f.a.depth, f.a.albedo, b->width, b->height, d,
                                 f.col, f.var, col, var, b->parts[0].stream, launches));
    }
    return RPTB_OK;
}

// A guided call's decision, enqueued on the stream of f's parts[0]: the filter over f (buffer_filter), then the guided
// mark kernel once per part of b -- into parts[0]'s own mask, flags and active count, and for every other part into the
// guide staging, whose mask and flags (tiles*132 bytes) and count then go to the part's device.  f is b itself
// (rptb_sample_into_guided), or the gathered whole buffer on the device of b, a shard (rptb_sample_into_guided_shard).
// Every later call on either buffer is ordered behind it.  Every part of b holds its select scratch.  `error`
// (rptb_sample_into_guided_error, a buffer with halves): the filter runs with the error estimate, and the mark tests E
// in place of v'.  *launches: kernels enqueued, the HALF plane's scatter aside.
static int guide_mark(rptb_buffer* f, rptb_buffer* b, const rptb_adaptive& crit, const rptb_denoise& d, uint32_t* launches, bool error) {
    BufferPart& q0 = f->parts[0];
    DeviceGuard g(q0.device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", q0.device);
    uint32_t most = 0, nl = 0;
    for (const BufferPart& q : f->parts) nl += q.tiles ? 1u : 0u;  // the gather's scatter
    for (size_t i = 1; i < b->parts.size(); i++) most = std::max(most, b->parts[i].tiles);
    if (most && !b->guide_mask) {
        CU(own(b->mem, &b->guide_mask, (size_t)most * 132u));
        CU(own(b->mem, &b->guide_active, sizeof(unsigned long long)));
    }
    Aov a;
    const double *icol, *ivar;
    uint32_t passes = 0;
    int rc = buffer_filter(f, d, error, &a, &icol, &ivar, &passes);
    if (rc != RPTB_OK) return rc;
    nl += 1u + passes;  // the features' resolve and the filter
    for (size_t i = 0; i < b->parts.size(); i++) {
        BufferPart& q = b->parts[i];
        uint8_t* mask = i == 0 ? q.mask : b->guide_mask;
        uint8_t* flags = i == 0 ? q.flags : b->guide_mask + (size_t)most * 128u;
        unsigned long long* active = i == 0 ? q.active : b->guide_active;
        CU(cudaStreamWaitEvent(q0.stream, q.done, 0));  // the part's last accumulate (and a shard's export) read its mask
        CU(launch_guided_mark(icol, ivar, a.albedo, f->rows.counts, f->width, f->height, q.index, q.count, q.tiles, d.albedo_eps, crit,
                              mask, flags, active, q0.stream));
        nl += q.tiles ? 1u : 0u;
        if (i == 0) continue;
        if (q.tiles) {
            CU(cudaMemcpyPeerAsync(q.mask, q.device, mask, q0.device, (size_t)q.tiles * 128u, q0.stream));
            CU(cudaMemcpyPeerAsync(q.flags, q.device, flags, q0.device, (size_t)q.tiles * 4u, q0.stream));
        }
        CU(cudaMemcpyPeerAsync(q.active, q.device, active, q0.device, sizeof(unsigned long long), q0.stream));
    }
    *launches = nl;
    rc = buffer_order_behind(b, q0.stream);
    if (rc == RPTB_OK && f != b) rc = buffer_order_behind(f, q0.stream);
    return rc;
}

static bool same_camera(const CameraRecord& a, const CameraRecord& b) {
    const ShardCamera x = shard_camera(a), y = shard_camera(b);
    return std::memcmp(&x, &y, sizeof(x)) == 0;
}

// What rptb_sample_into_guided_shard checks of `whole` (locked) once the filter runs: a one-part whole buffer on the
// shard's device, of its size, last written by an import of all the shards at the shard's current state -- which the
// shard still has, not having changed since its last export -- and check_guide_buffer's conditions.
static int check_guide_whole(const rptb_buffer* shard, const rptb_buffer* whole, const rptb_camera* cam) {
    if (!whole) return fail(RPTB_ERR_BAD_ARG, "null whole buffer: the shard has reached min_entries, so the filter runs over its gathered image");
    if (whole->shard) return fail(RPTB_ERR_BAD_ARG, "whole is a shard buffer: the filter needs every shard gathered (rptb_buffer_import_shards)");
    if (whole->parts.size() != 1)
        return fail(RPTB_ERR_UNSUPPORTED, "whole has %zu parts: a shard's filter runs over a one-part whole buffer", whole->parts.size());
    const BufferPart& q = shard->parts[0];
    if (whole->parts[0].device != q.device)
        return fail(RPTB_ERR_BAD_ARG, "whole is on device %d but the shard on device %d", whole->parts[0].device, q.device);
    if (whole->width != shard->width || whole->height != shard->height)
        return fail(RPTB_ERR_BAD_ARG, "whole is %ux%u but the shard %ux%u", whole->width, whole->height, shard->width, shard->height);
    if (shard->exported != shard->state)
        return fail(RPTB_ERR_BAD_ARG, "the shard changed since its last export: gather it into whole first (rptb_buffer_export_shard or "
                                      "rptb_buffer_export_delta)");
    if (whole->imported != whole->state || whole->imported_shards != q.count)
        return fail(RPTB_ERR_BAD_ARG, "whole was not last written by an import of the %u shards (rptb_buffer_import_shards or "
                                      "rptb_buffer_import_deltas)", q.count);
    if (whole->entries != shard->entries || whole->reprojected != shard->reprojected || whole->feature_rays != shard->feature_rays ||
        !same_camera(whole->entry_cam, shard->entry_cam) || !same_camera(whole->feat_cam, shard->feat_cam))
        return fail(RPTB_ERR_BAD_ARG,
                    "whole does not hold the shard's current state (entries %u / %u, reprojected %d / %d, feature rays %llu / %llu, or "
                    "cameras)", whole->entries, shard->entries, (int)whole->reprojected, (int)shard->reprojected,
                    (unsigned long long)whole->feature_rays, (unsigned long long)shard->feature_rays);
    return check_guide_buffer(whole, cam);
}

// rptb_sample_into (crit null), rptb_sample_into_adaptive (crit) and rptb_sample_into_guided (crit and guide; the
// filter runs when guide->iterations > 0).  shard_entry (rptb_sample_into_guided_shard): b is a shard buffer and the
// filter runs over `whole`.  error (rptb_sample_into_guided_error): b has halves, and the mark tests E.
static int sample_into_impl(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, const rptb_adaptive* crit,
                            const rptb_denoise* guide, rptb_buffer* b, uint64_t* out_active, rptb_stats* stats, bool shard_entry = false,
                            rptb_buffer* whole = nullptr, bool error = false) {
    int rc = check_render_into(s, cam, p, b);
    if (rc != RPTB_OK) return rc;
    if (crit && p->engine == RPTB_ENGINE_WAVEFRONT)
        return fail(RPTB_ERR_UNSUPPORTED, "adaptive sampling renders with the slot megakernel, not the wavefront engine");
    if (guide && b->shard && !shard_entry) return refuse_shard("guided adaptive sampling");
    if (error && !b->halves) return fail(RPTB_ERR_BAD_ARG, "the buffer has no halves (rptb_buffer_create_halves): no error estimate");
    if (shard_entry && !b->shard)
        return fail(RPTB_ERR_BAD_ARG, "not a shard buffer (rptb_buffer_create_shard): a whole buffer samples with rptb_sample_into_guided");
    const uint32_t nparts = (uint32_t)b->parts.size();
    std::lock_guard<std::mutex> bl(b->lock);
    if (b->entries == UINT32_MAX) return fail(RPTB_ERR_UNSUPPORTED, "too many entries");
    const bool filter = guide && guide->iterations > 0;
    if (filter) {
        rc = check_guide_buffer(b, cam);
        if (rc != RPTB_OK) return rc;
    }
    // While no pixel can hold min_entries (none holds more than b->entries), every pixel is active under either
    // criterion: the plain mark decides that without the filter.
    const bool marked = filter && b->entries >= crit->min_entries;
    std::unique_lock<std::mutex> wl;
    if (marked && shard_entry) {
        if (whole && whole != b) wl = std::unique_lock<std::mutex>(whole->lock);
        rc = check_guide_whole(b, whole, cam);
        if (rc != RPTB_OK) return rc;
    }
    uint32_t guide_launches = 0;
    if (marked) {
        for (BufferPart& q : b->parts) {
            DeviceGuard g(q.device);
            if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", q.device);
            rc = buffer_part_select_alloc(q);
            if (rc != RPTB_OK) return rc;
        }
        rc = guide_mark(shard_entry ? whole : b, b, *crit, *guide, &guide_launches, error);
        if (rc != RPTB_OK) return rc;
    }
    // every replica's share is enqueued before any is waited for, so the devices run concurrently
    std::vector<std::unique_lock<std::mutex>> locks;
    std::vector<uint32_t> launches(nparts, 0);
    for (uint32_t i = 0; i < nparts; i++) {
        rptb_scene* r = replica(s, i);
        locks.emplace_back(r->lock);
        rc = sample_part(r, cam, p, b->parts[i], stats != nullptr, &launches[i], crit, marked);
        if (rc != RPTB_OK) return nparts > 1 ? fail(rc, "device %d: %s", r->device, g_error.c_str()) : rc;
    }
    const CameraRecord cam_before = b->entry_cam;
    const uint32_t entries_before = b->entries;
    b->entries++;
    b->entry_cam.note(*cam);
    b->state++;
    // A delta block can carry this call when it was adaptive, and either kept the entry camera or made the first entry: an
    // importer then knows the camera before the call from the one after (rptb_buffer_import_deltas).
    const bool cam_known = same_camera(cam_before, b->entry_cam) || (cam_before.state == CameraRecord::NONE && entries_before == 0);
    b->masked = crit && cam_known ? b->state : UINT64_MAX;
    if (out_active) {
        uint64_t total = 0;
        for (uint32_t i = 0; i < nparts; i++) {
            rptb_scene* r = replica(s, i);
            DeviceGuard g(r->device);
            unsigned long long a = 0;
            CU(cudaMemcpyAsync(&a, b->parts[i].active, sizeof(a), cudaMemcpyDeviceToHost, r->stream));
            CU(cudaStreamSynchronize(r->stream));
            r->busy_pending = false;
            total += a;
        }
        *out_active = total;
    }
    if (!stats) return RPTB_OK;
    std::memset(stats, 0, sizeof(*stats));
    for (uint32_t i = 0; i < nparts; i++) {
        rptb_scene* r = replica(s, i);
        DeviceGuard g(r->device);
        DeviceCounters c;
        CU(cudaMemcpyAsync(&c, r->counters, sizeof(c), cudaMemcpyDeviceToHost, r->stream));
        CU(cudaStreamSynchronize(r->stream));
        r->busy_pending = false;
        rptb_stats st;
        std::memset(&st, 0, sizeof(st));
        read_stats(c, &st);
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, r->ev0, r->ev1));
        stats->segments += st.segments; stats->rays += st.rays;
        stats->node_visits += st.node_visits; stats->tri_tests += st.tri_tests;
        stats->mesh_hits += st.mesh_hits; stats->env_lookups += st.env_lookups;
        stats->object_tests += st.object_tests;
        stats->bvh_node_visits += st.bvh_node_visits; stats->bvh_tri_tests += st.bvh_tri_tests;
        stats->gpu_ms = std::max(stats->gpu_ms, (double)ms);  // the devices run concurrently
        stats->launches += launches[i];
    }
    stats->launches += guide_launches;
    stats->engine = !crit && use_wavefront(s, p) ? RPTB_ENGINE_WAVEFRONT : RPTB_ENGINE_MEGAKERNEL;
    return RPTB_OK;
}

int rptb_sample_into(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, rptb_buffer* b, rptb_stats* stats) {
    return sample_into_impl(s, cam, p, nullptr, nullptr, b, nullptr, stats);
}

static int check_adaptive(const rptb_adaptive* crit) {
    if (!crit) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (crit->min_entries < 2) return fail(RPTB_ERR_BAD_ARG, "min_entries %u < 2 (a pixel's variance needs two entries)", crit->min_entries);
    if (!(std::isfinite(crit->rel_tol) && crit->rel_tol >= 0.0) || !(std::isfinite(crit->abs_tol) && crit->abs_tol >= 0.0))
        return fail(RPTB_ERR_BAD_ARG, "tolerances must be finite and >= 0 (rel_tol %g, abs_tol %g)", crit->rel_tol, crit->abs_tol);
    return RPTB_OK;
}

static int check_denoise(const rptb_denoise* d) {
    if (!d) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (d->iterations > kDenoiseMaxIterations)
        return fail(RPTB_ERR_BAD_ARG, "iterations %u > %u", d->iterations, kDenoiseMaxIterations);
    if (!(std::isfinite(d->sigma_depth) && d->sigma_depth >= 0.0) || !(std::isfinite(d->sigma_luminance) && d->sigma_luminance >= 0.0) ||
        !(std::isfinite(d->albedo_eps) && d->albedo_eps >= 0.0))
        return fail(RPTB_ERR_BAD_ARG, "sigma_depth, sigma_luminance and albedo_eps must be finite and >= 0 (%g, %g, %g)", d->sigma_depth,
                    d->sigma_luminance, d->albedo_eps);
    return RPTB_OK;
}

int rptb_sample_into_adaptive(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, const rptb_adaptive* crit,
                              rptb_buffer* b, uint64_t* out_active, rptb_stats* stats) {
    const int rc = check_adaptive(crit);
    if (rc != RPTB_OK) return rc;
    return sample_into_impl(s, cam, p, crit, nullptr, b, out_active, stats);
}

int rptb_sample_into_guided(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, const rptb_adaptive* crit,
                            const rptb_denoise* guide, rptb_buffer* b, uint64_t* out_active, rptb_stats* stats) {
    int rc = check_adaptive(crit);
    if (rc == RPTB_OK) rc = check_denoise(guide);
    if (rc != RPTB_OK) return rc;
    return sample_into_impl(s, cam, p, crit, guide, b, out_active, stats);
}

int rptb_sample_into_guided_error(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, const rptb_adaptive* crit,
                                  const rptb_denoise* guide, rptb_buffer* b, uint64_t* out_active, rptb_stats* stats) {
    int rc = check_adaptive(crit);
    if (rc == RPTB_OK) rc = check_denoise(guide);
    if (rc != RPTB_OK) return rc;
    if (guide->iterations == 0) return fail(RPTB_ERR_BAD_ARG, "iterations 0: the error estimate needs at least one filter pass");
    return sample_into_impl(s, cam, p, crit, guide, b, out_active, stats, false, nullptr, true);
}

int rptb_sample_into_guided_shard(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, const rptb_adaptive* crit,
                                  const rptb_denoise* guide, rptb_buffer* shard, rptb_buffer* whole, uint64_t* out_active,
                                  rptb_stats* stats) {
    int rc = check_adaptive(crit);
    if (rc == RPTB_OK) rc = check_denoise(guide);
    if (rc != RPTB_OK) return rc;
    return sample_into_impl(s, cam, p, crit, guide, shard, out_active, stats, true, whole);
}

int rptb_buffer_add_samples(rptb_buffer* b, const double* rgb) {
    if (!b || !rgb) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (b->shard) return refuse_shard("add_samples");
    std::lock_guard<std::mutex> bl(b->lock);
    if (b->entries == UINT32_MAX) return fail(RPTB_ERR_UNSUPPORTED, "too many entries");
    const uint32_t nparts = (uint32_t)b->parts.size();
    const size_t nvals = (size_t)b->width * b->height * 3;
    for (uint32_t i = 0; i < nparts; i++) {
        BufferPart& q = b->parts[i];
        DeviceGuard g(q.device);
        if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", q.device);
        if (!q.upload) CU(own(q.mem, &q.upload, nvals * sizeof(double)));
        CU(cudaStreamWaitEvent(q.stream, q.done, 0));
        // pageable source: the call returns once the bytes are staged, `rgb` may be reused afterwards
        CU(cudaMemcpyAsync(q.upload, rgb, nvals * sizeof(double), cudaMemcpyHostToDevice, q.stream));
        CU(launch_buffer_accumulate(nullptr, q.upload, true, nullptr, (uint64_t)q.tiles * 128u, b->width, b->height, q.index, q.count,
                                    q.planes.sums, q.planes.m2, q.planes.counts, q.planes.half, q.stream));
        CU(cudaEventRecord(q.done, q.stream));
    }
    b->entries++;
    b->entry_cam.state = CameraRecord::UNKNOWN;
    b->state++;
    return RPTB_OK;
}

int rptb_buffer_image(rptb_buffer* b, uint8_t* out_rgb8) {
    if (!b || !out_rgb8) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (b->shard) return refuse_shard("image");
    std::lock_guard<std::mutex> bl(b->lock);
    if (b->entries == 0) return fail(RPTB_ERR_BAD_ARG, "Pixel found with no samples");  // buffer.rs:89
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    uint32_t least = 0;
    int rc = buffer_gather(b, 1u << SUMS | 1u << COUNTS);
    if (rc == RPTB_OK) rc = buffer_least_count(b, &least);
    if (rc != RPTB_OK) return rc;
    if (least == 0) return fail(RPTB_ERR_BAD_ARG, "Pixel found with no samples");  // buffer.rs:89
    const size_t nvals = (size_t)b->width * b->height * 3;
    CU(launch_film_resolve_counted(b->rows.sums, b->rows.counts, b->width, b->height, b->radius, b->rgb8, q0.stream));
    CU(cudaMemcpyAsync(out_rgb8, b->rgb8, nvals, cudaMemcpyDeviceToHost, q0.stream));
    CU(cudaStreamSynchronize(q0.stream));
    return RPTB_OK;
}

int rptb_buffer_variance(rptb_buffer* b, double* out) {
    if (!b || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (b->shard) return refuse_shard("variance");
    std::lock_guard<std::mutex> bl(b->lock);
    if (b->entries < 2) {  // n - 1 = 0: the reference divides by it
        *out = NAN;
        return RPTB_OK;
    }
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    uint32_t least = 0;
    int rc = buffer_gather(b, 1u << M2 | 1u << COUNTS);
    if (rc == RPTB_OK) rc = buffer_least_count(b, &least);
    if (rc != RPTB_OK) return rc;
    if (least < 2) {
        *out = NAN;
        return RPTB_OK;
    }
    const uint64_t npix = (uint64_t)b->width * b->height;
    double* total = b->partial + buffer_variance_blocks(npix);
    CU(launch_buffer_variance_sum(b->rows.m2, b->rows.counts, npix, b->partial, total, q0.stream));
    double sum = 0.0;
    CU(cudaMemcpyAsync(&sum, total, sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    CU(cudaStreamSynchronize(q0.stream));
    *out = sum / (double)npix;
    return RPTB_OK;
}

int rptb_buffer_sums(rptb_buffer* b, double* out_sums, uint32_t* out_entries) {
    if (!b || !out_sums) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (b->shard) return refuse_shard("sums");
    std::lock_guard<std::mutex> bl(b->lock);
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    const int rc = buffer_gather(b, 1u << SUMS | (out_entries ? 1u << COUNTS : 0u));
    if (rc != RPTB_OK) return rc;
    CU(cudaMemcpyAsync(out_sums, b->rows.sums, (size_t)b->width * b->height * 3 * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    std::vector<uint32_t> counts;
    if (out_entries) {
        counts.resize((size_t)b->width * b->height);
        CU(cudaMemcpyAsync(counts.data(), b->rows.counts, counts.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, q0.stream));
    }
    CU(cudaStreamSynchronize(q0.stream));
    if (out_entries) *out_entries = *std::max_element(counts.begin(), counts.end());
    return RPTB_OK;
}

int rptb_buffer_pixel_stats(rptb_buffer* b, double* sums, double* m2, uint32_t* counts) {
    if (!b) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (b->shard) return refuse_shard("pixel_stats");
    std::lock_guard<std::mutex> bl(b->lock);
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    const size_t npix = (size_t)b->width * b->height;
    const int rc = buffer_gather(b, (sums ? 1u << SUMS : 0u) | (m2 ? 1u << M2 : 0u) | (counts ? 1u << COUNTS : 0u));
    if (rc != RPTB_OK) return rc;
    if (sums) CU(cudaMemcpyAsync(sums, b->rows.sums, npix * 3 * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    if (m2) CU(cudaMemcpyAsync(m2, b->rows.m2, npix * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    if (counts) CU(cudaMemcpyAsync(counts, b->rows.counts, npix * sizeof(uint32_t), cudaMemcpyDeviceToHost, q0.stream));
    CU(cudaStreamSynchronize(q0.stream));
    return RPTB_OK;
}

int rptb_buffer_add_features(rptb_scene* s, const rptb_camera* cam, const rptb_render_params* p, rptb_buffer* b, rptb_stats* stats) {
    const int rc = check_render_into(s, cam, p, b);
    if (rc != RPTB_OK) return rc;
    const uint32_t nparts = (uint32_t)b->parts.size();
    std::lock_guard<std::mutex> bl(b->lock);
    if (b->feature_rays > UINT64_MAX / 2) return fail(RPTB_ERR_UNSUPPORTED, "too many feature rays");
    // every replica's share is enqueued before any is waited for
    std::vector<std::unique_lock<std::mutex>> locks;
    for (uint32_t i = 0; i < nparts; i++) {
        rptb_scene* r = replica(s, i);
        BufferPart& q = b->parts[i];
        locks.emplace_back(r->lock);
        DeviceGuard g(r->device);
        if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", r->device);
        const size_t nelem = (size_t)q.tiles * 128u;
        CU(cudaStreamWaitEvent(r->stream, q.done, 0));
        if (!q.planes.feat && nelem) {
            const int prc = planes_alloc(q.mem, q.planes, nelem, FEATURES);
            if (prc != RPTB_OK) return prc;
            CU(cudaMemsetAsync(q.planes.feat, 0, nelem * FEATURE_SUMS * sizeof(double), r->stream));
        }
        rptb_render_params qp = *p;
        qp.shard_index = q.index;
        qp.shard_count = q.count;
        if (stats) CU(cudaEventRecord(r->ev0, r->stream));
        if (p->precision == RPTB_PRECISION_F32) {
            RenderArgs<float> a;
            fill_args(cam, &qp, a);
            CU(launch_features_f32(r->view32, a, r->features, q.planes.feat, r->stream));
        } else {
            RenderArgs<double> a;
            fill_args(cam, &qp, a);
            CU(launch_features_f64(r->view64, a, r->features, q.planes.feat, r->stream));
        }
        if (stats) CU(cudaEventRecord(r->ev1, r->stream));
        CU(cudaEventRecord(q.done, r->stream));
    }
    b->feature_rays += p->iterations;
    b->feat_cam.note(*cam);
    b->state++;
    if (!stats) return RPTB_OK;
    std::memset(stats, 0, sizeof(*stats));
    for (uint32_t i = 0; i < nparts; i++) {
        rptb_scene* r = replica(s, i);
        DeviceGuard g(r->device);
        CU(cudaEventSynchronize(r->ev1));
        float ms = 0;
        CU(cudaEventElapsedTime(&ms, r->ev0, r->ev1));
        stats->gpu_ms = std::max(stats->gpu_ms, (double)ms);  // the devices run concurrently
        stats->launches += b->parts[i].tiles ? 1u : 0u;
    }
    uint64_t npix = (uint64_t)b->width * b->height;
    if (b->shard) {  // the pixels of the shard's own tiles
        const BufferPart& q = b->parts[0];
        const uint32_t tiles_x = (b->width + 15u) / 16u;
        npix = 0;
        for (uint32_t k = 0; k < q.tiles; k++) {
            const uint32_t t = q.index + k * q.count, x0 = t % tiles_x * 16u, y0 = t / tiles_x * 8u;
            npix += (uint64_t)std::min(16u, b->width - x0) * std::min(8u, b->height - y0);
        }
    }
    stats->rays = npix * p->iterations;
    stats->engine = RPTB_ENGINE_MEGAKERNEL;
    return RPTB_OK;
}

int rptb_buffer_features(rptb_buffer* b, double* normal, double* depth, double* albedo, double* hit_fraction) {
    if (!b) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (b->shard) return refuse_shard("features");
    std::lock_guard<std::mutex> bl(b->lock);
    if (b->feature_rays == 0) return fail(RPTB_ERR_BAD_ARG, "the buffer holds no features (rptb_buffer_add_features)");
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    const size_t npix = (size_t)b->width * b->height;
    const int rc = buffer_gather(b, FEATURES);
    if (rc != RPTB_OK) return rc;
    const Aov a = buffer_aov(b);
    CU(launch_features_resolve(feature_planes(b->rows.feat, npix), npix, (double)b->feature_rays, a, q0.stream));
    if (normal) CU(cudaMemcpyAsync(normal, a.normal, npix * 3 * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    if (albedo) CU(cudaMemcpyAsync(albedo, a.albedo, npix * 3 * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    if (depth) CU(cudaMemcpyAsync(depth, a.depth, npix * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    if (hit_fraction) CU(cudaMemcpyAsync(hit_fraction, a.frac, npix * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    CU(cudaStreamSynchronize(q0.stream));
    return RPTB_OK;
}

// What rptb_buffer_denoise, _variance and _error refuse before any device work.
static int check_denoise_entries(const rptb_buffer* b) {
    if (b->entries == 0) return fail(RPTB_ERR_BAD_ARG, "Pixel found with no samples");  // buffer.rs:89
    // Every pixel holds at least min(entries, 2) entries, so this is exact for any mix of calls: the first call of any
    // kind reaches every pixel (an adaptive one because n = 0 < min_entries); plain calls and add_samples reach every
    // pixel; and rptb_sample_into_adaptive refuses min_entries < 2, so a pixel with one entry is always active.
    if (b->entries < 2) return fail(RPTB_ERR_BAD_ARG, "a pixel has fewer than 2 entries (no variance to guide the filter)");
    if (b->feature_rays == 0) return fail(RPTB_ERR_BAD_ARG, "the buffer holds no features (rptb_buffer_add_features)");
    return RPTB_OK;
}

// ... and once the filter's gather has brought the counts: a reprojected buffer does not keep the invariant above, so
// its least count decides.
static int check_denoise_counts(rptb_buffer* b) {
    uint32_t least = 0;
    const int rc = buffer_least_count(b, &least);
    if (rc != RPTB_OK) return rc;
    if (least == 0) return fail(RPTB_ERR_BAD_ARG, "Pixel found with no samples");  // buffer.rs:89
    if (least < 2) return fail(RPTB_ERR_BAD_ARG, "a pixel has fewer than 2 entries (no variance to guide the filter)");
    return RPTB_OK;
}

int rptb_buffer_denoise(rptb_buffer* b, const rptb_denoise* d, double* out_rgb, uint8_t* out_rgb8) {
    if (!b) return fail(RPTB_ERR_BAD_ARG, "null argument");
    int rc = check_denoise(d);
    if (rc != RPTB_OK) return rc;
    if (b->shard) return refuse_shard("denoise");
    std::lock_guard<std::mutex> bl(b->lock);
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    FilterPlanes f;
    rc = check_denoise_entries(b);
    if (rc == RPTB_OK) rc = filter_planes(b, false, &f);
    if (rc == RPTB_OK) rc = check_denoise_counts(b);
    if (rc != RPTB_OK) return rc;
    const size_t npix = (size_t)b->width * b->height;
    uint32_t launches = 0;
    CU(launch_denoise(b->rows.sums, b->rows.m2, b->rows.counts, f.a.normal, f.a.depth, f.a.albedo, b->width, b->height, *d, f.col, f.var,
                      f.out, q0.stream, &launches));
    if (out_rgb) CU(cudaMemcpyAsync(out_rgb, f.out, npix * 3 * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    if (out_rgb8) {
        // the film resolve of one entry at radius 0: clamp, gamma and the truncating cast of Buffer::image
        CU(launch_film_resolve(f.out, 1u, b->width, b->height, 0u, b->rgb8, q0.stream));
        CU(cudaMemcpyAsync(out_rgb8, b->rgb8, npix * 3, cudaMemcpyDeviceToHost, q0.stream));
    }
    CU(cudaStreamSynchronize(q0.stream));
    return RPTB_OK;
}

// rptb_buffer_denoise_variance (v') and rptb_buffer_denoise_error (`error`: E), copied to out.
static int denoise_read(rptb_buffer* b, const rptb_denoise& d, bool error, double* out) {
    std::lock_guard<std::mutex> bl(b->lock);
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    Aov a;
    const double *icol, *ivar;
    uint32_t launches = 0;
    int rc = check_denoise_entries(b);
    if (rc == RPTB_OK) rc = buffer_filter(b, d, error, &a, &icol, &ivar, &launches);
    if (rc == RPTB_OK) rc = check_denoise_counts(b);
    if (rc != RPTB_OK) return rc;
    CU(cudaMemcpyAsync(out, ivar, (size_t)b->width * b->height * sizeof(double), cudaMemcpyDeviceToHost, q0.stream));
    CU(cudaStreamSynchronize(q0.stream));
    return RPTB_OK;
}

int rptb_buffer_denoise_variance(rptb_buffer* b, const rptb_denoise* d, double* out_var) {
    if (!b || !out_var) return fail(RPTB_ERR_BAD_ARG, "null argument");
    int rc = check_denoise(d);
    if (rc != RPTB_OK) return rc;
    if (b->shard) return refuse_shard("denoise_variance");
    return denoise_read(b, *d, false, out_var);
}

int rptb_buffer_half_sums(rptb_buffer* b, double* out) {
    if (!b || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (!b->halves) return fail(RPTB_ERR_BAD_ARG, "the buffer has no halves (rptb_buffer_create_halves)");
    std::lock_guard<std::mutex> bl(b->lock);
    BufferPart& q0 = b->parts[0];
    DeviceGuard g(q0.device);
    const int rc = buffer_gather(b, 1u << HALF);
    if (rc != RPTB_OK) return rc;
    CU(cudaMemcpyAsync(out, b->rows.half, plane_bytes(HALF, (size_t)b->width * b->height), cudaMemcpyDeviceToHost, q0.stream));
    CU(cudaStreamSynchronize(q0.stream));
    return RPTB_OK;
}

int rptb_buffer_denoise_error(rptb_buffer* b, const rptb_denoise* d, double* out) {
    if (!b || !out) return fail(RPTB_ERR_BAD_ARG, "null argument");
    int rc = check_denoise(d);
    if (rc != RPTB_OK) return rc;
    if (d->iterations == 0) return fail(RPTB_ERR_BAD_ARG, "iterations 0: the error estimate needs at least one filter pass");
    if (b->shard) return refuse_shard("denoise_error");
    if (!b->halves) return fail(RPTB_ERR_BAD_ARG, "the buffer has no halves (rptb_buffer_create_halves)");
    return denoise_read(b, *d, true, out);
}

// What a reprojection checks before it looks at the buffers: its arguments and parameters.
static int check_reproject_params(const rptb_buffer* dst, const rptb_buffer* src, const rptb_reproject* prm) {
    if (!dst || !src || !prm) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (dst == src) return fail(RPTB_ERR_BAD_ARG, "src and dst are the same buffer");
    if (!(std::isfinite(prm->depth_tol) && prm->depth_tol >= 0.0))
        return fail(RPTB_ERR_BAD_ARG, "depth_tol must be finite and >= 0 (%g)", prm->depth_tol);
    if (!(prm->normal_cos >= -1.0 && prm->normal_cos <= 1.0)) return fail(RPTB_ERR_BAD_ARG, "normal_cos must lie in [-1, 1] (%g)", prm->normal_cos);
    if (prm->max_history < 2) return fail(RPTB_ERR_BAD_ARG, "max_history %u < 2 (a pixel's variance needs two entries)", prm->max_history);
    return RPTB_OK;
}

// What a reprojection checks of the buffers (both locked): dst has no halves (history has none; a halves src is fine),
// features and no entries (a merge's dst: see check_merge_dst instead), src has entries and features made through one
// camera, and neither camera has an open aperture.
static int check_reproject_buffers(const rptb_buffer* dst, const rptb_buffer* src, bool merge) {
    if (dst->halves) return fail(RPTB_ERR_UNSUPPORTED, "dst has halves: reprojected history has no halves (a halves src is fine)");
    if (!merge && dst->entries) return fail(RPTB_ERR_BAD_ARG, "dst already holds entries");
    if (dst->feature_rays == 0) return fail(RPTB_ERR_BAD_ARG, "dst holds no features (rptb_buffer_add_features)");
    if (src->entries == 0) return fail(RPTB_ERR_BAD_ARG, "src holds no entries");
    if (src->feature_rays == 0) return fail(RPTB_ERR_BAD_ARG, "src holds no features (rptb_buffer_add_features)");
    const char* why[] = {"none", "one", "mixed (several cameras)", "unknown (a host entry)"};
    if (src->entry_cam.state != CameraRecord::ONE)
        return fail(RPTB_ERR_BAD_ARG, "src's entries have no single camera: %s", why[src->entry_cam.state]);
    if (src->feat_cam.state != CameraRecord::ONE)
        return fail(RPTB_ERR_BAD_ARG, "src's features have no single camera: %s", why[src->feat_cam.state]);
    if (dst->feat_cam.state != CameraRecord::ONE)
        return fail(RPTB_ERR_BAD_ARG, "dst's features have no single camera: %s", why[dst->feat_cam.state]);
    if (std::memcmp(&src->entry_cam.cam, &src->feat_cam.cam, sizeof(rptb_camera)) != 0)
        return fail(RPTB_ERR_BAD_ARG, "src's entries and features were made through different cameras");
    if (src->feat_cam.cam.aperture > 0.0 || dst->feat_cam.cam.aperture > 0.0)
        return fail(RPTB_ERR_UNSUPPORTED, "an open aperture: depth of field blurs the first hits, no one point to reproject");
    return RPTB_OK;
}

// What a merge checks of dst (locked) after check_reproject_buffers: fresh entries of its own view to test the history
// against -- at least 2 calls, so that every pixel of a never-reprojected buffer holds n_f >= 2 (rptb_buffer_denoise),
// none of them reprojected, all through dst's feature camera -- and room for the history's count.
static int check_merge_dst(const rptb_buffer* dst, const rptb_reproject* prm) {
    if (dst->entries < 2)
        return fail(RPTB_ERR_BAD_ARG, "dst holds %u entry calls: testing history needs >= 2 fresh ones (a mean and a variance)", dst->entries);
    if (dst->reprojected) return fail(RPTB_ERR_BAD_ARG, "dst is already reprojected: its entries are not all fresh");
    const char* why[] = {"none", "one", "mixed (several cameras)", "unknown (a host entry)"};
    if (dst->entry_cam.state != CameraRecord::ONE)
        return fail(RPTB_ERR_BAD_ARG, "dst's entries have no single camera: %s", why[dst->entry_cam.state]);
    if (std::memcmp(&dst->entry_cam.cam, &dst->feat_cam.cam, sizeof(rptb_camera)) != 0)
        return fail(RPTB_ERR_BAD_ARG, "dst's entries and features were made through different cameras");
    if (dst->entries > UINT32_MAX - prm->max_history) return fail(RPTB_ERR_UNSUPPORTED, "too many entries");
    return RPTB_OK;
}

// src's state and resolved features, row-major on its parts[0]'s device (current), enqueued on that part's stream with
// its `done` recorded behind them.
static int reproject_source(rptb_buffer* src, ReprojectSource* out) {
    BufferPart& s0 = src->parts[0];
    const size_t snpix = (size_t)src->width * src->height;
    const int rc = buffer_gather(src, COLOUR | FEATURES);
    if (rc != RPTB_OK) return rc;
    const Aov sa = buffer_aov(src);
    CU(launch_features_resolve(feature_planes(src->rows.feat, snpix), snpix, (double)src->feature_rays, sa, s0.stream));
    CU(cudaEventRecord(s0.done, s0.stream));
    *out = {src->rows.sums, src->rows.m2, src->rows.counts, sa.normal, sa.depth, sa.frac};
    return RPTB_OK;
}

// The counters (reused pixels, then a merge's rejected ones) and the least count of a reprojected buffer, on parts[0]'s
// device (current).
static int reproject_scratch_alloc(rptb_buffer* dst) {
    if (!dst->reused) CU(own(dst->mem, &dst->reused, 2 * sizeof(unsigned long long)));
    if (!dst->min_count) CU(own(dst->mem, &dst->min_count, sizeof(uint32_t)));
    return RPTB_OK;
}

// The state a reprojection leaves dst in, and its counts (waited for on `stream`) when asked: a reprojection's entries
// are max_history, a merge adds max_history to the fresh ones (both bounds); dst's entries now belong to its feature camera.
static int reproject_finish(rptb_buffer* dst, const rptb_reproject* prm, bool merge, uint64_t* out_reused, uint64_t* out_rejected,
                            cudaStream_t stream) {
    dst->entries = merge ? dst->entries + prm->max_history : prm->max_history;
    dst->reprojected = true;
    dst->entry_cam = dst->feat_cam;
    dst->state++;
    if (out_reused || out_rejected) {
        unsigned long long n[2] = {0, 0};
        CU(cudaMemcpyAsync(n, dst->reused, (merge ? 2 : 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
        if (out_reused) *out_reused = n[0];
        if (out_rejected) *out_rejected = n[1];
    }
    return RPTB_OK;
}

// rptb_buffer_reproject and rptb_buffer_reproject_shard (gamma null), rptb_buffer_reproject_merge and
// rptb_buffer_reproject_merge_shard (*gamma the test's threshold); shard_entry: the _shard entry points, whose dst is a
// shard buffer on src's first device.  Every dst part with tiles runs the per-element kernel over its own compact tiles
// against src's gathered row-major state: part 0 in place, any other (on another device, no peer access assumed) through
// the staging on parts[0]'s device.
static int reproject_impl(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* prm, const double* gamma, uint64_t* out_reused,
                          uint64_t* out_rejected, bool shard_entry) {
    int rc = check_reproject_params(dst, src, prm);
    if (rc != RPTB_OK) return rc;
    if (gamma && !(*gamma >= 0.0)) return fail(RPTB_ERR_BAD_ARG, "gamma must be >= 0 (%g)", *gamma);
    if (shard_entry && !dst->shard)
        return fail(RPTB_ERR_BAD_ARG, "dst is not a shard buffer (rptb_buffer_create_shard): a whole one reprojects with %s",
                    gamma ? "rptb_buffer_reproject_merge" : "rptb_buffer_reproject");
    if ((dst->shard && !shard_entry) || src->shard) return refuse_shard(gamma ? "reproject_merge" : "reproject");
    std::scoped_lock both(dst->lock, src->lock);
    BufferPart& d0 = dst->parts[0];
    BufferPart& s0 = src->parts[0];
    if (shard_entry && s0.device != d0.device)
        return fail(RPTB_ERR_BAD_ARG, "src's first device %d is not the shard's device %d", s0.device, d0.device);
    bool same = dst->parts.size() == src->parts.size();
    for (size_t i = 0; same && i < dst->parts.size(); i++) same = dst->parts[i].device == src->parts[i].device;
    if (!shard_entry && !same) return fail(RPTB_ERR_BAD_ARG, "the buffers were created on scenes with different device lists");
    rc = check_reproject_buffers(dst, src, gamma != nullptr);
    if (rc == RPTB_OK && gamma) rc = check_merge_dst(dst, prm);
    if (rc != RPTB_OK) return rc;
    DeviceGuard g(d0.device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", d0.device);
    rc = reproject_scratch_alloc(dst);
    if (rc != RPTB_OK) return rc;
    if (!d0.tiles) {  // a shard with no pixel to reproject: the state alone, so that its exchange block agrees with the others'
        if (out_reused) *out_reused = 0;
        if (out_rejected) *out_rejected = 0;
        return reproject_finish(dst, prm, gamma != nullptr, nullptr, nullptr, d0.stream);
    }
    size_t most = 0;  // the staging holds the largest other part
    for (size_t i = 1; i < dst->parts.size(); i++) most = std::max(most, (size_t)dst->parts[i].tiles * 128u);
    if (most) rc = planes_alloc(dst->mem, dst->staging, most, COLOUR | FEATURES);
    const bool count = out_reused || out_rejected;
    ReprojectSource sp;
    if (rc == RPTB_OK) rc = reproject_source(src, &sp);
    if (rc != RPTB_OK) return rc;
    CU(cudaStreamWaitEvent(d0.stream, s0.done, 0));
    if (count) CU(cudaMemsetAsync(dst->reused, 0, (gamma ? 2 : 1) * sizeof(unsigned long long), d0.stream));
    const ReprojectView dv = reproject_view(dst->feat_cam.cam, dst->width, dst->height);
    const ReprojectView sv = reproject_view(src->feat_cam.cam, src->width, src->height);
    const uint32_t in = gamma ? COLOUR | FEATURES : FEATURES;  // a merge reads the fresh colour; a reprojection writes it all
    for (size_t i = 0; rc == RPTB_OK && i < dst->parts.size(); i++) {
        const BufferPart& q = dst->parts[i];
        if (!q.tiles) continue;
        CU(cudaStreamWaitEvent(d0.stream, q.done, 0));
        const Planes& p = i == 0 ? q.planes : dst->staging;
        if (i > 0) rc = copy_planes(p.set(in), d0.device, q.planes.set(in), q.device, q.planes.n, d0.stream);
        if (rc != RPTB_OK) return rc;
        const FeaturePlanes f = feature_planes(p.feat, p.n);
        if (gamma)
            CU(launch_reproject_merge_part(dv, sv, sp, f, (double)dst->feature_rays, q.index, q.count, q.planes.n, *prm, *gamma, p.sums,
                                           p.m2, p.counts, count ? dst->reused : nullptr, d0.stream));
        else
            CU(launch_reproject_part(dv, sv, sp, f, (double)dst->feature_rays, q.index, q.count, q.planes.n, *prm, p.sums, p.m2, p.counts,
                                     count ? dst->reused : nullptr, d0.stream));
        if (i > 0) rc = copy_planes(q.planes.set(COLOUR), q.device, p.set(COLOUR), d0.device, q.planes.n, d0.stream);
    }
    // every later call on either buffer is ordered behind this one
    if (rc == RPTB_OK) rc = buffer_order_behind(dst, d0.stream);
    if (rc == RPTB_OK) rc = buffer_order_behind(src, d0.stream);
    if (rc != RPTB_OK) return rc;
    return reproject_finish(dst, prm, gamma != nullptr, out_reused, out_rejected, d0.stream);
}

int rptb_buffer_reproject(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* prm, uint64_t* out_reused) {
    return reproject_impl(dst, src, prm, nullptr, out_reused, nullptr, false);
}

int rptb_buffer_reproject_shard(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* prm, uint64_t* out_reused) {
    return reproject_impl(dst, src, prm, nullptr, out_reused, nullptr, true);
}

int rptb_buffer_reproject_merge(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* prm, double gamma, uint64_t* out_reused,
                                uint64_t* out_rejected) {
    return reproject_impl(dst, src, prm, &gamma, out_reused, out_rejected, false);
}

int rptb_buffer_reproject_merge_shard(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* prm, double gamma, uint64_t* out_reused,
                                      uint64_t* out_rejected) {
    return reproject_impl(dst, src, prm, &gamma, out_reused, out_rejected, true);
}

uint64_t rptb_buffer_shard_bytes(const rptb_buffer* b, uint32_t with_features) {
    if (!b || !b->shard) return 0;
    return shard_layout(b->width, b->height, b->parts[0].count, with_features != 0).bytes;
}

int rptb_buffer_export_shard(rptb_buffer* b, void* dst_device, uint32_t with_features, void* stream) {
    if (!b || !dst_device) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (!b->shard) return fail(RPTB_ERR_BAD_ARG, "not a shard buffer (rptb_buffer_create_shard)");
    std::lock_guard<std::mutex> bl(b->lock);
    if (with_features && b->feature_rays == 0) return fail(RPTB_ERR_BAD_ARG, "the buffer holds no features (rptb_buffer_add_features)");
    BufferPart& q = b->parts[0];
    DeviceGuard g(q.device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", q.device);
    const ShardLayout l = shard_layout(b->width, b->height, q.count, with_features != 0);
    ShardHeader h;
    std::memset(&h, 0, sizeof(h));
    h.magic = kShardMagic;
    h.with_features = with_features ? 1u : 0u;
    h.width = b->width;
    h.height = b->height;
    h.shard_index = q.index;
    h.shard_count = q.count;
    h.entries = b->entries;
    h.flags = b->reprojected ? kShardReprojected : 0u;
    h.feature_rays = b->feature_rays;
    h.entry_cam = shard_camera(b->entry_cam);
    h.feat_cam = shard_camera(b->feat_cam);
    cudaStream_t st = stream ? (cudaStream_t)stream : q.stream;
    CU(cudaStreamWaitEvent(st, q.done, 0));
    // pageable source: the call returns once the header is staged
    CU(cudaMemcpyAsync(dst_device, &h, sizeof(h), cudaMemcpyHostToDevice, st));
    // the part's planes are q.planes.n long, the block's l.slots
    const PlaneSet to = shard_planes(l, dst_device), from = q.planes.set(l.mask);
    for (int k = 0; k < NPLANES; k++)
        if (to.p[k] && q.tiles) CU(cudaMemcpyAsync(to.p[k], from.p[k], plane_bytes(k, q.planes.n), cudaMemcpyDeviceToDevice, st));
    // a later accumulate into the part waits until the block is read
    CU(cudaEventRecord(q.done, st));
    if (!stream) CU(cudaStreamSynchronize(st));
    b->exported = b->state;
    return RPTB_OK;
}

int rptb_buffer_import_shards(rptb_buffer* dst, const void* gathered_device, uint32_t shard_count, uint32_t with_features) {
    if (!dst || !gathered_device) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (shard_count == 0) return fail(RPTB_ERR_BAD_ARG, "shard_count 0");
    if (dst->shard) return fail(RPTB_ERR_BAD_ARG, "dst is a shard buffer: the shards gather into a whole buffer (rptb_buffer_create)");
    if (dst->halves) return fail(RPTB_ERR_UNSUPPORTED, "dst has halves: shards carry no halves");
    std::lock_guard<std::mutex> bl(dst->lock);
    BufferPart& d0 = dst->parts[0];
    DeviceGuard g(d0.device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", d0.device);
    const uint32_t W = dst->width, H = dst->height;
    const ShardLayout l = shard_layout(W, H, shard_count, with_features != 0);
    const char* in = (const char*)gathered_device;
    // header 0 first: only once it names dst's size, shard_count and with_features is the block stride known to be right
    std::vector<ShardHeader> hs(shard_count);
    CU(cudaMemcpyAsync(hs.data(), in, sizeof(ShardHeader), cudaMemcpyDeviceToHost, d0.stream));
    CU(cudaStreamSynchronize(d0.stream));
    const ShardHeader& h0 = hs[0];
    if (h0.magic != kShardMagic) return fail(RPTB_ERR_BAD_ARG, "block 0 is not a shard block (rptb_buffer_export_shard)");
    if (h0.width != W || h0.height != H)
        return fail(RPTB_ERR_BAD_ARG, "the shards are %ux%u but dst is %ux%u", h0.width, h0.height, W, H);
    if (h0.shard_count != shard_count) return fail(RPTB_ERR_BAD_ARG, "the shards are %u but shard_count is %u", h0.shard_count, shard_count);
    if (h0.with_features != (with_features ? 1u : 0u))
        return fail(RPTB_ERR_BAD_ARG, "the shards were exported %s features", h0.with_features ? "with" : "without");
    if (h0.flags & ~kShardReprojected) return fail(RPTB_ERR_BAD_ARG, "block 0 carries unknown flags 0x%x", h0.flags);
    if (shard_count > 1)
        CU(cudaMemcpy2DAsync(hs.data() + 1, sizeof(ShardHeader), in + l.bytes, l.bytes, sizeof(ShardHeader), shard_count - 1,
                             cudaMemcpyDeviceToHost, d0.stream));
    CU(cudaStreamSynchronize(d0.stream));
    for (uint32_t i = 0; i < shard_count; i++) {
        const ShardHeader& h = hs[i];
        if (h.magic != kShardMagic) return fail(RPTB_ERR_BAD_ARG, "block %u is not a shard block (rptb_buffer_export_shard)", i);
        if (h.shard_index != i) return fail(RPTB_ERR_BAD_ARG, "block %u holds shard %u: the shards must be in order 0..%u", i, h.shard_index, shard_count - 1);
        if (h.width != W || h.height != H || h.shard_count != shard_count || h.with_features != h0.with_features)
            return fail(RPTB_ERR_BAD_ARG, "block %u was exported from another image, shard count or feature choice", i);
        if (h.entries != h0.entries || h.flags != h0.flags || h.feature_rays != h0.feature_rays ||
            std::memcmp(&h.entry_cam, &h0.entry_cam, sizeof(ShardCamera)) != 0 ||
            std::memcmp(&h.feat_cam, &h0.feat_cam, sizeof(ShardCamera)) != 0)
            return fail(RPTB_ERR_BAD_ARG,
                        "shard %u received other calls than shard 0 (entries %u / %u, reprojected %u / %u, feature rays %llu / %llu, or "
                        "cameras)",
                        i, h.entries, h0.entries, h.flags & kShardReprojected, h0.flags & kShardReprojected,
                        (unsigned long long)h.feature_rays, (unsigned long long)h0.feature_rays);
    }
    // everything dst holds is overwritten: its earlier work finishes first
    dst->state++;
    for (BufferPart& q : dst->parts) CU(cudaStreamWaitEvent(d0.stream, q.done, 0));
    for (BufferPart& q : dst->parts) {
        DeviceGuard gq(q.device);
        if (with_features && q.tiles) {
            const int rc = planes_alloc(q.mem, q.planes, (size_t)q.tiles * 128u, FEATURES);
            if (rc != RPTB_OK) return rc;
        } else if (!with_features && q.planes.feat) {  // dst holds no features afterwards; the next feature pass starts from zero
            CU(cudaEventSynchronize(q.done));
            CU(cudaFree(q.planes.feat));
            q.mem.erase(std::find(q.mem.begin(), q.mem.end(), (void*)q.planes.feat));
            q.planes.feat = nullptr;
        }
    }
    // every block row-major on dst's first device, then back into dst's own parts; every later call on dst is ordered
    // behind this one
    const bool reprojected = (h0.flags & kShardReprojected) != 0;
    int rc = buffer_rows_alloc(dst, l.mask);
    if (rc == RPTB_OK && reprojected) rc = reproject_scratch_alloc(dst);
    for (uint32_t i = 0; rc == RPTB_OK && i < shard_count; i++)
        rc = buffer_scatter(dst, shard_planes(l, in + (size_t)i * l.bytes), l.mask, i, shard_count);
    if (rc == RPTB_OK) rc = buffer_write_back(dst, l.mask);
    if (rc == RPTB_OK) rc = buffer_order_behind(dst, d0.stream);
    if (rc != RPTB_OK) return rc;
    // the caller may reuse the gathered bytes when the call returns
    CU(cudaStreamSynchronize(d0.stream));
    dst->entries = h0.entries;
    dst->reprojected = reprojected;
    dst->entry_cam = camera_record(h0.entry_cam);
    dst->feature_rays = with_features ? h0.feature_rays : 0;
    dst->feat_cam = with_features ? camera_record(h0.feat_cam) : CameraRecord();
    dst->imported = dst->state;
    dst->imported_shards = shard_count;
    return RPTB_OK;
}

uint64_t rptb_delta_bytes(uint32_t capacity) { return delta_bytes(capacity); }

int rptb_buffer_export_delta(rptb_buffer* b, void* dst_device, uint32_t capacity, void* stream, uint32_t* out_pixels) {
    if (!b || !dst_device) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (!b->shard) return fail(RPTB_ERR_BAD_ARG, "not a shard buffer (rptb_buffer_create_shard)");
    std::lock_guard<std::mutex> bl(b->lock);
    if (b->masked != b->state || b->exported + 1 != b->state)
        return fail(RPTB_ERR_BAD_ARG, "no delta to export: the shard's last call must be an adaptive or guided entry made right after an "
                                      "export, keeping its entry camera; gather the full block (rptb_buffer_export_shard)");
    BufferPart& q = b->parts[0];
    DeviceGuard g(q.device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", q.device);
    cudaStream_t st = stream ? (cudaStream_t)stream : q.stream;
    CU(cudaStreamWaitEvent(st, q.done, 0));
    unsigned long long n = 0;  // the pixels the call changed: its active count
    CU(cudaMemcpyAsync(&n, q.active, sizeof(n), cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    if (n > capacity) return fail(RPTB_ERR_BAD_ARG, "capacity %u is below the %llu pixels the shard's last call changed", capacity, n);
    const uint64_t nelem = (uint64_t)q.tiles * 128u;
    if (nelem && !q.delta_len) {
        q.delta_temp_bytes = delta_temp_bytes(nelem);
        CU(own(q.mem, &q.delta_len, sizeof(uint32_t)));
        CU(own(q.mem, &q.delta_temp, q.delta_temp_bytes ? q.delta_temp_bytes : 1));
    }
    DeltaHeader h;
    std::memset(&h, 0, sizeof(h));
    h.magic = kDeltaMagic;
    h.width = b->width;
    h.height = b->height;
    h.shard_index = q.index;
    h.shard_count = q.count;
    h.entries_before = b->entries - 1;
    h.entries_after = b->entries;
    h.flags = b->reprojected ? kShardReprojected : 0u;
    h.feature_rays = b->feature_rays;
    h.entry_cam = shard_camera(b->entry_cam);
    h.feat_cam = shard_camera(b->feat_cam);
    h.pixels = (uint32_t)n;
    h.capacity = capacity;
    // pageable source: the call returns once the header is staged
    CU(cudaMemcpyAsync(dst_device, &h, sizeof(h), cudaMemcpyHostToDevice, st));
    CU(launch_delta_export(q.mask, nelem, q.planes.sums, q.planes.m2, q.planes.counts, dst_device, capacity, (uint32_t)n, q.delta_len,
                           q.delta_temp, q.delta_temp_bytes, st));
    // a later mark or accumulate into the part waits until the block is written
    CU(cudaEventRecord(q.done, st));
    if (!stream) CU(cudaStreamSynchronize(st));
    b->exported = b->state;
    if (out_pixels) *out_pixels = (uint32_t)n;
    return RPTB_OK;
}

int rptb_buffer_import_deltas(rptb_buffer* dst, const void* gathered_device, uint32_t shard_count, uint32_t capacity) {
    if (!dst || !gathered_device) return fail(RPTB_ERR_BAD_ARG, "null argument");
    if (shard_count == 0) return fail(RPTB_ERR_BAD_ARG, "shard_count 0");
    if (dst->shard) return fail(RPTB_ERR_BAD_ARG, "dst is a shard buffer: the deltas go into the shards' gathered whole buffer");
    if (dst->halves) return fail(RPTB_ERR_UNSUPPORTED, "dst has halves: shards carry no halves");
    if (dst->parts.size() != 1)
        return fail(RPTB_ERR_UNSUPPORTED, "dst has %zu parts: deltas are imported into a one-part whole buffer", dst->parts.size());
    std::lock_guard<std::mutex> bl(dst->lock);
    BufferPart& d0 = dst->parts[0];
    DeviceGuard g(d0.device);
    if (!g.ok) return fail(RPTB_ERR_CUDA, "cudaSetDevice(%d) failed", d0.device);
    const uint32_t W = dst->width, H = dst->height;
    const uint64_t bytes = delta_bytes(capacity);
    const char* in = (const char*)gathered_device;
    // header 0 first: only once it names dst's size, shard_count and capacity is the block stride known to be right
    std::vector<DeltaHeader> hs(shard_count);
    CU(cudaMemcpyAsync(hs.data(), in, sizeof(DeltaHeader), cudaMemcpyDeviceToHost, d0.stream));
    CU(cudaStreamSynchronize(d0.stream));
    const DeltaHeader& h0 = hs[0];
    if (h0.magic != kDeltaMagic) return fail(RPTB_ERR_BAD_ARG, "block 0 is not a delta block (rptb_buffer_export_delta)");
    if (h0.width != W || h0.height != H) return fail(RPTB_ERR_BAD_ARG, "the deltas are %ux%u but dst is %ux%u", h0.width, h0.height, W, H);
    if (h0.shard_count != shard_count) return fail(RPTB_ERR_BAD_ARG, "the deltas are of %u shards but shard_count is %u", h0.shard_count, shard_count);
    if (h0.capacity != capacity) return fail(RPTB_ERR_BAD_ARG, "the deltas have capacity %u but capacity is %u", h0.capacity, capacity);
    if (shard_count > 1)
        CU(cudaMemcpy2DAsync(hs.data() + 1, sizeof(DeltaHeader), in + bytes, bytes, sizeof(DeltaHeader), shard_count - 1,
                             cudaMemcpyDeviceToHost, d0.stream));
    CU(cudaStreamSynchronize(d0.stream));
    for (uint32_t i = 0; i < shard_count; i++) {
        const DeltaHeader& h = hs[i];
        if (h.magic != kDeltaMagic) return fail(RPTB_ERR_BAD_ARG, "block %u is not a delta block (rptb_buffer_export_delta)", i);
        if (h.shard_index != i)
            return fail(RPTB_ERR_BAD_ARG, "block %u holds shard %u: the shards must be in order 0..%u", i, h.shard_index, shard_count - 1);
        if (h.width != W || h.height != H || h.shard_count != shard_count || h.capacity != capacity)
            return fail(RPTB_ERR_BAD_ARG, "block %u was exported for another image, shard count or capacity", i);
        if (h.pixels > capacity) return fail(RPTB_ERR_BAD_ARG, "block %u holds %u pixels, more than its capacity %u", i, h.pixels, capacity);
        if (h.entries_before != h0.entries_before || h.entries_after != h0.entries_after || h.flags != h0.flags ||
            h.feature_rays != h0.feature_rays || std::memcmp(&h.entry_cam, &h0.entry_cam, sizeof(ShardCamera)) != 0 ||
            std::memcmp(&h.feat_cam, &h0.feat_cam, sizeof(ShardCamera)) != 0)
            return fail(RPTB_ERR_BAD_ARG,
                        "shard %u received other calls than shard 0 (entries %u -> %u / %u -> %u, reprojected %u / %u, feature rays "
                        "%llu / %llu, or cameras)",
                        i, h.entries_before, h.entries_after, h0.entries_before, h0.entries_after, h.flags & kShardReprojected,
                        h0.flags & kShardReprojected, (unsigned long long)h.feature_rays, (unsigned long long)h0.feature_rays);
    }
    // dst must hold the shards' state before the call: an import of them, untouched since.  The entry camera before the call
    // is the one after it, or none before the first entry (rptb_buffer_export_delta refuses any other change).
    const CameraRecord after_cam = camera_record(h0.entry_cam);
    const CameraRecord before_cam = h0.entries_before == 0 ? CameraRecord() : after_cam;
    const bool reprojected = (h0.flags & kShardReprojected) != 0;
    if (dst->imported != dst->state || dst->imported_shards != shard_count)
        return fail(RPTB_ERR_BAD_ARG, "dst was not last written by an import of the %u shards (rptb_buffer_import_shards or "
                                      "rptb_buffer_import_deltas); gather the full blocks", shard_count);
    if (dst->entries != h0.entries_before || dst->reprojected != reprojected || dst->feature_rays != h0.feature_rays ||
        !same_camera(dst->entry_cam, before_cam) || !same_camera(dst->feat_cam, camera_record(h0.feat_cam)))
        return fail(RPTB_ERR_BAD_ARG,
                    "dst is not at the shards' state before the call (entries %u / %u, reprojected %d / %d, feature rays %llu / %llu, or "
                    "cameras); gather the full blocks",
                    dst->entries, h0.entries_before, (int)dst->reprojected, (int)reprojected, (unsigned long long)dst->feature_rays,
                    (unsigned long long)h0.feature_rays);
    // in place in dst's compact planes; every later call on dst is ordered behind it
    dst->state++;
    CU(cudaStreamWaitEvent(d0.stream, d0.done, 0));
    CU(launch_delta_import(in, shard_count, capacity, d0.planes.sums, d0.planes.m2, d0.planes.counts, d0.stream));
    CU(cudaEventRecord(d0.done, d0.stream));
    // the caller may reuse the gathered bytes when the call returns
    CU(cudaStreamSynchronize(d0.stream));
    dst->entries = h0.entries_after;
    dst->entry_cam = after_cam;
    dst->imported = dst->state;
    return RPTB_OK;
}

}  // extern "C"
