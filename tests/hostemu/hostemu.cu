// hostemu.cu -- TEST INFRASTRUCTURE, NOT PRODUCT.  Never linked into librpt_b200.so, never loaded by
// rpt_b200/*: only tests/test_hostemu.py builds and loads it.
//
// The device functions of rpt_b200/csrc (geometry.cuh, shading.cuh: the code the CUDA kernels inline; and
// render_thread of integrator.cuh: the whole body of the path-tracing megakernel, run one lane at a time
// with a single-lane warp policy) compiled for the HOST with RPTB_HOST_EMU, over the very arrays
// rptb_scene_create would upload (flatten.h), so that their control flow -- kd traversal, the kd-tree of
// shapes, MonomialSurface, Transformed, finalize_hit, shape_sample -- can be checked against the oracle
// on a machine without a GPU.  It proves nothing about the kernels' scheduling, fast-math
// or memory behaviour; the `-m gpu` parity tests through the C ABI stay the gate.
//
// Built by `make hostemu` with nvcc (host pass) and -ffp-contract=off so Real = double rounds like the
// f64 parity kernels (-fmad=false).
#ifndef RPTB_HOST_EMU
#error "compile with -DRPTB_HOST_EMU"
#endif
#include <cstring>
#include <new>
#include <string>
#include <type_traits>

#include "../../rpt_b200/csrc/flatten.h"
#include "../../rpt_b200/csrc/integrator.cuh"
#include "../../rpt_b200/csrc/integrator_vx.cuh"
#include "../../rpt_b200/csrc/launch.h"

using namespace rptb;

namespace {

// bind_scene's "uploader": the arrays stay where they are
struct InPlace {
    uint64_t total = 0;
    template <class T>
    bool operator()(std::vector<T>& host, const T** where) {
        *where = host.empty() ? nullptr : host.data();
        total += host.size() * sizeof(T);
        return true;
    }
    uint64_t bytes() const { return total; }
};

// Shadow queries as sample_lights issues them (renderer.rs:190-197 through the megakernel's any-hit path):
// out[i] = 1 if something lies on ray i at t in [tmin, tmax[i]), found with `any` = true.
template <class R, int FEAT>
void occluded(const SceneView<R>& sv, const double* rays, const double* tmax, uint64_t n, double tmin, int32_t* out) {
#pragma omp parallel for schedule(static)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const double* r = rays + 6 * i;
        TravStats ts = {0, 0, 0, 0, 0};
        Hit<R> h;
        h.t = (R)tmax[i];
        closest_hit<R, false, FEAT>(sv, mk((R)r[0], (R)r[1], (R)r[2]), mk((R)r[3], (R)r[4], (R)r[5]), (R)tmin, true, h, ts);
        out[i] = h.obj >= 0 ? 1 : 0;
    }
}

template <class R, int FEAT>
void closest_hits(const SceneView<R>& sv, const double* rays, uint64_t n, double tmin, double* out_t, int32_t* out_obj,
                  double* out_n, uint32_t* out_aux, double* out_bvw, rptb_stats* stats) {
    unsigned long long nv = 0, tt = 0, ot = 0, bn = 0, bt = 0;
#pragma omp parallel for schedule(static) reduction(+ : nv, tt, ot, bn, bt)
    for (int64_t i = 0; i < (int64_t)n; i++) {  // body of closest_hit_kernel (integrator.cuh)
        const double* r = rays + 6 * i;
        const Vec3<R> o = {(R)r[0], (R)r[1], (R)r[2]};
        const Vec3<R> d = {(R)r[3], (R)r[4], (R)r[5]};
        TravStats ts = {0, 0, 0, 0, 0};
        Hit<R> h;
        h.t = M<R>::inf();
        closest_hit<R, true, FEAT>(sv, o, d, (R)tmin, false, h, ts);
        out_obj[i] = h.obj;
        out_t[i] = h.obj >= 0 ? (double)h.t : (double)INFINITY;
        if (out_aux) out_aux[i] = h.aux;  // which triangle / cube face: on a flat polygon the normal does not tell
        if (out_bvw) {
            out_bvw[2 * i] = (double)h.bv;
            out_bvw[2 * i + 1] = (double)h.bw;
        }
        if (out_n) {
            Vec3<R> nn = {(R)0, (R)0, (R)0};
            if (h.obj >= 0) nn = finalize_hit<R, FEAT>(sv, sv.objects[h.obj], o, d, h).n;
            out_n[3 * i] = (double)nn.x;
            out_n[3 * i + 1] = (double)nn.y;
            out_n[3 * i + 2] = (double)nn.z;
        }
        nv += ts.node_visits;
        tt += ts.tri_tests;
        ot += ts.object_tests;
        bn += ts.bvh_nodes;
        bt += ts.bvh_tris;
    }
    if (stats) {
        std::memset(stats, 0, sizeof(*stats));
        stats->rays = n;
        stats->node_visits = nv;
        stats->tri_tests = tt;
        stats->object_tests = ot;
        stats->bvh_node_visits = bn;
        stats->bvh_tri_tests = bt;
    }
}

template <class R>
void illuminations(const SceneView<R>& sv, uint32_t light, const double* pos, uint64_t n, uint64_t seed, double* out_i,
                   double* out_wi, double* out_dist) {
    for (uint64_t i = 0; i < n; i++) {  // same stream as oracle_illuminate: key (seed), pixel i, sample 0
        Rng<R> rng;
        rng.init(seed, (uint32_t)i, 0);
        Vec3<R> I, wi;
        R dist;
        illuminate<R, F_EVERY>(sv, sv.lights[light], mk((R)pos[3 * i], (R)pos[3 * i + 1], (R)pos[3 * i + 2]), rng, I, wi, dist);
        out_i[3 * i] = (double)I.x; out_i[3 * i + 1] = (double)I.y; out_i[3 * i + 2] = (double)I.z;
        out_wi[3 * i] = (double)wi.x; out_wi[3 * i + 1] = (double)wi.y; out_wi[3 * i + 2] = (double)wi.z;
        out_dist[i] = (double)dist;
    }
}

// The megakernel's warp policy for one lane run on its own: a vote over the warp is the lane's own
// predicate, a reduction its own value.  (The kernel's warp-level structure -- slot schedule, reconvergence,
// the shared Philox refill -- only changes WHEN lanes do things, never what a lane computes.)
struct HostLane {
    static __host__ __device__ unsigned activemask() { return 1u; }
    static __host__ __device__ bool all(unsigned, bool p) { return p; }
    static __host__ __device__ bool any(unsigned, bool p) { return p; }
    static constexpr uint32_t width = 1u;
    static __host__ __device__ unsigned ballot(unsigned, bool p) { return p ? 1u : 0u; }
    static __host__ __device__ uint32_t rank(unsigned, uint32_t) { return 0u; }  // lanes below me among the voters: none
    static __host__ __device__ uint32_t popc(unsigned v) { uint32_t c = 0; while (v) { c += v & 1u; v >>= 1; } return c; }
    static __host__ __device__ void sync(unsigned) {}
    static __host__ __device__ uint32_t reduce_add(unsigned, uint32_t v) { return v; }
    static __host__ __device__ bool is_leader(unsigned, uint32_t) { return true; }
    static __host__ __device__ void add(unsigned long long* p, unsigned long long v) {
#ifndef __CUDA_ARCH__
#pragma omp atomic
        *p += v;
#else
        (void)p, (void)v;
#endif
    }
};

template <class R, int MAXD, bool STATS, int FEAT>
void run_grid(const SceneView<R>& sv, const RenderArgs<R>& a) {
    const int64_t nblocks = (int64_t)a.ntiles_mine * a.ngroups;
#pragma omp parallel for schedule(dynamic, 1)
    for (int64_t b = 0; b < nblocks; b++) {
        const uint32_t bx = (uint32_t)(b % a.ntiles_mine), by = (uint32_t)(b / a.ntiles_mine);
        for (uint32_t t = 0; t < (uint32_t)RENDER_THREADS; t++) render_thread<R, MAXD, STATS, FEAT, HostLane>(sv, a, bx, by, t);
    }
    if (a.nchunks > 1) {
#pragma omp parallel for schedule(static)
        for (int64_t bx = 0; bx < (int64_t)a.ntiles_mine; bx++)
            for (uint32_t t = 0; t < (uint32_t)RENDER_THREADS; t++) resolve_chunks_thread<R>(a, (uint32_t)bx, t);
    }
}

// The vertex-at-once engine (integrator_vx.cuh), one lane at a time: the "warp" is one lane wide, so the compacted work
// list of a mesh holds just this lane's rays -- what a lane computes for a ray is what any lane of a real warp would.
template <bool STATS, int FEAT>
void run_grid_vx(const SceneView<float>& sv, const RenderArgs<float>& a) {
    const int64_t nblocks = (int64_t)a.ntiles_mine * a.ngroups;
    const size_t words = vx_shared_words(a.ks + 1u);
#pragma omp parallel for schedule(dynamic, 1)
    for (int64_t b = 0; b < nblocks; b++) {
        std::vector<float4> smem((words + 3) / 4);  // 16-byte aligned
        const uint32_t bx = (uint32_t)(b % a.ntiles_mine), by = (uint32_t)(b / a.ntiles_mine);
        for (uint32_t t = 0; t < (uint32_t)RENDER_THREADS; t++)
            render_thread_vx<STATS, FEAT, HostLane>(sv, a, bx, by, t, reinterpret_cast<uint32_t*>(smem.data()));
    }
    if (a.nchunks > 1) {
#pragma omp parallel for schedule(static)
        for (int64_t bx = 0; bx < (int64_t)a.ntiles_mine; bx++)
            for (uint32_t t = 0; t < (uint32_t)RENDER_THREADS; t++) resolve_chunks_thread<float>(a, (uint32_t)bx, t);
    }
}

// launch_render_vx_f32's dispatch (kernels_vx.cu, through launch.h).  Returns the FEAT it ran, -1 if that variant is not
// compiled.
inline int run_render_vx(const SceneView<float>& sv, const RenderArgs<float>& a, int stats, int features) {
    const Variant v = pick_render_vx(features, stats);
    if (!visit(RenderVariantsVx{}, v, [&](auto t) { using T = decltype(t); run_grid_vx<T::stats, T::feat>(sv, a); })) return -1;
    return v.feat;
}

// launch_render_impl's dispatch (launch_impl.cuh, through launch.h).  Returns the FEAT it ran, -1 if that variant is not
// compiled.
template <class R>
int run_render(const SceneView<R>& sv, const RenderArgs<R>& a, int stats, int features) {
    using List = std::conditional_t<M<R>::literal, RenderVariantsF64, RenderVariantsF32>;
    const Variant v = pick_render(features, stats, M<R>::literal, a.max_bounces);
    if (!visit(List{}, v, [&](auto t) { using T = decltype(t); run_grid<R, T::maxd, T::stats, T::feat>(sv, a); })) return -1;
    return v.feat;
}

// launch_closest_hit_impl's choice for rptb_closest_hit without counters (the any-hit queries take the same walk); the
// emulation always counts.  Returns the FEAT it ran, -1 if that variant is not compiled.
template <class R>
int run_closest_hits(const SceneView<R>& sv, int features, const double* rays, uint64_t n, double tmin, double* out_t,
                     int32_t* out_obj, double* out_n, uint32_t* out_aux, double* out_bvw, rptb_stats* stats) {
    using List = std::conditional_t<M<R>::literal, HitVariantsF64, HitVariantsF32>;
    const Variant v = pick_closest_hit(features, 0, M<R>::literal);
    if (!visit(List{}, v, [&](auto t) { closest_hits<R, decltype(t)::feat>(sv, rays, n, tmin, out_t, out_obj, out_n, out_aux, out_bvw, stats); }))
        return -1;
    return v.feat;
}

template <class R>
int run_occluded(const SceneView<R>& sv, int features, const double* rays, const double* tmax, uint64_t n, double tmin, int32_t* out) {
    using List = std::conditional_t<M<R>::literal, HitVariantsF64, HitVariantsF32>;
    const Variant v = pick_closest_hit(features, 0, M<R>::literal);
    if (!visit(List{}, v, [&](auto t) { occluded<R, decltype(t)::feat>(sv, rays, tmax, n, tmin, out); })) return -1;
    return v.feat;
}

template <class R>
int render_impl(const SceneView<R>& sv, const rptb_camera* cam, const rptb_render_params* p, int features, uint32_t sampled_lights,
                double* out_rgb, rptb_stats* stats) {
    RenderArgs<R> a;
    fill_args(cam, p, a);
    const size_t nvals = (size_t)p->width * p->height * 3;
    std::vector<R> out(nvals, (R)0);  // pixels of other shards stay zero (clear_kernel)
    std::vector<double> partial;
    if (a.nchunks > 1) partial.assign((size_t)a.nchunks * a.ntiles_mine * RENDER_THREADS * 3, 0.0);
    DeviceCounters counters;
    std::memset(&counters, 0, sizeof(counters));
    a.out = out.data();
    a.partial = partial.empty() ? nullptr : partial.data();
    a.counters = &counters;
    int feat = -1;
    if (a.ntiles_mine > 0) {
        bool vx = false;
        if constexpr (!M<R>::literal) {  // api.cu, render_launch: the vertex-at-once engine unless RPTB_VX=0 or a kd counting pass
            const char* e = getenv("RPTB_VX");
            a.ks = sampled_lights;
            vx = e && std::strcmp(e, "1") == 0 && sampled_lights <= VX_MAX_SHADOW && p->collect_stats != 2;
            if (vx) feat = run_render_vx(sv, a, (int)p->collect_stats, features);
        }
        if (!vx) feat = run_render<R>(sv, a, (int)p->collect_stats, features);
    }
    for (size_t i = 0; i < nvals; i++) out_rgb[i] = (double)out[i];
    if (stats) {
        std::memset(stats, 0, sizeof(*stats));
        stats->segments = counters.segments; stats->rays = counters.rays; stats->node_visits = counters.node_visits;
        stats->tri_tests = counters.tri_tests; stats->mesh_hits = counters.mesh_hits; stats->env_lookups = counters.env_lookups;
        stats->object_tests = counters.object_tests;
        stats->bvh_node_visits = counters.bvh_node_visits; stats->bvh_tri_tests = counters.bvh_tri_tests;
        stats->engine = RPTB_ENGINE_MEGAKERNEL;
    }
    return feat;
}

}  // namespace

extern "C" {

struct hostemu_scene {
    HostScene hs;
    SceneView<float> v32;
    SceneView<double> v64;
    int features;
};

// Returns NULL and writes the flattener's message to `err` on a bad description.
// The BVH of the f32 path is built iff desc->accel == RPTB_ACCEL_BVH (no environment, no default here).
hostemu_scene* hostemu_scene_create(const rptb_scene_desc* desc, char* err, size_t errlen) {
    hostemu_scene* s = new (std::nothrow) hostemu_scene();
    if (!s) return nullptr;
    std::memset(&s->v32, 0, sizeof(s->v32));
    std::memset(&s->v64, 0, sizeof(s->v64));
    std::string msg;
    if (flatten_scene(desc, s->hs, msg, desc->accel == RPTB_ACCEL_BVH) != RPTB_OK) {
        if (err && errlen) {
            std::strncpy(err, msg.c_str(), errlen - 1);
            err[errlen - 1] = 0;
        }
        delete s;
        return nullptr;
    }
    InPlace put;
    uint64_t f32_bytes = 0;
    bind_scene(s->hs, put, false, s->v32, s->v64, f32_bytes);
    s->features = kernel_features(s->hs);
    return s;
}

void hostemu_scene_destroy(hostemu_scene* s) { delete s; }

int hostemu_scene_features(const hostemu_scene* s) { return s->features; }

// precision: 0 = Real float, 1 = Real double (rptb_precision).  out_aux (n) and out_bvw (n x 2) may be null: the hit
// triangle or cube face, and the barycentrics (v, w) of a triangle hit.  Returns the FEAT of the walk, -1 if it is not
// compiled.
int hostemu_closest_hit(const hostemu_scene* s, const double* rays, uint64_t n, double t_min, uint32_t precision,
                        double* out_t, int32_t* out_object, double* out_normal, uint32_t* out_aux, double* out_bvw, rptb_stats* stats) {
    if (precision == RPTB_PRECISION_F64)
        return run_closest_hits<double>(s->v64, s->features, rays, n, t_min, out_t, out_object, out_normal, out_aux, out_bvw, stats);
    return run_closest_hits<float>(s->v32, s->features, rays, n, t_min, out_t, out_object, out_normal, out_aux, out_bvw, stats);
}

// The packed primitive table (scene_dev.cuh, F_FLAT) as built, whether or not the scene is traced through it, and what it
// was built from.  info = {words, flat_ok, objects, triangles over all meshes}; each pointer may be null:
// words (4 x info[0] 32-bit words), inv (12 floats per object: the f32 ObjectRec's inverse-transform rows),
// tri48 (12 floats per triangle, the meshes in order).
void hostemu_flat_table(const hostemu_scene* s, uint64_t* info, uint32_t* words, float* inv, float* tri48) {
    const HostScene& hs = s->hs;
    uint64_t ntris = 0;
    for (const HostMesh& hm : hs.meshes) ntris += hm.tri48.size() / 3;
    info[0] = hs.flat.size();
    info[1] = hs.flat_ok ? 1u : 0u;
    info[2] = hs.t32.objects.size();
    info[3] = ntris;
    if (words && !hs.flat.empty()) std::memcpy(words, hs.flat.data(), hs.flat.size() * sizeof(float4));
    if (inv)
        for (size_t i = 0; i < hs.t32.objects.size(); i++) std::memcpy(inv + 12 * i, hs.t32.objects[i].inv, 12 * sizeof(float));
    if (tri48)
        for (const HostMesh& hm : hs.meshes) {
            if (!hm.tri48.empty()) std::memcpy(tri48, hm.tri48.data(), hm.tri48.size() * sizeof(float4));
            tri48 += 4 * hm.tri48.size();
        }
}

// The variant the launchers pick (launch.h).  engine: 0 = render_kernel (slot engine), 1 = render_kernel_vx, 2 =
// closest_hit_kernel.  out = {STATS, FEAT, MAXD}; returns 1 if that variant is in the list of compiled ones, else 0.
int hostemu_pick_variant(int engine, int features, int stats, uint32_t precision, uint32_t max_bounces, int32_t* out) {
    const bool f64 = precision == RPTB_PRECISION_F64;
    Variant v;
    bool compiled;
    if (engine == 0) {
        v = pick_render(features, stats, f64, max_bounces);
        compiled = f64 ? RenderVariantsF64::has(v) : RenderVariantsF32::has(v);
    } else if (engine == 1) {
        v = pick_render_vx(features, stats);
        compiled = RenderVariantsVx::has(v);
    } else {
        v = pick_closest_hit(features, stats, f64);
        compiled = f64 ? HitVariantsF64::has(v) : HitVariantsF32::has(v);
    }
    out[0] = v.stats ? 1 : 0;
    out[1] = v.feat;
    out[2] = v.maxd;
    return compiled ? 1 : 0;
}

// Structural check of the BVH of mesh `mesh`: out = {nodes, leaves, largest leaf, depth, distinct triangles
// referenced, violations}.  A violation is a triangle vertex (as the kernels see it: float) outside the box
// its parent stores for its leaf, a child box that sticks out of its parent's, or a malformed leaf code.
// Renderer::sample through the megakernel's thread body (every lane run on its own; see HostLane).  Same contract
// as rptb_render_samples; returns the FEAT bits of the kernel instantiation that was emulated, or -1 on bad params.
// ext_bvh: what RPTB_EXT_BVH=1 asks of the library (mesh children of kd-trees of shapes through their BVH).
int hostemu_render(const hostemu_scene* s, const rptb_camera* cam, const rptb_render_params* p, int ext_bvh, double* out_rgb,
                   rptb_stats* stats) {
    if (!s || !cam || !p || !out_rgb || p->width == 0 || p->height == 0 || p->iterations == 0 ||
        p->max_bounces > MAX_BOUNCES_SUPPORTED)
        return -1;
    if (p->precision == RPTB_PRECISION_F64) return render_impl<double>(s->v64, cam, p, s->features, s->hs.sampled_lights, out_rgb, stats);
    int feats = s->features;
    if ((feats & F_EXT) && !ext_bvh) feats &= ~F_BVH;
    return render_impl<float>(s->v32, cam, p, feats, s->hs.sampled_lights, out_rgb, stats);
}

// The eight-wide collapse of mesh `mesh` against its binary BVH, ray by ray (mesh-local rays, n x 6 doubles): the scalar
// walk of Bvh8Node (geometry.cuh, bvh8_intersect_scalar) must find the binary tree's hits.  out_t / out_tri are n x 2
// (binary, eight-wide); out_info = {8-wide nodes, max children used, empty child slots, binary node visits, 8-wide node visits}.
int hostemu_bvh8_probe(const hostemu_scene* s, uint32_t mesh, const double* rays, uint64_t n, int any, double* out_t, int64_t* out_tri,
                       uint64_t* out_info) {
    if (mesh >= s->hs.t32.meshes.size()) return -1;
    const MeshRec<float>& m = s->v32.meshes[mesh];
    if (!m.bvh_nodes || !m.bvh8_nodes) return -1;
    const HostMesh& hm = s->hs.meshes[mesh];
    uint64_t used_max = 0, empty = 0;
    for (const Bvh8Node& nd : hm.bvh8_nodes) {
        uint64_t used = 0;
        for (int k = 0; k < 8; k++) used += nd.c[k].code != BVH8_EMPTY;
        used_max = std::max(used_max, used);
        empty += 8 - used;
    }
    unsigned long long v2 = 0, v8 = 0;
#pragma omp parallel for schedule(static) reduction(+ : v2, v8)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const double* r = rays + 6 * i;
        const Vec3<float> o = {(float)r[0], (float)r[1], (float)r[2]}, d = {(float)r[3], (float)r[4], (float)r[5]};
        for (int w = 0; w < 2; w++) {
            TravStats ts = {0, 0, 0, 0, 0};
            Hit<float> h;
            h.t = INFINITY; h.obj = -1; h.aux = 0xFFFFFFFFu; h.bv = h.bw = 0.0f;
            const bool hit = w == 0 ? bvh_intersect<true>(m, o, d, 1e-12f, any != 0, h, ts) : bvh8_intersect_scalar<true>(m, o, d, 1e-12f, any != 0, h, ts);
            out_t[2 * i + w] = hit ? (double)h.t : (double)INFINITY;
            out_tri[2 * i + w] = hit ? (int64_t)h.aux : -1;
            (w == 0 ? v2 : v8) += ts.bvh_nodes;
        }
    }
    out_info[0] = hm.bvh8_nodes.size(); out_info[1] = used_max; out_info[2] = empty; out_info[3] = v2; out_info[4] = v8 / 4;
    return 0;
}

// The four-wide collapse (what one lane per ray traverses: geometry.cuh, bvh4_intersect) against the binary tree, ray by
// ray, same layout of the outputs; out_info = {4-wide nodes, empty child slots, binary node visits, 4-wide node visits,
// binary triangle tests, 4-wide triangle tests}.
int hostemu_bvh4_probe(const hostemu_scene* s, uint32_t mesh, const double* rays, uint64_t n, int any, double* out_t, int64_t* out_tri,
                       uint64_t* out_info) {
    if (mesh >= s->hs.t32.meshes.size()) return -1;
    const MeshRec<float>& m = s->v32.meshes[mesh];
    if (!m.bvh_nodes || !m.bvh4_nodes) return -1;
    const HostMesh& hm = s->hs.meshes[mesh];
    uint64_t empty = 0;
    for (const Bvh4Node& nd : hm.bvh4_nodes)
        empty += (nd.code.x == BVH8_EMPTY) + (nd.code.y == BVH8_EMPTY) + (nd.code.z == BVH8_EMPTY) + (nd.code.w == BVH8_EMPTY);
    unsigned long long v2 = 0, v4 = 0, t2 = 0, t4 = 0;
#pragma omp parallel for schedule(static) reduction(+ : v2, v4, t2, t4)
    for (int64_t i = 0; i < (int64_t)n; i++) {
        const double* r = rays + 6 * i;
        const Vec3<float> o = {(float)r[0], (float)r[1], (float)r[2]}, d = {(float)r[3], (float)r[4], (float)r[5]};
        for (int w = 0; w < 2; w++) {
            TravStats ts = {0, 0, 0, 0, 0};
            Hit<float> h;
            h.t = INFINITY; h.obj = -1; h.aux = 0xFFFFFFFFu; h.bv = h.bw = 0.0f;
            const bool hit = w == 0 ? bvh_intersect<true>(m, o, d, 1e-12f, any != 0, h, ts) : bvh4_intersect<true>(m, o, d, 1e-12f, any != 0, h, ts);
            out_t[2 * i + w] = hit ? (double)h.t : (double)INFINITY;
            out_tri[2 * i + w] = hit ? (int64_t)h.aux : -1;
            (w == 0 ? v2 : v4) += ts.bvh_nodes;
            (w == 0 ? t2 : t4) += ts.bvh_tris;
        }
    }
    out_info[0] = hm.bvh4_nodes.size(); out_info[1] = empty; out_info[2] = v2; out_info[3] = v4 / 2; out_info[4] = t2; out_info[5] = t4;
    return 0;
}

int hostemu_bvh_check(const hostemu_scene* s, uint32_t mesh, uint64_t* out) {
    const HostMesh& hm = s->hs.meshes[mesh];
    for (int i = 0; i < 6; i++) out[i] = 0;
    if (hm.bvh_nodes.empty()) return -1;
    std::vector<uint8_t> seen(hm.ntris, 0);
    uint64_t leaves = 0, max_leaf = 0, depth = 0, violations = 0;
    struct Item { int32_t code; float lo[3], hi[3]; uint32_t depth; };
    std::vector<Item> stack;
    Item root;
    root.code = 0;
    root.depth = 0;
    for (int a = 0; a < 3; a++) root.lo[a] = -INFINITY, root.hi[a] = INFINITY;
    stack.push_back(root);
    while (!stack.empty()) {
        const Item it = stack.back();
        stack.pop_back();
        depth = std::max<uint64_t>(depth, it.depth);
        if (it.code >= 0) {
            if ((size_t)it.code >= hm.bvh_nodes.size()) { violations++; continue; }
            const BvhNodeDev& n = hm.bvh_nodes[it.code];
            Item c[2];
            c[0].code = n.child0; c[1].code = n.child1;
            c[0].lo[0] = n.c0xy.x; c[0].hi[0] = n.c0xy.y; c[0].lo[1] = n.c0xy.z; c[0].hi[1] = n.c0xy.w; c[0].lo[2] = n.cz.x; c[0].hi[2] = n.cz.y;
            c[1].lo[0] = n.c1xy.x; c[1].hi[0] = n.c1xy.y; c[1].lo[1] = n.c1xy.z; c[1].hi[1] = n.c1xy.w; c[1].lo[2] = n.cz.z; c[1].hi[2] = n.cz.w;
            for (int k = 0; k < 2; k++) {
                c[k].depth = it.depth + 1;
                // child boxes are padded independently of the parent's: allow the pad (relative 1e-5)
                for (int a = 0; a < 3; a++) {
                    const float tol = 1e-5f * std::fmax(1e-3f, std::fmax(std::fabs(c[k].lo[a]), std::fabs(c[k].hi[a])));
                    if (c[k].lo[a] < it.lo[a] - tol || c[k].hi[a] > it.hi[a] + tol) violations++;
                }
                stack.push_back(c[k]);
            }
        } else {
            const uint32_t code = (uint32_t)~it.code;
            const uint32_t first = code >> 3, count = (code & 7u) + 1u;
            leaves++;
            max_leaf = std::max<uint64_t>(max_leaf, count);
            if (count > (uint32_t)BVH_LEAF_MAX || (uint64_t)first + count > hm.ntris) { violations++; continue; }
            for (uint32_t k = first; k < first + count; k++) {
                const uint32_t id = hm.bvh_ids[k];
                if (id >= hm.ntris) { violations++; continue; }
                seen[id]++;
                for (int v = 0; v < 3; v++)
                    for (int a = 0; a < 3; a++) {
                        const float x = hm.verts32[9 * (size_t)id + 3 * v + a];
                        if (x < it.lo[a] || x > it.hi[a]) violations++;
                    }
                // the permuted triangle data is the original's
                for (int j = 0; j < 3; j++)
                    if (std::memcmp(&hm.bvh_tri48[3 * (size_t)k + j], &hm.tri48[3 * (size_t)id + j], sizeof(float4)) != 0) violations++;
            }
        }
    }
    uint64_t distinct = 0;
    for (uint8_t c : seen) {
        distinct += c != 0;
        if (c > 1) violations++;  // every triangle in exactly one leaf
    }
    out[0] = hm.bvh_nodes.size(); out[1] = leaves; out[2] = max_leaf; out[3] = depth; out[4] = distinct; out[5] = violations;
    return 0;
}

// precision as above; use_bvh: take the BVH where the scene has one (f32 only).  Returns the FEAT of the walk, -1 if it
// is not compiled.
int hostemu_occluded(const hostemu_scene* s, const double* rays, const double* tmax, uint64_t n, double t_min, uint32_t precision,
                     int use_bvh, int32_t* out) {
    if (precision == RPTB_PRECISION_F64) return run_occluded<double>(s->v64, s->features, rays, tmax, n, t_min, out);
    return run_occluded<float>(s->v32, use_bvh ? s->features : s->features & ~(int)F_BVH, rays, tmax, n, t_min, out);
}

int hostemu_illuminate(const hostemu_scene* s, uint32_t light, const double* pos, uint64_t n, uint64_t seed, uint32_t precision,
                       double* out_intensity, double* out_wi, double* out_dist) {
    if (precision == RPTB_PRECISION_F64) illuminations<double>(s->v64, light, pos, n, seed, out_intensity, out_wi, out_dist);
    else illuminations<float>(s->v32, light, pos, n, seed, out_intensity, out_wi, out_dist);
    return 0;
}

// The first n draws of stream (seed, pixel, sample) as every generator of rng.cuh hands them out: out64 = the f64
// generator's 64-bit draws; out32 = 4 x n words, row k = Rng buffering k (BUF_PAIR, BUF_FOUR, BUF_EIGHT) and row 3 the
// shared-memory ring's host form.  `ensure_every` > 0: ensure() is called before every ensure_every-th draw, as the
// integrator does at its converged points (the buffers must hand out the same words whenever they are refilled).
void hostemu_draws(uint64_t seed, uint32_t pixel, uint64_t sample, uint32_t n, uint32_t ensure_every, uint64_t* out64, uint32_t* out32) {
    Rng<double> r64;
    r64.init(seed, pixel, sample);
    for (uint32_t i = 0; i < n; i++) out64[i] = r64.p.next_u64();
    RngF32<BUF_PAIR> a;
    RngF32<BUF_FOUR> b;
    RngF32<BUF_EIGHT> c;
    RngRing d;
    a.init(seed, pixel, sample);
    b.init(seed, pixel, sample);
    c.init(seed, pixel, sample);
    d.bind(nullptr, 0);
    d.init(seed, pixel, sample);
    for (uint32_t i = 0; i < n; i++) {
        if (ensure_every && i % ensure_every == 0) {
            a.ensure();
            b.ensure();
            c.ensure();
            d.ensure<HostLane>(1u, 1u + (i / ensure_every) % 8u);
        }
        out32[i] = a.next32();
        out32[n + i] = b.next32();
        out32[2 * n + i] = c.next32();
        out32[3 * n + i] = d.next32();
    }
}

}  // extern "C"
