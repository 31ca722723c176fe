// wavefront.cuh -- the wavefront engine: the same integrator as integrator.cuh's
// megakernel, scheduled as two kernels per path vertex with the path state in HBM.
//
// Why a second schedule: on kd-tree scenes (teapot, dragon) the work of one
// get_closest_hit varies by two orders of magnitude between the rays of a warp (a ray
// that misses the mesh AABB costs nothing, one that grazes the dragon visits > 1000
// triangles).  In the megakernel a lane is tied to its pixel, so a warp's trace takes as
// long as its slowest ray: on the dragon proxy about a quarter of the lanes are active.
// Here the rays of all paths go through a PERSISTENT TRACE KERNEL whose lanes fetch a new
// ray the moment theirs is finished (Aila & Laine's persistent while-while with dynamic
// fetch), while a SHADE KERNEL advances every path by one vertex per step:
//
//   step:  shade(p)  consumes the answers of the rays path p emitted in the previous step
//                    (shadow rays of the current vertex in light order, then the bounce /
//                    camera ray), finishes paths (per-level clamp), regenerates camera
//                    rays, shades the new vertex: Le, one light sample per sampled light
//                    (illuminate + bsdf -> pending contribution + shadow ray),
//                    Material::sample_f + bsdf -> pending level weight + bounce ray;
//                    appends the ray slots it wrote to a compact list (warp-aggregated
//                    atomic);
//          trace     persistent CTAs drain that list.
//
// Per path the sequence of operations and of random draws is trace_ray's
// (src/renderer.rs:145-174), exactly as in the megakernel, so both engines render the
// same image up to the compiler's FMA contraction; every pixel is still accumulated by
// one owner in sample order (bit-reproducible, shard-independent).
#pragma once
#include "integrator.cuh"

namespace rptb {

constexpr int WF_THREADS = 128;
constexpr int WF_MAX_SHADOW = 8;
#ifndef WF_TRACE_MIN_BLOCKS
#define WF_TRACE_MIN_BLOCKS 8  // resident CTAs/SM the trace kernel is compiled for (64 registers; latency bound: 8 measured best of 7/8/10)
#endif  // sampled (non-ambient) lights per scene the wavefront engine handles

struct __align__(16) WfRay {
    float ox, oy, oz, tmax;
    float dx, dy, dz;
    uint32_t any;  // 1 = shadow query
};
struct __align__(16) WfHit {
    float t;
    int obj;
    uint32_t aux;
    float bv;
    float bw;
    uint32_t _pad[3];
};

enum : uint32_t {
    WF_FRESH = 0,   // needs a camera ray
    WF_CAMERA = 1,  // camera ray in flight
    WF_VERTEX = 2,  // at a vertex, its shadow / bounce rays in flight
    WF_DONE = 3
};

struct __align__(16) WfPath {
    float pos[3], err_scale;
    float n[3];
    uint32_t mat_id;
    float ng[3];
    uint32_t status;
    float wo[3];
    uint32_t s;
    float color[3];
    uint32_t depth;
    float w[3];  // weight of the pending bounce level
    uint32_t flags;  // bit0 dead, bit1 sample_f returned a direction, bit2 bounce ray emitted, bit3 fwd_ok, bits 8.. shadow mask
    float fwdA[3], fwdT0;
    float fwdT12[2], fwdTmin[2];
    float fwdTmin2;
    uint32_t chunk_id;  // sample chunk this path is summing (scene_dev.cuh: RenderArgs::chunk)
    uint32_t rng_block, rng_avail;
    uint32_t rng_q[8];  // the generator's buffered draws (Rng<float>::save)
    double acc[3];
    double _pad1;
};

struct WfBuffers {
    WfPath* paths;
    float* contrib;   // npaths * Ks * 3
    float* levels;    // npaths * maxd * 6
    WfRay* rays;      // npaths * (Ks + 1)
    WfHit* hits;      // npaths * (Ks + 1)
    uint32_t* list;   // compact list of live ray slots
    uint32_t* count;  // [0] rays emitted this step, [1] fetch cursor of the trace kernel
    // npaths = npix * G: every owned pixel slot has G paths in flight, path (slot, g) sums the sample
    // chunks g, g + G, g + 2G, ... one after the other (the chunk sums are resolved in chunk order, so
    // the image does not depend on G -- which is chosen per launch to keep ~2M paths in flight)
    uint32_t npaths, npix, G, Ks, maxd;
};

RPTB_D void wf_pixel_of(const RenderArgs<float>& a, uint32_t slot, uint32_t& x, uint32_t& y) {
    const uint32_t k = slot / RENDER_THREADS, tid = slot % RENDER_THREADS;
    const uint32_t tile = a.shard_index + k * a.shard_count;
    const uint32_t tx = tile % a.tiles_x, ty = tile / a.tiles_x;
    const uint32_t warp = tid >> 5, lane = tid & 31u;
    x = tx * TILE_W + (warp & 1u) * 8u + (lane & 7u);
    y = ty * TILE_H + (warp >> 1) * 4u + (lane >> 3);
}

__global__ void wf_init_kernel(const RenderArgs<float> a, const WfBuffers b) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= b.npaths) return;
    uint32_t x, y;
    wf_pixel_of(a, p % b.npix, x, y);
    WfPath st;
    memset(&st, 0, sizeof(st));
    st.chunk_id = p / b.npix;
    st.s = st.chunk_id * a.chunk;
    st.status = (x < a.width && y < a.height && st.s < a.iterations) ? WF_FRESH : WF_DONE;
    st.fwdT0 = 1.0f;
    st.fwdT12[0] = st.fwdT12[1] = 1.0f;
    st.fwdTmin[0] = st.fwdTmin[1] = st.fwdTmin2 = 1.0f;
    st.flags = 8u;  // fwd_ok
    b.paths[p] = st;
}

// Append `slot` to the compact ray list (one atomic per warp).
RPTB_D void wf_emit(const WfBuffers& b, bool pred, uint32_t slot) {
    const unsigned m = __ballot_sync(__activemask(), pred);
    if (!pred) return;
    const unsigned peers = m;
    const int leader = __ffs(peers) - 1;
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t base = 0;
    if ((int)lane == leader) base = atomicAdd(b.count, (uint32_t)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    b.list[base + __popc(peers & ((1u << lane) - 1u))] = slot;
}

template <bool STATS>
__global__ void __launch_bounds__(WF_THREADS) wf_shade_kernel(const SceneView<float> sv, const RenderArgs<float> a,
                                                              const WfBuffers b) {
    typedef float R;
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in_range = p < b.npaths;
    const uint32_t Ks = b.Ks, nslot = Ks + 1;
    WfPath st;
    if (in_range) {
        st = b.paths[p];
    } else {
        memset(&st, 0, sizeof(st));
        st.status = WF_DONE;
    }
    // `live` threads run the whole step; finished paths only take part in the warp votes
    const bool live = st.status != WF_DONE;

    uint32_t x = 0, y = 0;
    if (in_range) wf_pixel_of(a, p % b.npix, x, y);
    const uint32_t pix = y * a.width + x;
    Rng<R> rng;
    rng.init(a.seed, pix, a.first_sample + st.s);
    rng.half = st.rng_block;
    rng.avail = st.rng_avail;
    rng.load(st.rng_q);

    uint32_t n_seg = 0, n_mesh = 0, n_env = 0, n_rays = 0;
    Vec3<R> color = {st.color[0], st.color[1], st.color[2]};
    Vec3<R> fwdA = {st.fwdA[0], st.fwdA[1], st.fwdA[2]};
    Vec3<R> fwdT = {st.fwdT0, st.fwdT12[0], st.fwdT12[1]};
    Vec3<R> fwdTmin = {st.fwdTmin[0], st.fwdTmin[1], st.fwdTmin2};
    bool fwd_ok = (st.flags & 8u) != 0;
    Vec3<R> Lterm = {0.f, 0.f, 0.f};
    bool finish = false, new_vertex = false;
    Hit<R> h;
    h.t = M<R>::inf(); h.obj = -1; h.aux = 0; h.bv = h.bw = 0.f;
    Vec3<R> ro = {0.f, 0.f, 0.f}, rd = {0.f, 0.f, 1.f};
    float* lev = b.levels + (size_t)p * b.maxd * 6;

    if (live) {
        // ============ 1. the answers to last step's rays =================================
        bool seg_ray = false;
        if (st.status == WF_VERTEX) {
            const MaterialRec<R> mat = sv.materials[st.mat_id];
            uint32_t k = 0;
            for (uint32_t li = 0; li < sv.nlights; li++) {  // sample_lights, list order
                const LightRec<R>& l = sv.lights[li];
                if (l.kind == LIGHT_AMBIENT) {
                    color = color + cmul(mk(l.color[0], l.color[1], l.color[2]), mat_color(mat));
                } else {
                    if ((st.flags >> (8 + k)) & 1u) {
                        if (b.hits[(size_t)p * nslot + k].obj < 0) {
                            const float* c = b.contrib + ((size_t)p * Ks + k) * 3;
                            color = color + mk(c[0], c[1], c[2]);
                        }
                    }
                    k++;
                }
            }
            if (st.flags & 2u) {  // sample_f produced a direction: the level exists
                const Vec3<R> w = {st.w[0], st.w[1], st.w[2]};
                float* lv = lev + (size_t)st.depth * 6;
                lv[0] = color.x; lv[1] = color.y; lv[2] = color.z;
                lv[3] = w.x; lv[4] = w.y; lv[5] = w.z;
                fwd_ok = fwd_ok && color.x >= 0.f && color.y >= 0.f && color.z >= 0.f;
                fwdTmin = {fminf(fwdTmin.x, fwdT.x), fminf(fwdTmin.y, fwdT.y), fminf(fwdTmin.z, fwdT.z)};
                fwdA = fwdA + cmul(fwdT, color);
                fwdT = cmul(fwdT, w);
            }
            if (st.flags & 4u) {
                st.depth++;
                seg_ray = true;
            } else {
                Lterm = color;
                finish = true;
            }
        } else if (st.status == WF_CAMERA) {
            seg_ray = true;
        }
        if (seg_ray) {
            n_seg++;  // one trace_ray invocation
            const WfRay r = b.rays[(size_t)p * nslot + Ks];
            const WfHit hh = b.hits[(size_t)p * nslot + Ks];
            ro = {r.ox, r.oy, r.oz};
            rd = {r.dx, r.dy, r.dz};
            if (hh.obj < 0) {
                if (sv.env.kind != 0) n_env++;
                Lterm = env_color(sv.env, rd);
                finish = true;
            } else {
                h.t = hh.t; h.obj = hh.obj; h.aux = hh.aux; h.bv = hh.bv; h.bw = hh.bw;
                new_vertex = true;
            }
        }

        // ============ 2. finish the path (per-level clamp), start the next sample ========
        if (finish) {
            Vec3<R> L = Lterm;
            const Vec3<R> y0 = fwdA + cmul(fwdT, Lterm);
            const bool fast = fwd_ok && Lterm.x >= 0.f && Lterm.y >= 0.f && Lterm.z >= 0.f &&
                              y0.x <= 100.f * fwdTmin.x && y0.y <= 100.f * fwdTmin.y && y0.z <= 100.f * fwdTmin.z;
            if (fast) {
                L = y0;
            } else {
                for (int k = (int)st.depth - 1; k >= 0; k--) {
                    const float* lv = lev + (size_t)k * 6;
                    L = {lv[0] + fminf(lv[3] * L.x, 100.f), lv[1] + fminf(lv[4] * L.y, 100.f), lv[2] + fminf(lv[5] * L.z, 100.f)};
                }
            }
            fwdA = {0.f, 0.f, 0.f};
            fwdT = {1.f, 1.f, 1.f};
            fwdTmin = {1.f, 1.f, 1.f};
            fwd_ok = true;
            st.acc[0] += (double)L.x;
            st.acc[1] += (double)L.y;
            st.acc[2] += (double)L.z;
            st.s++;
            if (a.nchunks > 1) {
                const uint32_t cend = min((st.chunk_id + 1u) * a.chunk, a.iterations);
                if (st.s >= cend) {  // chunk complete: publish its sum, move on to this path's next chunk
                    double* o = a.partial + ((size_t)st.chunk_id * b.npix + (p % b.npix)) * 3;
                    o[0] = st.acc[0]; o[1] = st.acc[1]; o[2] = st.acc[2];
                    st.acc[0] = st.acc[1] = st.acc[2] = 0.0;
                    st.chunk_id += b.G;
                    st.s = st.chunk_id * a.chunk;  // >= iterations when no chunk is left
                }
            }
            st.status = WF_FRESH;
        }
    }

    // ============ 3. the rays of this step ================================================
    bool emit_seg = false;
    uint32_t shadow_mask = 0;
    if (live && st.status == WF_FRESH) {
        if (st.s >= a.iterations) {
            st.status = WF_DONE;
        } else {
            rng.init(a.seed, pix, a.first_sample + st.s);
            rng.ensure();
            const R dim = (R)max(a.width, a.height);
            const R xn = ((R)(2u * x + 1u) - (R)a.width) / dim;
            const R yn = ((R)(2u * (a.height - y) - 1u) - (R)a.height) / dim;
            const R dx = gen_range(rng, (R)-1 / dim, (R)1 / dim);
            const R dy = gen_range(rng, (R)-1 / dim, (R)1 / dim);
            const Vec3<R> eye = {a.cam.eye[0], a.cam.eye[1], a.cam.eye[2]};
            const Vec3<R> cdir = {a.cam.direction[0], a.cam.direction[1], a.cam.direction[2]};
            const Vec3<R> cup = {a.cam.up[0], a.cam.up[1], a.cam.up[2]};
            const Vec3<R> cright = {a.cam.right[0], a.cam.right[1], a.cam.right[2]};
            const R cx = xn + dx, cy = yn + dy;
            Vec3<R> origin = eye;
            Vec3<R> new_dir = a.cam.d * cdir + cx * cright + cy * cup;
            if (a.cam.aperture > (R)0) {
                const Vec3<R> focal_point = origin + M<R>::normalize(new_dir) * a.cam.focal_distance;
                R ax, ay;
                unit_disc(rng, ax, ay);
                origin = origin + (ax * cright + ay * cup) * a.cam.aperture;
                new_dir = focal_point - origin;
            }
            const Vec3<R> dirn = M<R>::normalize(new_dir);
            WfRay r;
            r.ox = origin.x; r.oy = origin.y; r.oz = origin.z; r.tmax = M<R>::inf();
            r.dx = dirn.x; r.dy = dirn.y; r.dz = dirn.z; r.any = 0;
            b.rays[(size_t)p * nslot + Ks] = r;
            emit_seg = true;
            st.depth = 0;
            st.status = WF_CAMERA;
        }
    } else if (live && new_vertex) {
        const ObjectRec<R>& ob = sv.objects[h.obj];
        const Surface<R> sf = finalize_hit(sv, ob, ro, rd, h);
        if (sf.on_mesh) n_mesh++;
        const Vec3<R> pos = ro + h.t * rd;
        const Vec3<R> n = sf.n, ng = sf.ng;
        const Vec3<R> wo = -M<R>::normalize(rd);
        const MaterialRec<R> mat = sv.materials[ob.material];
        const R err_scale = M<R>::max(max_abs3(pos), max_abs3(ro));
        color = mat.emittance * mat_color(mat);
        const bool dead = !mat.transparent && M<R>::signbit(dot(n, wo));
        rng.ensure();
        // sample_lights: one draw set per sampled light, in list order
        if (!dead) {
            uint32_t k = 0;
            for (uint32_t li = 0; li < sv.nlights; li++) {
                const LightRec<R>& l = sv.lights[li];
                if (l.kind == LIGHT_AMBIENT) continue;
                Vec3<R> intensity, wi;
                R dist;
                illuminate(sv, l, pos, rng, intensity, wi, dist);
                const bool zero_i = intensity.x == 0.f && intensity.y == 0.f && intensity.z == 0.f;
                if (!(zero_i || (!mat.transparent && M<R>::signbit(dot(n, wi))))) {
                    const Vec3<R> f = bsdf(mat, n, wo, wi);
                    const Vec3<R> c = cmul(f, intensity) * dot(wi, n);
                    float* cp = b.contrib + ((size_t)p * Ks + k) * 3;
                    cp[0] = c.x; cp[1] = c.y; cp[2] = c.z;
                    const Vec3<R> o2 = offset_origin(pos, ng, wi, err_scale);
                    WfRay r;
                    r.ox = o2.x; r.oy = o2.y; r.oz = o2.z; r.tmax = M<R>::next_up(dist);
                    r.dx = wi.x; r.dy = wi.y; r.dz = wi.z; r.any = 1;
                    b.rays[(size_t)p * nslot + k] = r;
                    shadow_mask |= 1u << k;
                }
                k++;
                rng.ensure();
            }
        }
        // Material::sample_f for the bounce
        uint32_t fl = dead ? 1u : 0u;
        if (st.depth < a.max_bounces && !dead) {
            Vec3<R> wi;
            R pdf;
            if (sample_f(mat, n, wo, rng, wi, pdf)) {
                const Vec3<R> f = bsdf(mat, n, wo, wi);
                const R abscos = M<R>::abs(dot(wi, n));
                const R kk = pdf > 0.f ? abscos / pdf : 0.f;
                const Vec3<R> w = {f.x * kk, f.y * kk, f.z * kk};
                st.w[0] = w.x; st.w[1] = w.y; st.w[2] = w.z;
                fl |= 2u;
                if (!(w.x == 0.f && w.y == 0.f && w.z == 0.f)) {
                    fl |= 4u;
                    const Vec3<R> o2 = offset_origin(pos, ng, wi, err_scale);
                    WfRay r;
                    r.ox = o2.x; r.oy = o2.y; r.oz = o2.z; r.tmax = M<R>::inf();
                    r.dx = wi.x; r.dy = wi.y; r.dz = wi.z; r.any = 0;
                    b.rays[(size_t)p * nslot + Ks] = r;
                    emit_seg = true;
                }
            }
        }
        st.flags = fl | (shadow_mask << 8);
        st.pos[0] = pos.x; st.pos[1] = pos.y; st.pos[2] = pos.z;
        st.err_scale = err_scale;
        st.n[0] = n.x; st.n[1] = n.y; st.n[2] = n.z;
        st.ng[0] = ng.x; st.ng[1] = ng.y; st.ng[2] = ng.z;
        st.wo[0] = wo.x; st.wo[1] = wo.y; st.wo[2] = wo.z;
        st.mat_id = ob.material;
        st.status = WF_VERTEX;
    }

    // compact list of the live ray slots (votes: every thread of the warp takes part)
    for (uint32_t k = 0; k < Ks; k++) wf_emit(b, (shadow_mask >> k) & 1u, p * nslot + k);
    wf_emit(b, emit_seg, p * nslot + Ks);
    n_rays = __popc(shadow_mask) + (emit_seg ? 1u : 0u);

    if (live) {
        st.color[0] = color.x; st.color[1] = color.y; st.color[2] = color.z;
        st.fwdA[0] = fwdA.x; st.fwdA[1] = fwdA.y; st.fwdA[2] = fwdA.z;
        st.fwdT0 = fwdT.x; st.fwdT12[0] = fwdT.y; st.fwdT12[1] = fwdT.z;
        st.fwdTmin[0] = fwdTmin.x; st.fwdTmin[1] = fwdTmin.y; st.fwdTmin2 = fwdTmin.z;
        st.flags = (st.flags & ~8u) | (fwd_ok ? 8u : 0u);
        st.rng_block = rng.half;
        st.rng_avail = rng.avail;
        rng.save(st.rng_q);
        b.paths[p] = st;
    }

    if (a.counters) {
        const unsigned m = __activemask();
        const uint32_t v0 = __reduce_add_sync(m, n_seg), v1 = __reduce_add_sync(m, n_rays);
        const uint32_t v2 = __reduce_add_sync(m, n_mesh), v3 = __reduce_add_sync(m, n_env);
        if ((threadIdx.x & 31u) == (uint32_t)(__ffs(m) - 1)) {
            if (v0) atomicAdd(&a.counters->segments, (unsigned long long)v0);
            if (v1) atomicAdd(&a.counters->rays, (unsigned long long)v1);
            if (v2) atomicAdd(&a.counters->mesh_hits, (unsigned long long)v2);
            if (v3) atomicAdd(&a.counters->env_lookups, (unsigned long long)v3);
        }
    }
}

// ---- the persistent trace kernel --------------------------------------------------------
// Every lane owns at most one ray; a lane whose ray is finished fetches the next slot from
// the compact list at the top of the loop (warp-aggregated atomic cursor), so the warp's
// traversal loops stay populated however uneven the rays are.  The traversal is the explicit
// state machine of geometry.cuh's kd_intersect: scene.objects are walked in order; analytic
// shapes and single-leaf meshes are intersected on the spot, a kd-tree mesh switches the
// lane into the TRAVERSE state, where each loop iteration descends to one leaf, tests its
// triangles and pops.
// BVH = true: a mesh with a real tree is traversed through its BVH (scene_dev.cuh, F_BVH) instead --
// same state machine, each loop iteration descends to one BVH leaf, tests its <= 4 triangles and pops.
template <bool STATS, bool BVH>
__global__ void __launch_bounds__(WF_THREADS, WF_TRACE_MIN_BLOCKS) wf_trace_kernel(const SceneView<float> sv, const WfBuffers b,
                                                              const uint32_t* __restrict__ list,
                                                              DeviceCounters* counters) {
    typedef float R;
    const R tmin = (R)1e-12;
    const uint32_t total = b.count[0];
    const uint32_t lane = threadIdx.x & 31u;
    TravStats ts = {0, 0, 0, 0, 0};

    bool have = false, exhausted = false;
    uint32_t slot = 0;
    bool any = false;
    Vec3<R> wo_ = {0.f, 0.f, 0.f}, wd_ = {0.f, 0.f, 1.f};  // world ray
    Hit<R> h;
    h.t = 0.f; h.obj = -1; h.aux = 0; h.bv = h.bw = 0.f;
    uint32_t oi = 0;
    // TRAVERSE state (mesh-local ray)
    bool trav = false;
    Vec3<R> lo_o = wo_, lo_d = wd_, inv = wd_;
    const MeshRec<R>* mesh = nullptr;
    uint32_t node = 0;
    R lo = 0.f, hi = 0.f;
    int sp = 0;
    bool mesh_hit = false;
    uint32_t st_node[BVH ? 1 : KD_STACK];
    R st_lo[BVH ? 1 : KD_STACK], st_hi[BVH ? 1 : KD_STACK];
    int32_t bstack[BVH ? BVH_STACK : 1];  // BVH mode: pending far children
    int32_t cur = 0;
    Vec3<R> oinv = wd_;                   // BVH mode: o / d per axis

    while (true) {
        // ---- fetch -----------------------------------------------------------------------
        {
            const bool want = !have && !exhausted;
            const unsigned m = __ballot_sync(0xffffffffu, want);
            if (m) {
                const int leader = __ffs(m) - 1;
                uint32_t base = 0;
                if ((int)lane == leader) base = atomicAdd(b.count + 1, (uint32_t)__popc(m));
                base = __shfl_sync(0xffffffffu, base, leader);
                if (want) {
                    const uint32_t idx = base + __popc(m & ((1u << lane) - 1u));
                    if (idx < total) {
                        slot = list[idx];
                        const WfRay r = b.rays[slot];
                        wo_ = {r.ox, r.oy, r.oz};
                        wd_ = {r.dx, r.dy, r.dz};
                        any = r.any != 0;
                        h.t = r.tmax; h.obj = -1; h.aux = 0; h.bv = h.bw = 0.f;
                        oi = 0;
                        trav = false;
                        have = true;
                    } else {
                        exhausted = true;
                    }
                }
            }
            if (__all_sync(0xffffffffu, !have)) break;
        }
        // ---- walk scene.objects up to the next kd-tree mesh (or the end of the ray) ------
        if (have && !trav) {
            bool done = false;
            while (!done) {
                if (oi >= sv.nobjects) { done = true; break; }
                const ObjectRec<R>& ob = sv.objects[oi];
                if (STATS) ts.object_tests++;
                if (ob.kind == SHAPE_MESH && !sv.meshes[ob.mesh].root_is_leaf) {
                    Vec3<R> o = wo_, d = wd_;
                    if (ob.has_transform) {
                        o = xform_point(ob.inv, wo_);
                        d = xform_dir(ob.inv, wd_);
                    }
                    const MeshRec<R>& mm = sv.meshes[ob.mesh];
                    const Vec3<R> iv = {M<R>::rcp(d.x), M<R>::rcp(d.y), M<R>::rcp(d.z)};
                    const R x1 = (mm.bmin[0] - o.x) * iv.x, x2 = (mm.bmax[0] - o.x) * iv.x;
                    const R y1 = (mm.bmin[1] - o.y) * iv.y, y2 = (mm.bmax[1] - o.y) * iv.y;
                    const R z1 = (mm.bmin[2] - o.z) * iv.z, z2 = (mm.bmax[2] - o.z) * iv.z;
                    const R l0 = fmaxf(fmaxf(fminf(x1, x2), fminf(y1, y2)), fminf(z1, z2));
                    const R h0 = fminf(fminf(fmaxf(x1, x2), fmaxf(y1, y2)), fmaxf(z1, z2));
                    if (fmaxf(l0, tmin) > fminf(h0, h.t)) {  // root cull (kdtree.rs:130-134)
                        oi++;
                        continue;
                    }
                    lo_o = o; lo_d = d; inv = iv;
                    mesh = &mm;
                    node = 0; lo = l0; hi = h0; sp = 0;
                    if (BVH) {
                        cur = 0;
                        inv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};  // finite even for a zero component (geometry.cuh)
                        oinv = {o.x * inv.x, o.y * inv.y, o.z * inv.z};
                    }
                    mesh_hit = false;
                    trav = true;
                    break;
                }
                if (object_intersect<R, STATS>(sv, ob, wo_, wd_, tmin, any, h, ts)) {
                    h.obj = (int)oi;
                    if (any) { done = true; break; }
                }
                oi++;
            }
            if (done) {  // ray finished: publish the hit
                WfHit out;
                out.t = h.t; out.obj = h.obj; out.aux = h.aux; out.bv = h.bv; out.bw = h.bw;
                out._pad[0] = out._pad[1] = out._pad[2] = 0;
                b.hits[slot] = out;
                have = false;
            }
        }
        // ---- one round of the kd traversal: descend to a leaf, test it, pop ---------------
        // ("while-while".  A finer-grained "if-if" schedule -- a few node steps, then one 4-triangle
        // batch per loop iteration -- was measured on the dragon proxy and lost: a third more instructions
        // for one or two more active lanes.)
        if (BVH && have && trav) {
            // ---- one round of the BVH traversal (geometry.cuh, bvh_intersect) -----------------
            bool mesh_done = false;
            while (cur >= 0) {
                if (STATS) ts.node_visits++;
                const BvhNodeDev n = load_bvh_node(mesh->bvh_nodes + cur);
                const float ax0 = fmaf(n.c0xy.x, inv.x, -oinv.x), ax1 = fmaf(n.c0xy.y, inv.x, -oinv.x);
                const float ay0 = fmaf(n.c0xy.z, inv.y, -oinv.y), ay1 = fmaf(n.c0xy.w, inv.y, -oinv.y);
                const float az0 = fmaf(n.cz.x, inv.z, -oinv.z), az1 = fmaf(n.cz.y, inv.z, -oinv.z);
                const float bx0 = fmaf(n.c1xy.x, inv.x, -oinv.x), bx1 = fmaf(n.c1xy.y, inv.x, -oinv.x);
                const float by0 = fmaf(n.c1xy.z, inv.y, -oinv.y), by1 = fmaf(n.c1xy.w, inv.y, -oinv.y);
                const float bz0 = fmaf(n.cz.z, inv.z, -oinv.z), bz1 = fmaf(n.cz.w, inv.z, -oinv.z);
                const float an = fmaxf(fmaxf(fminf(ax0, ax1), fminf(ay0, ay1)), fmaxf(fminf(az0, az1), tmin));
                const float af = fminf(fminf(fmaxf(ax0, ax1), fmaxf(ay0, ay1)), fminf(fmaxf(az0, az1), h.t));
                const float bn = fmaxf(fmaxf(fminf(bx0, bx1), fminf(by0, by1)), fmaxf(fminf(bz0, bz1), tmin));
                const float bf = fminf(fminf(fmaxf(bx0, bx1), fmaxf(by0, by1)), fminf(fmaxf(bz0, bz1), h.t));
                const bool ha = an <= af, hb = bn <= bf;
                if (ha && hb) {
                    const bool a_first = an <= bn;
                    bstack[sp++] = a_first ? n.child1 : n.child0;
                    cur = a_first ? n.child0 : n.child1;
                } else if (ha) {
                    cur = n.child0;
                } else if (hb) {
                    cur = n.child1;
                } else {
                    if (sp == 0) { mesh_done = true; break; }
                    cur = bstack[--sp];
                }
            }
            if (!mesh_done) {  // cur is a leaf
                const uint32_t code = (uint32_t)~cur;
                const uint32_t first = code >> 3, cnt = (code & 7u) + 1u;
                const float4* T = mesh->bvh_tri48 + 3 * (size_t)first;
                float4 q0[BVH_LEAF_MAX];
#pragma unroll
                for (uint32_t j = 0; j < (uint32_t)BVH_LEAF_MAX; j++) q0[j] = __ldg(T + 3 * min(j, cnt - 1u));
#pragma unroll
                for (uint32_t j = 0; j < (uint32_t)BVH_LEAF_MAX; j++) {
                    if (j >= cnt) break;
                    if (STATS) ts.tri_tests++;
                    const float cosine = q0[j].x * lo_d.x + q0[j].y * lo_d.y + q0[j].z * lo_d.z;
                    if (fabsf(cosine) < 1e-8f) continue;
                    const float time = __fdividef(q0[j].w - (q0[j].x * lo_o.x + q0[j].y * lo_o.y + q0[j].z * lo_o.z), cosine);
                    if (time < tmin || time >= h.t) continue;
                    const float4 q1 = __ldg(T + 3 * j + 1);
                    const float4 q2 = __ldg(T + 3 * j + 2);
                    const float px = fmaf(time, lo_d.x, lo_o.x), py = fmaf(time, lo_d.y, lo_o.y), pz = fmaf(time, lo_d.z, lo_o.z);
                    const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
                    const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
                    const float u = 1.0f - v - w;
                    if (u >= 0.0f && v >= 0.0f && w >= 0.0f) {
                        h.t = time;
                        h.bv = v;
                        h.bw = w;
                        h.aux = __ldg(mesh->bvh_ids + first + j);
                        mesh_hit = true;
                    }
                }
                if ((any && mesh_hit) || sp == 0) mesh_done = true;
                else cur = bstack[--sp];
            }
            if (mesh_done) {  // back to the object walk (next object, or the end of the ray)
                if (mesh_hit) h.obj = (int)oi;
                trav = false;
                if (any && mesh_hit) oi = sv.nobjects;
                else oi++;
            }
        }
        if (!BVH && have && trav) {
            auto nd = load_node(mesh->nodes + node);
            while ((nd.word & 3u) != 3u) {
                if (STATS) ts.node_visits++;
                const uint32_t axis = nd.word & 3u;
                const uint32_t right = nd.word >> 2;
                const R split = nd.split;
                const R oa = comp(lo_o, (int)axis), ia = comp(inv, (int)axis);
                const R sd = split - oa;
                const R t_split = sd * ia;
                // (o < split) || (o == split && d <= 0); sign(1/d) == sign(d)
                const bool left_first = (sd > (R)0) || (sd == (R)0 && ia <= (R)0);
                const uint32_t first = left_first ? node + 1u : right;
                const uint32_t second = left_first ? right : node + 1u;
                if (t_split > fminf(hi, h.t) || t_split <= (R)0) {
                    node = first;
                } else if (t_split < fmaxf(lo, tmin)) {
                    node = second;
                } else {
                    st_node[sp] = second; st_lo[sp] = t_split; st_hi[sp] = hi;
                    sp++;
                    node = first;
                    hi = t_split;
                }
                nd = load_node(mesh->nodes + node);
            }
            if (STATS) ts.node_visits++;
            {
                // Leaf: every referenced triangle is considered (kdtree.rs:162-171), four at a time so
                // that the index and plane loads of a batch are in flight together (the kernel is
                // bound by L2 latency, not by arithmetic).  A plane hit outside this cell's interval
                // [lo, hi] is left to the cell that contains it -- the triangle is referenced there
                // too (inclusive partition, kdtree.rs:270-281) -- which saves the barycentric half of
                // the test and its 32 bytes for most triangles of a leaf.
                const uint32_t first_ref = nd.first_ref;
                const uint32_t cnt = nd.word >> 2;
                const float4* T = mesh->tri48;
                const float4* LP = mesh->leaf_planes + first_ref;  // this leaf's planes, contiguous
                const R slack = (fabsf(lo) + fabsf(hi)) * 1e-4f + 1e-6f;
                const R c_lo = fmaxf(lo - slack, tmin), c_hi = hi + slack;
                for (uint32_t i = 0; i < cnt; i += 4) {
                    const uint32_t n4 = min(4u, cnt - i);
                    float4 q0[4];
#pragma unroll
                    for (uint32_t j = 0; j < 4; j++) q0[j] = __ldg(LP + i + min(j, n4 - 1u));
#pragma unroll
                    for (uint32_t j = 0; j < 4; j++) {
                        if (j >= n4) break;
                        if (STATS) ts.tri_tests++;
                        const float cosine = q0[j].x * lo_d.x + q0[j].y * lo_d.y + q0[j].z * lo_d.z;
                        if (fabsf(cosine) < 1e-8f) continue;
                        const float time = __fdividef(q0[j].w - (q0[j].x * lo_o.x + q0[j].y * lo_o.y + q0[j].z * lo_o.z), cosine);
                        if (time < c_lo || time >= h.t || time > c_hi) continue;
                        const uint32_t tri = __ldg(mesh->refs + first_ref + i + j);
                        const float4 q1 = __ldg(T + 3 * (size_t)tri + 1);
                        const float4 q2 = __ldg(T + 3 * (size_t)tri + 2);
                        const float px = fmaf(time, lo_d.x, lo_o.x), py = fmaf(time, lo_d.y, lo_o.y), pz = fmaf(time, lo_d.z, lo_o.z);
                        const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
                        const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
                        const float u = 1.0f - v - w;
                        if (u >= 0.0f && v >= 0.0f && w >= 0.0f) {
                            h.t = time;
                            h.bv = v;
                            h.bw = w;
                            h.aux = tri;
                            mesh_hit = true;
                        }
                    }
                }
            }
            bool mesh_done = any && mesh_hit;
            if (!mesh_done) {
                while (true) {
                    if (sp == 0) { mesh_done = true; break; }
                    sp--;
                    node = st_node[sp]; lo = st_lo[sp]; hi = st_hi[sp];
                    if (!(h.t < lo)) break;
                }
            }
            if (mesh_done) {  // back to the object walk (next object, or the end of the ray)
                if (mesh_hit) h.obj = (int)oi;
                trav = false;
                if (any && mesh_hit) oi = sv.nobjects;
                else oi++;
            }
        }
    }

    if (counters) {
        atomicAdd(&counters->node_visits, (unsigned long long)ts.node_visits);
        atomicAdd(&counters->tri_tests, (unsigned long long)ts.tri_tests);
        atomicAdd(&counters->object_tests, (unsigned long long)ts.object_tests);
    }
}

__global__ void wf_finish_kernel(const RenderArgs<float> a, const WfBuffers b) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= b.npaths) return;  // (nchunks == 1 only: npaths == npix; otherwise resolve_chunks_kernel)
    uint32_t x, y;
    wf_pixel_of(a, p, x, y);
    if (x >= a.width || y >= a.height) return;
    const WfPath& st = b.paths[p];
    const double it = (double)a.iterations;
    float* out = a.out + 3 * (a.compact ? (size_t)p : (size_t)y * a.width + x);  // path p of a one-chunk render = pixel slot p
    out[0] = (float)(st.acc[0] / it * (double)a.exposure_scale);
    out[1] = (float)(st.acc[1] / it * (double)a.exposure_scale);
    out[2] = (float)(st.acc[2] / it * (double)a.exposure_scale);
}

}  // namespace rptb
