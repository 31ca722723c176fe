// integrator.cuh -- the path-tracing megakernel and the diagnostic kernels.
//
// Reference loop being replaced (ekzhang/rpt @815b21c):
//   Renderer::sample        src/renderer.rs:117-129   rayon over rows, one StdRng per row
//   Renderer::get_color     src/renderer.rs:131-142   for _ in 0..iterations { jitter; cast_ray; trace_ray }
//   Camera::cast_ray        src/camera.rs:64-81
//   Renderer::trace_ray     src/renderer.rs:145-174   recursive, per-level firefly clamp
//   Renderer::sample_lights src/renderer.rs:177-204
//   Renderer::get_closest_hit src/renderer.rs:211-220
//
// Design: one thread owns one pixel for all `iterations` samples and sums them
// in sample order, so the image is bit-reproducible and independent of how pixel
// tiles are sharded over GPUs (no atomics on the film).  A warp covers an 8x4 pixel
// block, a CTA a 16x8 tile; tiles are dealt round-robin to shards.  The recursion
// of trace_ray is flattened into ONE loop whose body is one path segment: a lane
// whose path ended regenerates its next camera ray at the top of the same loop
// instead of idling until the longest path of the warp finishes (persistent-lane
// path regeneration).  The per-level clamp `min(indirect, 100)` makes the estimator
// non-linear.  The f64 parity gate keeps each level's (local radiance, throughput) on a small
// per-thread stack and unwinds it when the path ends -- literally the reference's recursion.  The
// f32 product path needs no stack: a level is the map x -> a + min(w x, 100) of the radiance x coming
// back from below, and such maps compose into one of the same shape, A + min(W x, C), so the path carries
// nine floats forward and the value is exact (see `render_thread`).
#pragma once
#include "shading.cuh"

namespace rptb {

constexpr int RENDER_THREADS = 128;  // 4 warps: a 16x8 pixel tile
// Resident CTAs/SM each instantiation is compiled for (register cap = 65536 / (128 * blocks); the
// H100 has the same 64 K registers per SM as the GPU these were tuned on, not yet re-tuned on it).
// Measured: the full-feature kernel (glass) is fastest at 5, the feature-free kernel (Cornell) at 8.
#ifndef RPTB_MIN_BLOCKS
#define RPTB_MIN_BLOCKS 5
#endif
#ifndef RPTB_MIN_BLOCKS_LITE
#define RPTB_MIN_BLOCKS_LITE 8
#endif
#ifndef RPTB_MIN_BLOCKS_TREE
#define RPTB_MIN_BLOCKS_TREE 8   // F_TREE only (teapot: fastest of 5 / 6 / 8)
#endif
#ifndef RPTB_MIN_BLOCKS_GLASS
#define RPTB_MIN_BLOCKS_GLASS 5  // F_TRANSP | F_HDRI, no trees (glass: flat across 5 / 6 / 8)
#endif
#ifndef RPTB_MIN_BLOCKS_BVH
#define RPTB_MIN_BLOCKS_BVH 8    // F_BVH: the node loop is latency bound at 5-6 lanes, more resident warps help more than the spills of the 64-register
                                 // build hurt (8 beat 6 and 7 on teapot, dragon-proxy and knot)
#endif
#ifndef RPTB_MIN_BLOCKS_EXT
#define RPTB_MIN_BLOCKS_EXT 4    // F_EVERY (two nested traversal stacks in local memory): not tuned on hardware yet
#endif
constexpr int render_min_blocks(int feat) {
    if (feat & F_EXT) return RPTB_MIN_BLOCKS_EXT;
    if (feat & F_BVH) return RPTB_MIN_BLOCKS_BVH;
    const int base = feat & F_ALL;  // F_SMALL does not change the register budget
    return base == 0 ? RPTB_MIN_BLOCKS_LITE : base == F_TREE ? RPTB_MIN_BLOCKS_TREE : base == (F_TRANSP | F_HDRI) ? RPTB_MIN_BLOCKS_GLASS : RPTB_MIN_BLOCKS;
}
constexpr int TILE_W = 16, TILE_H = 8;

template <class R>
struct Level;
template <>
struct Level<float> {  // throughput pre-multiplied: w = f * (|cos| / pdf)
    float local[3], w[3];
};
template <>
struct Level<double> {  // literal: indirect = 1/pdf * (f (.) L) * |cos|
    double local[3], f[3], inv_pdf, abscos;
};

RPTB_D Vec3<float> unwind(const Level<float>& l, Vec3<float> L) {
    return {l.local[0] + fminf(l.w[0] * L.x, 100.0f), l.local[1] + fminf(l.w[1] * L.y, 100.0f),
            l.local[2] + fminf(l.w[2] * L.z, 100.0f)};
}
RPTB_D Vec3<double> unwind(const Level<double>& l, Vec3<double> L) {
    const double ix = l.inv_pdf * (l.f[0] * L.x) * l.abscos;
    const double iy = l.inv_pdf * (l.f[1] * L.y) * l.abscos;
    const double iz = l.inv_pdf * (l.f[2] * L.z) * l.abscos;
    return {l.local[0] + fmin(ix, 100.0), l.local[1] + fmin(iy, 100.0), l.local[2] + fmin(iz, 100.0)};
}

struct PathCounters {
    uint32_t segments, rays, mesh_hits, env_lookups;
    TravStats ts;
};

// scene.lights[i]: from parameter space when the scene's tables ride in the kernel parameters
template <int FEAT, class R>
RPTB_D const LightRec<R>& scene_light(const SceneView<R>& sv, uint32_t i) {
    if constexpr ((FEAT & F_SMALL) != 0 && !M<R>::literal) return sv.small.lights[i];
    else return sv.lights[i];
}

// Per-lane status in the flattened trace_ray recursion.
enum : int {
    ST_FRESH = 0,   // needs a camera ray (start of get_color's next sample)
    ST_VERTEX = 1,  // at a surface: lights are walked in the light slots, the bounce in the segment slot
    ST_FINISH = 2,  // path ended with radiance Lterm: unwind the per-level clamps at the next segment slot
    ST_IDLE = 3     // all samples of this pixel are done; waiting for the rest of the warp
};

// The warp runs a fixed slot schedule: slot j < Ks traces the shadow ray of the j-th
// sampled (non-ambient) light for every lane standing at a vertex, slot Ks traces the
// segment rays (Material::sample_f bounces and fresh camera rays).  The slot counter is
// warp-uniform, so all lanes execute the same shading code in the same iteration and meet
// at the single get_closest_hit site; a lane with nothing to do in a slot (light sample
// with provably zero contribution, path just ended) sits that trace out.  Per lane the
// order of operations -- and of random draws -- is exactly trace_ray's.
//
// The body is `render_thread`: one thread's whole life, written against a warp policy W.  On the device W is
// DeviceWarp (the real votes and reductions) and render_kernel is a one-line wrapper, so the generated code is
// what it was when the body lived in the kernel.  tests/hostemu instantiates the same body with a
// single-lane policy to run the integrator on the host against the oracle (test infrastructure).
#ifdef __CUDACC__
struct DeviceWarp {
    static __device__ __forceinline__ unsigned activemask() { return __activemask(); }
    static __device__ __forceinline__ bool all(unsigned m, bool p) { return __all_sync(m, p); }
    static __device__ __forceinline__ bool any(unsigned m, bool p) { return __any_sync(m, p); }
    static constexpr uint32_t width = 32u;
    static __device__ __forceinline__ unsigned ballot(unsigned m, bool p) { return __ballot_sync(m, p); }
    static __device__ __forceinline__ uint32_t rank(unsigned votes, uint32_t lane) { return (uint32_t)__popc(votes & ((1u << lane) - 1u)); }
    static __device__ __forceinline__ uint32_t popc(unsigned v) { return (uint32_t)__popc(v); }
    static __device__ __forceinline__ void sync(unsigned m) { __syncwarp(m); }
    static __device__ __forceinline__ uint32_t reduce_add(unsigned m, uint32_t v) { return __reduce_add_sync(m, v); }
    static __device__ __forceinline__ bool is_leader(unsigned m, uint32_t lane) { return (int)lane == __ffs(m) - 1; }
    static __device__ __forceinline__ void add(unsigned long long* p, unsigned long long v) { atomicAdd(p, v); }
};
#endif

// The generator the megakernel draws from: f64 the oracle's; f32 the same stream buffered in registers the way that
// suits the instantiation (rng.cuh: the 64-register F_BVH kernels take the smallest buffer), or the shared-memory ring
template <class R, int FEAT>
struct MegaRng { typedef Rng<R> type; };
#if RPTB_RNG_FIFO
template <int FEAT>
struct MegaRng<float, FEAT> { typedef RngF32<(FEAT & F_BVH) ? RPTB_FIFO_MODE_BVH : RPTB_FIFO_MODE> type; };
#else
template <int FEAT>
struct MegaRng<float, FEAT> { typedef RngRing type; };
#endif

// `rng_ring`: RNG_RING * RENDER_THREADS words of shared memory (f32 on the device; null otherwise).
// `coop`: this warp's CoopWarp block (geometry.cuh) when meshes are traversed by lane groups (F_BVH on the device), else null.
template <class R, int MAXD, bool STATS, int FEAT, class W>
RPTB_D void render_thread(const SceneView<R>& sv, const RenderArgs<R>& a, const uint32_t block_x, const uint32_t block_y,
                          const uint32_t thread_x, uint32_t* rng_ring = nullptr, void* coop = nullptr) {
    const uint32_t tile = a.shard_index + block_x * a.shard_count;
    const uint32_t tx = tile % a.tiles_x, ty = tile / a.tiles_x;
    const uint32_t warp = thread_x >> 5, lane = thread_x & 31u;
    const uint32_t x = tx * TILE_W + (warp & 1u) * 8u + (lane & 7u);
    const uint32_t y = ty * TILE_H + (warp >> 1) * 4u + (lane >> 3);
    if (x >= a.width || y >= a.height) return;
    const uint32_t pix = y * a.width + x;
    // The lanes of this warp that own a pixel.  They stay together until all of them have
    // finished their samples (independent thread scheduling gives no such guarantee).
    const unsigned wmask = W::activemask();

    const R tmin = (R)1e-12;  // EPSILON, renderer.rs:14
    const R dim = (R)max(a.width, a.height);
    const R xn = ((R)(2u * x + 1u) - (R)a.width) / dim;
    const R yn = ((R)(2u * (a.height - y) - 1u) - (R)a.height) / dim;

    uint32_t Ks = 0;        // lights that need a shadow ray (warp-uniform)
    uint32_t draw_hint = 0;  // 4 bits per sampled light (the first 8): draws its sample typically takes
    for (uint32_t i = 0; i < sv.nlights; i++) {
        const LightRec<R>& l = scene_light<FEAT>(sv, i);
        if (l.kind == LIGHT_AMBIENT) continue;
        if (Ks < 8u) draw_hint |= light_draws_hint(l) << (4u * Ks);
        Ks++;
    }

    PathCounters pc = {0, 0, 0, 0, {0, 0, 0, 0, 0}};
    double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0;
    Level<R> stack[M<R>::literal ? MAXD : 1];  // f64 gate only
    typename MegaRng<R, FEAT>::type rng;
    rng.bind(rng_ring ? rng_ring + thread_x : nullptr, RENDER_THREADS);
    rng.init(a.seed, pix, a.first_sample);

    // current ray
    Vec3<R> ro = {(R)0, (R)0, (R)0}, rd = {(R)0, (R)0, (R)1};
    R tmax = M<R>::inf();
    // surface context of the vertex being shaded (valid in ST_VERTEX)
    Vec3<R> pos = ro, n = rd, ng = rd, wo = rd;
    Vec3<R> color = {(R)0, (R)0, (R)0};    // Le + direct light gathered so far at this vertex
    Vec3<R> contrib = {(R)0, (R)0, (R)0};  // f (.) I (wi.n) of the light sample whose shadow ray is in flight
    Vec3<R> Lterm = {(R)0, (R)0, (R)0};
    R err_scale = (R)0;
    uint32_t mat_id = 0, li = 0;
    bool dead = false;
    // this thread's run of samples: [s, s_end) of [0, iterations) = chunks_per_group whole chunks
    uint32_t s = block_y * a.chunks_per_group * a.chunk;
    const uint32_t s_end = min(s + a.chunks_per_group * a.chunk, a.iterations);
    uint32_t chunk_id = block_y * a.chunks_per_group, chunk_left = a.chunk;
    const size_t pslot = (size_t)block_x * RENDER_THREADS + thread_x;
    const size_t pstride = (size_t)a.ntiles_mine * RENDER_THREADS;
    int depth = 0;
    int status = ST_FRESH;
    // f32 only: trace_ray's value as a function of the radiance x that comes back from below the deepest level
    // reached so far, per channel:  L(x) = fwdA + min(fwdT x, fwdC).  A level contributes x -> a + min(w x, 100)
    // (renderer.rs:153-167: a = Le + direct light, w = f |cos| / pdf >= 0), and for W >= 0
    //     A + min(W (a + min(w x, 100)), C)  =  (A + W a) + min(W w x, min(100 W, C - W a)),
    // so the composite keeps its shape: exact per-level clamps with nine floats and no stack.
    const R clamp_inf = M<R>::inf();
    Vec3<R> fwdA = {(R)0, (R)0, (R)0}, fwdT = {(R)1, (R)1, (R)1}, fwdC = {clamp_inf, clamp_inf, clamp_inf};
    uint32_t slot = Ks;  // every lane starts with a camera ray

    while (true) {
        const bool light_slot = slot < Ks;
        // (Measured and dropped: moving the generator of a lane that is certain to regenerate in this slot --
        // ST_FINISH, or a vertex that is dead or at max_bounces -- to its next sample HERE, so that the sample's first
        // Philox block is computed with everybody else's refill instead of on demand by the one lane in five that starts a
        // sample: bit-identical images, slower on every config.  The extra state test at the top of every slot costs more
        // than the refills it merges.)
        {   // converged here: the lanes that are short of draws for this slot compute their Philox blocks together
            uint32_t need = 0;
            if (status == ST_VERTEX && !dead) {
                if (light_slot) need = slot < 8u ? (draw_hint >> (4u * slot)) & 15u : 4u;
                else if ((uint32_t)depth < a.max_bounces) need = 4u;  // gen_bool + Beckmann (1 + UnitCircle) or UnitDisc
            }
            rng.template ensure<W>(wmask, need);
        }
        bool active = false;  // this lane sends a ray through the trace site in this slot

        if (light_slot) {
            // ================= sample_lights, one sampled light per slot ==================
            if (status == ST_VERTEX && !dead) {
                const MaterialRec<R> mat = sv.materials[mat_id];
                while (scene_light<FEAT>(sv, li).kind == LIGHT_AMBIENT) {  // ambient lights listed before it
                    const LightRec<R>& l = scene_light<FEAT>(sv, li);
                    color = color + cmul(mk(l.color[0], l.color[1], l.color[2]), mat_color(mat));
                    li++;
                }
                const LightRec<R>& l = scene_light<FEAT>(sv, li);
                li++;
                Vec3<R> intensity, wi;
                R dist;
                illuminate<R, FEAT>(sv, l, pos, rng, intensity, wi, dist);
                bool skip = false;
                if (!M<R>::literal) {
                    // provably zero contribution: no shadow ray (the draws above are still consumed)
                    const bool zero_i = intensity.x == (R)0 && intensity.y == (R)0 && intensity.z == (R)0;
                    skip = zero_i || (!mat.transparent && M<R>::signbit(dot(n, wi)));
                }
                if (!skip) {
                    const Vec3<R> f = bsdf<R, FEAT>(mat, n, wo, wi);
                    contrib = cmul(f, intensity) * dot(wi, n);  // renderer.rs:198-199 (signed cosine)
                    tmax = M<R>::next_up(dist);  // occluded iff some hit has t <= dist (renderer.rs:197)
                    ro = offset_origin(pos, ng, wi, err_scale);
                    rd = wi;
                    active = true;
                }
            }
        } else {
            // ================= segment slot: bounce, finish, regenerate ====================
            if (status == ST_VERTEX) {
                const MaterialRec<R> mat = sv.materials[mat_id];
                while (li < sv.nlights) {  // trailing ambient lights (and, for a dead vertex, all of them)
                    const LightRec<R>& l = scene_light<FEAT>(sv, li);
                    if (l.kind == LIGHT_AMBIENT) color = color + cmul(mk(l.color[0], l.color[1], l.color[2]), mat_color(mat));
                    li++;
                }
                Vec3<R> wi = rd;
                R pdf = (R)1;
                bool bounce = false;
                if ((uint32_t)depth < a.max_bounces && !dead) bounce = sample_f<R, FEAT>(mat, n, wo, rng, wi, pdf);
                if (bounce) {  // renderer.rs:157-164
                    const Vec3<R> f = bsdf<R, FEAT>(mat, n, wo, wi);
                    const R abscos = M<R>::abs(dot(wi, n));
                    if constexpr (M<R>::literal) {
                        Level<R>& lv = stack[depth];
                        lv.local[0] = color.x; lv.local[1] = color.y; lv.local[2] = color.z;
                        lv.f[0] = f.x; lv.f[1] = f.y; lv.f[2] = f.z;
                        lv.inv_pdf = (R)1 / pdf;
                        lv.abscos = abscos;
                    } else {
                        // exp() underflows in f32 long before it does in f64: a pdf of exactly 0 can only
                        // pair with a direction whose true weight is negligible -> weight 0, not 0/0.  The same for
                        // a weight that is not >= 0 (NaN from 0/0 in the BSDF): the composition below needs W >= 0.
                        const R k = pdf > (R)0 ? abscos / pdf : (R)0;
                        Vec3<R> w = {f.x * k, f.y * k, f.z * k};
                        w = {w.x >= (R)0 ? w.x : (R)0, w.y >= (R)0 ? w.y : (R)0, w.z >= (R)0 ? w.z : (R)0};
                        // compose this level (a = color, w) under the levels above it
                        const Vec3<R> Wa = cmul(fwdT, color);
                        fwdC = {M<R>::min((R)100 * fwdT.x, fwdC.x - Wa.x), M<R>::min((R)100 * fwdT.y, fwdC.y - Wa.y),
                                M<R>::min((R)100 * fwdT.z, fwdC.z - Wa.z)};
                        fwdA = fwdA + Wa;
                        fwdT = cmul(fwdT, w);
                        // an exactly zero weight (direction sampled below an opaque surface): the whole
                        // subtree is multiplied by 0 -- do not trace it
                        bounce = !(w.x == (R)0 && w.y == (R)0 && w.z == (R)0);
                    }
                    if (bounce) {
                        depth++;
                        tmax = M<R>::inf();
                        ro = offset_origin(pos, ng, wi, err_scale);
                        rd = wi;
                        active = true;
                    }
                }
                if (!bounce) {
                    // (after a zero-weight sample: depth was not advanced; f32: fwdT is 0 and fwdA already holds
                    // this vertex's colour, so the composite evaluates to it whatever Lterm is; f64: the level at
                    // stack[depth] is not unwound, Lterm = color is the value of this vertex)
                    Lterm = color;
                    status = ST_FINISH;
                }
            }
            if (status == ST_FINISH) {
                Vec3<R> L = Lterm;
                if constexpr (!M<R>::literal) {
                    // the composite of every level's clamp, applied to what came back from the last ray
                    // (0 * inf cannot occur: fwdT = 0 pairs with a finite Lterm = colour of the last vertex)
                    L = {fwdA.x + M<R>::min(fwdT.x * Lterm.x, fwdC.x), fwdA.y + M<R>::min(fwdT.y * Lterm.y, fwdC.y),
                         fwdA.z + M<R>::min(fwdT.z * Lterm.z, fwdC.z)};
                    fwdA = {(R)0, (R)0, (R)0};
                    fwdT = {(R)1, (R)1, (R)1};
                    fwdC = {clamp_inf, clamp_inf, clamp_inf};
                } else {
                    for (int k = depth - 1; k >= 0; k--) L = unwind(stack[k], L);
                }
                acc0 += (double)L.x;
                acc1 += (double)L.y;
                acc2 += (double)L.z;
                s++;
                if (a.nchunks > 1 && (--chunk_left == 0 || s == s_end)) {  // chunk complete: publish its sum
                    double* o = a.partial + ((size_t)chunk_id * pstride + pslot) * 3;
                    o[0] = acc0; o[1] = acc1; o[2] = acc2;
                    acc0 = acc1 = acc2 = 0.0;
                    chunk_id++;
                    chunk_left = a.chunk;
                }
                status = ST_FRESH;
            }
            if (status == ST_FRESH) {
                if (s >= s_end) {
                    status = ST_IDLE;
                } else {
                    rng.init(a.seed, pix, a.first_sample + s);
                    const R dx = gen_range(rng, (R)-1 / dim, (R)1 / dim);
                    const R dy = gen_range(rng, (R)-1 / dim, (R)1 / dim);
                    // Camera::cast_ray (camera.rs:64-81)
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
                    ro = origin;
                    rd = M<R>::normalize(new_dir);
                    tmax = M<R>::inf();
                    depth = 0;
                    active = true;
                }
            }
        }

        // ================= the single get_closest_hit site ==============================
        if (W::all(wmask, status == ST_IDLE)) break;  // also re-converges the warp
        Hit<R> h;
        h.t = tmax;
        h.obj = -1;
        bool traced = false;
#if defined(__CUDACC__) && !defined(RPTB_HOST_EMU)
        if constexpr (!M<R>::literal && (FEAT & F_BVH) != 0 && W::width == 32u && RPTB_COOP_MAX > 0) {
            // meshes through the eight-wide BVH, eight lanes per ray (every lane of the warp takes part, with or without a ray
            // of its own); a warp at the image's edge, with fewer than 32 lanes, keeps the per-lane binary traversal
            if (coop != nullptr && wmask == 0xffffffffu) {
                if (active) pc.rays++;
                closest_hit_coop<STATS, FEAT>(sv, active, ro, rd, tmin, light_slot, h, pc.ts, lane, *static_cast<CoopWarp*>(coop));
                traced = true;
            }
        }
#endif
        if (!traced && active) {
            pc.rays++;
            closest_hit<R, STATS, FEAT>(sv, ro, rd, tmin, light_slot, h, pc.ts);
        }

        // ================= consume the answer ============================================
        if (active) {
            if (light_slot) {
                if (h.obj < 0) color = color + contrib;
            } else {
                pc.segments++;  // one trace_ray invocation
                if (h.obj < 0) {
                    if ((FEAT & F_HDRI) && sv.env.kind != 0) pc.env_lookups++;
                    Lterm = env_color<R, FEAT>(sv.env, rd);
                    status = ST_FINISH;
                } else {
                    const ObjectRec<R>& ob = sv.objects[h.obj];
                    const Surface<R> sf = finalize_hit<R, FEAT>(sv, ob, ro, rd, h);
                    if (sf.on_mesh) pc.mesh_hits++;
                    pos = ro + h.t * rd;
                    n = sf.n;
                    ng = sf.ng;
                    wo = -M<R>::normalize(rd);
                    mat_id = ob.material;
                    const MaterialRec<R> mat = sv.materials[mat_id];
                    err_scale = M<R>::literal ? (R)0 : M<R>::max(max_abs3(pos), max_abs3(ro));
                    color = mat.emittance * mat_color(mat);
                    // opaque surface seen from its back: bsdf == 0 for every wi (material.rs:130-133),
                    // so neither the lights nor the bounce can contribute (f32 only; f64 stays literal)
                    dead = !M<R>::literal && !mat.transparent && M<R>::signbit(dot(n, wo));
                    li = 0;
                    status = ST_VERTEX;
                }
            }
        }
        slot = slot >= Ks ? 0u : slot + 1u;
    }

    // color / iterations * 2^EV  (renderer.rs:141)
    if (a.nchunks > 1) {
        // the chunk sums were published as they completed; resolve_chunks_kernel finishes the pixel
    } else {
        const double it = (double)a.iterations;
        R* out = a.out + 3 * (a.compact ? pslot : (size_t)pix);
        out[0] = (R)(acc0 / it * (double)a.exposure_scale);
        out[1] = (R)(acc1 / it * (double)a.exposure_scale);
        out[2] = (R)(acc2 / it * (double)a.exposure_scale);
    }

    if (a.counters) {
        const unsigned m = W::activemask();
        const uint32_t v0 = W::reduce_add(m, pc.segments), v1 = W::reduce_add(m, pc.rays);
        const uint32_t v2 = W::reduce_add(m, pc.mesh_hits), v3 = W::reduce_add(m, pc.env_lookups);
        // node/tri counters can exceed 2^32 per warp on long renders: reduce in two halves
        const uint32_t n_lo = W::reduce_add(m, pc.ts.node_visits & 0xFFFFu), n_hi = W::reduce_add(m, pc.ts.node_visits >> 16);
        const uint32_t t_lo = W::reduce_add(m, pc.ts.tri_tests & 0xFFFFu), t_hi = W::reduce_add(m, pc.ts.tri_tests >> 16);
        const uint32_t o_lo = W::reduce_add(m, pc.ts.object_tests & 0xFFFFu), o_hi = W::reduce_add(m, pc.ts.object_tests >> 16);
        const uint32_t bn_lo = W::reduce_add(m, pc.ts.bvh_nodes & 0xFFFFu), bn_hi = W::reduce_add(m, pc.ts.bvh_nodes >> 16);
        const uint32_t bt_lo = W::reduce_add(m, pc.ts.bvh_tris & 0xFFFFu), bt_hi = W::reduce_add(m, pc.ts.bvh_tris >> 16);
        if (W::is_leader(m, lane)) {
            W::add(&a.counters->segments, (unsigned long long)v0);
            W::add(&a.counters->rays, (unsigned long long)v1);
            W::add(&a.counters->mesh_hits, (unsigned long long)v2);
            W::add(&a.counters->env_lookups, (unsigned long long)v3);
            if (STATS) {
                W::add(&a.counters->node_visits, (unsigned long long)n_lo + ((unsigned long long)n_hi << 16));
                W::add(&a.counters->tri_tests, (unsigned long long)t_lo + ((unsigned long long)t_hi << 16));
                W::add(&a.counters->object_tests, (unsigned long long)o_lo + ((unsigned long long)o_hi << 16));
                if ((FEAT & F_BVH) != 0) {
                    W::add(&a.counters->bvh_node_visits, (unsigned long long)bn_lo + ((unsigned long long)bn_hi << 16));
                    W::add(&a.counters->bvh_tri_tests, (unsigned long long)bt_lo + ((unsigned long long)bt_hi << 16));
                }
            }
        }
    }
}

#ifdef __CUDACC__
template <class R, int MAXD, bool STATS, int FEAT = F_ALL>
__global__ void __launch_bounds__(RENDER_THREADS, render_min_blocks(FEAT)) render_kernel(const __grid_constant__ SceneView<R> sv, const __grid_constant__ RenderArgs<R> a) {
    if constexpr (M<R>::literal) {
        render_thread<R, MAXD, STATS, FEAT, DeviceWarp>(sv, a, blockIdx.x, blockIdx.y, threadIdx.x);
    } else {
        __shared__ uint32_t rng_ring[RNG_RING * RENDER_THREADS];  // 4 KB: every thread's 8 buffered draws, one bank per lane
#ifndef RPTB_HOST_EMU
        if constexpr ((FEAT & F_BVH) != 0 && RPTB_COOP_MAX > 0) {
            __shared__ CoopWarp coop[RENDER_THREADS / 32];  // 3 KB per warp: compacted rays, answers, the lane groups' stacks
            render_thread<R, MAXD, STATS, FEAT, DeviceWarp>(sv, a, blockIdx.x, blockIdx.y, threadIdx.x, rng_ring, &coop[threadIdx.x >> 5]);
        } else
#endif
        {
            render_thread<R, MAXD, STATS, FEAT, DeviceWarp>(sv, a, blockIdx.x, blockIdx.y, threadIdx.x, rng_ring);
        }
    }
}
#endif

// Add the chunk sums of every pixel in chunk order and apply 1/iterations * 2^EV (renderer.rs:141).
template <class R>
RPTB_D void resolve_chunks_thread(const RenderArgs<R>& a, const uint32_t block_x, const uint32_t thread_x) {
    const uint32_t tile = a.shard_index + block_x * a.shard_count;
    const uint32_t tx = tile % a.tiles_x, ty = tile / a.tiles_x;
    const uint32_t warp = thread_x >> 5, lane = thread_x & 31u;
    const uint32_t x = tx * TILE_W + (warp & 1u) * 8u + (lane & 7u);
    const uint32_t y = ty * TILE_H + (warp >> 1) * 4u + (lane >> 3);
    if (x >= a.width || y >= a.height) return;
    const size_t slot = (size_t)block_x * RENDER_THREADS + thread_x;
    const size_t stride = (size_t)a.ntiles_mine * RENDER_THREADS;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (uint32_t c = 0; c < a.nchunks; c++) {
        const double* p = a.partial + ((size_t)c * stride + slot) * 3;
        s0 += p[0]; s1 += p[1]; s2 += p[2];
    }
    const double it = (double)a.iterations;
    R* out = a.out + 3 * (a.compact ? slot : (size_t)y * a.width + x);
    out[0] = (R)(s0 / it * (double)a.exposure_scale);
    out[1] = (R)(s1 / it * (double)a.exposure_scale);
    out[2] = (R)(s2 / it * (double)a.exposure_scale);
}
#ifdef __CUDACC__
template <class R>
__global__ void resolve_chunks_kernel(const RenderArgs<R> a) {
    resolve_chunks_thread<R>(a, blockIdx.x, threadIdx.x);
}
#endif

// Zero the pixels of tiles that belong to other shards (so an all-reduce(sum) of the
// shard buffers is the full image, bit-identical for any shard count).
template <class R>
__global__ void clear_kernel(R* out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (R)0;
}

// ---- K2: Renderer::get_closest_hit for a batch of world rays -----------------------
template <class R, bool STATS, int FEAT>
__global__ void closest_hit_kernel(const SceneView<R> sv, const double* __restrict__ rays, uint64_t n, double tmin_d,
                                   double* __restrict__ out_t, int32_t* __restrict__ out_obj,
                                   double* __restrict__ out_n, DeviceCounters* counters) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    TravStats ts = {0, 0, 0, 0, 0};
    if (i < n) {
        const double* r = rays + 6 * i;
        const Vec3<R> o = {(R)r[0], (R)r[1], (R)r[2]};
        const Vec3<R> d = {(R)r[3], (R)r[4], (R)r[5]};
        Hit<R> h;
        h.t = M<R>::inf();
        closest_hit<R, STATS, FEAT>(sv, o, d, (R)tmin_d, false, h, ts);
        out_obj[i] = h.obj;
        out_t[i] = h.obj >= 0 ? (double)h.t : (double)INFINITY;
        if (out_n) {
            Vec3<R> nn = {(R)0, (R)0, (R)0};
            if (h.obj >= 0) nn = finalize_hit<R, FEAT>(sv, sv.objects[h.obj], o, d, h).n;
            out_n[3 * i] = (double)nn.x;
            out_n[3 * i + 1] = (double)nn.y;
            out_n[3 * i + 2] = (double)nn.z;
        }
    }
    if (counters) {
        if (i < n) atomicAdd(&counters->rays, 1ull);
        if (STATS && i < n) {
            atomicAdd(&counters->node_visits, (unsigned long long)ts.node_visits);
            atomicAdd(&counters->tri_tests, (unsigned long long)ts.tri_tests);
            atomicAdd(&counters->object_tests, (unsigned long long)ts.object_tests);
            if ((FEAT & F_BVH) != 0) {
                atomicAdd(&counters->bvh_node_visits, (unsigned long long)ts.bvh_nodes);
                atomicAdd(&counters->bvh_tri_tests, (unsigned long long)ts.bvh_tris);
            }
        }
    }
}

#if defined(__CUDACC__) && !defined(RPTB_HOST_EMU)
// The same query through the product path's mesh traversal: every warp takes 32 rays, meshes are entered by lane groups
// over the eight-wide BVH (geometry.cuh, closest_hit_coop).  f32 scenes with a BVH.
template <bool STATS, int FEAT>
__global__ void __launch_bounds__(128) closest_hit_coop_kernel(const SceneView<float> sv, const double* __restrict__ rays, uint64_t n,
                                                               double tmin_d, double* __restrict__ out_t, int32_t* __restrict__ out_obj,
                                                               double* __restrict__ out_n, DeviceCounters* counters) {
    __shared__ CoopWarp coop[4];
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < n;  // nobody leaves: the traversal needs whole warps
    TravStats ts = {0, 0, 0, 0, 0};
    Vec3<float> o = {0.f, 0.f, 0.f}, d = {0.f, 0.f, 1.f};
    if (active) {
        const double* r = rays + 6 * i;
        o = {(float)r[0], (float)r[1], (float)r[2]};
        d = {(float)r[3], (float)r[4], (float)r[5]};
    }
    Hit<float> h;
    h.t = INFINITY;
    closest_hit_coop<STATS, FEAT>(sv, active, o, d, (float)tmin_d, false, h, ts, threadIdx.x & 31u, coop[threadIdx.x >> 5]);
    if (active) {
        out_obj[i] = h.obj;
        out_t[i] = h.obj >= 0 ? (double)h.t : (double)INFINITY;
        if (out_n) {
            Vec3<float> nn = {0.f, 0.f, 0.f};
            if (h.obj >= 0) nn = finalize_hit<float, FEAT>(sv, sv.objects[h.obj], o, d, h).n;
            out_n[3 * i] = (double)nn.x;
            out_n[3 * i + 1] = (double)nn.y;
            out_n[3 * i + 2] = (double)nn.z;
        }
    }
    if (counters) {
        if (active) atomicAdd(&counters->rays, 1ull);
        if (STATS) {
            atomicAdd(&counters->node_visits, (unsigned long long)ts.node_visits);
            atomicAdd(&counters->tri_tests, (unsigned long long)ts.tri_tests);
            atomicAdd(&counters->object_tests, (unsigned long long)ts.object_tests);
            atomicAdd(&counters->bvh_node_visits, (unsigned long long)ts.bvh_nodes);
            atomicAdd(&counters->bvh_tri_tests, (unsigned long long)ts.bvh_tris);
        }
    }
}
#endif

// ---- point-wise Material::bsdf / sample_f ------------------------------------------------
template <class R>
__global__ void bsdf_kernel(const MaterialRec<R> m, const double* __restrict__ dirs, uint64_t n, double* __restrict__ out) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* d = dirs + 9 * i;
    const Vec3<R> f = bsdf(m, mk((R)d[0], (R)d[1], (R)d[2]), mk((R)d[3], (R)d[4], (R)d[5]), mk((R)d[6], (R)d[7], (R)d[8]));
    out[3 * i] = (double)f.x;
    out[3 * i + 1] = (double)f.y;
    out[3 * i + 2] = (double)f.z;
}

template <class R>
__global__ void sample_f_kernel(const MaterialRec<R> m, const double* __restrict__ dirs, uint64_t n, uint64_t seed,
                                double* __restrict__ out_wi, double* __restrict__ out_pdf) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* d = dirs + 6 * i;
    Rng<R> rng;
    rng.init(seed, (uint32_t)i, 0);
    Vec3<R> wi = {(R)0, (R)0, (R)0};
    R pdf = (R)-1;
    if (!sample_f(m, mk((R)d[0], (R)d[1], (R)d[2]), mk((R)d[3], (R)d[4], (R)d[5]), rng, wi, pdf)) {
        wi = mk((R)0, (R)0, (R)0);
        pdf = (R)-1;
    }
    out_wi[3 * i] = (double)wi.x;
    out_wi[3 * i + 1] = (double)wi.y;
    out_wi[3 * i + 2] = (double)wi.z;
    out_pdf[i] = (double)pdf;
}

// ---- point-wise Light::illuminate (light.rs:23-47), Shape::sample of the light's object included ----------
// Stream i = Philox(seed, i, sample 0), like sample_f_kernel.  Ambient returns (color, 0, 0) as the reference does.
template <class R, int FEAT>
__global__ void illuminate_kernel(const SceneView<R> sv, uint32_t light, const double* __restrict__ pos, uint64_t n, uint64_t seed,
                                  double* __restrict__ out_i, double* __restrict__ out_wi, double* __restrict__ out_dist) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const LightRec<R>& l = sv.lights[light];
    Vec3<R> I = mk(l.color[0], l.color[1], l.color[2]), wi = mk((R)0, (R)0, (R)0);
    R dist = (R)0;
    if (l.kind != LIGHT_AMBIENT) {
        Rng<R> rng;
        rng.init(seed, (uint32_t)i, 0);
        illuminate<R, FEAT>(sv, l, mk((R)pos[3 * i], (R)pos[3 * i + 1], (R)pos[3 * i + 2]), rng, I, wi, dist);
    }
    out_i[3 * i] = (double)I.x; out_i[3 * i + 1] = (double)I.y; out_i[3 * i + 2] = (double)I.z;
    out_wi[3 * i] = (double)wi.x; out_wi[3 * i + 1] = (double)wi.y; out_wi[3 * i + 2] = (double)wi.z;
    out_dist[i] = (double)dist;
}

}  // namespace rptb
