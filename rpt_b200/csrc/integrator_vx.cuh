// integrator_vx.cuh -- the f32 product megakernel, "vertex at once".
//
// Same estimator and the same per-path sequence of operations and random draws as integrator.cuh's slot
// engine (which stays: it is the f64 parity gate and the fallback for scenes with more than VX_MAX_SHADOW
// sampled lights) -- Renderer::get_color / trace_ray / sample_lights of ekzhang/rpt src/renderer.rs:131-204 --
// scheduled differently:
//
//   slot engine   one ray per lane per loop iteration: shadow ray of light 0, ..., shadow ray of light Ks-1,
//                 bounce ray; Ks + 1 trips through the single get_closest_hit site per path vertex
//   this engine   one loop iteration per path vertex.  A lane at a vertex draws ALL its light samples and its
//                 BSDF sample first (the reference's draw order: sample_lights never depends on a shadow
//                 ray's answer), writes up to Ks + 1 rays into SHARED memory, and the warp traces them in one
//                 pass.  The shadow answers are applied before the level is closed, so the value is the same.
//
// Why (ncu, round 2): on mesh scenes 70 % of the slot engine's warp instructions were the BVH node loop at
// 5.3 of 32 lanes -- in any one slot only a few lanes of a warp hold a ray that enters the mesh's box, and the
// warp pays for the longest of them three times per vertex.  Here the rays of a warp that pass a mesh's root
// box (from all Ks + 1 slots of all 32 lanes) are COMPACTED by warp votes into a work list in shared memory and
// traversed 32 at a time by whichever lanes are free: a lane traverses rays that belong to other lanes' pixels
// and writes the hit back to the owner's record.  Analytic shapes and one-leaf meshes are intersected by the
// owning lane, for all its rays in one walk over scene.objects.
//
// Shared memory per thread (words): 8 per ray slot (origin, tmax, direction, flags), 2 per slot of hit record
// (t, object) + 4 for the segment slot (triangle / face code, barycentrics, group child), 3 per shadow slot
// (the light sample's pending contribution), 1 per slot of work list, 8 of RNG ring = 14 (Ks + 1) + 9.
#pragma once
#include "integrator.cuh"

namespace rptb {

constexpr uint32_t VX_MAX_SHADOW = 3;  // sampled lights this engine handles (one shared-memory ray slot each)

RPTB_HD uint32_t vx_shared_words(uint32_t k1) { return (uint32_t)RENDER_THREADS * (14u * k1 + 9u); }

struct VxShared {
    float4* ra;  // [k1][128]  origin, tmax
    float4* rb;  // [k1][128]  direction, unused
    float* ht;   // [k1][128]  closest t so far (HitRecord::time)
    int* hobj;   // [k1][128]  object index or -1
    uint32_t* haux;    // [128]  segment slot only: Hit::aux, bv, bw, child
    float* hbv;
    float* hbw;
    uint32_t* hchild;
    float* cx;   // [k1 - 1][128] pending contribution f (.) I (wi.n) of each light sample
    float* cy;
    float* cz;
    uint32_t* work;  // [4 warps][k1 * 32] compacted list of ray slots that enter the current mesh
    uint32_t* rng;   // [RNG_RING][128]
};

RPTB_D VxShared vx_carve(uint32_t* base, uint32_t k1) {
    VxShared s;
    const uint32_t T = (uint32_t)RENDER_THREADS;
    uint32_t* p = base;
    s.ra = reinterpret_cast<float4*>(p); p += 4u * k1 * T;
    s.rb = reinterpret_cast<float4*>(p); p += 4u * k1 * T;
    s.ht = reinterpret_cast<float*>(p); p += k1 * T;
    s.hobj = reinterpret_cast<int*>(p); p += k1 * T;
    s.haux = p; p += T;
    s.hbv = reinterpret_cast<float*>(p); p += T;
    s.hbw = reinterpret_cast<float*>(p); p += T;
    s.hchild = p; p += T;
    s.cx = reinterpret_cast<float*>(p); p += (k1 - 1u) * T;
    s.cy = reinterpret_cast<float*>(p); p += (k1 - 1u) * T;
    s.cz = reinterpret_cast<float*>(p); p += (k1 - 1u) * T;
    s.work = p; p += k1 * T;
    s.rng = p;
    return s;
}

template <int FEAT>
RPTB_D const ObjectRec<float>& vx_object(const SceneView<float>& sv, uint32_t i) {
    if constexpr ((FEAT & F_SMALL) != 0) return sv.small.objects[i];
    else return sv.objects[i];
}
template <int FEAT>
RPTB_D const MeshRec<float>& vx_mesh(const SceneView<float>& sv, uint32_t i) {
    if constexpr ((FEAT & F_SMALL) != 0) return sv.small.meshes[i];
    else return sv.meshes[i];
}

// get_closest_hit (renderer.rs:211-220) for every ray slot of every lane of the warp.  `valid` bit j: this lane's
// slot j holds a ray.  Slots 0 .. k1-2 are shadow queries (any hit with t < tmax ends them), slot k1-1 is the
// segment ray.  On return ht / hobj (and, for the segment slot, haux / hbv / hbw / hchild) hold the answers.
template <bool STATS, int FEAT, class W>
RPTB_D void vx_trace(const SceneView<float>& sv, const VxShared& S, const uint32_t k1, const uint32_t valid, const uint32_t me,
                     const uint32_t lane, const uint32_t warp, const unsigned wmask, TravStats& ts) {
    const float tmin = 1e-12f;  // EPSILON, renderer.rs:14
    const uint32_t T = (uint32_t)RENDER_THREADS, seg = k1 - 1u;
    for (uint32_t j = 0; j < k1; j++)
        if ((valid >> j) & 1u) {
            S.ht[j * T + me] = S.ra[j * T + me].w;
            S.hobj[j * T + me] = -1;
        }
    if ((valid >> seg) & 1u) {
        S.haux[me] = 0u;
        S.hbv[me] = 0.0f;
        S.hbw[me] = 0.0f;
        S.hchild[me] = 0u;
    }
    const uint32_t nobj = sv.nobjects;
    for (uint32_t i = 0; i < nobj; i++) {
        const ObjectRec<float>& ob = vx_object<FEAT>(sv, i);
        bool coop = false;  // warp-uniform: every lane looks at the same object
        if constexpr ((FEAT & F_BVH) != 0) coop = ob.kind == SHAPE_MESH && !vx_mesh<FEAT>(sv, ob.mesh).root_is_leaf;
        if (coop) {
            // ---- a mesh with a BVH: compact the rays that enter its box, traverse them with whatever lanes are free
            const MeshRec<float>& mm = sv.meshes[ob.mesh];
            uint32_t* work = S.work + warp * (k1 * 32u);
            uint32_t count = 0;
            for (uint32_t j = 0; j < k1; j++) {
                bool pred = ((valid >> j) & 1u) != 0u;
                if (pred && j != seg && S.hobj[j * T + me] >= 0) pred = false;  // an occluded shadow ray is finished
                if (pred) {
                    if (STATS) ts.object_tests++;
                    const float4 A = S.ra[j * T + me], B = S.rb[j * T + me];
                    Vec3<float> o = {A.x, A.y, A.z}, d = {B.x, B.y, B.z};
                    if (ob.has_transform) {
                        const Vec3<float> lo = xform_point(ob.inv, o), ld = xform_dir(ob.inv, d);
                        o = lo;
                        d = ld;
                    }
                    // root cull: BoundingBox::intersect of KdTree::bounds (kdtree.rs:130-134) against [tmin, closest so far]
                    const Vec3<float> iv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};
                    const float x1 = (mm.bmin[0] - o.x) * iv.x, x2 = (mm.bmax[0] - o.x) * iv.x;
                    const float y1 = (mm.bmin[1] - o.y) * iv.y, y2 = (mm.bmax[1] - o.y) * iv.y;
                    const float z1 = (mm.bmin[2] - o.z) * iv.z, z2 = (mm.bmax[2] - o.z) * iv.z;
                    const float l0 = fmaxf(fmaxf(fminf(x1, x2), fminf(y1, y2)), fminf(z1, z2));
                    const float h0 = fminf(fminf(fmaxf(x1, x2), fmaxf(y1, y2)), fmaxf(z1, z2));
                    pred = !(fmaxf(l0, tmin) > fminf(h0, S.ht[j * T + me]));
                }
                const unsigned m = W::ballot(wmask, pred);
                if (pred) work[count + W::rank(m, lane)] = j * T + me;
                count += W::popc(m);
            }
            W::sync(wmask);
            // (a warp at the image's edge has fewer than 32 lanes: stride by the lanes that exist, index by rank among them)
            const uint32_t nact = W::popc(wmask), myrank = W::rank(wmask, lane);
            for (uint32_t b = 0; b < count; b += nact) {
                const uint32_t it = b + myrank;
                if (it < count) {
                    const uint32_t id = work[it];  // slot * 128 + owner thread: possibly another lane's ray
                    const bool any = (id / T) != seg;
                    const float4 A = S.ra[id], B = S.rb[id];
                    Vec3<float> o = {A.x, A.y, A.z}, d = {B.x, B.y, B.z};
                    if (ob.has_transform) {
                        const Vec3<float> lo = xform_point(ob.inv, o), ld = xform_dir(ob.inv, d);
                        o = lo;
                        d = ld;
                    }
                    Hit<float> h;
                    h.t = S.ht[id];
                    h.obj = -1;
                    h.aux = 0;
                    h.bv = h.bw = 0.0f;
                    if (bvh_intersect<STATS>(mm, o, d, tmin, any, h, ts)) {
                        S.ht[id] = h.t;
                        S.hobj[id] = (int)i;
                        if (!any) {
                            const uint32_t own = id % T;
                            S.haux[own] = h.aux;
                            S.hbv[own] = h.bv;
                            S.hbw[own] = h.bw;
                        }
                    }
                }
            }
            W::sync(wmask);
        } else {
            // ---- analytic shapes, one-leaf meshes, kd-trees of shapes: the owning lane, all of its rays
            for (uint32_t j = 0; j < k1; j++) {
                if (!((valid >> j) & 1u)) continue;
                const bool any = j != seg;
                if (any && S.hobj[j * T + me] >= 0) continue;
                if (STATS) ts.object_tests++;
                const float4 A = S.ra[j * T + me], B = S.rb[j * T + me];
                Hit<float> h;
                h.t = S.ht[j * T + me];
                h.obj = -1;
                h.aux = 0;
                h.bv = h.bw = 0.0f;
                if constexpr ((FEAT & F_GROUP) != 0) h.child = 0;
                if (object_intersect<float, STATS, FEAT>(sv, ob, mk(A.x, A.y, A.z), mk(B.x, B.y, B.z), tmin, any, h, ts)) {
                    S.ht[j * T + me] = h.t;
                    S.hobj[j * T + me] = (int)i;
                    if (!any) {
                        S.haux[me] = h.aux;
                        S.hbv[me] = h.bv;
                        S.hbw[me] = h.bw;
                        if constexpr ((FEAT & F_GROUP) != 0) S.hchild[me] = h.child;
                    }
                }
            }
        }
    }
}

template <bool STATS, int FEAT, class W>
RPTB_D void render_thread_vx(const SceneView<float>& sv, const RenderArgs<float>& a, const uint32_t block_x, const uint32_t block_y,
                             const uint32_t thread_x, uint32_t* smem) {
    typedef float R;
    const uint32_t T = (uint32_t)RENDER_THREADS;
    const uint32_t tile = a.shard_index + block_x * a.shard_count;
    const uint32_t tx = tile % a.tiles_x, ty = tile / a.tiles_x;
    const uint32_t warp = thread_x >> 5, lane = W::width == 1u ? 0u : (thread_x & 31u);
    const uint32_t x = tx * TILE_W + (warp & 1u) * 8u + (thread_x & 7u);
    const uint32_t y = ty * TILE_H + (warp >> 1) * 4u + ((thread_x & 31u) >> 3);
    if (x >= a.width || y >= a.height) return;
    const uint32_t pix = y * a.width + x;
    const unsigned wmask = W::activemask();  // the lanes of this warp that own a pixel stay together to the end
    const uint32_t me = thread_x;

    const R dim = (R)max(a.width, a.height);
    const R xn = ((R)(2u * x + 1u) - (R)a.width) / dim;
    const R yn = ((R)(2u * (a.height - y) - 1u) - (R)a.height) / dim;
    const uint32_t Ks = a.ks, k1 = Ks + 1u;  // sampled (non-ambient) lights; ray slots
    uint32_t lights_need = 0;  // draws the light samples of one vertex typically take (refill hint, rng.cuh)
    for (uint32_t i = 0; i < sv.nlights; i++) lights_need += light_draws_hint(scene_light<FEAT>(sv, i));
    const VxShared S = vx_carve(smem, k1);

    PathCounters pc = {0, 0, 0, 0, {0, 0, 0, 0, 0}};
    double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0;
    RngRing rng;
    rng.bind(S.rng + me, T);
    rng.init(a.seed, pix, a.first_sample);

    // the vertex being shaded (status == ST_VERTEX)
    Vec3<R> pos = {0, 0, 0}, n = {0, 0, 1}, ng = {0, 0, 1}, wo = {0, 0, 1}, color = {0, 0, 0};
    R err_scale = (R)0;
    uint32_t mat_id = 0;
    bool dead = false;
    // this thread's run of samples: [s, s_end) of [0, iterations) = chunks_per_group whole chunks; `s` is the sample in
    // flight (ST_VERTEX) or the next one to start (ST_FRESH)
    uint32_t s = block_y * a.chunks_per_group * a.chunk;
    const uint32_t s_end = min(s + a.chunks_per_group * a.chunk, a.iterations);
    uint32_t chunk_id = block_y * a.chunks_per_group, chunk_left = a.chunk;
    const size_t pslot = (size_t)block_x * T + thread_x;
    const size_t pstride = (size_t)a.ntiles_mine * T;
    uint32_t depth = 0;
    int status = s < s_end ? ST_FRESH : ST_IDLE;
    // trace_ray's value as a function of the radiance x coming back from below the deepest level so far:
    // L(x) = fwdA + min(fwdT x, fwdC) per channel (integrator.cuh, render_thread)
    const R clamp_inf = M<R>::inf();
    Vec3<R> fwdA = {(R)0, (R)0, (R)0}, fwdT = {(R)1, (R)1, (R)1}, fwdC = {clamp_inf, clamp_inf, clamp_inf};

    auto finish_sample = [&](Vec3<R> Lterm) {  // the path ended with radiance Lterm below its deepest level
        const R lx = fwdA.x + M<R>::min(fwdT.x * Lterm.x, fwdC.x), ly = fwdA.y + M<R>::min(fwdT.y * Lterm.y, fwdC.y),
                lz = fwdA.z + M<R>::min(fwdT.z * Lterm.z, fwdC.z);
        acc0 += (double)lx;
        acc1 += (double)ly;
        acc2 += (double)lz;
        fwdA = {(R)0, (R)0, (R)0};
        fwdT = {(R)1, (R)1, (R)1};
        fwdC = {clamp_inf, clamp_inf, clamp_inf};
        s++;
        if (a.nchunks > 1 && (--chunk_left == 0 || s == s_end)) {  // chunk complete: publish its sum
            double* o = a.partial + ((size_t)chunk_id * pstride + pslot) * 3;
            o[0] = acc0; o[1] = acc1; o[2] = acc2;
            acc0 = acc1 = acc2 = 0.0;
            chunk_id++;
            chunk_left = a.chunk;
        }
    };

    while (true) {
        if (W::all(wmask, status == ST_IDLE)) break;  // also re-converges the warp
        uint32_t valid = 0;    // bit j: ray slot j of this lane holds a ray in this iteration
        bool ending = false;   // the path in flight ends at this vertex (no bounce); finished after the shadow answers
        bool camera = false;   // the segment slot holds a fresh camera ray (not a bounce of the path in flight)
        Vec3<R> w = {(R)0, (R)0, (R)0};  // weight f |cos| / pdf of the bounce

        // ================= sample_lights: every light's sample, in list order (renderer.rs:177-204) ==========
        rng.template ensure<W>(wmask, status == ST_VERTEX && !dead ? lights_need : 0u);
        if (status == ST_VERTEX) {
            const MaterialRec<R> mat = sv.materials[mat_id];
            uint32_t jj = 0;
            for (uint32_t li = 0; li < sv.nlights; li++) {
                const LightRec<R>& l = scene_light<FEAT>(sv, li);
                if (l.kind == LIGHT_AMBIENT) {
                    color = color + cmul(mk(l.color[0], l.color[1], l.color[2]), mat_color(mat));
                    continue;
                }
                if (!dead) {
                    Vec3<R> intensity, wi;
                    R dist;
                    illuminate<R, FEAT>(sv, l, pos, rng, intensity, wi, dist);
                    // provably zero contribution: no shadow ray (the draws above are still consumed)
                    const bool zero_i = intensity.x == (R)0 && intensity.y == (R)0 && intensity.z == (R)0;
                    if (!(zero_i || (!mat.transparent && M<R>::signbit(dot(n, wi))))) {
                        const Vec3<R> f = bsdf<R, FEAT>(mat, n, wo, wi);
                        const Vec3<R> c = cmul(f, intensity) * dot(wi, n);  // renderer.rs:198-199 (signed cosine)
                        S.cx[jj * T + me] = c.x;
                        S.cy[jj * T + me] = c.y;
                        S.cz[jj * T + me] = c.z;
                        const Vec3<R> ro = offset_origin(pos, ng, wi, err_scale);
                        // occluded iff some hit has t <= dist (renderer.rs:197)
                        S.ra[jj * T + me] = make_float4(ro.x, ro.y, ro.z, M<R>::next_up(dist));
                        S.rb[jj * T + me] = make_float4(wi.x, wi.y, wi.z, 0.0f);
                        valid |= 1u << jj;
                    }
                }
                jj++;
            }
        }
        // ================= Material::sample_f: the bounce (renderer.rs:156-164) ==============================
        rng.template ensure<W>(wmask, status == ST_VERTEX && !dead && depth < a.max_bounces ? 4u : 0u);
        if (status == ST_VERTEX) {
            bool bounce = false;
            if (depth < a.max_bounces && !dead) {
                const MaterialRec<R> mat = sv.materials[mat_id];
                Vec3<R> wi = {(R)0, (R)0, (R)1};
                R pdf = (R)1;
                if (sample_f<R, FEAT>(mat, n, wo, rng, wi, pdf)) {
                    const Vec3<R> f = bsdf<R, FEAT>(mat, n, wo, wi);
                    const R abscos = M<R>::abs(dot(wi, n));
                    // a pdf of exactly 0 (exp underflow) or a weight that is not >= 0 (0/0 in the BSDF): weight 0
                    const R k = pdf > (R)0 ? abscos / pdf : (R)0;
                    w = {f.x * k, f.y * k, f.z * k};
                    w = {w.x >= (R)0 ? w.x : (R)0, w.y >= (R)0 ? w.y : (R)0, w.z >= (R)0 ? w.z : (R)0};
                    // an exactly zero weight (direction sampled below an opaque surface) multiplies its whole subtree
                    // by 0: the vertex's value is its own colour -- it ends the path without a ray
                    if (!(w.x == (R)0 && w.y == (R)0 && w.z == (R)0)) {
                        const Vec3<R> ro = offset_origin(pos, ng, wi, err_scale);
                        S.ra[Ks * T + me] = make_float4(ro.x, ro.y, ro.z, M<R>::inf());
                        S.rb[Ks * T + me] = make_float4(wi.x, wi.y, wi.z, 0.0f);
                        valid |= 1u << Ks;
                        bounce = true;
                    }
                }
            }
            ending = !bounce;
        }
        // ================= get_color's next sample: a camera ray for a lane whose path is over ==============
        // (a lane whose path ends at this vertex starts its next sample in the same iteration: the path in flight
        // draws nothing more, so the generator can move on before that path's shadow answers are in)
        const uint32_t s_cam = ending ? s + 1u : s;
        const bool want_cam = (status == ST_FRESH || ending) && s_cam < s_end;
        if (want_cam) rng.init(a.seed, pix, a.first_sample + s_cam);
        rng.template ensure<W>(wmask, want_cam ? (a.cam.aperture > (R)0 ? 4u : 2u) : 0u);
        if (want_cam) {
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
            const Vec3<R> rd = M<R>::normalize(new_dir);
            S.ra[Ks * T + me] = make_float4(origin.x, origin.y, origin.z, M<R>::inf());
            S.rb[Ks * T + me] = make_float4(rd.x, rd.y, rd.z, 0.0f);
            valid |= 1u << Ks;
            camera = true;
        }

        // ================= get_closest_hit for every ray of the warp =========================================
        pc.rays += W::popc(valid);
        vx_trace<STATS, FEAT, W>(sv, S, k1, valid, me, lane, warp, wmask, pc.ts);

        // ================= consume the answers ================================================================
        if (status == ST_VERTEX) {
            for (uint32_t jj = 0; jj < Ks; jj++)
                if (((valid >> jj) & 1u) && S.hobj[jj * T + me] < 0)
                    color = color + mk(S.cx[jj * T + me], S.cy[jj * T + me], S.cz[jj * T + me]);  // unoccluded (renderer.rs:197-200)
            if (ending) {
                finish_sample(color);
                status = ST_FRESH;
            } else {
                // close this level: x -> color + min(w x, 100) under the levels above it
                const Vec3<R> Wa = cmul(fwdT, color);
                fwdC = {M<R>::min((R)100 * fwdT.x, fwdC.x - Wa.x), M<R>::min((R)100 * fwdT.y, fwdC.y - Wa.y),
                        M<R>::min((R)100 * fwdT.z, fwdC.z - Wa.z)};
                fwdA = fwdA + Wa;
                fwdT = cmul(fwdT, w);
                depth++;
            }
        }
        if ((valid >> Ks) & 1u) {  // a segment was traced: one trace_ray invocation
            pc.segments++;
            if (camera) depth = 0;
            const float4 A = S.ra[Ks * T + me], B = S.rb[Ks * T + me];
            const Vec3<R> ro = {A.x, A.y, A.z}, rd = {B.x, B.y, B.z};
            Hit<R> h;
            h.t = S.ht[Ks * T + me];
            h.obj = S.hobj[Ks * T + me];
            if (h.obj < 0) {
                if ((FEAT & F_HDRI) && sv.env.kind != 0) pc.env_lookups++;
                finish_sample(env_color<R, FEAT>(sv.env, rd));
                status = ST_FRESH;
            } else {
                h.aux = S.haux[me];
                h.bv = S.hbv[me];
                h.bw = S.hbw[me];
                if constexpr ((FEAT & F_GROUP) != 0) h.child = S.hchild[me];
                const ObjectRec<R>& ob = sv.objects[h.obj];
                const Surface<R> sf = finalize_hit<R, FEAT>(sv, ob, ro, rd, h);
                if (sf.on_mesh) pc.mesh_hits++;
                pos = ro + h.t * rd;
                n = sf.n;
                ng = sf.ng;
                wo = -M<R>::normalize(rd);
                mat_id = ob.material;
                const MaterialRec<R> mat = sv.materials[mat_id];
                err_scale = M<R>::max(M<R>::max(max_abs3(pos), max_abs3(ro)), ob.err_mag);
                color = mat.emittance * mat_color(mat);
                // opaque surface seen from its back: bsdf == 0 for every wi (material.rs:130-133)
                dead = !mat.transparent && M<R>::signbit(dot(n, wo));
                status = ST_VERTEX;
            }
        }
        if (status == ST_FRESH && s >= s_end) status = ST_IDLE;
    }

    // color / iterations * 2^EV  (renderer.rs:141)
    if (a.nchunks <= 1) {
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
        const uint32_t n_lo = W::reduce_add(m, pc.ts.node_visits & 0xFFFFu), n_hi = W::reduce_add(m, pc.ts.node_visits >> 16);
        const uint32_t t_lo = W::reduce_add(m, pc.ts.tri_tests & 0xFFFFu), t_hi = W::reduce_add(m, pc.ts.tri_tests >> 16);
        const uint32_t o_lo = W::reduce_add(m, pc.ts.object_tests & 0xFFFFu), o_hi = W::reduce_add(m, pc.ts.object_tests >> 16);
        const uint32_t bn_lo = W::reduce_add(m, pc.ts.bvh_nodes & 0xFFFFu), bn_hi = W::reduce_add(m, pc.ts.bvh_nodes >> 16);
        const uint32_t bt_lo = W::reduce_add(m, pc.ts.bvh_tris & 0xFFFFu), bt_hi = W::reduce_add(m, pc.ts.bvh_tris >> 16);
        if (W::is_leader(m, thread_x & 31u)) {
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
#ifndef RPTB_VX_BLOCKS_LITE
#define RPTB_VX_BLOCKS_LITE 8
#endif
#ifndef RPTB_VX_BLOCKS_BVH
#define RPTB_VX_BLOCKS_BVH 6
#endif
constexpr int vx_min_blocks(int feat) {
    if (feat & F_EXT) return RPTB_MIN_BLOCKS_EXT;
    if (feat & F_BVH) return RPTB_VX_BLOCKS_BVH;
    const int base = feat & F_ALL;
    return base == 0 ? RPTB_VX_BLOCKS_LITE : base == F_TREE ? RPTB_MIN_BLOCKS_TREE : base == (F_TRANSP | F_HDRI) ? RPTB_MIN_BLOCKS_GLASS : RPTB_MIN_BLOCKS;
}
template <bool STATS, int FEAT>
__global__ void __launch_bounds__(RENDER_THREADS, vx_min_blocks(FEAT)) render_kernel_vx(const __grid_constant__ SceneView<float> sv,
                                                                                       const __grid_constant__ RenderArgs<float> a) {
    extern __shared__ __align__(16) uint32_t vx_smem[];
    render_thread_vx<STATS, FEAT, DeviceWarp>(sv, a, blockIdx.x, blockIdx.y, threadIdx.x, vx_smem);
}
#endif

}  // namespace rptb
