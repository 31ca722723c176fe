// geometry.cuh -- ray/shape intersection on the device.
//
// Reference functions restated (file:line in ekzhang/rpt @815b21c):
//   Ray::apply_transform             src/shape.rs:64-72
//   Transformed<T>::intersect        src/shape.rs:128-137
//   Sphere::intersect                src/shape/sphere.rs:13-45
//   Plane::intersect                 src/shape/plane.rs:17-32
//   Cube::intersect                  src/shape/cube.rs:20-72
//   Triangle::intersect              src/shape/mesh.rs:49-82
//   BoundingBox::intersect           src/kdtree.rs:54-68
//   KdTree::intersect/_subtree       src/kdtree.rs:129-136,151-223  (over triangles, and over whole shapes)
//   MonomialSurface::intersect       src/shape/monomial_surface.rs:21-105
//   Renderer::get_closest_hit        src/renderer.rs:211-220
//
// Design (not a port): the reference recurses through a pointer tree carrying a
// child AABB per call and re-slabbing it at every node (6 divisions).  Here the
// tree is a flat 8-byte-node array in DFS order and the traversal carries only the
// ray's parametric interval [lo, hi] inside the current cell on a small per-thread
// stack; the three pruning rules of kdtree.rs:207-222 are kept verbatim, so the
// set of leaves visited -- and therefore the closest hit -- is the reference's
// (SURVEY 8a a-TRAV).  Hit normals are *deferred*: the loop tracks (t, object,
// triangle, barycentrics / face code) and the normal of the winner is computed
// once, which is what the reference's repeated overwrites of `record.normal`
// amount to.
#pragma once
#include "scene_dev.cuh"

namespace rptb {

template <class R>
struct Hit {
    R t;           // HitRecord::time
    int obj;       // index into scene.objects, -1 = miss
    uint32_t aux;  // MESH: triangle index; CUBE: axis*2 + (normal positive ? 1 : 0)
    R bv, bw;      // MESH: barycentrics v, w
    uint32_t child;  // GROUP: which child of the kd-tree of shapes was hit (aux/bv/bw then describe the child's hit)
};

struct TravStats {
    uint32_t node_visits, tri_tests, object_tests;  // the reference-shaped kd-trees (kdtree.rs:151, mesh.rs:49) and Shape::intersect dispatches
    uint32_t bvh_nodes, bvh_tris;                   // the f32 path's BVH: 64-byte nodes fetched, triangles tested
};

template <class R>
RPTB_D Vec3<R> xform_point(const R* m, Vec3<R> p) {  // rows of a 3x4
    return {m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3], m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7],
            m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11]};
}
template <class R>
RPTB_D Vec3<R> xform_dir(const R* m, Vec3<R> d) {
    return {m[0] * d.x + m[1] * d.y + m[2] * d.z, m[4] * d.x + m[5] * d.y + m[6] * d.z,
            m[8] * d.x + m[9] * d.y + m[10] * d.z};
}
template <class R>
RPTB_D Vec3<R> xform3(const R* m, Vec3<R> d) {  // rows of a 3x3
    return {m[0] * d.x + m[1] * d.y + m[2] * d.z, m[3] * d.x + m[4] * d.y + m[5] * d.z,
            m[6] * d.x + m[7] * d.y + m[8] * d.z};
}

// ---------------------------------------------------------------- sphere ------
template <class R>
RPTB_D bool sphere_intersect(Vec3<R> o, Vec3<R> d, R tmin, R& rec_t) {
    const R a = length2(d);
    const R b = dot(d, o);
    R disc;
    if (M<R>::literal) {
        const R c = length2(o) - (R)1;
        disc = b * b - a * c;
    } else {
        // same quantity, b^2 - a(|o|^2 - 1) = a (1 - |o - (b/a) d|^2), without the f32 cancellation
        const R k = b / a;
        const Vec3<R> q = o - k * d;
        disc = a * ((R)1 - length2(q));
    }
    if (M<R>::signbit(disc)) return false;
    const R sd = M<R>::sqrt(disc);
    R t;
    const R t_minus = (-b - sd) / a;
    if (t_minus < tmin) {
        const R t_plus = (-b + sd) / a;
        if (t_plus < tmin) return false;
        t = t_plus;
    } else {
        t = t_minus;
    }
    if (t < rec_t) {
        rec_t = t;
        return true;
    }
    return false;
}

// ----------------------------------------------------------------- plane ------
template <class R>
RPTB_D bool plane_intersect(const R* n, R value, Vec3<R> o, Vec3<R> d, R tmin, R& rec_t) {
    const Vec3<R> nn = {n[0], n[1], n[2]};
    const R cosine = dot(nn, d);
    if (M<R>::abs(cosine) < (R)1e-8) return false;
    const R time = (value - dot(nn, o)) / cosine;
    if (time >= tmin && time < rec_t) {
        rec_t = time;
        return true;
    }
    return false;
}

// ------------------------------------------------------------------ cube ------
template <class R>
RPTB_D bool cube_intersect(Vec3<R> o, Vec3<R> d, R tmin, R& rec_t, uint32_t& code) {
    R lo[3], hi[3];
    bool swapped[3];
#pragma unroll
    for (int dim = 0; dim < 3; dim++) {
        const R oo = comp(o, dim), dd = comp(d, dim);
        R x1 = ((R)-0.5 - oo) / dd;
        R x2 = ((R)0.5 - oo) / dd;
        swapped[dim] = x1 > x2;
        if (swapped[dim]) {
            const R tmp = x1;
            x1 = x2;
            x2 = tmp;
        }
        lo[dim] = x1;
        hi[dim] = x2;
    }
    // entry face normal is -1 along dim unless swapped; exit face normal is +1 unless swapped
    R start, end;
    uint32_t sc, ec;
    if (lo[0] > lo[1] && lo[0] > lo[2]) { start = lo[0]; sc = 0u * 2u + (swapped[0] ? 1u : 0u); }
    else if (lo[1] > lo[2]) { start = lo[1]; sc = 1u * 2u + (swapped[1] ? 1u : 0u); }
    else { start = lo[2]; sc = 2u * 2u + (swapped[2] ? 1u : 0u); }
    if (hi[0] < hi[1] && hi[0] < hi[2]) { end = hi[0]; ec = 0u * 2u + (swapped[0] ? 0u : 1u); }
    else if (hi[1] < hi[2]) { end = hi[1]; ec = 1u * 2u + (swapped[1] ? 0u : 1u); }
    else { end = hi[2]; ec = 2u * 2u + (swapped[2] ? 0u : 1u); }
    if (start > end || end < tmin) return false;
    R time;
    uint32_t c;
    if (start < tmin) { time = end; c = ec; }
    else { time = start; c = sc; }
    if (time < rec_t) {
        rec_t = time;
        code = c;
        return true;
    }
    return false;
}

// ------------------------------------------------------- monomial surface ------
// y = height * (x^2 + z^2)^2 over the unit disc, the reference's scheme kept step for step: slab test of
// the bounding box, Newton towards the maximum of dist(t) when the ray starts below the surface, then 60
// bisections between t_min and that point (or t = 10000).  Which crossing it returns depends on t_min;
// callers inside a kd-tree pass the cell's t_min exactly as KdTree::intersect_subtree does.
template <class R>
RPTB_D bool monomial_intersect(R height, Vec3<R> o, Vec3<R> d, R tmin, R& rec_t) {
    R b_min, b_max;
    {
        const R x1 = ((R)-1 - o.x) / d.x, x2 = ((R)1 - o.x) / d.x;
        const R y1 = ((R)0 - o.y) / d.y, y2 = (height - o.y) / d.y;
        const R z1 = ((R)-1 - o.z) / d.z, z2 = ((R)1 - o.z) / d.z;
        b_min = M<R>::max(M<R>::max(M<R>::min(x1, x2), M<R>::min(y1, y2)), M<R>::min(z1, z2));
        b_max = M<R>::min(M<R>::min(M<R>::max(x1, x2), M<R>::max(y1, y2)), M<R>::max(z1, z2));
    }
    if (M<R>::max(b_min, tmin) > M<R>::min(b_max, rec_t)) return false;
    auto dist = [&](R t) {
        const R x = o.x + t * d.x, y = o.y + t * d.y, z = o.z + t * d.z;
        const R r2 = x * x + z * z;
        return y - height * (r2 * r2);
    };
    const R coef0 = o.x * o.x + o.z * o.z;
    const R coef1 = (R)2 * (o.x * d.x + o.z * d.z);
    const R coef2 = d.x * d.x + d.z * d.z;
    auto deriv = [&](R t) {
        const R dy = (R)2 * coef0 * coef1 + (R)2 * t * (coef1 * coef1 + (R)2 * coef0 * coef2) +
                     (R)3 * (t * t) * (R)2 * coef1 * coef2 + (R)4 * (t * (t * t)) * coef2 * coef2;
        return d.y - height * dy;
    };
    auto deriv2 = [&](R t) {
        const R dy = (R)2 * (coef1 * coef1 + (R)2 * coef0 * coef2) + (R)3 * (R)2 * t * (R)2 * coef1 * coef2 +
                     (R)4 * (R)3 * (t * t) * coef2 * coef2;
        return -height * dy;
    };
    const bool maximize = dist(tmin) < (R)0;
    R t_max;
    if (maximize) {
        R cur = (b_min + b_max) / (R)2;
        for (int it = 0; it < 10; it++) {
            if (dist(cur) > (R)0) break;
            cur -= deriv(cur) / deriv2(cur);
        }
        t_max = cur;
        if (t_max < tmin) return false;
    } else {
        t_max = (R)10000;
    }
    if ((dist(tmin) < (R)0) == (dist(t_max) < (R)0)) return false;
    R l = tmin, r = t_max;
    for (int it = 0; it < 60; it++) {
        const R m = (l + r) / (R)2;
        if ((dist(m) >= (R)0) == maximize) r = m;
        else l = m;
    }
    if (r > rec_t) return false;
    const R px = o.x + r * d.x, pz = o.z + r * d.z;
    if (px * px + pz * pz > (R)1) return false;  // beyond the rim
    rec_t = r;
    return true;
}

// -------------------------------------------------------------- triangle ------
// f64: the reference's formulas verbatim from the three vertices.
RPTB_D bool tri_intersect(const MeshRec<double>& m, uint32_t tri, Vec3<double> o, Vec3<double> d, double tmin,
                          double& rec_t, double& bv, double& bw) {
    const double* p = m.verts + 9 * (size_t)tri;
    const Vec3<double> v1 = {p[0], p[1], p[2]}, v2 = {p[3], p[4], p[5]}, v3 = {p[6], p[7], p[8]};
    const Vec3<double> d0 = v2 - v1, d1 = v3 - v1;
    const Vec3<double> pn = M<double>::normalize(cross(d0, d1));
    const double cosine = dot(pn, d);
    if (fabs(cosine) < 1e-8) return false;
    const double time = dot(pn, v1 - o) / cosine;
    if (time < tmin || time >= rec_t) return false;
    const Vec3<double> d2 = (o + time * d) - v1;
    const double d00 = dot(d0, d0), d01 = dot(d0, d1), d11 = dot(d1, d1);
    const double d20 = dot(d2, d0), d21 = dot(d2, d1);
    const double denom = d00 * d11 - d01 * d01;
    const double v = (d11 * d20 - d01 * d21) / denom;
    const double w = (d00 * d21 - d01 * d20) / denom;
    const double u = 1.0 - v - w;
    if (u >= 0.0 && v >= 0.0 && w >= 0.0) {
        rec_t = time;
        bv = v;
        bw = w;
        return true;
    }
    return false;
}
// f32: the same plane-hit + dot-product barycentrics, with everything that depends
// only on the triangle folded into 48 bytes on the host (in double):
//   q0 = (pn, pn.v1)   q1 = (A, -A.v1)   q2 = (B, -B.v1)
//   A = (d11 d0 - d01 d1)/denom, B = (d00 d1 - d01 d0)/denom  =>  v = A.(P - v1), w = B.(P - v1)
RPTB_D bool tri_intersect(const MeshRec<float>& m, uint32_t tri, Vec3<float> o, Vec3<float> d, float tmin,
                          float& rec_t, float& bv, float& bw) {
    const float4* q = m.tri48 + 3 * (size_t)tri;
    const float4 q0 = ldg(q);
    const float cosine = q0.x * d.x + q0.y * d.y + q0.z * d.z;
    if (fabsf(cosine) < 1e-8f) return false;
    const float time = fdividef(q0.w - (q0.x * o.x + q0.y * o.y + q0.z * o.z), cosine);
    if (time < tmin || time >= rec_t) return false;
    const float4 q1 = ldg(q + 1);
    const float4 q2 = ldg(q + 2);
    const float px = fmaf(time, d.x, o.x), py = fmaf(time, d.y, o.y), pz = fmaf(time, d.z, o.z);
    const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
    const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
    const float u = 1.0f - v - w;
    if (u >= 0.0f && v >= 0.0f && w >= 0.0f) {
        rec_t = time;
        bv = v;
        bw = w;
        return true;
    }
    return false;
}

// ----------------------------------------------------------- BVH traversal -----
// The f32 path's own structure (bvhbuild.cpp): a binary SAH BVH, both child boxes in the parent's 64-byte
// node, every triangle in exactly one leaf of <= 4.  Same query as KdTree::intersect -- closest triangle hit
// in [tmin, h.t), or any hit for a shadow ray -- and the same triangle test (tri48); only the set of
// triangles a ray has to look at shrinks (dragon proxy: 419 -> ~10 per ray).  Exact ties in t between two
// triangles (shared edges) may resolve to the other triangle than in the reference's leaf order.
// 1/x for slab tests written as b * (1/d) - o * (1/d): an exactly zero direction component would make both
// products infinite and their difference NaN, and fminf/fmaxf over ONE NaN plane silently shrink the interval
// (a box the ray is inside of gets culled).  A component of magnitude < 1e-30 is treated as +-1e-30: every
// product stays finite, and the error this makes in t is far below the padding of the boxes.
RPTB_D float slab_rcp(float x) { return M<float>::rcp(fabsf(x) < 1e-30f ? copysignf(1e-30f, x) : x); }

RPTB_D BvhNodeDev load_bvh_node(const BvhNodeDev* p) {
    BvhNodeDev n;
    const float4* q = reinterpret_cast<const float4*>(p);
    n.c0xy = ldg(q);
    n.c1xy = ldg(q + 1);
    n.cz = ldg(q + 2);
    const int4 w = ldg(reinterpret_cast<const int4*>(q + 3));
    n.child0 = w.x;
    n.child1 = w.y;
    return n;
}

template <bool STATS>
RPTB_D bool bvh_intersect(const MeshRec<float>& m, Vec3<float> o, Vec3<float> d, float tmin, bool any, Hit<float>& h,
                          TravStats& ts) {
    const Vec3<float> inv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};
    // o * inv per axis, so that a slab is one FMA: (b - o) * inv = b * inv - o * inv
    const Vec3<float> oi = {o.x * inv.x, o.y * inv.y, o.z * inv.z};
    int32_t stack[BVH_STACK];
    int sp = 0;
    int32_t cur = 0;  // the root is always an inner node
    bool hit = false;
    while (true) {
        while (cur >= 0) {  // inner node: test both children
            if (STATS) ts.bvh_nodes++;
            const BvhNodeDev n = load_bvh_node(m.bvh_nodes + cur);
            const float ax0 = fmaf(n.c0xy.x, inv.x, -oi.x), ax1 = fmaf(n.c0xy.y, inv.x, -oi.x);
            const float ay0 = fmaf(n.c0xy.z, inv.y, -oi.y), ay1 = fmaf(n.c0xy.w, inv.y, -oi.y);
            const float az0 = fmaf(n.cz.x, inv.z, -oi.z), az1 = fmaf(n.cz.y, inv.z, -oi.z);
            const float bx0 = fmaf(n.c1xy.x, inv.x, -oi.x), bx1 = fmaf(n.c1xy.y, inv.x, -oi.x);
            const float by0 = fmaf(n.c1xy.z, inv.y, -oi.y), by1 = fmaf(n.c1xy.w, inv.y, -oi.y);
            const float bz0 = fmaf(n.cz.z, inv.z, -oi.z), bz1 = fmaf(n.cz.w, inv.z, -oi.z);
            const float an = fmaxf(fmaxf(fminf(ax0, ax1), fminf(ay0, ay1)), fmaxf(fminf(az0, az1), tmin));
            const float af = fminf(fminf(fmaxf(ax0, ax1), fmaxf(ay0, ay1)), fminf(fmaxf(az0, az1), h.t));
            const float bn = fmaxf(fmaxf(fminf(bx0, bx1), fminf(by0, by1)), fmaxf(fminf(bz0, bz1), tmin));
            const float bf = fminf(fminf(fmaxf(bx0, bx1), fmaxf(by0, by1)), fminf(fmaxf(bz0, bz1), h.t));
            const bool ha = an <= af, hb = bn <= bf;
#if defined(__CUDA_ARCH__) && RPTB_BVH_PREFETCH
            // the loop is bound by the latency of one dependent node fetch per step (ncu: long_scoreboard on top): ask L1 for
            // both children's lines now, whichever is taken first (the other usually follows from the stack)
            if (ha && n.child0 >= 0) asm volatile("prefetch.global.L1 [%0];" ::"l"(m.bvh_nodes + n.child0));
            if (hb && n.child1 >= 0) asm volatile("prefetch.global.L1 [%0];" ::"l"(m.bvh_nodes + n.child1));
#endif
            if (ha && hb) {
                const bool a_first = an <= bn;
                stack[sp++] = a_first ? n.child1 : n.child0;
                cur = a_first ? n.child0 : n.child1;
            } else if (ha) {
                cur = n.child0;
            } else if (hb) {
                cur = n.child1;
            } else {
                if (sp == 0) return hit;
                cur = stack[--sp];
            }
        }
        // leaf: ~cur = (first << 3) | (count - 1)
        {
            const uint32_t code = (uint32_t)~cur;
            const uint32_t first = code >> 3, count = (code & 7u) + 1u;
            for (uint32_t k = first; k < first + count; k++) {
                if (STATS) ts.bvh_tris++;
                const float4* q = m.bvh_tri48 + 3 * (size_t)k;
                const float4 q0 = ldg(q);
                const float cosine = q0.x * d.x + q0.y * d.y + q0.z * d.z;
                if (fabsf(cosine) < 1e-8f) continue;
                const float time = fdividef(q0.w - (q0.x * o.x + q0.y * o.y + q0.z * o.z), cosine);
                if (time < tmin || time >= h.t) continue;
                const float4 q1 = ldg(q + 1);
                const float4 q2 = ldg(q + 2);
                const float px = fmaf(time, d.x, o.x), py = fmaf(time, d.y, o.y), pz = fmaf(time, d.z, o.z);
                const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
                const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
                const float u = 1.0f - v - w;
                if (u >= 0.0f && v >= 0.0f && w >= 0.0f) {
                    h.t = time;
                    h.bv = v;
                    h.bw = w;
                    h.aux = ldg(m.bvh_ids + k);
                    hit = true;
                }
            }
        }
        if (any && hit) return true;
        if (sp == 0) return hit;
        cur = stack[--sp];
    }
}
template <bool STATS>
RPTB_D bool bvh_intersect(const MeshRec<double>&, Vec3<double>, Vec3<double>, double, bool, Hit<double>&, TravStats&) {
    return false;  // the f64 gate never uses the BVH
}

// ------------------------------------------------- the four-wide BVH ---------
// One lane per ray through Bvh4Node: all four child boxes decided from one 112-byte fetch, the hit children sorted by
// entry distance (a five-exchange network on (t, code) pairs), the nearest followed and the others stacked farthest
// first WITH their entry distance, so that a popped entry the ray has meanwhile found a closer hit than is dropped
// without a fetch.  Same leaves, same triangle test and the same answer as bvh_intersect (ties in t aside).
#define RPTB_CSWAP(i, j)                                   \
    {                                                      \
        const bool s_ = tn[j] < tn[i];                     \
        const float ta_ = s_ ? tn[j] : tn[i];              \
        const float tb_ = s_ ? tn[i] : tn[j];              \
        const int32_t ca_ = s_ ? cd[j] : cd[i];            \
        const int32_t cb_ = s_ ? cd[i] : cd[j];            \
        tn[i] = ta_, tn[j] = tb_, cd[i] = ca_, cd[j] = cb_; \
    }
template <bool STATS>
RPTB_D bool bvh4_intersect(const MeshRec<float>& m, Vec3<float> o, Vec3<float> d, float tmin, bool any, Hit<float>& h,
                           TravStats& ts) {
    const Vec3<float> inv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};
    const Vec3<float> oi = {o.x * inv.x, o.y * inv.y, o.z * inv.z};
    const float inf = M<float>::inf();
    int32_t scode[BVH4_STACK];
    float stn[BVH4_STACK];
    int sp = 0;
    int32_t cur = 0;  // the root is always an inner node
    bool hit = false;
    while (true) {
        while (cur >= 0) {
            if (STATS) ts.bvh_nodes += 2;  // counted in 64-byte units, like the binary tree's nodes
            const float4* q = reinterpret_cast<const float4*>(m.bvh4_nodes + cur);
            const float4 lox = ldg(q), hix = ldg(q + 1), loy = ldg(q + 2), hiy = ldg(q + 3), loz = ldg(q + 4), hiz = ldg(q + 5);
            const int4 code = ldg(reinterpret_cast<const int4*>(q + 6));
            const float lx[4] = {lox.x, lox.y, lox.z, lox.w}, hx[4] = {hix.x, hix.y, hix.z, hix.w};
            const float ly[4] = {loy.x, loy.y, loy.z, loy.w}, hy[4] = {hiy.x, hiy.y, hiy.z, hiy.w};
            const float lz[4] = {loz.x, loz.y, loz.z, loz.w}, hz[4] = {hiz.x, hiz.y, hiz.z, hiz.w};
            float tn[4];
            int32_t cd[4] = {code.x, code.y, code.z, code.w};
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
            for (int k = 0; k < 4; k++) {
                const float x0 = fmaf(lx[k], inv.x, -oi.x), x1 = fmaf(hx[k], inv.x, -oi.x);
                const float y0 = fmaf(ly[k], inv.y, -oi.y), y1 = fmaf(hy[k], inv.y, -oi.y);
                const float z0 = fmaf(lz[k], inv.z, -oi.z), z1 = fmaf(hz[k], inv.z, -oi.z);
                const float nr = fmaxf(fmaxf(fminf(x0, x1), fminf(y0, y1)), fmaxf(fminf(z0, z1), tmin));
                const float fr = fminf(fminf(fmaxf(x0, x1), fmaxf(y0, y1)), fminf(fmaxf(z0, z1), h.t));
                tn[k] = (nr <= fr && cd[k] != BVH8_EMPTY) ? nr : inf;
            }
            RPTB_CSWAP(0, 1)
            RPTB_CSWAP(2, 3)
            RPTB_CSWAP(0, 2)
            RPTB_CSWAP(1, 3)
            RPTB_CSWAP(1, 2)
            if (tn[0] == inf) {  // nothing hit: back to the nearest pending entry still in range
                cur = BVH8_EMPTY;
                while (sp > 0) {
                    --sp;
                    if (stn[sp] < h.t) {
                        cur = scode[sp];
                        break;
                    }
                }
                if (cur == BVH8_EMPTY) return hit;
                continue;
            }
            if (tn[3] < inf) scode[sp] = cd[3], stn[sp] = tn[3], sp++;
            if (tn[2] < inf) scode[sp] = cd[2], stn[sp] = tn[2], sp++;
            if (tn[1] < inf) scode[sp] = cd[1], stn[sp] = tn[1], sp++;
            cur = cd[0];
        }
        {  // leaf: ~cur = (first << 3) | (count - 1)
            const uint32_t lcode = (uint32_t)~cur;
            const uint32_t first = lcode >> 3, count = (lcode & 7u) + 1u;
            for (uint32_t k = first; k < first + count; k++) {
                if (STATS) ts.bvh_tris++;
                const float4* q = m.bvh_tri48 + 3 * (size_t)k;
                const float4 q0 = ldg(q);
                const float cosine = q0.x * d.x + q0.y * d.y + q0.z * d.z;
                if (fabsf(cosine) < 1e-8f) continue;
                const float time = fdividef(q0.w - (q0.x * o.x + q0.y * o.y + q0.z * o.z), cosine);
                if (time < tmin || time >= h.t) continue;
                const float4 q1 = ldg(q + 1);
                const float4 q2 = ldg(q + 2);
                const float px = fmaf(time, d.x, o.x), py = fmaf(time, d.y, o.y), pz = fmaf(time, d.z, o.z);
                const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
                const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
                const float u = 1.0f - v - w;
                if (u >= 0.0f && v >= 0.0f && w >= 0.0f) {
                    h.t = time;
                    h.bv = v;
                    h.bw = w;
                    h.aux = ldg(m.bvh_ids + k);
                    hit = true;
                }
            }
        }
        if (any && hit) return true;
        cur = BVH8_EMPTY;
        while (sp > 0) {
            --sp;
            if (stn[sp] < h.t) {
                cur = scode[sp];
                break;
            }
        }
        if (cur == BVH8_EMPTY) return hit;
    }
}
#undef RPTB_CSWAP
template <bool STATS>
RPTB_D bool bvh4_intersect(const MeshRec<double>&, Vec3<double>, Vec3<double>, double, bool, Hit<double>&, TravStats&) {
    return false;
}

// what a mesh with a BVH is traversed through: the four-wide tree where the scene has one, else the binary tree
template <bool STATS, typename R>
RPTB_D bool bvh_query(const MeshRec<R>& m, Vec3<R> o, Vec3<R> d, R tmin, bool any, Hit<R>& h, TravStats& ts) {
#if RPTB_BVH4
    if (m.bvh4_nodes) return bvh4_intersect<STATS>(m, o, d, tmin, any, h, ts);
#endif
    return bvh_intersect<STATS>(m, o, d, tmin, any, h, ts);
}

// ------------------------------------------------- the eight-wide BVH --------
// Per-lane (scalar) traversal of the collapsed tree: test infrastructure for the builder (tests/hostemu checks its hits
// against the binary tree's) -- the product traverses Bvh8Node with groups of eight lanes, below.
template <bool STATS>
RPTB_D bool bvh8_intersect_scalar(const MeshRec<float>& m, Vec3<float> o, Vec3<float> d, float tmin, bool any, Hit<float>& h,
                                  TravStats& ts) {
    const Vec3<float> inv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};
    const Vec3<float> oi = {o.x * inv.x, o.y * inv.y, o.z * inv.z};
    int32_t stack[8 * BVH8_STACK];
    int sp = 0;
    stack[sp++] = 0;
    bool hit = false;
    while (sp > 0) {
        const int32_t cur = stack[--sp];
        if (cur >= 0) {
            if (STATS) ts.bvh_nodes += 4;
            const Bvh8Node& n = m.bvh8_nodes[cur];
            for (int k = 0; k < 8; k++) {
                const Bvh8Child& c = n.c[k];
                if (c.code == BVH8_EMPTY) continue;
                const float x0 = fmaf(c.lo[0], inv.x, -oi.x), x1 = fmaf(c.hi[0], inv.x, -oi.x);
                const float y0 = fmaf(c.lo[1], inv.y, -oi.y), y1 = fmaf(c.hi[1], inv.y, -oi.y);
                const float z0 = fmaf(c.lo[2], inv.z, -oi.z), z1 = fmaf(c.hi[2], inv.z, -oi.z);
                const float tn = fmaxf(fmaxf(fminf(x0, x1), fminf(y0, y1)), fmaxf(fminf(z0, z1), tmin));
                const float tf = fminf(fminf(fmaxf(x0, x1), fmaxf(y0, y1)), fminf(fmaxf(z0, z1), h.t));
                if (tn <= tf && sp < 8 * BVH8_STACK) stack[sp++] = c.code;
            }
            continue;
        }
        const uint32_t code = (uint32_t)~cur;
        const uint32_t first = code >> 3, count = (code & 7u) + 1u;
        for (uint32_t k = first; k < first + count; k++) {
            if (STATS) ts.bvh_tris++;
            const float4* q = m.bvh_tri48 + 3 * (size_t)k;
            const float4 q0 = ldg(q);
            const float cosine = q0.x * d.x + q0.y * d.y + q0.z * d.z;
            if (fabsf(cosine) < 1e-8f) continue;
            const float time = fdividef(q0.w - (q0.x * o.x + q0.y * o.y + q0.z * o.z), cosine);
            if (time < tmin || time >= h.t) continue;
            const float4 q1 = ldg(q + 1), q2 = ldg(q + 2);
            const float px = fmaf(time, d.x, o.x), py = fmaf(time, d.y, o.y), pz = fmaf(time, d.z, o.z);
            const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
            const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
            if (1.0f - v - w >= 0.0f && v >= 0.0f && w >= 0.0f) {
                h.t = time; h.bv = v; h.bw = w; h.aux = ldg(m.bvh_ids + k);
                hit = true;
            }
        }
        if (any && hit) return true;
    }
    return hit;
}

#if defined(__CUDACC__) && !defined(RPTB_HOST_EMU)
// ---- traversal by groups of eight lanes ---------------------------------------------------------------------------
// ncu (round 2, dragon configs): with one ray per lane the binary-BVH node loop ran at 5-6 of 32 lanes however the
// rays were scheduled -- the rays of a warp that enter a mesh at all are few, and their traversal lengths spread over
// two orders of magnitude, so a warp spends its time walking the one or two longest rays with everybody else idle.
// The idle width is therefore spent INSIDE a ray: the warp's rays that pass the mesh's root box are compacted (warp
// vote) into this per-warp block of shared memory, and each group of eight lanes takes one ray at a time off that list
// (an atomic cursor in shared memory: the four groups balance themselves).  Per node, lane k of the group loads child k
// (one coalesced 256-byte request per group), tests its box, and three votes later the group knows which children are
// hit, which is nearest, and in what order the others go on the group's stack (shared memory, nearest on top).  A leaf's
// <= 4 triangles are tested one per lane.  A ray walks ~3x fewer, fatter steps than in the binary tree, and four rays
// advance per warp instruction instead of "the slowest of 32".
struct __align__(16) CoopWarp {
    float4 ra[32];   // compacted rays, mesh-local: origin, closest t so far
    float4 rb[32];   // direction
    float4 res[32];  // answer: t (< 0: no hit; -2: stack overflow, redo with the binary tree), bv, bw, triangle id bits
    uint2 stack[4][BVH8_STACK];  // per group: (child code, entry t bits)
    uint32_t next;   // cursor into the list
    uint32_t _pad[3];
};

template <bool STATS>
__device__ __forceinline__ void bvh8_group_trace(const MeshRec<float>& m, CoopWarp& cw, const uint32_t count, const bool any,
                                                 const uint32_t lane, TravStats& ts) {
    const float tmin = 1e-12f;
    const uint32_t k = lane & 7u, gbase = lane & ~7u;
    const unsigned gmask = 0xFFu << gbase;
    uint2* const stack = cw.stack[lane >> 3];
    while (true) {
        uint32_t it = 0;
        if (k == 0u) it = atomicAdd(&cw.next, 1u);
        it = __shfl_sync(gmask, it, gbase);
        if (it >= count) break;
        const float4 A = cw.ra[it], B = cw.rb[it];
        const Vec3<float> o = {A.x, A.y, A.z}, d = {B.x, B.y, B.z};
        const Vec3<float> inv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};
        const Vec3<float> oi = {o.x * inv.x, o.y * inv.y, o.z * inv.z};
        float ht = A.w;  // everything below that is not per-child is identical in the eight lanes of the group
        bool hit = false, overflow = false, done = false;
        int32_t cur = 0;
        int sp = 0;
        while (!done) {
            bool pop = false;
            if (cur >= 0) {
                if (STATS && k == 0u) ts.bvh_nodes += 4;  // 256 bytes = four 64-byte units of the bytes model
                const float4* c = reinterpret_cast<const float4*>(&m.bvh8_nodes[cur].c[k]);
                const float4 c0 = ldg(c), c1 = ldg(c + 1);  // lo.x lo.y lo.z hi.x | hi.y hi.z code pad
                const int32_t code = __float_as_int(c1.z);
                const float x0 = fmaf(c0.x, inv.x, -oi.x), x1 = fmaf(c0.w, inv.x, -oi.x);
                const float y0 = fmaf(c0.y, inv.y, -oi.y), y1 = fmaf(c1.x, inv.y, -oi.y);
                const float z0 = fmaf(c0.z, inv.z, -oi.z), z1 = fmaf(c1.y, inv.z, -oi.z);
                const float tn = fmaxf(fmaxf(fminf(x0, x1), fminf(y0, y1)), fmaxf(fminf(z0, z1), tmin));
                const float tf = fminf(fminf(fmaxf(x0, x1), fmaxf(y0, y1)), fminf(fmaxf(z0, z1), ht));
                const bool hc = code != BVH8_EMPTY && tn <= tf;
                const unsigned hm = (__ballot_sync(gmask, hc) >> gbase) & 0xFFu;
                if (hm == 0u) {
                    pop = true;
                } else {
                    const uint32_t key = hc ? __float_as_uint(tn) : 0xFFFFFFFFu;  // tn >= tmin > 0: the bits order like the value
                    const uint32_t kmin = __reduce_min_sync(gmask, key);
                    const unsigned nm = (__ballot_sync(gmask, key == kmin) >> gbase) & 0xFFu;
                    const int nl = __ffs(nm) - 1;  // the nearest child's lane
                    const int32_t ncode = __shfl_sync(gmask, code, gbase + nl);
                    const int nh = __popc(hm);
                    if (nh > 1) {
                        if (sp + nh - 1 > BVH8_STACK) {
                            overflow = true;
                            done = true;
                        } else {
                            // position on the stack: the farther, the deeper (so the nearest of the rest is popped first)
                            uint32_t rank = 0;
#pragma unroll
                            for (int j = 0; j < 8; j++) {
                                const uint32_t kj = __shfl_sync(gmask, key, gbase + j);
                                if (j != nl && ((hm >> j) & 1u) && (kj > key || (kj == key && j > (int)k))) rank++;
                            }
                            if (hc && (int)k != nl) stack[sp + rank] = make_uint2((uint32_t)code, key);
                            sp += nh - 1;
                            __syncwarp(gmask);
                        }
                    }
                    cur = ncode;
                }
            } else {
                // leaf: ~cur = (first << 3) | (count - 1); one triangle per lane (Triangle::intersect as in tri_intersect)
                const uint32_t code = (uint32_t)~cur;
                const uint32_t first = code >> 3, cnt = (code & 7u) + 1u;
                if (STATS && k == 0u) ts.bvh_tris += cnt;
                uint32_t key = 0xFFFFFFFFu;
                float bv = 0.0f, bw = 0.0f;
                if (k < cnt) {
                    const float4* q = m.bvh_tri48 + 3 * (size_t)(first + k);
                    const float4 q0 = ldg(q);
                    const float cosine = q0.x * d.x + q0.y * d.y + q0.z * d.z;
                    if (!(fabsf(cosine) < 1e-8f)) {
                        const float time = __fdividef(q0.w - (q0.x * o.x + q0.y * o.y + q0.z * o.z), cosine);
                        if (!(time < tmin || time >= ht)) {
                            const float4 q1 = ldg(q + 1), q2 = ldg(q + 2);
                            const float px = fmaf(time, d.x, o.x), py = fmaf(time, d.y, o.y), pz = fmaf(time, d.z, o.z);
                            const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
                            const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
                            if (1.0f - v - w >= 0.0f && v >= 0.0f && w >= 0.0f) {
                                key = __float_as_uint(time);
                                bv = v;
                                bw = w;
                            }
                        }
                    }
                }
                const uint32_t kmin = __reduce_min_sync(gmask, key);
                if (kmin != 0xFFFFFFFFu) {
                    const unsigned wm = (__ballot_sync(gmask, key == kmin) >> gbase) & 0xFFu;
                    ht = __uint_as_float(kmin);
                    hit = true;
                    if ((int)k == __ffs(wm) - 1)  // the first of equal times wins, like the binary tree's leaf loop
                        cw.res[it] = make_float4(ht, bv, bw, __uint_as_float(ldg(m.bvh_ids + first + k)));
                }
                if (any && hit) done = true;
                else pop = true;
            }
            if (pop && !done) {
                while (true) {
                    if (sp == 0) {
                        done = true;
                        break;
                    }
                    sp--;
                    const uint2 e = stack[sp];  // one address for the eight lanes: a broadcast
                    if (__uint_as_float(e.y) < ht) {  // entered before the closest hit so far
                        cur = (int32_t)e.x;
                        break;
                    }
                }
            }
        }
        if (overflow && k == 0u) cw.res[it].x = -2.0f;
        __syncwarp(gmask);
    }
}

#endif

// ------------------------------------------------------------ kd traversal -----
RPTB_D KdNodeDev load_node(const KdNodeDev* p) {
    const uint2 v = ldg(reinterpret_cast<const uint2*>(p));
    KdNodeDev n;
    n.first_ref = v.x;
    n.word = v.y;
    return n;
}
RPTB_D KdNodeDev64 load_node(const KdNodeDev64* p) { return *p; }
RPTB_D float node_split(const KdNodeDev& n) { return n.split; }
RPTB_D double node_split(const KdNodeDev64& n) { return n.split; }
RPTB_D uint32_t node_first_ref(const KdNodeDev& n) { return n.first_ref; }
RPTB_D uint32_t node_first_ref(const KdNodeDev64& n) { return n.first_ref; }

// KdTree::intersect.  `o`,`d` are in the mesh's local space (d not normalised, so
// t is the world t).  Returns true if some triangle tightened h.t.  `any` = shadow
// query: return at the first leaf that produced a hit.
template <class R, bool STATS, int FEAT = F_ALL>
RPTB_D bool kd_intersect(const SceneView<R>& sv, const MeshRec<R>& m, Vec3<R> o, Vec3<R> d, R tmin, bool any, Hit<R>& h,
                         TravStats& ts) {
    if constexpr ((FEAT & F_SMALL) != 0 && !M<R>::literal) if (m.root_is_leaf) {
        // one-leaf mesh, triangles in parameter space: Triangle::intersect as in tri_intersect(float)
        bool hit = false;
        if (STATS) ts.node_visits++;
        const uint32_t base = m.small_tri_base;
        for (uint32_t tri = 0; tri < m.ntris; tri++) {
            if (STATS) ts.tri_tests++;
            const float4 q0 = sv.small.tri48[3 * (base + tri)];
            const float cosine = q0.x * d.x + q0.y * d.y + q0.z * d.z;
            if (fabsf(cosine) < 1e-8f) continue;
            const float time = fdividef(q0.w - (q0.x * o.x + q0.y * o.y + q0.z * o.z), cosine);
            if (time < tmin || time >= h.t) continue;
            const float4 q1 = sv.small.tri48[3 * (base + tri) + 1];
            const float4 q2 = sv.small.tri48[3 * (base + tri) + 2];
            const float px = fmaf(time, d.x, o.x), py = fmaf(time, d.y, o.y), pz = fmaf(time, d.z, o.z);
            const float v = fmaf(q1.x, px, fmaf(q1.y, py, fmaf(q1.z, pz, q1.w)));
            const float w = fmaf(q2.x, px, fmaf(q2.y, py, fmaf(q2.z, pz, q2.w)));
            const float u = 1.0f - v - w;
            if (u >= 0.0f && v >= 0.0f && w >= 0.0f) {
                h.t = time;
                h.bv = v;
                h.bw = w;
                h.aux = tri;
                hit = true;
            }
        }
        return hit;
    }
    if (!M<R>::literal && (m.root_is_leaf || !(FEAT & F_TREE))) {
        // f32 only (the f64 gate keeps the reference's control flow).  A tree that is one leaf (e.g. every `polygon` of the Cornell box): the root cull
        // of kdtree.rs:130-134 can only prune, never change the hit, so all lanes test the
        // few triangles directly -- no divergent slab test.
        bool hit = false;
        if (STATS) ts.node_visits++;
        for (uint32_t tri = 0; tri < m.ntris; tri++) {
            if (STATS) ts.tri_tests++;
            if (tri_intersect(m, tri, o, d, tmin, h.t, h.bv, h.bw)) {
                h.aux = tri;
                hit = true;
            }
        }
        return hit;
    }
    if constexpr (!(FEAT & F_TREE) && !M<R>::literal) return false;  // (unreachable: compiled for tree-less scenes)
    if constexpr ((FEAT & F_BVH) != 0 && !M<R>::literal) return bvh_query<STATS>(m, o, d, tmin, any, h, ts);
    // root cull: BoundingBox::intersect of `bounds` (kdtree.rs:130-134)
    R lo, hi;
    Vec3<R> inv;
    {
        if (M<R>::literal) {
            inv = {(R)0, (R)0, (R)0};
            const R x1 = (m.bmin[0] - o.x) / d.x, x2 = (m.bmax[0] - o.x) / d.x;
            const R y1 = (m.bmin[1] - o.y) / d.y, y2 = (m.bmax[1] - o.y) / d.y;
            const R z1 = (m.bmin[2] - o.z) / d.z, z2 = (m.bmax[2] - o.z) / d.z;
            lo = M<R>::max(M<R>::max(M<R>::min(x1, x2), M<R>::min(y1, y2)), M<R>::min(z1, z2));
            hi = M<R>::min(M<R>::min(M<R>::max(x1, x2), M<R>::max(y1, y2)), M<R>::max(z1, z2));
        } else {
            inv = {M<R>::rcp(d.x), M<R>::rcp(d.y), M<R>::rcp(d.z)};
            const R x1 = (m.bmin[0] - o.x) * inv.x, x2 = (m.bmax[0] - o.x) * inv.x;
            const R y1 = (m.bmin[1] - o.y) * inv.y, y2 = (m.bmax[1] - o.y) * inv.y;
            const R z1 = (m.bmin[2] - o.z) * inv.z, z2 = (m.bmax[2] - o.z) * inv.z;
            lo = M<R>::max(M<R>::max(M<R>::min(x1, x2), M<R>::min(y1, y2)), M<R>::min(z1, z2));
            hi = M<R>::min(M<R>::min(M<R>::max(x1, x2), M<R>::max(y1, y2)), M<R>::max(z1, z2));
        }
        if (M<R>::max(lo, tmin) > M<R>::min(hi, h.t)) return false;
    }

    uint32_t st_node[KD_STACK];
    R st_lo[KD_STACK], st_hi[KD_STACK];
    int sp = 0;
    uint32_t node = 0;
    bool hit = false;

    while (true) {
        auto nd = load_node(m.nodes + node);
        while ((nd.word & 3u) != 3u) {
            if (STATS) ts.node_visits++;
            const uint32_t axis = nd.word & 3u;
            const uint32_t right = nd.word >> 2;
            const R split = node_split(nd);
            const R oa = comp(o, (int)axis), da = comp(d, (int)axis);
            R t_split;
            if (M<R>::literal) t_split = (split - oa) / da;
            else t_split = (split - oa) * comp(inv, (int)axis);
            const bool left_first = (oa < split) || (oa == split && da <= (R)0);
            const uint32_t first = left_first ? node + 1u : right;
            const uint32_t second = left_first ? right : node + 1u;
            if (t_split > M<R>::min(hi, h.t) || t_split <= (R)0) {
                node = first;  // (i) near only
            } else if (t_split < M<R>::max(lo, tmin)) {
                node = second;  // (ii) far only
            } else {  // (iii) near, then far with the cell clipped at t_split
                st_node[sp] = second;
                st_lo[sp] = t_split;
                st_hi[sp] = hi;
                sp++;
                node = first;
                hi = t_split;
            }
            nd = load_node(m.nodes + node);
        }
        // leaf: every referenced triangle, no early out (kdtree.rs:162-171)
        if (STATS) ts.node_visits++;
        {
            const uint32_t first_ref = node_first_ref(nd);
            const uint32_t count = nd.word >> 2;
            for (uint32_t i = 0; i < count; i++) {
                const uint32_t tri = ldg(m.refs + first_ref + i);
                if (STATS) ts.tri_tests++;
                if (tri_intersect(m, tri, o, d, tmin, h.t, h.bv, h.bw)) {
                    h.aux = tri;
                    hit = true;
                }
            }
        }
        if (any && hit) return true;
        // pop; skip far cells that start beyond the hit found so far (kdtree.rs:212-213)
        while (true) {
            if (sp == 0) return hit;
            sp--;
            node = st_node[sp];
            lo = st_lo[sp];
            hi = st_hi[sp];
            if (!(h.t < lo)) break;
        }
    }
}

// ------------------------------------------------------- object dispatch ------
template <class R, bool STATS, int FEAT>
RPTB_D bool group_intersect(const SceneView<R>& sv, const GroupRec<R>& g, Vec3<R> o, Vec3<R> d, R tmin, bool any, Hit<R>& h,
                            TravStats& ts);

template <class R, bool STATS, int FEAT = F_ALL>
RPTB_D bool object_intersect(const SceneView<R>& sv, const ObjectRec<R>& ob, Vec3<R> o, Vec3<R> d, R tmin, bool any,
                             Hit<R>& h, TravStats& ts) {
    if (ob.has_transform) {  // Ray::apply_transform(inverse_transform)
        const Vec3<R> lo = xform_point(ob.inv, o);
        const Vec3<R> ld = xform_dir(ob.inv, d);
        o = lo;
        d = ld;
    }
    if constexpr ((FEAT & F_MONO) != 0)
        if (ob.kind == SHAPE_MONOMIAL) return monomial_intersect(ob.plane_v, o, d, tmin, h.t);
    if constexpr ((FEAT & F_GROUP) != 0)
        if (ob.kind == SHAPE_GROUP) return group_intersect<R, STATS, FEAT>(sv, sv.groups[ob.mesh], o, d, tmin, any, h, ts);
    switch (ob.kind) {
        case SHAPE_SPHERE: return sphere_intersect(o, d, tmin, h.t);
        case SHAPE_PLANE: return plane_intersect(ob.plane_n, ob.plane_v, o, d, tmin, h.t);
        case SHAPE_CUBE: return cube_intersect(o, d, tmin, h.t, h.aux);
        default:
            if constexpr ((FEAT & F_SMALL) != 0 && !M<R>::literal) return kd_intersect<R, STATS, FEAT>(sv, sv.small.meshes[ob.mesh], o, d, tmin, any, h, ts);
            else return kd_intersect<R, STATS, FEAT>(sv, sv.meshes[ob.mesh], o, d, tmin, any, h, ts);
    }
}

// KdTree<Box<dyn Bounded>>::intersect (src/kdtree.rs:129-136,151-223) over whole shapes: the traversal of
// kd_intersect, with two differences the reference's recursion implies once the leaves hold arbitrary
// shapes instead of triangles.  (1) A child is intersected with the t_min its cell received: the far
// child of a straddled split gets t_min := t_split (kdtree.rs:219), and MonomialSurface::intersect is
// sensitive to it.  (2) A child is a full shape: its own transform, and for a mesh its own kd-tree
// (kd_intersect with its own stack) -- the two-level instancing of examples/fractal_teapots.rs.
template <class R, bool STATS, int FEAT>
RPTB_D bool group_intersect(const SceneView<R>& sv, const GroupRec<R>& g, Vec3<R> o, Vec3<R> d, R tmin, bool any, Hit<R>& h,
                            TravStats& ts) {
    constexpr int CHILD = FEAT & ~F_GROUP;  // children are never groups
    R lo, hi;
    Vec3<R> inv = {(R)0, (R)0, (R)0};
    if constexpr (!M<R>::literal) inv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};  // for the child-box cull below
    {  // root cull: BoundingBox::intersect of `bounds` (kdtree.rs:130-134)
        const R x1 = (g.bmin[0] - o.x) / d.x, x2 = (g.bmax[0] - o.x) / d.x;
        const R y1 = (g.bmin[1] - o.y) / d.y, y2 = (g.bmax[1] - o.y) / d.y;
        const R z1 = (g.bmin[2] - o.z) / d.z, z2 = (g.bmax[2] - o.z) / d.z;
        lo = M<R>::max(M<R>::max(M<R>::min(x1, x2), M<R>::min(y1, y2)), M<R>::min(z1, z2));
        hi = M<R>::min(M<R>::min(M<R>::max(x1, x2), M<R>::max(y1, y2)), M<R>::max(z1, z2));
        if (M<R>::max(lo, tmin) > M<R>::min(hi, h.t)) return false;
    }
    uint32_t st_node[GROUP_STACK];
    R st_lo[GROUP_STACK], st_hi[GROUP_STACK], st_tmin[GROUP_STACK];
    int sp = 0;
    uint32_t node = 0;
    R cur_tmin = tmin;
    bool hit = false;
    while (true) {
        auto nd = load_node(g.nodes + node);
        while ((nd.word & 3u) != 3u) {
            if (STATS) ts.node_visits++;
            const uint32_t axis = nd.word & 3u;
            const uint32_t right = nd.word >> 2;
            const R split = node_split(nd);
            const R oa = comp(o, (int)axis), da = comp(d, (int)axis);
            const R t_split = (split - oa) / da;
            const bool left_first = (oa < split) || (oa == split && da <= (R)0);
            const uint32_t first = left_first ? node + 1u : right;
            const uint32_t second = left_first ? right : node + 1u;
            if (t_split > M<R>::min(hi, h.t) || t_split <= (R)0) {
                node = first;  // (i) near only
            } else if (t_split < M<R>::max(lo, cur_tmin)) {
                node = second;  // (ii) far only
            } else {  // (iii) near, then far with t_min := t_split
                st_node[sp] = second;
                st_lo[sp] = t_split;
                st_hi[sp] = hi;
                st_tmin[sp] = t_split;
                sp++;
                node = first;
                hi = t_split;
            }
            nd = load_node(g.nodes + node);
        }
        if (STATS) ts.node_visits++;
        {
            const uint32_t first_ref = node_first_ref(nd);
            const uint32_t count = nd.word >> 2;
            for (uint32_t i = 0; i < count; i++) {
                const uint32_t c = ldg(g.refs + first_ref + i);
                if constexpr (!M<R>::literal) {
                    // f32 only (the f64 gate calls every child, like the reference): a ray that misses the
                    // child's bounding box cannot hit the child, so skip the change of space, the three
                    // reciprocals and the slab test of the instance's own root (fractal_teapots: ~40 children
                    // tested per ray, most of them missed)
                    const float4 bl = ldg(g.child_box + 2 * c), bh = ldg(g.child_box + 2 * c + 1);
                    const R x1 = ((R)bl.x - o.x) * inv.x, x2 = ((R)bh.x - o.x) * inv.x;
                    const R y1 = ((R)bl.y - o.y) * inv.y, y2 = ((R)bh.y - o.y) * inv.y;
                    const R z1 = ((R)bl.z - o.z) * inv.z, z2 = ((R)bh.z - o.z) * inv.z;
                    const R c0 = M<R>::max(M<R>::max(M<R>::min(x1, x2), M<R>::min(y1, y2)), M<R>::min(z1, z2));
                    const R c1 = M<R>::min(M<R>::min(M<R>::max(x1, x2), M<R>::max(y1, y2)), M<R>::max(z1, z2));
                    if (M<R>::max(c0, cur_tmin) > M<R>::min(c1, h.t)) continue;
                }
                if (STATS) ts.object_tests++;
                if (object_intersect<R, STATS, CHILD>(sv, g.children[c], o, d, cur_tmin, any, h, ts)) {
                    h.child = c;
                    hit = true;
                }
            }
        }
        if (any && hit) return true;
        while (true) {  // pop; a far cell is skipped when the near side hit before its split (kdtree.rs:212-213)
            if (sp == 0) return hit;
            sp--;
            node = st_node[sp];
            lo = st_lo[sp];
            hi = st_hi[sp];
            cur_tmin = st_tmin[sp];
            if (!(h.t < lo)) break;
        }
    }
}

// Surface data of the winning hit, computed once.
template <class R>
struct Surface {
    Vec3<R> n;   // shading normal == HitRecord::normal
    Vec3<R> ng;  // geometric normal (f32 ray-offset policy only)
    bool on_mesh;
};

template <class R, int FEAT = F_ALL>
RPTB_D Surface<R> finalize_hit(const SceneView<R>& sv, const ObjectRec<R>& ob, Vec3<R> o, Vec3<R> d, const Hit<R>& h) {
    Surface<R> s;
    if (ob.has_transform) {
        const Vec3<R> lo = xform_point(ob.inv, o);
        const Vec3<R> ld = xform_dir(ob.inv, d);
        o = lo;
        d = ld;
    }
    Vec3<R> n, ng;
    s.on_mesh = false;
    if constexpr ((FEAT & F_GROUP) != 0)
        if (ob.kind == SHAPE_GROUP) {
            // the hit child finishes its own normal (its transform included); the group's transform, if
            // any, is applied on top -- Transformed<KdTree<..>>::intersect wrapping the child's intersect
            s = finalize_hit<R, FEAT & ~F_GROUP>(sv, sv.groups[ob.mesh].children[h.child], o, d, h);
            if (ob.has_transform) {
                s.n = M<R>::normalize(xform3(ob.nrm, s.n));
                s.ng = M<R>::literal ? s.n : M<R>::normalize(xform3(ob.nrm, s.ng));
            }
            return s;
        }
    if constexpr ((FEAT & F_MONO) != 0)
        if (ob.kind == SHAPE_MONOMIAL) {  // monomial_surface.rs:93-103
            const Vec3<R> pos = o + h.t * d;
            const R r2 = pos.x * pos.x + pos.z * pos.z;
            n = M<R>::normalize(mk(ob.plane_v * (R)4 * pos.x * r2, (R)-1, ob.plane_v * (R)4 * pos.z * r2));
            if (dot(n, d) > (R)0) n = -n;  // two-sided
            if (ob.has_transform) n = M<R>::normalize(xform3(ob.nrm, n));
            s.n = n;
            s.ng = n;
            return s;
        }
    switch (ob.kind) {
        case SHAPE_SPHERE:
            n = M<R>::normalize(o + h.t * d);  // sphere.rs:40
            ng = n;
            break;
        case SHAPE_PLANE: {
            const Vec3<R> pn = {ob.plane_n[0], ob.plane_n[1], ob.plane_n[2]};
            const R cosine = dot(pn, d);
            if (M<R>::literal) n = -M<R>::normalize(pn) * signum(cosine);  // plane.rs:27
            else n = -mk(ob.plane_unit[0], ob.plane_unit[1], ob.plane_unit[2]) * signum(cosine);
            ng = n;
            break;
        }
        case SHAPE_CUBE: {
            const uint32_t axis = h.aux >> 1;
            const R sgn = (h.aux & 1u) ? (R)1 : (R)-1;
            n = mk(axis == 0 ? sgn : (R)0, axis == 1 ? sgn : (R)0, axis == 2 ? sgn : (R)0);
            ng = n;
            break;
        }
        default: {
            const MeshRec<R>& m = sv.meshes[ob.mesh];
            const R* p = m.norms + 9 * (size_t)h.aux;
            const R u = (R)1 - h.bv - h.bw;
            const Vec3<R> n1 = {p[0], p[1], p[2]}, n2 = {p[3], p[4], p[5]}, n3 = {p[6], p[7], p[8]};
            n = M<R>::normalize(u * n1 + h.bv * n2 + h.bw * n3);  // mesh.rs:77
            if (!M<R>::literal) {
                const float4 q0 = ldg(m.tri48 + 3 * (size_t)h.aux);
                ng = mk((R)q0.x, (R)q0.y, (R)q0.z);
            } else {
                ng = n;
            }
            s.on_mesh = true;
        }
    }
    if (ob.has_transform) {  // shape.rs:132
        n = M<R>::normalize(xform3(ob.nrm, n));
        if (!M<R>::literal) ng = M<R>::normalize(xform3(ob.nrm, ng));
        else ng = n;
    }
    s.n = n;
    s.ng = ng;
    return s;
}

// get_closest_hit: linear scan of scene.objects.  `any` = shadow query (the first
// object with a hit at t < h.t ends the scan; the caller preloads h.t with the light
// distance).
template <class R, bool STATS, int FEAT = F_ALL>
RPTB_D void closest_hit(const SceneView<R>& sv, Vec3<R> o, Vec3<R> d, R tmin, bool any, Hit<R>& h, TravStats& ts) {
    h.obj = -1;
    h.aux = 0;
    h.bv = h.bw = (R)0;
    if constexpr ((FEAT & F_GROUP) != 0) h.child = 0;
    const uint32_t n = sv.nobjects;
    for (uint32_t i = 0; i < n; i++) {
        if (STATS) ts.object_tests++;
        bool hit;
        if constexpr ((FEAT & F_SMALL) != 0 && !M<R>::literal) hit = object_intersect<R, STATS, FEAT>(sv, sv.small.objects[i], o, d, tmin, any, h, ts);
        else hit = object_intersect<R, STATS, FEAT>(sv, sv.objects[i], o, d, tmin, any, h, ts);
        if (hit) {
            h.obj = (int)i;
            if (any) return;
        }
    }
}

#if defined(__CUDACC__) && !defined(RPTB_HOST_EMU)
// get_closest_hit (renderer.rs:211-220) for the warp: every lane with `active` holds a world ray (ro, rd) and its
// h.t = tmax.  Analytic shapes, one-leaf meshes and kd-trees of shapes are intersected by the lane that owns the ray;
// a mesh with a BVH is entered through the lane-group traversal above.  Called by ALL 32 lanes of a full warp.
template <bool STATS, int FEAT>
__device__ __forceinline__ void closest_hit_coop(const SceneView<float>& sv, const bool active, const Vec3<float> ro, const Vec3<float> rd,
                                                 const float tmin, const bool any, Hit<float>& h, TravStats& ts, const uint32_t lane,
                                                 CoopWarp& cw) {
    h.obj = -1;
    h.aux = 0;
    h.bv = h.bw = 0.0f;
    if constexpr ((FEAT & F_GROUP) != 0) h.child = 0;
    const uint32_t n = sv.nobjects;
    for (uint32_t i = 0; i < n; i++) {
        const ObjectRec<float>& ob = sv.objects[i];
        const bool live = active && !(any && h.obj >= 0);  // a shadow ray ends at its first hit
        if (ob.kind == SHAPE_MESH && !sv.meshes[ob.mesh].root_is_leaf) {  // warp-uniform
            const MeshRec<float>& mm = sv.meshes[ob.mesh];
            bool pred = live;
            Vec3<float> o = ro, d = rd;
            if (pred) {
                if (STATS) ts.object_tests++;
                if (ob.has_transform) {
                    o = xform_point(ob.inv, ro);
                    d = xform_dir(ob.inv, rd);
                }
                // root cull: BoundingBox::intersect of KdTree::bounds (kdtree.rs:130-134) against [tmin, closest so far]
                const Vec3<float> iv = {slab_rcp(d.x), slab_rcp(d.y), slab_rcp(d.z)};
                const float x1 = (mm.bmin[0] - o.x) * iv.x, x2 = (mm.bmax[0] - o.x) * iv.x;
                const float y1 = (mm.bmin[1] - o.y) * iv.y, y2 = (mm.bmax[1] - o.y) * iv.y;
                const float z1 = (mm.bmin[2] - o.z) * iv.z, z2 = (mm.bmax[2] - o.z) * iv.z;
                const float l0 = fmaxf(fmaxf(fminf(x1, x2), fminf(y1, y2)), fminf(z1, z2));
                const float h0 = fminf(fminf(fmaxf(x1, x2), fmaxf(y1, y2)), fmaxf(z1, z2));
                pred = !(fmaxf(l0, tmin) > fminf(h0, h.t));
            }
            const unsigned m = __ballot_sync(0xffffffffu, pred);
            if (__popc(m) > RPTB_COOP_MAX) {
                // many rays of the warp enter the mesh (coherent camera or shadow rays): one ray per lane fills the warp
                if (pred && bvh_query<STATS>(mm, o, d, tmin, any, h, ts)) h.obj = (int)i;
            } else if (m != 0u) {
                const uint32_t pos = (uint32_t)__popc(m & ((1u << lane) - 1u));
                if (pred) {
                    cw.ra[pos] = make_float4(o.x, o.y, o.z, h.t);
                    cw.rb[pos] = make_float4(d.x, d.y, d.z, 0.0f);
                    cw.res[pos] = make_float4(-1.0f, 0.0f, 0.0f, 0.0f);
                }
                if (lane == 0u) cw.next = 0u;
                __syncwarp();
                bvh8_group_trace<STATS>(mm, cw, (uint32_t)__popc(m), any, lane, ts);
                __syncwarp();
                if (pred) {
                    const float4 r = cw.res[pos];
                    if (r.x == -2.0f) {  // the group's stack overflowed (a pathological tree): the binary BVH has no such limit
                        if (bvh_query<STATS>(mm, o, d, tmin, any, h, ts)) h.obj = (int)i;
                    } else if (r.x >= 0.0f) {
                        h.t = r.x;
                        h.bv = r.y;
                        h.bw = r.z;
                        h.aux = __float_as_uint(r.w);
                        h.obj = (int)i;
                    }
                }
                __syncwarp();  // the answers are read before the next mesh reuses the block
            }
        } else if (live) {
            if (STATS) ts.object_tests++;
            if (object_intersect<float, STATS, FEAT>(sv, ob, ro, rd, tmin, any, h, ts)) h.obj = (int)i;
        }
    }
}
#endif

// f32 only: start the next ray a few ulps off the surface, on the side it leaves from.
// The reference restarts exactly at the hit point with t_min = 1e-12, which only works
// in f64 (SURVEY section 7, "f64 -> f32").
RPTB_D Vec3<float> offset_origin(Vec3<float> p, Vec3<float> ng, Vec3<float> dir, float scale) {
    const float delta = 1.9073486e-6f * scale;  // 32 * 2^-24 * max |coordinate| involved
    const float s = dot(dir, ng) >= 0.0f ? delta : -delta;
    return {fmaf(s, ng.x, p.x), fmaf(s, ng.y, p.y), fmaf(s, ng.z, p.z)};
}
RPTB_D Vec3<double> offset_origin(Vec3<double> p, Vec3<double>, Vec3<double>, double) { return p; }

template <class R>
RPTB_D R max_abs3(Vec3<R> a) { return M<R>::max(M<R>::max(M<R>::abs(a.x), M<R>::abs(a.y)), M<R>::abs(a.z)); }

}  // namespace rptb
