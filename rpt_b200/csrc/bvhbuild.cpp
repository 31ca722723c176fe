// bvhbuild.cpp -- host-side builder of the f32 path's own acceleration structure.
//
// The reference intersects a Mesh through KdTree<Triangle> (ekzhang/rpt src/kdtree.rs:99-223), built by a
// spatial-median `construct` whose inclusive two-sided partition references a triangle in every cell its
// box touches (SURVEY Appendix A #16: 5-7.5x duplication, leaves of up to 30+ triangles).  The closest hit
// of a ray does not depend on the structure that finds it, only its cost does: on the 871 k-triangle
// dragon proxy the reference-shaped tree costs 152 node visits and 419 triangle tests per ray.  The f64
// parity gate keeps that tree node for node; the f32 product path may use this one instead: a binary BVH,
// binned surface-area heuristic (16 bins over the centroid bounds), every triangle in exactly one leaf of at
// most BVH_LEAF_MAX triangles.  What stays the reference's is the triangle test itself (tri48).
//
// Output: nodes in the two-boxes-per-node layout of BvhNodeDev (scene_dev.cuh) and the permutation that
// puts the triangles in leaf order.  Boxes are rounded outward to float and padded, so the slab test can
// never reject a ray the f32 triangle test would accept.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#include <vector_types.h>

#include "scene_dev.cuh"

namespace {

using rptb::BvhNodeDev;
using rptb::Bvh8Node;
using rptb::Bvh4Node;

struct Box {
    float lo[3], hi[3];
    void reset() {
        for (int a = 0; a < 3; a++) lo[a] = INFINITY, hi[a] = -INFINITY;
    }
    void grow(const Box& b) {
        for (int a = 0; a < 3; a++) lo[a] = std::fmin(lo[a], b.lo[a]), hi[a] = std::fmax(hi[a], b.hi[a]);
    }
    void grow(const float* p) {
        for (int a = 0; a < 3; a++) lo[a] = std::fmin(lo[a], p[a]), hi[a] = std::fmax(hi[a], p[a]);
    }
    float half_area() const {
        const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        return dx * dy + dy * dz + dz * dx;
    }
};

struct Prim {
    Box box;
    float c[3];
    uint32_t id;
};

struct Node {
    Box box;
    std::unique_ptr<Node> kid[2];
    uint32_t first = 0, count = 0;  // leaf: range in `prims`
};

constexpr int BINS = 16;

// Builds the subtree over prims[first, first + count) in place (the range is partitioned recursively).
std::unique_ptr<Node> build(std::vector<Prim>& prims, uint32_t first, uint32_t count, int depth) {
    auto node = std::make_unique<Node>();
    node->box.reset();
    Box cb;
    cb.reset();
    for (uint32_t i = first; i < first + count; i++) {
        node->box.grow(prims[i].box);
        cb.grow(prims[i].c);
    }
    auto make_leaf = [&]() {
        node->first = first;
        node->count = count;
        return std::move(node);
    };
    if (count == 1) return make_leaf();
    const bool must_split = count > (uint32_t)rptb::BVH_LEAF_MAX;
    // binned SAH over the centroid bounds, best of the three axes
    float best_cost = INFINITY;
    int best_axis = -1, best_bin = -1;
    for (int a = 0; a < 3; a++) {
        const float ext = cb.hi[a] - cb.lo[a];
        if (!(ext > 0.0f)) continue;
        Box bb[BINS];
        uint32_t bn[BINS];
        for (int b = 0; b < BINS; b++) bb[b].reset(), bn[b] = 0;
        const float scale = (float)BINS / ext;
        for (uint32_t i = first; i < first + count; i++) {
            int b = (int)((prims[i].c[a] - cb.lo[a]) * scale);
            b = b < 0 ? 0 : (b >= BINS ? BINS - 1 : b);
            bb[b].grow(prims[i].box);
            bn[b]++;
        }
        float right_area[BINS];
        uint32_t right_n[BINS];
        Box acc;
        acc.reset();
        uint32_t n = 0;
        for (int b = BINS - 1; b > 0; b--) {
            acc.grow(bb[b]);
            n += bn[b];
            right_area[b] = acc.half_area();
            right_n[b] = n;
        }
        acc.reset();
        n = 0;
        for (int b = 0; b < BINS - 1; b++) {
            acc.grow(bb[b]);
            n += bn[b];
            if (n == 0 || right_n[b + 1] == 0) continue;
            const float cost = acc.half_area() * (float)n + right_area[b + 1] * (float)right_n[b + 1];
            if (cost < best_cost) best_cost = cost, best_axis = a, best_bin = b;
        }
    }
    uint32_t mid;
    if (best_axis < 0) {
        // all centroids coincide: nothing to bin
        if (!must_split) return make_leaf();
        mid = first + count / 2;
    } else {
        // SAH termination: a leaf costs `count` triangle tests, a split one node visit (~1 test) plus the
        // expected tests below it
        const float leaf_cost = (float)count;
        const float split_cost = 1.0f + best_cost / std::fmax(node->box.half_area(), 1e-30f);
        if (!must_split && split_cost >= leaf_cost) return make_leaf();
        const float ext = cb.hi[best_axis] - cb.lo[best_axis];
        const float scale = (float)BINS / ext;
        auto it = std::partition(prims.begin() + first, prims.begin() + first + count, [&](const Prim& p) {
            int b = (int)((p.c[best_axis] - cb.lo[best_axis]) * scale);
            b = b < 0 ? 0 : (b >= BINS ? BINS - 1 : b);
            return b <= best_bin;
        });
        mid = (uint32_t)(it - prims.begin());
        if (mid == first || mid == first + count) mid = first + count / 2;  // numerical corner: fall back to halves
    }
    if (depth >= rptb::BVH_STACK - 34) {
        // pathological input (SAH peeling off one triangle per level): the traversal stack is bounded, so from
        // here on split by index median, which halves the count per level -- at most 31 more levels
        mid = first + count / 2;
    }
    const uint32_t nl = mid - first, nr = count - nl;
    Node* np = node.get();
    if (count > 50000) {
#pragma omp task shared(prims) firstprivate(np, first, nl, depth) untied
        np->kid[0] = build(prims, first, nl, depth + 1);
#pragma omp task shared(prims) firstprivate(np, mid, nr, depth) untied
        np->kid[1] = build(prims, mid, nr, depth + 1);
#pragma omp taskwait
    } else {
        np->kid[0] = build(prims, first, nl, depth + 1);
        np->kid[1] = build(prims, mid, nr, depth + 1);
    }
    return node;
}

// Round a box outward and pad it: the f32 triangle test works on o + t d evaluated in float, which can
// land a few ulps outside the exact triangle, and the slab test evaluates (b - o)/d as b*(1/d) - o*(1/d), whose
// rounding error is ~6e-8 |o| in space whatever the box.  The pad therefore scales with the larger of the box's own
// coordinate and the MESH's extent (g_root_mag, set per build), including boxes that hug a coordinate plane (where
// |b| alone would give no pad).  Measured against a scan of every triangle (tests/test_hostemu_placement.py): the BVH
// returns every hit well inside a triangle from ray origins up to 1e3 mesh extents away.  At 1e5 extents, where t itself
// is resolved to ~1 % of the mesh, 0.8 % of those hits differ -- the same with a pad 100x smaller, so there it is the
// rounding of t, not the boxes, that decides.
float g_root_mag = 0.0f;
#pragma omp threadprivate(g_root_mag)
void pad(const Box& b, float* lo, float* hi) {
    for (int a = 0; a < 3; a++) {
        const float mag = std::fmax(std::fmax(std::fmax(std::fabs(b.lo[a]), std::fabs(b.hi[a])), g_root_mag), 1e-3f);
        const float eps = 4e-6f * mag;
        lo[a] = std::nextafterf(b.lo[a] - eps, -INFINITY);
        hi[a] = std::nextafterf(b.hi[a] + eps, INFINITY);
    }
}

int32_t child_code(const Node& n, std::vector<BvhNodeDev>& out, uint32_t depth, uint32_t& max_depth);

int32_t emit_inner(const Node& n, std::vector<BvhNodeDev>& out, uint32_t depth, uint32_t& max_depth) {
    const size_t me = out.size();
    out.emplace_back();
    std::memset(&out[me], 0, sizeof(BvhNodeDev));
    max_depth = std::max(max_depth, depth);
    float lo0[3], hi0[3], lo1[3], hi1[3];
    pad(n.kid[0]->box, lo0, hi0);
    pad(n.kid[1]->box, lo1, hi1);
    const int32_t c0 = child_code(*n.kid[0], out, depth + 1, max_depth);
    const int32_t c1 = child_code(*n.kid[1], out, depth + 1, max_depth);
    BvhNodeDev& d = out[me];
    d.c0xy = make_float4(lo0[0], hi0[0], lo0[1], hi0[1]);
    d.c1xy = make_float4(lo1[0], hi1[0], lo1[1], hi1[1]);
    d.cz = make_float4(lo0[2], hi0[2], lo1[2], hi1[2]);
    d.child0 = c0;
    d.child1 = c1;
    return (int32_t)me;
}

int32_t child_code(const Node& n, std::vector<BvhNodeDev>& out, uint32_t depth, uint32_t& max_depth) {
    if (n.count) return ~(int32_t)((n.first << 3) | (n.count - 1u));
    return emit_inner(n, out, depth, max_depth);
}

// ---- the eight-wide form: collapse the binary tree --------------------------------------------------------------
// Starting from a node's two children, the inner child with the largest surface area is replaced by its own two
// children until there are eight (or only leaves are left): the usual greedy collapse.  Leaves are kept as they are.
int32_t emit8(const Node& n, std::vector<Bvh8Node>& out, uint32_t depth, uint32_t& max_depth) {
    const size_t me = out.size();
    out.emplace_back();
    max_depth = std::max(max_depth, depth);
    const Node* kids[8];
    int nk = 2;
    kids[0] = n.kid[0].get();
    kids[1] = n.kid[1].get();
    while (nk < 8) {
        int best = -1;
        float best_area = -1.0f;
        for (int i = 0; i < nk; i++)
            if (!kids[i]->count && kids[i]->box.half_area() > best_area) best_area = kids[i]->box.half_area(), best = i;
        if (best < 0) break;
        const Node* open = kids[best];
        kids[best] = open->kid[0].get();
        kids[nk++] = open->kid[1].get();
    }
    Bvh8Node node;
    std::memset(&node, 0, sizeof(node));
    for (int i = 0; i < 8; i++) {
        rptb::Bvh8Child& c = node.c[i];
        if (i >= nk) {
            c.code = rptb::BVH8_EMPTY;
            continue;
        }
        pad(kids[i]->box, c.lo, c.hi);
        c.code = kids[i]->count ? ~(int32_t)((kids[i]->first << 3) | (kids[i]->count - 1u)) : emit8(*kids[i], out, depth + 1, max_depth);
    }
    out[me] = node;
    return (int32_t)me;
}

// ---- the four-wide form: the same greedy collapse, stopped at four children ----------------------------------------
int32_t emit4(const Node& n, std::vector<Bvh4Node>& out, uint32_t depth, uint32_t& max_depth) {
    const size_t me = out.size();
    out.emplace_back();
    max_depth = std::max(max_depth, depth);
    const Node* kids[4];
    int nk = 2;
    kids[0] = n.kid[0].get();
    kids[1] = n.kid[1].get();
    while (nk < 4) {
        int best = -1;
        float best_area = -1.0f;
        for (int i = 0; i < nk; i++)
            if (!kids[i]->count && kids[i]->box.half_area() > best_area) best_area = kids[i]->box.half_area(), best = i;
        if (best < 0) break;
        const Node* open = kids[best];
        kids[best] = open->kid[0].get();
        kids[nk++] = open->kid[1].get();
    }
    float lo[4][3], hi[4][3];
    int32_t code[4];
    for (int i = 0; i < 4; i++) {
        if (i >= nk) {  // an empty slot: a box nothing can enter, and a code the traversal never follows
            // (both planes at +inf: every slab product is +inf or -inf on BOTH planes, never NaN, and near > far)
            for (int a = 0; a < 3; a++) lo[i][a] = INFINITY, hi[i][a] = INFINITY;
            code[i] = rptb::BVH8_EMPTY;
            continue;
        }
        pad(kids[i]->box, lo[i], hi[i]);
        code[i] = kids[i]->count ? ~(int32_t)((kids[i]->first << 3) | (kids[i]->count - 1u)) : emit4(*kids[i], out, depth + 1, max_depth);
    }
    Bvh4Node node;
    std::memset(&node, 0, sizeof(node));
    node.lox = make_float4(lo[0][0], lo[1][0], lo[2][0], lo[3][0]);
    node.hix = make_float4(hi[0][0], hi[1][0], hi[2][0], hi[3][0]);
    node.loy = make_float4(lo[0][1], lo[1][1], lo[2][1], lo[3][1]);
    node.hiy = make_float4(hi[0][1], hi[1][1], hi[2][1], hi[3][1]);
    node.loz = make_float4(lo[0][2], lo[1][2], lo[2][2], lo[3][2]);
    node.hiz = make_float4(hi[0][2], hi[1][2], hi[2][2], hi[3][2]);
    node.code = make_int4(code[0], code[1], code[2], code[3]);
    out[me] = node;
    return (int32_t)me;
}

}  // namespace

namespace rptb {

// tris: ntris x 18 doubles (v1 v2 v3 n1 n2 n3).  `order[k]` = original index of the k-th triangle in leaf
// order.  1 <= ntris < 2^28; returns 0, or -1 outside that range.  The root is always an inner node: a mesh the
// SAH would leave as one leaf (a caller-supplied kd-tree may split over four triangles or fewer) becomes a root
// whose two children are the halves of that leaf (the same leaf twice for a single triangle -- the second test of a
// triangle can never tighten the hit, `time >= h.t` rejects it).
int build_bvh_host(const double* tris, uint64_t ntris, std::vector<BvhNodeDev>& nodes, std::vector<uint32_t>& order,
                   uint32_t& depth, std::vector<Bvh8Node>* nodes8, std::vector<Bvh4Node>* nodes4) {
    if (ntris == 0 || ntris >= (1ull << 28)) return -1;
    std::vector<Prim> prims(ntris);
    for (uint64_t i = 0; i < ntris; i++) {
        const double* t = tris + 18 * i;
        Prim& p = prims[i];
        p.id = (uint32_t)i;
        p.box.reset();
        for (int k = 0; k < 3; k++) {
            // outward-rounded float box of the double vertices
            float v[3];
            for (int a = 0; a < 3; a++) v[a] = (float)t[3 * k + a];
            for (int a = 0; a < 3; a++) {
                const float f = v[a];
                const float lo = (double)f > t[3 * k + a] ? std::nextafterf(f, -INFINITY) : f;
                const float hi = (double)f < t[3 * k + a] ? std::nextafterf(f, INFINITY) : f;
                p.box.lo[a] = std::fmin(p.box.lo[a], lo);
                p.box.hi[a] = std::fmax(p.box.hi[a], hi);
            }
        }
        for (int a = 0; a < 3; a++) p.c[a] = 0.5f * (p.box.lo[a] + p.box.hi[a]);
    }
    std::unique_ptr<Node> root;
#pragma omp parallel
#pragma omp single
    root = build(prims, 0, (uint32_t)ntris, 0);
    nodes.clear();
    depth = 0;
    g_root_mag = 0.0f;
    for (int a = 0; a < 3; a++) g_root_mag = std::fmax(g_root_mag, std::fmax(std::fabs(root->box.lo[a]), std::fabs(root->box.hi[a])));
    if (root->count) {  // the whole mesh is one leaf: give the root two leaf children
        const uint32_t n = root->count, h = n > 1 ? n / 2 : 1;
        for (int k = 0; k < 2; k++) {
            auto kid = std::make_unique<Node>();
            kid->first = (k == 0 || n == 1) ? 0 : h;
            kid->count = n == 1 ? 1 : (k == 0 ? h : n - h);
            kid->box.reset();
            for (uint32_t i = kid->first; i < kid->first + kid->count; i++) kid->box.grow(prims[i].box);
            root->kid[k] = std::move(kid);
        }
        root->count = 0;
    }
    emit_inner(*root, nodes, 0, depth);
    if (nodes8) {
        nodes8->clear();
        uint32_t depth8 = 0;
        emit8(*root, *nodes8, 0, depth8);
    }
    if (nodes4) {
        nodes4->clear();
        uint32_t depth4 = 0;
        emit4(*root, *nodes4, 0, depth4);
        // a ray pushes at most three entries per level it descends
        if (3 * (depth4 + 1) > (uint32_t)rptb::BVH4_STACK) nodes4->clear();
    }
    order.resize(ntris);
    for (uint64_t i = 0; i < ntris; i++) order[i] = prims[i].id;
    return 0;
}

}  // namespace rptb
