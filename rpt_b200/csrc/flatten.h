// flatten.h -- rptb_scene_desc -> the arrays the kernels read, built on the host (no CUDA calls).
//
// What is flattened (ekzhang/rpt @815b21c): Scene{objects, lights, environment} (src/scene.rs:7-18),
// Object{shape: Box<dyn Shape>, material} (src/object.rs:10-16), Transformed<T> (src/shape.rs:99-125:
// the inverse, the normal matrix and det(linear) are precomputed exactly as Transformed::new does),
// KdTree<Triangle> and KdTree<Box<dyn Bounded>> (src/kdtree.rs:99-119,226-233: re-serialised in DFS
// pre-order, left child = node + 1), Triangle (src/shape/mesh.rs:7-22: plus the per-triangle invariants
// of Triangle::intersect folded into 48 bytes).
//
// Two consumers: api.cu uploads the vectors (bind_scene with an uploader that copies to the device);
// tests/hostemu binds the same vectors in place so the device functions can be run on the host.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/rpt_b200.h"
#include "scene_dev.cuh"

namespace rptb {

int build_kdtree_host(const double* tris, uint64_t ntris, std::vector<rptb_kdnode>& nodes, std::vector<uint32_t>& refs,
                      uint32_t& depth, uint32_t& max_leaf);
int build_kdtree_boxes_host(const double* boxes, uint64_t nboxes, std::vector<rptb_kdnode>& nodes, std::vector<uint32_t>& refs,
                            uint32_t& depth, uint32_t& max_leaf);
int build_bvh_host(const double* tris, uint64_t ntris, std::vector<BvhNodeDev>& nodes, std::vector<uint32_t>& order, uint32_t& depth,
                   std::vector<Bvh8Node>* nodes8 = nullptr, std::vector<Bvh4Node>* nodes4 = nullptr);

inline int flat_fail(std::string& err, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    err = buf;
    return code;
}

// ---- small double-precision matrix helpers (column-major 4x4 in) -------------------
struct Xf {
    double fwd[12];  // rows of the 3x4
    double inv[12];
    double nrm[9];   // rows of (L^-1)^T
    double det;
};

inline bool invert4(const double* m /*col-major*/, double* out /*col-major*/) {
    double w[4][8];
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) {
            w[r][c] = m[c * 4 + r];
            w[r][c + 4] = r == c ? 1.0 : 0.0;
        }
    for (int i = 0; i < 4; i++) {
        int p = i;
        for (int r = i + 1; r < 4; r++)
            if (std::fabs(w[r][i]) > std::fabs(w[p][i])) p = r;
        if (w[p][i] == 0.0) return false;
        if (p != i)
            for (int c = 0; c < 8; c++) std::swap(w[i][c], w[p][c]);
        const double piv = w[i][i];
        for (int c = 0; c < 8; c++) w[i][c] /= piv;
        for (int r = 0; r < 4; r++)
            if (r != i && w[r][i] != 0.0) {
                const double f = w[r][i];
                for (int c = 0; c < 8; c++) w[r][c] -= f * w[i][c];
            }
    }
    for (int r = 0; r < 4; r++)
        for (int c = 0; c < 4; c++) out[c * 4 + r] = w[r][c + 4];
    return true;
}

// Transformed::new (src/shape.rs:111-124)
inline bool make_xf(const double* t /*col-major 4x4*/, Xf& x) {
    double inv[16];
    if (!invert4(t, inv)) return false;
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 4; c++) {
            x.fwd[r * 4 + c] = t[c * 4 + r];
            x.inv[r * 4 + c] = inv[c * 4 + r];
        }
    // linear = upper-left 3x3; L(r,c) = t[c*4+r]
    auto L = [&](int r, int c) { return t[c * 4 + r]; };
    const double det = L(0, 0) * (L(1, 1) * L(2, 2) - L(1, 2) * L(2, 1)) - L(0, 1) * (L(1, 0) * L(2, 2) - L(1, 2) * L(2, 0)) +
                       L(0, 2) * (L(1, 0) * L(2, 1) - L(1, 1) * L(2, 0));
    x.det = det;
    // inverse transpose = cofactor matrix / det
    double cof[3][3];
    cof[0][0] = L(1, 1) * L(2, 2) - L(1, 2) * L(2, 1);
    cof[0][1] = -(L(1, 0) * L(2, 2) - L(1, 2) * L(2, 0));
    cof[0][2] = L(1, 0) * L(2, 1) - L(1, 1) * L(2, 0);
    cof[1][0] = -(L(0, 1) * L(2, 2) - L(0, 2) * L(2, 1));
    cof[1][1] = L(0, 0) * L(2, 2) - L(0, 2) * L(2, 0);
    cof[1][2] = -(L(0, 0) * L(2, 1) - L(0, 1) * L(2, 0));
    cof[2][0] = L(0, 1) * L(1, 2) - L(0, 2) * L(1, 1);
    cof[2][1] = -(L(0, 0) * L(1, 2) - L(0, 2) * L(1, 0));
    cof[2][2] = L(0, 0) * L(1, 1) - L(0, 1) * L(1, 0);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) x.nrm[r * 3 + c] = cof[r][c] / det;
    return true;
}

template <class R>
void fill_object(const rptb_object& o, ObjectRec<R>& rec) {
    std::memset(&rec, 0, sizeof(rec));
    rec.kind = o.kind;
    rec.material = o.material;
    rec.mesh = o.mesh;
    rec.has_transform = o.has_transform ? 1u : 0u;
    Xf x;
    static const double ident[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    make_xf(o.has_transform ? o.transform : ident, x);
    for (int i = 0; i < 12; i++) {
        rec.inv[i] = (R)x.inv[i];
        rec.fwd[i] = (R)x.fwd[i];
    }
    for (int i = 0; i < 9; i++) rec.nrm[i] = (R)x.nrm[i];
    rec.det = (R)x.det;
    const double len = std::sqrt(o.plane_normal[0] * o.plane_normal[0] + o.plane_normal[1] * o.plane_normal[1] +
                                 o.plane_normal[2] * o.plane_normal[2]);
    for (int i = 0; i < 3; i++) {
        rec.plane_n[i] = (R)o.plane_normal[i];
        rec.plane_unit[i] = (R)(len > 0 ? o.plane_normal[i] / len : 0.0);
    }
    rec.plane_v = (R)o.plane_value;
    if (o.kind == RPTB_SHAPE_MONOMIAL) {  // MonomialSurface{height, exp} rides in the plane slots
        rec.plane_v = (R)o.monomial_height;
        rec.plane_n[0] = (R)o.monomial_exp;
    }
}

template <class R>
void fill_material(const rptb_material& m, MaterialRec<R>& rec) {
    for (int i = 0; i < 3; i++) rec.color[i] = (R)m.color[i];
    rec.index = (R)m.index;
    rec.roughness = (R)m.roughness;
    rec.metallic = (R)m.metallic;
    rec.emittance = (R)m.emittance;
    rec.transparent = m.transparent ? 1u : 0u;
}

// A kd-tree re-serialised for the device, in both node formats.
struct FlatTree {
    std::vector<KdNodeDev> nodes32;
    std::vector<KdNodeDev64> nodes64;
    std::vector<uint32_t> refs;
    uint32_t depth = 0;
};

// One flattened mesh on the host, before upload.
struct HostMesh : FlatTree {
    std::vector<float4> tri48;
    std::vector<float4> leaf_planes;
    std::vector<BvhNodeDev> bvh_nodes;  // F_BVH: the f32 path's own structure over the same triangles
    std::vector<Bvh8Node> bvh8_nodes;   // ... collapsed to eight children per node
    std::vector<Bvh4Node> bvh4_nodes;   // ... and to four
    std::vector<float4> bvh_tri48;
    std::vector<uint32_t> bvh_ids;
    std::vector<float> verts32, norms32;
    std::vector<double> verts64, norms64;
    double bmin[3], bmax[3];
    uint32_t ntris = 0;
};

// Re-serialise the boundary tree in DFS pre-order (left child = node + 1) into both node formats.
inline int flatten_nodes(const rptb_kdnode* in, uint64_t nnodes, const uint32_t* in_refs, uint64_t nrefs, uint64_t ntris,
                         FlatTree& hm, std::string& err) {
    struct Item {
        uint32_t src;
        uint32_t depth;
        int64_t parent;  // dst index of the parent waiting for its right-child index, -1 if none
    };
    std::vector<Item> stack;
    stack.push_back({0, 0, -1});
    hm.depth = 0;
    while (!stack.empty()) {
        const Item it = stack.back();
        stack.pop_back();
        if (it.src >= nnodes) return flat_fail(err, RPTB_ERR_BAD_ARG, "kd node index %u out of range (%llu nodes)", it.src, (unsigned long long)nnodes);
        if (hm.nodes32.size() > nnodes) return flat_fail(err, RPTB_ERR_BAD_ARG, "kd tree is not a tree (cycle?)");
        const rptb_kdnode& s = in[it.src];
        const uint32_t dst = (uint32_t)hm.nodes32.size();
        if (it.parent >= 0) {  // we are the right child of `parent`
            hm.nodes32[it.parent].word |= dst << 2;
            hm.nodes64[it.parent].word |= dst << 2;
        }
        hm.depth = std::max(hm.depth, it.depth);
        KdNodeDev n32;
        KdNodeDev64 n64;
        if (s.kind == 3) {
            if ((uint64_t)s.first_ref + s.num_refs > nrefs) return flat_fail(err, RPTB_ERR_BAD_ARG, "kd leaf refs out of range");
            if (s.num_refs >= (1u << 30)) return flat_fail(err, RPTB_ERR_UNSUPPORTED, "kd leaf too large");
            const uint32_t first = (uint32_t)hm.refs.size();
            for (uint32_t i = 0; i < s.num_refs; i++) {
                const uint32_t t = in_refs[s.first_ref + i];
                if (t >= ntris) return flat_fail(err, RPTB_ERR_BAD_ARG, "kd leaf references object %u of %llu", t, (unsigned long long)ntris);
                hm.refs.push_back(t);
            }
            n32.first_ref = first;
            n32.word = (s.num_refs << 2) | 3u;
            n64.split = 0.0;
            n64.first_ref = first;
            n64.word = n32.word;
            hm.nodes32.push_back(n32);
            hm.nodes64.push_back(n64);
        } else if (s.kind <= 2) {
            n32.split = (float)s.split;
            n32.word = s.kind;  // right child patched in when it is emitted
            n64.split = s.split;
            n64.first_ref = 0;
            n64.word = s.kind;
            hm.nodes32.push_back(n32);
            hm.nodes64.push_back(n64);
            // pre-order: left next (pushed last), right later with a back-pointer to us
            stack.push_back({s.right, it.depth + 1, (int64_t)dst});
            stack.push_back({s.left, it.depth + 1, -1});
        } else {
            return flat_fail(err, RPTB_ERR_BAD_ARG, "kd node kind %u", s.kind);
        }
    }
    if (hm.nodes32.size() >= (1u << 30)) return flat_fail(err, RPTB_ERR_UNSUPPORTED, "kd tree has too many nodes");
    return RPTB_OK;
}

inline int flatten_mesh(const rptb_mesh& m, HostMesh& hm, std::string& err) {
    if (m.ntris == 0 || m.tris == nullptr) return flat_fail(err, RPTB_ERR_BAD_ARG, "mesh without triangles");
    if (m.ntris >= (1ull << 31)) return flat_fail(err, RPTB_ERR_UNSUPPORTED, "mesh too large");
    hm.ntris = (uint32_t)m.ntris;
    int rc;
    if (m.nodes == nullptr) {
        std::vector<rptb_kdnode> nodes;
        std::vector<uint32_t> refs;
        uint32_t depth, max_leaf;
        build_kdtree_host(m.tris, m.ntris, nodes, refs, depth, max_leaf);
        rc = flatten_nodes(nodes.data(), nodes.size(), refs.data(), refs.size(), m.ntris, hm, err);
    } else {
        rc = flatten_nodes(m.nodes, m.nnodes, m.refs, m.nrefs, m.ntris, hm, err);
    }
    if (rc != RPTB_OK) return rc;
    if (hm.depth >= (uint32_t)KD_STACK) return flat_fail(err, RPTB_ERR_UNSUPPORTED, "kd tree depth %u exceeds the traversal stack (%d)", hm.depth, KD_STACK);

    for (int a = 0; a < 3; a++) {
        hm.bmin[a] = INFINITY;
        hm.bmax[a] = -INFINITY;
    }
    hm.tri48.resize(3 * (size_t)m.ntris);
    hm.verts32.resize(9 * (size_t)m.ntris);
    hm.norms32.resize(9 * (size_t)m.ntris);
    hm.verts64.resize(9 * (size_t)m.ntris);
    hm.norms64.resize(9 * (size_t)m.ntris);
    for (uint64_t i = 0; i < m.ntris; i++) {
        const double* t = m.tris + 18 * i;
        for (int k = 0; k < 9; k++) {
            hm.verts64[9 * i + k] = t[k];
            hm.verts32[9 * i + k] = (float)t[k];
            hm.norms64[9 * i + k] = t[9 + k];
            hm.norms32[9 * i + k] = (float)t[9 + k];
        }
        for (int a = 0; a < 3; a++) {  // KdTree::bounds = merge of Triangle::bounding_box
            hm.bmin[a] = std::fmin(hm.bmin[a], std::fmin(std::fmin(t[a], t[3 + a]), t[6 + a]));
            hm.bmax[a] = std::fmax(hm.bmax[a], std::fmax(std::fmax(t[a], t[3 + a]), t[6 + a]));
        }
        // the per-triangle invariants of Triangle::intersect (mesh.rs:50-72), folded in double
        const double d0[3] = {t[3] - t[0], t[4] - t[1], t[5] - t[2]};
        const double d1[3] = {t[6] - t[0], t[7] - t[1], t[8] - t[2]};
        double pn[3] = {d0[1] * d1[2] - d0[2] * d1[1], d0[2] * d1[0] - d0[0] * d1[2], d0[0] * d1[1] - d0[1] * d1[0]};
        const double len = std::sqrt(pn[0] * pn[0] + pn[1] * pn[1] + pn[2] * pn[2]);
        for (int a = 0; a < 3; a++) pn[a] /= len;
        const double d00 = d0[0] * d0[0] + d0[1] * d0[1] + d0[2] * d0[2];
        const double d01 = d0[0] * d1[0] + d0[1] * d1[1] + d0[2] * d1[2];
        const double d11 = d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2];
        const double denom = d00 * d11 - d01 * d01;
        double A[3], B[3];
        for (int a = 0; a < 3; a++) {
            A[a] = (d11 * d0[a] - d01 * d1[a]) / denom;
            B[a] = (d00 * d1[a] - d01 * d0[a]) / denom;
        }
        const double pnv1 = pn[0] * t[0] + pn[1] * t[1] + pn[2] * t[2];
        const double a0 = -(A[0] * t[0] + A[1] * t[1] + A[2] * t[2]);
        const double b0 = -(B[0] * t[0] + B[1] * t[1] + B[2] * t[2]);
        hm.tri48[3 * i + 0] = make_float4((float)pn[0], (float)pn[1], (float)pn[2], (float)pnv1);
        hm.tri48[3 * i + 1] = make_float4((float)A[0], (float)A[1], (float)A[2], (float)a0);
        hm.tri48[3 * i + 2] = make_float4((float)B[0], (float)B[1], (float)B[2], (float)b0);
    }
    return RPTB_OK;
}


// One flattened kd-tree over whole shapes (rptb_group).
struct HostGroup : FlatTree {
    std::vector<float4> kid_boxes;  // 2 per child: Bounded::bounding_box in the group's space, widened for f32
    std::vector<ObjectRec<float>> kids32;
    std::vector<ObjectRec<double>> kids64;
    double bmin[3], bmax[3];
};

template <class R>
struct Tables {
    std::vector<ObjectRec<R>> objects;
    std::vector<LightRec<R>> lights;
    std::vector<MaterialRec<R>> materials;
    std::vector<MeshRec<R>> meshes;
    std::vector<GroupRec<R>> groups;
};

struct HostScene {
    std::vector<HostMesh> meshes;
    std::vector<HostGroup> groups;
    Tables<float> t32;
    Tables<double> t64;
    std::vector<float4> env32;
    std::vector<double> env64;
    EnvRec<float> envrec32;
    EnvRec<double> envrec64;
    std::vector<float4> small_tris;  // tri48 of the one-leaf meshes, for SmallTables
    bool small_ok = false;
    std::vector<float4> flat;  // the packed primitive table (scene_dev.cuh, F_FLAT)
    bool flat_ok = false;      // the scene qualifies for it: the render and hit kernels walk `flat` (F_FLAT)
    int features = 0;         // F_TREE | F_TRANSP | F_HDRI | F_SMALL | F_GROUP | F_MONO actually present
    bool has_tree = false;     // some mesh's kd-tree is more than one leaf
    uint64_t tree_nodes = 0;   // kd nodes over all meshes
    double wlo[3] = {INFINITY, INFINITY, INFINITY}, whi[3] = {-INFINITY, -INFINITY, -INFINITY};  // world bounds of the meshes
    uint32_t sampled_lights = 0;  // non-ambient lights
};

// ---- Bounded::bounding_box (src/kdtree.rs:8-12 and the impls it cites) ---------------------------
inline void transform_box(const double* t /*col-major 4x4*/, const double* lo, const double* hi, double* olo, double* ohi) {
    for (int a = 0; a < 3; a++) {
        olo[a] = INFINITY;
        ohi[a] = -INFINITY;
    }
    for (int c = 0; c < 8; c++) {  // src/shape.rs:153-175: the box of the 8 transformed corners
        const double p[3] = {(c & 4) ? hi[0] : lo[0], (c & 2) ? hi[1] : lo[1], (c & 1) ? hi[2] : lo[2]};
        for (int r = 0; r < 3; r++) {
            const double v = t[0 * 4 + r] * p[0] + t[1 * 4 + r] * p[1] + t[2 * 4 + r] * p[2] + t[3 * 4 + r];
            olo[r] = std::fmin(olo[r], v);
            ohi[r] = std::fmax(ohi[r], v);
        }
    }
}

// false = the shape is not Bounded here (Plane, or a group inside a group)
inline bool shape_box(const rptb_object& o, const std::vector<HostMesh>& meshes, double* lo, double* hi) {
    double blo[3], bhi[3];
    switch (o.kind) {
        case RPTB_SHAPE_SPHERE:  // src/shape/sphere.rs:67-74
            for (int a = 0; a < 3; a++) blo[a] = -1.0, bhi[a] = 1.0;
            break;
        case RPTB_SHAPE_CUBE:  // src/shape/cube.rs:10-17
            for (int a = 0; a < 3; a++) blo[a] = -0.5, bhi[a] = 0.5;
            break;
        case RPTB_SHAPE_MONOMIAL:  // src/shape/monomial_surface.rs:179-186
            blo[0] = -1.0, blo[1] = 0.0, blo[2] = -1.0;
            bhi[0] = 1.0, bhi[1] = o.monomial_height, bhi[2] = 1.0;
            break;
        case RPTB_SHAPE_MESH:  // KdTree::bounds, src/kdtree.rs:122-126
            for (int a = 0; a < 3; a++) blo[a] = meshes[o.mesh].bmin[a], bhi[a] = meshes[o.mesh].bmax[a];
            break;
        default: return false;
    }
    if (o.has_transform) transform_box(o.transform, blo, bhi, lo, hi);
    else
        for (int a = 0; a < 3; a++) lo[a] = blo[a], hi[a] = bhi[a];
    return true;
}

inline int validate_object(const rptb_scene_desc* d, const rptb_object& o, const char* what, uint64_t i, bool in_group, std::string& err) {
    if (o.kind > RPTB_SHAPE_GROUP) return flat_fail(err, RPTB_ERR_BAD_ARG, "%s %llu: bad shape kind %u", what, (unsigned long long)i, o.kind);
    if (in_group && o.kind == RPTB_SHAPE_PLANE)
        return flat_fail(err, RPTB_ERR_BAD_ARG, "%s %llu: a Plane is not Bounded and cannot be a kd-tree child", what, (unsigned long long)i);
    if (in_group && o.kind == RPTB_SHAPE_GROUP)
        return flat_fail(err, RPTB_ERR_UNSUPPORTED, "%s %llu: a kd-tree of shapes inside a kd-tree of shapes is not supported", what, (unsigned long long)i);
    if (!in_group && o.material >= d->nmaterials)
        return flat_fail(err, RPTB_ERR_BAD_ARG, "%s %llu: material %u out of range", what, (unsigned long long)i, o.material);
    if (o.kind == RPTB_SHAPE_MESH && o.mesh >= d->nmeshes)
        return flat_fail(err, RPTB_ERR_BAD_ARG, "%s %llu: mesh %u out of range", what, (unsigned long long)i, o.mesh);
    if (o.kind == RPTB_SHAPE_GROUP && (o.mesh >= d->ngroups || d->groups == nullptr))
        return flat_fail(err, RPTB_ERR_BAD_ARG, "%s %llu: group %u out of range", what, (unsigned long long)i, o.mesh);
    if (o.has_transform) {
        Xf x;
        if (!make_xf(o.transform, x)) return flat_fail(err, RPTB_ERR_BAD_ARG, "%s %llu: singular transform", what, (unsigned long long)i);
    }
    return RPTB_OK;
}

inline int flatten_group(const rptb_scene_desc* d, const rptb_group& g, uint32_t gi, const std::vector<HostMesh>& meshes,
                         HostGroup& hg, std::string& err) {
    if (g.nchildren == 0 || g.children == nullptr) return flat_fail(err, RPTB_ERR_BAD_ARG, "group %u without children", gi);
    if (g.nchildren >= (1ull << 30)) return flat_fail(err, RPTB_ERR_UNSUPPORTED, "group %u too large", gi);
    std::vector<double> boxes(6 * (size_t)g.nchildren);
    hg.kids32.resize((size_t)g.nchildren);
    hg.kids64.resize((size_t)g.nchildren);
    for (int a = 0; a < 3; a++) hg.bmin[a] = INFINITY, hg.bmax[a] = -INFINITY;
    for (uint64_t i = 0; i < g.nchildren; i++) {
        const rptb_object& c = g.children[i];
        const int rc = validate_object(d, c, "group child", i, true, err);
        if (rc != RPTB_OK) return rc;
        shape_box(c, meshes, &boxes[6 * i], &boxes[6 * i + 3]);
        for (int a = 0; a < 3; a++) {  // KdTree::new: bounds = fold(merge), src/kdtree.rs:110-113
            hg.bmin[a] = std::fmin(hg.bmin[a], boxes[6 * i + a]);
            hg.bmax[a] = std::fmax(hg.bmax[a], boxes[6 * i + 3 + a]);
        }
        fill_object(c, hg.kids32[i]);
        fill_object(c, hg.kids64[i]);
        // the f32 path culls a child by this box before entering its space; widen it by more than the
        // f32 rounding of the child's own transform can move a hit point (|x| * 2^-23 per operation)
        float mag = 1.0f;
        for (int a = 0; a < 6; a++) mag = std::fmax(mag, std::fabs((float)boxes[6 * i + a]));
        const float eps = 8e-6f * mag;
        hg.kid_boxes.push_back(make_float4((float)boxes[6 * i + 0] - eps, (float)boxes[6 * i + 1] - eps, (float)boxes[6 * i + 2] - eps, 0.0f));
        hg.kid_boxes.push_back(make_float4((float)boxes[6 * i + 3] + eps, (float)boxes[6 * i + 4] + eps, (float)boxes[6 * i + 5] + eps, 0.0f));
    }
    int rc;
    if (g.nodes == nullptr) {
        std::vector<rptb_kdnode> nodes;
        std::vector<uint32_t> refs;
        uint32_t depth, max_leaf;
        build_kdtree_boxes_host(boxes.data(), g.nchildren, nodes, refs, depth, max_leaf);
        rc = flatten_nodes(nodes.data(), nodes.size(), refs.data(), refs.size(), g.nchildren, hg, err);
    } else {
        rc = flatten_nodes(g.nodes, g.nnodes, g.refs, g.nrefs, g.nchildren, hg, err);
    }
    if (rc != RPTB_OK) return rc;
    if (hg.depth >= (uint32_t)GROUP_STACK)
        return flat_fail(err, RPTB_ERR_UNSUPPORTED, "group %u: kd tree depth %u exceeds the traversal stack (%d)", gi, hg.depth, GROUP_STACK);
    return RPTB_OK;
}

template <class R>
void fill_tables(const rptb_scene_desc* d, Tables<R>& t) {
    t.objects.resize(d->nobjects);
    for (uint32_t i = 0; i < d->nobjects; i++) fill_object(d->objects[i], t.objects[i]);
    t.materials.resize(d->nmaterials);
    for (uint32_t i = 0; i < d->nmaterials; i++) fill_material(d->materials[i], t.materials[i]);
    t.lights.resize(d->nlights);
    for (uint32_t i = 0; i < d->nlights; i++) {
        const rptb_light& l = d->lights[i];
        LightRec<R>& r = t.lights[i];
        std::memset(&r, 0, sizeof(r));
        r.kind = l.kind;
        for (int k = 0; k < 3; k++) {
            r.color[k] = (R)l.color[k];
            r.vec[k] = (R)l.vec[k];
        }
        if (l.kind == RPTB_LIGHT_OBJECT) {
            fill_object(l.object, r.object);
            const rptb_material& m = d->materials[l.object.material];
            for (int k = 0; k < 3; k++) r.radiance[k] = (R)(m.color[k] * m.emittance);  // light.rs:42
        }
    }
}

// ObjectRec::err_mag.  A hit is computed on object-space coordinates (M^-1 o, the tri48 plane word pn . v1, q0.w - pn . o),
// which round relative to the object's own extent, and the rounding reaches world space through the transform's linear
// part L.  So the f32 path's restart offset (offset_origin) is sized from max(|world coordinates|, err_mag) with
// err_mag = ||L||_inf * (largest |coordinate| of the object's bounds in its own space) / 8: offset_origin's 32 ulp of it are
// 4 ulp of the object-space magnitude, what the chain M^-1 o, pn . o, q0.w - pn . o and the plane word rounds
// (tests/test_hostemu_placement.py measures the choice).  A mesh whose vertices sit far
// from its local origin and are pulled back by its transform (scanned, CAD and georeferenced files) has world
// coordinates ~1 but object-space ones ~1e4: the world term alone leaves its restarted rays re-hitting their own face.
// Without a transform the object-space coordinates are the world ones: 0.  A kd-tree of shapes: its children's terms.
inline double object_err_mag(const rptb_scene_desc* d, const rptb_object& o, const std::vector<HostMesh>& meshes,
                             const std::vector<HostGroup>& groups) {
    double mag = 0.0, inner = 0.0;
    switch (o.kind) {
        case RPTB_SHAPE_SPHERE: mag = 1.0; break;
        case RPTB_SHAPE_CUBE: mag = 0.5; break;
        case RPTB_SHAPE_MONOMIAL: mag = std::fmax(1.0, std::fabs(o.monomial_height)); break;
        case RPTB_SHAPE_PLANE: {
            const double len = std::sqrt(o.plane_normal[0] * o.plane_normal[0] + o.plane_normal[1] * o.plane_normal[1] +
                                         o.plane_normal[2] * o.plane_normal[2]);
            mag = len > 0.0 ? std::fabs(o.plane_value) / len : 0.0;
            break;
        }
        case RPTB_SHAPE_MESH:
            for (int a = 0; a < 3; a++) mag = std::fmax(mag, std::fmax(std::fabs(meshes[o.mesh].bmin[a]), std::fabs(meshes[o.mesh].bmax[a])));
            break;
        case RPTB_SHAPE_GROUP: {
            const HostGroup& g = groups[o.mesh];
            for (int a = 0; a < 3; a++) mag = std::fmax(mag, std::fmax(std::fabs(g.bmin[a]), std::fabs(g.bmax[a])));
            const rptb_group& dg = d->groups[o.mesh];
            for (uint64_t i = 0; i < dg.nchildren; i++) inner = std::fmax(inner, object_err_mag(d, dg.children[i], meshes, groups));
            break;
        }
        default: break;
    }
    if (!o.has_transform) return inner;
    double norm = 0.0;  // ||L||_inf: the largest absolute row sum of the linear part
    for (int r = 0; r < 3; r++)
        norm = std::fmax(norm, std::fabs(o.transform[r]) + std::fabs(o.transform[4 + r]) + std::fabs(o.transform[8 + r]));
    return norm * std::fmax(mag, inner) / 8.0;
}

// f32 bounds must contain what f32 arithmetic makes of the contents: widen by one ulp outward
inline void widen_bounds(const double* lo, const double* hi, float* flo, float* fhi) {
    for (int k = 0; k < 3; k++) {
        flo[k] = std::nextafterf((float)lo[k], -INFINITY);
        fhi[k] = std::nextafterf((float)hi[k], INFINITY);
    }
}

inline void grow_world_bounds(HostScene& hs, const rptb_object& o, const double* blo, const double* bhi) {
    double lo[3], hi[3];
    static const double ident[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    transform_box(o.has_transform ? o.transform : ident, blo, bhi, lo, hi);
    for (int r = 0; r < 3; r++) {
        hs.wlo[r] = std::fmin(hs.wlo[r], lo[r]);
        hs.whi[r] = std::fmax(hs.whi[r], hi[r]);
    }
}

// Indices, enums and transforms of a description (no allocation: rptb_scene_create runs this before it
// even looks for a device, so a bad scene is a BAD_ARG on every box).
inline int validate_scene(const rptb_scene_desc* d, std::string& err) {
    if (d->nobjects && !d->objects) return flat_fail(err, RPTB_ERR_BAD_ARG, "objects is null");
    if (d->nlights && !d->lights) return flat_fail(err, RPTB_ERR_BAD_ARG, "lights is null");
    if (d->nmaterials && !d->materials) return flat_fail(err, RPTB_ERR_BAD_ARG, "materials is null");
    if (d->nmeshes && !d->meshes) return flat_fail(err, RPTB_ERR_BAD_ARG, "meshes is null");
    if (d->ngroups && !d->groups) return flat_fail(err, RPTB_ERR_BAD_ARG, "groups is null");
    for (uint32_t i = 0; i < d->nobjects; i++) {
        const int rc = validate_object(d, d->objects[i], "object", i, false, err);
        if (rc != RPTB_OK) return rc;
    }
    for (uint32_t i = 0; i < d->nlights; i++) {
        if (d->lights[i].kind > RPTB_LIGHT_OBJECT) return flat_fail(err, RPTB_ERR_BAD_ARG, "light %u: bad kind %u", i, d->lights[i].kind);
        if (d->lights[i].kind == RPTB_LIGHT_OBJECT) {
            const int rc = validate_object(d, d->lights[i].object, "light object", i, false, err);
            if (rc != RPTB_OK) return rc;
        }
    }
    for (uint32_t g = 0; g < d->ngroups; g++) {
        if (d->groups[g].nchildren == 0 || d->groups[g].children == nullptr) return flat_fail(err, RPTB_ERR_BAD_ARG, "group %u without children", g);
        for (uint64_t i = 0; i < d->groups[g].nchildren; i++) {
            const int rc = validate_object(d, d->groups[g].children[i], "group child", i, true, err);
            if (rc != RPTB_OK) return rc;
        }
    }
    if (d->environment.kind > RPTB_ENV_HDRI) return flat_fail(err, RPTB_ERR_BAD_ARG, "bad environment kind %u", d->environment.kind);
    if (d->accel > RPTB_ACCEL_BVH) return flat_fail(err, RPTB_ERR_BAD_ARG, "bad accel %u", d->accel);
    return RPTB_OK;
}

// The packed primitive table of scene_dev.cuh (F_FLAT) from the f32 object records, for scenes without kd-trees,
// BVHs, groups or monomials.  A one-leaf mesh becomes one record per run of consecutive triangles whose planes q0 are
// bitwise equal (Cornell: the two triangles of every polygon): the run's plane test gives the same time for each of
// them, so it is done once, and the barycentric tests still go in triangle order.
inline void build_flat_table(HostScene& hs) {
    hs.flat.clear();
    hs.flat_ok = false;
    if (hs.features & (F_TREE | F_EXT | F_BVH)) return;
    auto header = [&](uint32_t kind, uint32_t obj, uint32_t k, uint32_t first) {
        float4 w;
        const uint32_t v[4] = {kind, obj, k, first};
        std::memcpy(&w, v, sizeof(w));
        hs.flat.push_back(w);
    };
    for (uint32_t i = 0; i < (uint32_t)hs.t32.objects.size(); i++) {
        const ObjectRec<float>& ob = hs.t32.objects[i];
        const uint32_t tf = ob.has_transform ? FLAT_TF : 0u;
        auto rows = [&] {
            if (tf)
                for (int r = 0; r < 3; r++) hs.flat.push_back(make_float4(ob.inv[4 * r], ob.inv[4 * r + 1], ob.inv[4 * r + 2], ob.inv[4 * r + 3]));
        };
        if (ob.kind == SHAPE_SPHERE || ob.kind == SHAPE_CUBE) {
            header(ob.kind | tf, i, 0, 0);
            rows();
        } else if (ob.kind == SHAPE_PLANE) {
            header(ob.kind | tf, i, 0, 0);
            rows();
            hs.flat.push_back(make_float4(ob.plane_n[0], ob.plane_n[1], ob.plane_n[2], ob.plane_v));
        } else if (ob.kind == SHAPE_MESH) {
            if (!hs.t32.meshes[ob.mesh].root_is_leaf) {  // (excluded by F_TREE above)
                hs.flat.clear();
                return;
            }
            const std::vector<float4>& q = hs.meshes[ob.mesh].tri48;
            const uint32_t ntris = hs.t32.meshes[ob.mesh].ntris;
            for (uint32_t first = 0; first < ntris;) {
                uint32_t k = 1;
                while (first + k < ntris && std::memcmp(&q[3 * (size_t)(first + k)], &q[3 * (size_t)first], sizeof(float4)) == 0) k++;
                header(SHAPE_MESH | tf, i, k, first);
                rows();
                hs.flat.push_back(q[3 * (size_t)first]);
                for (uint32_t j = first; j < first + k; j++) {
                    hs.flat.push_back(q[3 * (size_t)j + 1]);
                    hs.flat.push_back(q[3 * (size_t)j + 2]);
                }
                first += k;
            }
        } else {  // (excluded by F_EXT above)
            hs.flat.clear();
            return;
        }
    }
    hs.flat_ok = true;
}

// Validates `d` and fills every host-side array; pointers inside the MeshRec / GroupRec / EnvRec tables
// stay null until bind_scene.
inline int flatten_scene(const rptb_scene_desc* d, HostScene& hs, std::string& err, bool want_bvh = false) {
    {
        const int rc = validate_scene(d, err);
        if (rc != RPTB_OK) return rc;
    }
    fill_tables(d, hs.t32);
    fill_tables(d, hs.t64);

    hs.meshes.resize(d->nmeshes);
    hs.t32.meshes.resize(d->nmeshes);
    hs.t64.meshes.resize(d->nmeshes);
    for (uint32_t i = 0; i < d->nmeshes; i++) {
        HostMesh& hm = hs.meshes[i];
        const int rc = flatten_mesh(d->meshes[i], hm, err);
        if (rc != RPTB_OK) return rc;
        MeshRec<float>& a = hs.t32.meshes[i];
        MeshRec<double>& b = hs.t64.meshes[i];
        std::memset(&a, 0, sizeof(a));
        std::memset(&b, 0, sizeof(b));
        const bool leaf = (hm.nodes32[0].word & 3u) == 3u;
        if (!leaf) {  // a real tree: planes in leaf order for the trace kernel
            hm.leaf_planes.resize(hm.refs.size());
            for (size_t k = 0; k < hm.refs.size(); k++) hm.leaf_planes[k] = hm.tri48[3 * (size_t)hm.refs[k]];
        }
        if (!leaf && want_bvh) {  // the f32 path's own BVH over the same triangles (bvhbuild.cpp)
            uint32_t bvh_depth = 0;
            if (build_bvh_host(d->meshes[i].tris, d->meshes[i].ntris, hm.bvh_nodes, hm.bvh_ids, bvh_depth, RPTB_BUILD_BVH8 ? &hm.bvh8_nodes : nullptr, RPTB_BUILD_BVH4 ? &hm.bvh4_nodes : nullptr) != 0)
                return flat_fail(err, RPTB_ERR_UNSUPPORTED, "mesh %u: cannot build a BVH over %llu triangles", i, (unsigned long long)d->meshes[i].ntris);
            if (bvh_depth + 2 >= (uint32_t)BVH_STACK)
                return flat_fail(err, RPTB_ERR_UNSUPPORTED, "mesh %u: BVH depth %u exceeds the traversal stack (%d)", i, bvh_depth, BVH_STACK);
            hm.bvh_tri48.resize(3 * (size_t)hm.ntris);
            for (size_t k = 0; k < hm.ntris; k++)
                for (int j = 0; j < 3; j++) hm.bvh_tri48[3 * k + j] = hm.tri48[3 * (size_t)hm.bvh_ids[k] + j];
        }
        for (int k = 0; k < 3; k++) {
            b.bmin[k] = hm.bmin[k];
            b.bmax[k] = hm.bmax[k];
        }
        widen_bounds(hm.bmin, hm.bmax, a.bmin, a.bmax);
        a.ntris = b.ntris = hm.ntris;
        a.root_is_leaf = b.root_is_leaf = leaf;
        if (leaf) {
            a.small_tri_base = (uint32_t)(hs.small_tris.size() / 3);
            hs.small_tris.insert(hs.small_tris.end(), hm.tri48.begin(), hm.tri48.end());
        } else {
            hs.has_tree = true;
        }
        hs.tree_nodes += hm.nodes32.size();
        // world-space bounds of every object that uses this mesh, for the ray sort keys
        for (uint32_t oi = 0; oi < d->nobjects; oi++)
            if (d->objects[oi].kind == RPTB_SHAPE_MESH && d->objects[oi].mesh == i) grow_world_bounds(hs, d->objects[oi], hm.bmin, hm.bmax);
    }

    hs.groups.resize(d->ngroups);
    hs.t32.groups.resize(d->ngroups);
    hs.t64.groups.resize(d->ngroups);
    bool has_mono = false;
    for (uint32_t i = 0; i < d->ngroups; i++) {
        HostGroup& hg = hs.groups[i];
        const int rc = flatten_group(d, d->groups[i], i, hs.meshes, hg, err);
        if (rc != RPTB_OK) return rc;
        GroupRec<float>& a = hs.t32.groups[i];
        GroupRec<double>& b = hs.t64.groups[i];
        std::memset(&a, 0, sizeof(a));
        std::memset(&b, 0, sizeof(b));
        for (int k = 0; k < 3; k++) {
            b.bmin[k] = hg.bmin[k];
            b.bmax[k] = hg.bmax[k];
        }
        widen_bounds(hg.bmin, hg.bmax, a.bmin, a.bmax);
        a.nchildren = b.nchildren = (uint32_t)hg.kids32.size();
        a.root_is_leaf = b.root_is_leaf = (hg.nodes32[0].word & 3u) == 3u;
        for (uint64_t c = 0; c < d->groups[i].nchildren; c++) has_mono |= d->groups[i].children[c].kind == RPTB_SHAPE_MONOMIAL;
    }
    for (uint32_t i = 0; i < d->nobjects; i++) hs.t32.objects[i].err_mag = (float)object_err_mag(d, d->objects[i], hs.meshes, hs.groups);
    for (uint32_t i = 0; i < d->nobjects; i++) has_mono |= d->objects[i].kind == RPTB_SHAPE_MONOMIAL;
    for (uint32_t i = 0; i < d->nlights; i++)
        if (d->lights[i].kind == RPTB_LIGHT_OBJECT) has_mono |= d->lights[i].object.kind == RPTB_SHAPE_MONOMIAL;

    // environment
    std::memset(&hs.envrec32, 0, sizeof(hs.envrec32));
    std::memset(&hs.envrec64, 0, sizeof(hs.envrec64));
    hs.envrec32.kind = hs.envrec64.kind = d->environment.kind;
    for (int k = 0; k < 3; k++) {
        hs.envrec32.color[k] = (float)d->environment.color[k];
        hs.envrec64.color[k] = d->environment.color[k];
    }
    if (d->environment.kind == RPTB_ENV_HDRI) {
        const uint32_t w = d->environment.width, h = d->environment.height;
        if (w == 0 || h == 0 || d->environment.texels == nullptr) return flat_fail(err, RPTB_ERR_BAD_ARG, "HDRI without texels");
        const size_t n = (size_t)w * h;
        hs.env32.resize(n);
        for (size_t i = 0; i < n; i++)
            hs.env32[i] = make_float4((float)d->environment.texels[3 * i], (float)d->environment.texels[3 * i + 1],
                                      (float)d->environment.texels[3 * i + 2], 0.0f);
        hs.env64.assign(d->environment.texels, d->environment.texels + 3 * n);
        hs.envrec32.width = hs.envrec64.width = w;
        hs.envrec32.height = hs.envrec64.height = h;
    }

    for (uint32_t i = 0; i < d->nlights; i++)
        if (d->lights[i].kind != RPTB_LIGHT_AMBIENT) hs.sampled_lights++;
    if (hs.has_tree) hs.features |= F_TREE;
    if (hs.has_tree && want_bvh) hs.features |= F_BVH;  // every mesh with a real tree has its BVH
    for (uint32_t i = 0; i < d->nmaterials; i++)
        if (d->materials[i].transparent) hs.features |= F_TRANSP;
    if (d->environment.kind == RPTB_ENV_HDRI) hs.features |= F_HDRI;
    if (d->ngroups) hs.features |= F_GROUP;
    if (has_mono) hs.features |= F_MONO;
    // small scenes: the uniform tables also ride in the kernel parameters (scene_dev.cuh, SmallTables)
    // ... but only when what a ray actually walks (objects + lights + one-leaf triangles) stays within
    // ~1 KB: the constant cache in front of parameter space is tiny.  Measured: the sphere scene (0.6 KB)
    // got faster, Cornell (2.1 KB walked per ray) slower -- so Cornell stays on L1.
    // The packed primitive table (F_FLAT, 608 B for Cornell) lives in global memory only.  Measured on one H100 80GB HBM3
    // at a 400 W power limit, megakernel time at the bench size (Cornell 800x800, 512 spp, max_bounces 6): 253.3 ms with
    // the object scan, 238.6 ms with the table through L1, 243.9 ms with the same table in kernel-parameter space.
    const size_t walked = d->nobjects * sizeof(ObjectRec<float>) + d->nlights * sizeof(LightRec<float>) + hs.small_tris.size() * sizeof(float4);
    hs.small_ok = d->nobjects <= (uint32_t)SMALL_OBJECTS && d->nlights <= (uint32_t)SMALL_LIGHTS && d->nmeshes <= (uint32_t)SMALL_MESHES &&
                  hs.small_tris.size() <= (size_t)3 * SMALL_TRIS && walked <= 1024 && !(hs.features & F_EXT);
    build_flat_table(hs);
    // A/B switches, read when a scene is created: RPTB_NO_SMALL keeps the tables out of kernel-parameter space, RPTB_NO_FLAT
    // traces a flat scene through the scan over scene.objects instead of the packed table (which is still built)
    if (getenv("RPTB_NO_SMALL") != nullptr) hs.small_ok = false;
    if (getenv("RPTB_NO_FLAT") != nullptr) hs.flat_ok = false;
    return RPTB_OK;
}

// The feature bits the launchers dispatch on (launch.h) once bind_scene has run: what the scene has (hs.features, F_SMALL
// included), plus F_FLAT when it is traced through the packed primitive table.
inline int kernel_features(const HostScene& hs) { return hs.features | (hs.flat_ok ? (int)F_FLAT : 0); }

// Hands every array to `put` (which returns where the kernels will find it) and fills the SceneViews.
// Put:  template <class T> bool operator()(std::vector<T>& host, const T** where);   uint64_t bytes() const;
// `release` = the host copy of the big per-mesh arrays is dropped as soon as it is handed over.
template <class Put>
bool bind_scene(HostScene& hs, Put& put, bool release, SceneView<float>& v32, SceneView<double>& v64, uint64_t& f32_bytes) {
    f32_bytes = 0;
    for (size_t i = 0; i < hs.meshes.size(); i++) {
        HostMesh& hm = hs.meshes[i];
        MeshRec<float>& a = hs.t32.meshes[i];
        MeshRec<double>& b = hs.t64.meshes[i];
        const uint64_t before = put.bytes();
        if (!put(hm.nodes32, &a.nodes) || !put(hm.refs, &a.refs) || !put(hm.tri48, &a.tri48) || !put(hm.leaf_planes, &a.leaf_planes) ||
            !put(hm.verts32, &a.verts) || !put(hm.norms32, &a.norms) || !put(hm.bvh_nodes, &a.bvh_nodes) || !put(hm.bvh8_nodes, &a.bvh8_nodes) || !put(hm.bvh4_nodes, &a.bvh4_nodes) ||
            !put(hm.bvh_tri48, &a.bvh_tri48) || !put(hm.bvh_ids, &a.bvh_ids))
            return false;
        f32_bytes += put.bytes() - before;
        if (!put(hm.nodes64, &b.nodes) || !put(hm.verts64, &b.verts) || !put(hm.norms64, &b.norms)) return false;
        b.refs = a.refs;
        b.tri48 = nullptr;
        if (release) {
            std::vector<KdNodeDev>().swap(hm.nodes32);
            std::vector<KdNodeDev64>().swap(hm.nodes64);
            std::vector<uint32_t>().swap(hm.refs);
            std::vector<float4>().swap(hm.tri48);
            std::vector<float4>().swap(hm.leaf_planes);
            std::vector<BvhNodeDev>().swap(hm.bvh_nodes);
            std::vector<Bvh8Node>().swap(hm.bvh8_nodes);
            std::vector<Bvh4Node>().swap(hm.bvh4_nodes);
            std::vector<float4>().swap(hm.bvh_tri48);
            std::vector<uint32_t>().swap(hm.bvh_ids);
            std::vector<float>().swap(hm.verts32);
            std::vector<float>().swap(hm.norms32);
            std::vector<double>().swap(hm.verts64);
            std::vector<double>().swap(hm.norms64);
        }
    }
    for (size_t i = 0; i < hs.groups.size(); i++) {
        HostGroup& hg = hs.groups[i];
        GroupRec<float>& a = hs.t32.groups[i];
        GroupRec<double>& b = hs.t64.groups[i];
        const uint64_t before = put.bytes();
        if (!put(hg.nodes32, &a.nodes) || !put(hg.refs, &a.refs) || !put(hg.kids32, &a.children) || !put(hg.kid_boxes, &a.child_box)) return false;
        f32_bytes += put.bytes() - before;
        if (!put(hg.nodes64, &b.nodes) || !put(hg.kids64, &b.children)) return false;
        b.refs = a.refs;
    }
    {
        const uint64_t before = put.bytes();
        if (!put(hs.t32.objects, &v32.objects) || !put(hs.t32.lights, &v32.lights) || !put(hs.t32.materials, &v32.materials) ||
            !put(hs.t32.meshes, &v32.meshes) || !put(hs.t32.groups, &v32.groups) || !put(hs.flat, &v32.flat))
            return false;
        v32.env = hs.envrec32;
        if (!put(hs.env32, &v32.env.texels_f4)) return false;
        f32_bytes += put.bytes() - before;
        if (!put(hs.t64.objects, &v64.objects) || !put(hs.t64.lights, &v64.lights) || !put(hs.t64.materials, &v64.materials) ||
            !put(hs.t64.meshes, &v64.meshes) || !put(hs.t64.groups, &v64.groups))
            return false;
        v64.env = hs.envrec64;
        if (!put(hs.env64, &v64.env.texels_f64)) return false;
    }
    v32.nobjects = v64.nobjects = (uint32_t)hs.t32.objects.size();
    v32.nlights = v64.nlights = (uint32_t)hs.t32.lights.size();
    v32.nmaterials = v64.nmaterials = (uint32_t)hs.t32.materials.size();
    v32.nmeshes = v64.nmeshes = (uint32_t)hs.t32.meshes.size();
    v32.ngroups = v64.ngroups = (uint32_t)hs.t32.groups.size();
    v32.tables_in_const = v64.tables_in_const = 0;
    if (hs.small_ok) {
        SmallTables<float>& sm = v32.small;
        std::memset(&sm, 0, sizeof(sm));
        for (size_t i = 0; i < hs.t32.objects.size(); i++) sm.objects[i] = hs.t32.objects[i];
        for (size_t i = 0; i < hs.t32.lights.size(); i++) sm.lights[i] = hs.t32.lights[i];
        for (size_t i = 0; i < hs.t32.meshes.size(); i++) sm.meshes[i] = hs.t32.meshes[i];
        for (size_t i = 0; i < hs.small_tris.size(); i++) sm.tri48[i] = hs.small_tris[i];
        v32.tables_in_const = 1;
        hs.features |= F_SMALL;
    }
    v32.flat_words = (uint32_t)hs.flat.size();
    return true;
}

// rptb_camera + rptb_render_params -> the kernel arguments (everything but the output / partial pointers).
template <class R>
void fill_args(const rptb_camera* cam, const rptb_render_params* p, RenderArgs<R>& a) {
    std::memset(&a, 0, sizeof(a));
    // Camera::cast_ray invariants (src/camera.rs:66-67)
    const double d = 1.0 / std::tan(cam->fov / 2.0);
    const double* di = cam->direction;
    const double* up = cam->up;
    double right[3] = {di[1] * up[2] - di[2] * up[1], di[2] * up[0] - di[0] * up[2], di[0] * up[1] - di[1] * up[0]};
    const double len = std::sqrt(right[0] * right[0] + right[1] * right[1] + right[2] * right[2]);
    for (int k = 0; k < 3; k++) {
        a.cam.eye[k] = (R)cam->eye[k];
        a.cam.direction[k] = (R)di[k];
        a.cam.up[k] = (R)up[k];
        a.cam.right[k] = (R)(right[k] / len);
    }
    a.cam.d = (R)d;
    a.cam.aperture = (R)cam->aperture;
    a.cam.focal_distance = (R)cam->focal_distance;
    a.width = p->width;
    a.height = p->height;
    a.iterations = p->iterations;
    a.max_bounces = p->max_bounces;
    a.exposure_scale = (R)std::pow(2.0, p->exposure_value);
    a.seed = p->seed;
    a.first_sample = p->first_sample;
    a.shard_count = p->shard_count ? p->shard_count : 1;
    a.shard_index = p->shard_index;
    a.tiles_x = (p->width + 15) / 16;
    a.tiles_y = (p->height + 7) / 8;
    const uint32_t ntiles = a.tiles_x * a.tiles_y;
    a.ntiles_mine = ntiles > a.shard_index ? (ntiles - a.shard_index + a.shard_count - 1) / a.shard_count : 0;
    sample_chunks(p->iterations, a.nchunks, a.chunk);
    sample_groups(a.ntiles_mine, a.nchunks, a.ngroups, a.chunks_per_group);
    if (const char* g = getenv("RPTB_GROUPS")) {  // tuning aid: force the number of sample groups
        uint32_t want = (uint32_t)atoi(g);
        if (want < 1) want = 1;
        if (want > a.nchunks) want = a.nchunks;
        a.chunks_per_group = (a.nchunks + want - 1) / want;
        a.ngroups = (a.nchunks + a.chunks_per_group - 1) / a.chunks_per_group;
    }
    a.partial = nullptr;
}


}  // namespace rptb
