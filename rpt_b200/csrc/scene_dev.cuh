// scene_dev.cuh -- the flattened scene as the kernels see it (HBM layout).
//
// Reference structures being flattened:
//   Scene{objects, lights, environment}   src/scene.rs:7-18
//   Object{shape: Box<dyn Shape>, material} src/object.rs:10-16
//   Transformed<T>{transform, linear, inverse_transform, normal_transform, scale} src/shape.rs:99-125
//   KdTree<Triangle>{root, objects, bounds} src/kdtree.rs:99-104,226-233
//   Triangle{v1,v2,v3,n1,n2,n3}           src/shape/mesh.rs:7-22
//   Material (6 fields)                   src/material.rs:7-26
//   Light                                 src/light.rs:7-19
//   Hdri{width,height,buf}                src/environment.rs:4-14
//
// Layout (R = float unless the parity gate asks for double):
//   objects[]   ObjectRec<R>   one per scene object, uniform access -> __constant__ when it fits
//   lights[]    LightRec<R>
//   materials[] MaterialRec<R> divergent access -> global (L1-resident)
//   per mesh:   nodes[]  KdNodeDev (8 B: split f32 | (child<<2 | axis), leaf: first_ref | (count<<2 | 3))
//                        for double: KdNodeDev64 (16 B)
//               refs[]   u32 triangle indices, leaf order of the reference (ascending)
//               tri48[]  3 x float4 per triangle (f32 only): plane + two barycentric functionals
//               leaf_planes[] float4 per leaf ref (f32): the plane of refs[k], so a leaf's planes are one
//                        contiguous stream instead of one dependent gather per triangle
//               verts[]  9 R per triangle  (v1,v2,v3)  -- f64 intersect, light sampling
//               norms[]  9 R per triangle  (n1,n2,n3)  -- fetched once per final hit
#pragma once
#include "vec.cuh"

namespace rptb {

enum : uint32_t { SHAPE_SPHERE = 0, SHAPE_PLANE = 1, SHAPE_CUBE = 2, SHAPE_MESH = 3, SHAPE_MONOMIAL = 4, SHAPE_GROUP = 5 };
enum : uint32_t { LIGHT_POINT = 0, LIGHT_AMBIENT = 1, LIGHT_DIRECTIONAL = 2, LIGHT_OBJECT = 3 };

// Scene features a render kernel instantiation is compiled for.  The megakernel's hot loop is bound
// by instruction issue and its instruction cache (ncu: `no_instruction` is the #2 stall), so scenes
// that provably lack a feature run a variant with that code compiled out.
enum : int {
    F_TREE = 1 /* kd-trees beyond one leaf */, F_TRANSP = 2 /* transparent materials */, F_HDRI = 4, F_ALL = 7,
    F_SMALL = 8 /* the scene tables fit SmallTables: read them from kernel-parameter (constant) space */,
    F_GROUP = 16 /* kd-trees over whole shapes (KdTree<Box<dyn Bounded>>) */, F_MONO = 32 /* MonomialSurface */,
    F_EXT = F_GROUP | F_MONO, F_EVERY = F_ALL | F_EXT /* the one instantiation that knows every shape */,
    F_BVH = 64 /* f32 only: meshes are traversed through their BVH (MeshRec::bvh_*) instead of the reference-shaped kd-tree */,
    F_FLAT = 128 /* f32 only: get_closest_hit walks the packed primitive table (SceneView::flat) instead of the objects */
};

// Two experiments on the mesh configs (teapot / dragon-proxy / dragon-knot), both measured slower than what they were
// meant to improve and therefore off (measured before the port to the H100; not re-measured there):
//   RPTB_BVH_PREFETCH  prefetch.global.L1 of both children's lines once their boxes are hit -- the loop is latency bound,
//                      but the extra requests cost more than the early lines save
//   RPTB_COOP_MAX      the warp's rays that enter a mesh are traversed by groups of eight lanes over the eight-wide tree
//                      when there are at most this many of them (closest_hit_coop): slower at every limit tried.
//                      0 = never, and the code is compiled out
#ifndef RPTB_BVH_PREFETCH
#define RPTB_BVH_PREFETCH 0
#endif
#ifndef RPTB_COOP_MAX
#define RPTB_COOP_MAX 0
#endif
#ifndef RPTB_BUILD_BVH8
#define RPTB_BUILD_BVH8 (RPTB_COOP_MAX > 0)  // the eight-wide tree is built and uploaded only when something traverses it (tests/hostemu does)
#endif

constexpr int KD_STACK = 64;          // max kd-tree depth the traversal stack holds
constexpr int GROUP_STACK = 32;       // same, for a kd-tree over whole shapes (a few thousand children at most)
constexpr int MAX_CONST_OBJECTS = 96;  // tables up to this size live in __constant__ memory
constexpr int MAX_CONST_LIGHTS = 16;

struct KdNodeDev {  // 8 B
    union {
        float split;         // interior
        uint32_t first_ref;  // leaf
    };
    uint32_t word;  // interior: (right_child << 2) | axis ; leaf: (num_refs << 2) | 3
};
struct KdNodeDev64 {  // 16 B, parity gate
    double split;
    uint32_t word;       // as above
    uint32_t first_ref;  // leaf
};
template <class R>
struct NodeOf;
template <>
struct NodeOf<float> { typedef KdNodeDev type; };
template <>
struct NodeOf<double> { typedef KdNodeDev64 type; };

// A node of the f32 path's own acceleration structure: a binary BVH built with the surface-area
// heuristic (bvhbuild.cpp).  The node carries the boxes of BOTH children, so one 64-byte fetch decides
// which of them the ray enters.  child >= 0: index of an inner node; child < 0: a leaf,
// ~child = (first << 3) | (count - 1), naming triangles [first, first + count) in BVH order.
struct BvhNodeDev {
    float4 c0xy;  // child 0: lo.x, hi.x, lo.y, hi.y
    float4 c1xy;  // child 1
    float4 cz;    // lo0.z, hi0.z, lo1.z, hi1.z
    int32_t child0, child1;
    uint32_t _pad[2];
};
// The same tree collapsed to eight children per node, for traversal by GROUPS OF EIGHT LANES (geometry.cuh,
// bvh8_group_trace): lane k of a group fetches child k -- the group reads the 256-byte node as one coalesced
// request -- tests its box, and the group's votes pick the nearest.  A child is 32 bytes: its box (rounded outward,
// padded like the binary node's) and a code: >= 0 inner node, BVH8_EMPTY no child, otherwise a leaf with the
// binary tree's code ~((first << 3) | (count - 1)) (the leaves, hence bvh_tri48 / bvh_ids, are the binary tree's).
struct Bvh8Child {
    float lo[3], hi[3];
    int32_t code;
    uint32_t _pad;
};
struct Bvh8Node {
    Bvh8Child c[8];
};
constexpr int32_t BVH8_EMPTY = (int32_t)0x80000000;

// The four-wide form for ONE lane per ray (geometry.cuh, bvh4_intersect): a node holds the boxes of four children as
// six float4 (one per box plane, child k in component k), so the slab test of all four is 24 FMAs on whole vectors and a
// ray takes half as many dependent fetches as through the binary tree -- the node loop is latency bound (ncu:
// long_scoreboard on top at 5-6 active lanes).  Child codes as in Bvh8Node (>= 0 inner, BVH8_EMPTY none, else leaf).
#ifndef RPTB_BUILD_BVH4
#define RPTB_BUILD_BVH4 RPTB_BVH4  // the builder makes the four-wide tree only for a build that walks it (tests/hostemu sets it on its own)
#endif
struct __align__(16) Bvh4Node {
    float4 lox, hix, loy, hiy, loz, hiz;
    int4 code;
    int4 _pad;
};
#ifndef RPTB_BVH4
#define RPTB_BVH4 0  // 1: meshes with a BVH are traversed through the four-wide tree.  Measured slower than the binary tree on every mesh
                     // config at 8, 6 and 5 CTAs per SM (before the port to the H100): 0.45x the dependent fetches (tests/test_hostemu.py) but
                     // 24 slab FMAs + a sorting network per step whether one child is hit or four: the loop is bound by issue slots at 5-6
                     // active lanes, not by the fetch latency alone, so the binary tree stays the default.
#endif
constexpr int BVH8_STACK = 48;     // entries of a group's traversal stack in shared memory (overflow -> the ray falls back to the binary BVH)
constexpr int BVH4_STACK = 64;     // (code, entry t) pairs of the four-wide traversal; the builder drops the four-wide tree of a mesh too deep for it
constexpr int BVH_STACK = 96;      // traversal stack entries; the builder keeps the depth below it (bvhbuild.cpp)
constexpr int BVH_LEAF_MAX = 4;    // triangles per leaf (3 bits in the leaf code would allow 8)

template <class R>
struct MeshRec {
    const typename NodeOf<R>::type* nodes;
    const uint32_t* refs;
    const float4* tri48;  // f32 only (null for double)
    const float4* leaf_planes;  // f32, kd-tree meshes only: tri48[3*refs[k]] for every leaf ref k (planes in leaf order)
    const BvhNodeDev* bvh_nodes;  // f32, when the scene was created with the BVH (F_BVH): node 0 is the root
    const Bvh8Node* bvh8_nodes;   // the same tree, eight children per node (node 0 = root), for the lane-group traversal
    const Bvh4Node* bvh4_nodes;   // the same tree, four children per node: what one lane per ray traverses (RPTB_BVH4)
    const float4* bvh_tri48;      // tri48 permuted into BVH leaf order (a leaf's triangles are contiguous)
    const uint32_t* bvh_ids;      // original triangle index of each BVH-order triangle (normals, Hit::aux)
    const R* verts;       // 9 per triangle
    const R* norms;       // 9 per triangle
    R bmin[3], bmax[3];   // KdTree::bounds
    uint32_t ntris;
    uint32_t root_is_leaf;
    uint32_t small_tri_base;  // first triangle of this mesh in SmallTables::tri48 (one-leaf meshes, F_SMALL)
    uint32_t _pad;
};

template <class R>
struct ObjectRec {
    uint32_t kind, material, mesh /* MESH: mesh index; GROUP: group index */, has_transform;
    R inv[12];  // rows of inverse_transform (3x4): local = inv * (p,1)
    R nrm[9];   // rows of normal_transform M^-T (3x3)
    R fwd[12];  // rows of transform (3x4), for Transformed::sample
    R det;      // `scale` = det(linear)
    R plane_n[3];     // PLANE: normal.  MONOMIAL: plane_n[0] = exp
    R plane_v;        // PLANE: value.   MONOMIAL: height
    R plane_unit[3];  // normalize(plane normal), precomputed
    R _pad;
};

// KdTree<Box<dyn Bounded>> (src/kdtree.rs:99-104 over shapes): the tree's refs index `children`, each a
// Bounded shape with its own transform (a mesh child = one instance of meshes[child.mesh]).
template <class R>
struct GroupRec {
    const typename NodeOf<R>::type* nodes;
    const uint32_t* refs;
    const ObjectRec<R>* children;
    const float4* child_box;  // f32 only: (lo.xyz, hi.xyz) of every child in the group's space, widened -- see group_intersect
    R bmin[3], bmax[3];  // KdTree::bounds = merge of the children's bounding boxes
    uint32_t nchildren;
    uint32_t root_is_leaf;
};

template <class R>
struct MaterialRec {
    R color[3];
    R index, roughness, metallic, emittance;
    uint32_t transparent;
};

template <class R>
struct LightRec {
    uint32_t kind, _pad;
    R color[3];
    R vec[3];
    R radiance[3];  // OBJECT: material.color * material.emittance
    ObjectRec<R> object;
};

template <class R>
struct EnvRec {
    uint32_t kind, width, height, _pad;
    R color[3];
    const float4* texels_f4;  // f32: rgb + pad
    const double* texels_f64; // f64: packed rgb
};

// A small scene's warp-uniform tables, carried IN the kernel parameters (constant bank, up to 32 KB per
// launch on sm_90): every lane of a warp walks scene.objects / scene.lights in lock step and tests
// the same few triangles of one-leaf meshes, so these reads are uniform -- from parameter space they
// are constant-cache broadcasts that need no LSU slot, no L1 tag look-up and no address registers.
// Divergent accesses (the object / material of a lane's own hit) keep using the global copies.
constexpr int SMALL_OBJECTS = 16, SMALL_LIGHTS = 4, SMALL_MESHES = 16, SMALL_TRIS = 64;
template <class R>
struct SmallTables {};  // f64 parity gate: not used
template <>
struct SmallTables<float> {
    ObjectRec<float> objects[SMALL_OBJECTS];
    LightRec<float> lights[SMALL_LIGHTS];
    MeshRec<float> meshes[SMALL_MESHES];
    float4 tri48[3 * SMALL_TRIS];  // one-leaf meshes only; MeshRec::small_tri_base indexes it
};

// The packed primitive table (F_FLAT): what get_closest_hit walks for an f32 scene whose objects are all spheres, planes,
// cubes and one-leaf meshes (no kd-tree, BVH, group or monomial).  One record per object -- per coplanar triangle run
// for a mesh -- in object order, so that the first object wins ties exactly as in the scan over scene.objects:
//   header  int4 {kind | FLAT_TF if transformed, object index, k = triangles in the run, first triangle of the run}
//   FLAT_TF     3 words: the rows of inverse_transform
//   PLANE       1 word:  (normal, value)
//   MESH        1 word:  q0, the plane the run's k triangles share bitwise (one plane test for all of them);
//               k x 2 words: q1, q2 of each triangle (tri48 without its q0)
// Every word is read by the whole warp at once; a ray walks the table with no dependent ObjectRec -> MeshRec -> tri48 loads.
// Cornell's table is 38 words (608 B) against the ~2.2 KB of records and triangles the scan reads per ray.
enum : uint32_t { FLAT_TF = 0x100u };

template <class R>
struct SceneView {
    const ObjectRec<R>* objects;  // global copies (always valid)
    const LightRec<R>* lights;
    const MaterialRec<R>* materials;
    const MeshRec<R>* meshes;
    uint32_t nobjects, nlights, nmaterials, nmeshes;
    uint32_t tables_in_const;  // F_SMALL: `small` is filled
    uint32_t ngroups;
    const GroupRec<R>* groups;  // F_GROUP
    EnvRec<R> env;
    SmallTables<R> small;
    const float4* flat;   // F_FLAT (f32): the packed primitive table, read through L1
    uint32_t flat_words;  // its length in float4
};

// Camera with the per-render invariants hoisted (src/camera.rs:64-81 recomputes
// d, right per sample; the values are identical).
template <class R>
struct CameraRec {
    R eye[3], direction[3], up[3], right[3];
    R d;  // 1 / tan(fov / 2)
    R aperture, focal_distance;
};

struct DeviceCounters {
    unsigned long long segments, rays, node_visits, tri_tests, mesh_hits, env_lookups, object_tests;
    unsigned long long bvh_node_visits, bvh_tri_tests;  // the f32 path's own structure (F_BVH), counted when it is what was traversed
};

template <class R>
struct RenderArgs {
    CameraRec<R> cam;
    uint32_t width, height, iterations, max_bounces;
    R exposure_scale;  // 2^EV
    uint64_t seed, first_sample;
    uint32_t shard_index, shard_count;
    uint32_t tiles_x, tiles_y, ntiles_mine;
    R* out;  // width*height*3
    DeviceCounters* counters;
    // Sample chunks: the `iterations` samples of a pixel are cut into `nchunks` runs of `chunk`
    // samples; each run is summed sequentially into partial[(c * npix_slots + slot) * 3] (double)
    // and resolve adds the chunk sums in chunk order.  The cut depends on `iterations` only, so the
    // image is bit-identical however the work is spread: a thread takes `chunks_per_group`
    // consecutive chunks (grid = tiles x groups), and that number IS chosen per launch -- few groups
    // when the shard has many tiles (long runs, little tail), many when it has few.
    uint32_t nchunks, chunk, ngroups, chunks_per_group;
    double* partial;  // nchunks > 1 only
    // compact = 1: `out` holds ntiles_mine * 128 * 3 values in tile-major order (owned tile k, thread j of the
    // CTA -> out[(k * 128 + j) * 3]); nothing is written for other shards' pixels.  The multi-device handle
    // copies exactly its own pixels back this way (api.cu); 0 = the full row-major width * height * 3 image.
    uint32_t compact;
    uint32_t ks;  // sampled (non-ambient) lights of the scene: the vertex-at-once engine's shadow ray slots (integrator_vx.cuh)
};

// chunk = max(64, ceil(iterations / 32)) samples, so at most 32 chunks
inline void sample_chunks(uint32_t iterations, uint32_t& nchunks, uint32_t& chunk) {
    chunk = (iterations + 31u) / 32u;
    if (chunk < 64u) chunk = 64u;
    nchunks = (iterations + chunk - 1u) / chunk;
    if (nchunks < 1u) nchunks = 1u;
}
// groups so that tiles * groups is about 10 waves of resident CTAs (H100: 132 SMs x 8 CTAs): more CTAs
// shorten the grid's tail, longer runs per thread shorten the warp's.  The image does not depend on it.
inline void sample_groups(uint32_t ntiles, uint32_t nchunks, uint32_t& ngroups, uint32_t& chunks_per_group) {
    const uint32_t want = ntiles ? (10560u + ntiles - 1u) / ntiles : 1u;
    ngroups = want < 1u ? 1u : (want > nchunks ? nchunks : want);
    chunks_per_group = (nchunks + ngroups - 1u) / ngroups;
    ngroups = (nchunks + chunks_per_group - 1u) / chunks_per_group;
}

}  // namespace rptb
