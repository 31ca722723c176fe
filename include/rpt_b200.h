/*
 * rpt_b200.h -- C ABI of the H100-native path-tracing core that stands where
 * rpt's private `Renderer::sample` stands today.
 *
 * Every entry point cites the reference interface it replaces.  Citations are
 * relative to the reference checkout (ekzhang/rpt @ 815b21c):
 *
 *   Renderer::sample / get_color / trace_ray   src/renderer.rs:117-174
 *   Renderer::sample_lights / get_closest_hit  src/renderer.rs:177-220
 *   Scene / Object / Light / Environment       src/scene.rs:7-41, src/object.rs:10-32,
 *                                              src/light.rs:7-19, src/environment.rs:4-14,55-63
 *   Material                                   src/material.rs:7-26
 *   Camera                                     src/camera.rs:8-26
 *   KdTree<Triangle> (= Mesh)                  src/kdtree.rs:99-119,226-233, src/shape/mesh.rs:7-22,102
 *   Buffer::image / variance, color_bytes      src/buffer.rs:43-93, src/color.rs:17-23
 *
 * All structs are plain-old-data; all pointers are caller-owned host memory
 * unless the name says `_device`.  Values cross the boundary as `double`
 * because every quantity in the reference is `f64` (src/color.rs:2); the
 * library converts to its device layout (f32 SoA, or f64 for the parity gate)
 * inside rptb_scene_create.
 *
 * Error model: every function returning `int` returns RPTB_OK (0) or a
 * negative rptb_status; the message is available from rptb_last_error()
 * (thread-local).  Nothing unwinds or aborts across the boundary.  NaN/inf in
 * inputs are passed through -- the reference does not validate them either.
 *
 * Threading: a rptb_scene is immutable after creation (the reference shares
 * `&Scene` read-only across rayon workers, src/shape.rs:18 `Send + Sync`).
 * Render calls on one handle are serialised internally.
 */
#ifndef RPT_B200_H
#define RPT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RPTB_VERSION 100

typedef enum rptb_status {
    RPTB_OK = 0,
    RPTB_ERR_BAD_ARG = -1,   /* null pointer, out-of-range index, bad enum   */
    RPTB_ERR_CUDA = -2,      /* a CUDA runtime call failed (message has it)  */
    RPTB_ERR_NO_DEVICE = -3, /* no usable sm_90 device / extension missing   */
    RPTB_ERR_OOM = -4,       /* host or device allocation failed             */
    RPTB_ERR_UNSUPPORTED = -5
} rptb_status;

/* ---- Material: src/material.rs:7-26 (six fields, same meaning) ---------- */
typedef struct rptb_material {
    double color[3];
    double index;
    double roughness;
    double metallic;
    double emittance;
    uint32_t transparent; /* bool */
    uint32_t _pad;
} rptb_material;

/* ---- KdTree<Triangle>: src/kdtree.rs:99-104,226-233 ---------------------
 * The reference's pointer tree is serialised in depth-first pre-order.
 * kind 0/1/2 = SplitX/SplitY/SplitZ(split, left, right); kind 3 = Leaf whose
 * triangle indices are refs[first_ref .. first_ref+num_refs) in the order of
 * the reference's Vec<usize> (ascending triangle index, src/kdtree.rs:270-281).
 */
typedef struct rptb_kdnode {
    double split;
    uint32_t kind;
    uint32_t left;      /* node index of the left child  (kind 0..2) */
    uint32_t right;     /* node index of the right child (kind 0..2) */
    uint32_t first_ref; /* kind 3 */
    uint32_t num_refs;  /* kind 3 */
    uint32_t _pad;
} rptb_kdnode;

/* Mesh = KdTree<Triangle>; a triangle is 18 doubles v1,v2,v3,n1,n2,n3
 * (src/shape/mesh.rs:7-22).  If `nodes` is NULL the library builds the
 * reference-shaped tree itself (rptb_build_kdtree, src/kdtree.rs:235-355). */
typedef struct rptb_mesh {
    const double* tris;
    uint64_t ntris;
    const rptb_kdnode* nodes;
    uint64_t nnodes;
    const uint32_t* refs;
    uint64_t nrefs;
} rptb_mesh;

/* ---- Object { shape: Box<dyn Shape>, material }: src/object.rs:10-16 ----
 * The type-erased shape is made explicit.  `has_transform` distinguishes a
 * bare shape from Transformed<T> (src/shape.rs:99-137); `transform` is the
 * composed column-major 4x4 `Transformed::transform`.                        */
typedef enum rptb_shape_kind {
    RPTB_SHAPE_SPHERE = 0, /* src/shape/sphere.rs:13-64 */
    RPTB_SHAPE_PLANE = 1,  /* src/shape/plane.rs:17-32  */
    RPTB_SHAPE_CUBE = 2,   /* src/shape/cube.rs:20-87   */
    RPTB_SHAPE_MESH = 3,   /* src/kdtree.rs:129-143 + src/shape/mesh.rs:49-98 */
    RPTB_SHAPE_MONOMIAL = 4, /* MonomialSurface{height, exp}: src/shape/monomial_surface.rs:13-123 */
    RPTB_SHAPE_GROUP = 5   /* KdTree<Box<dyn Bounded>> over shapes: src/kdtree.rs:99-223 as used by
                              examples/fractal_spheres.rs:43-47 and examples/fractal_teapots.rs:53-59 */
} rptb_shape_kind;

typedef struct rptb_object {
    uint32_t kind;          /* rptb_shape_kind */
    uint32_t material;      /* index into rptb_scene_desc.materials */
    uint32_t mesh;          /* MESH: index into rptb_scene_desc.meshes; GROUP: index into .groups */
    uint32_t has_transform; /* 0 = bare shape, 1 = Transformed<T> */
    double transform[16];   /* column-major */
    double plane_normal[3]; /* PLANE only: x . normal = value */
    double plane_value;
    double monomial_height; /* MONOMIAL only: y = height * (x^2 + z^2)^(exp/2), x^2 + z^2 <= 1 */
    double monomial_exp;    /* MONOMIAL only; the reference's intersect/normal assume 4       */
} rptb_object;

/* ---- KdTree<T: Bounded> over whole shapes (two-level instancing) -----------
 * `children` are the tree's `objects` (src/kdtree.rs:100-104): Bounded shapes only -- SPHERE, CUBE,
 * MESH, MONOMIAL, bare or Transformed (Plane has no bounding box; a GROUP inside a GROUP is
 * RPTB_ERR_UNSUPPORTED).  Their `material` is ignored: the tree is ONE shape of ONE Object.  Many
 * children may name the same mesh (the reference shares it through Arc<Mesh>).  `nodes`/`refs` are
 * the tree serialised as in rptb_kdnode, refs = child indices; if `nodes` is NULL the library
 * builds it with the reference's `construct` over the children's bounding boxes
 * (Sphere [-1,1]^3, Cube [-.5,.5]^3, MonomialSurface (-1,0,-1)..(1,height,1), KdTree::bounds,
 * Transformed = box of the 8 transformed corners, src/shape.rs:153-175).                      */
typedef struct rptb_group {
    const struct rptb_object* children;
    uint64_t nchildren;
    const rptb_kdnode* nodes;
    uint64_t nnodes;
    const uint32_t* refs;
    uint64_t nrefs;
} rptb_group;

/* ---- Light: src/light.rs:7-19 -------------------------------------------- */
typedef enum rptb_light_kind {
    RPTB_LIGHT_POINT = 0,       /* Point(color, location)        */
    RPTB_LIGHT_AMBIENT = 1,     /* Ambient(color)                */
    RPTB_LIGHT_DIRECTIONAL = 2, /* Directional(color, direction) */
    RPTB_LIGHT_OBJECT = 3       /* Object(Object) -- invisible emitter */
} rptb_light_kind;

typedef struct rptb_light {
    uint32_t kind;
    uint32_t _pad;
    double color[3];
    double vec[3];      /* location (POINT) or direction (DIRECTIONAL) */
    rptb_object object; /* OBJECT only; its material holds colour/emittance */
} rptb_light;

/* ---- Environment: src/environment.rs:4-14,55-63 --------------------------- */
typedef enum rptb_env_kind { RPTB_ENV_COLOR = 0, RPTB_ENV_HDRI = 1 } rptb_env_kind;

typedef struct rptb_env {
    uint32_t kind;
    uint32_t width, height; /* HDRI */
    uint32_t _pad;
    double color[3];        /* COLOR */
    const double* texels;   /* HDRI: width*height*3, row-major, row 0 = +y pole */
} rptb_env;

/* How the f32 product path finds the closest triangle of a Mesh.  The closest hit of a ray does not depend
 * on it (up to which of two triangles wins an exact tie in t on a shared edge); the cost does.
 *   KDTREE  the reference-shaped KdTree<Triangle> (src/kdtree.rs:99-223), node for node -- what the f64
 *           parity gate, rptb_closest_hit with stats, and the traversal counters of rptb_stats always use
 *   BVH     a binary SAH BVH built by the library over the same triangles, each in exactly one leaf
 * AUTO = the library's default, BVH (environment variable RPTB_ACCEL=kdtree|bvh overrides it).         */
typedef enum rptb_accel { RPTB_ACCEL_AUTO = 0, RPTB_ACCEL_KDTREE = 1, RPTB_ACCEL_BVH = 2 } rptb_accel;

/* ---- Scene: src/scene.rs:7-18 ---------------------------------------------- */
typedef struct rptb_scene_desc {
    const rptb_material* materials;
    uint32_t nmaterials;
    const rptb_mesh* meshes;
    uint32_t nmeshes;
    const rptb_object* objects; /* scene.objects, in order */
    uint32_t nobjects;
    const rptb_light* lights;   /* scene.lights, in order */
    uint32_t nlights;
    rptb_env environment;
    const rptb_group* groups;   /* targets of GROUP objects (may be NULL when ngroups == 0) */
    uint32_t ngroups;
    uint32_t accel;             /* rptb_accel: what the f32 path traverses meshes with */
} rptb_scene_desc;

/* ---- Camera: src/camera.rs:8-26 (same six fields) -------------------------- */
typedef struct rptb_camera {
    double eye[3];
    double direction[3];
    double up[3];
    double fov;
    double aperture;
    double focal_distance;
} rptb_camera;

/* ---- Renderer parameters: src/renderer.rs:18-57 ----------------------------
 * width/height/max_bounces/exposure_value are the builder fields; `iterations`
 * is the argument of Renderer::sample.  The reference seeds every row from OS
 * entropy (src/renderer.rs:121); here the stream is Philox4x32-10 keyed by
 * (seed, pixel, first_sample + i), so iterative_render passes an advancing
 * first_sample to get the disjoint streams fresh entropy gave it.            */
typedef enum rptb_precision {
    RPTB_PRECISION_F32 = 0, /* the product path */
    RPTB_PRECISION_F64 = 1  /* parity gate: literal f64 semantics, no ray offsets */
} rptb_precision;

/* How the integrator is scheduled on the device (results agree to f32 rounding):
 *   MEGAKERNEL  one thread per pixel, whole path in registers -- best when rays are cheap
 *               (analytic shapes, tiny meshes: sphere, cornell, glass)
 *   WAVEFRONT   path state in HBM, a shade kernel and a persistent trace kernel per path
 *               vertex -- best when kd-tree traversal dominates (teapot, dragon)
 * AUTO picks WAVEFRONT iff the scene was created with RPTB_ACCEL_KDTREE and its kd-trees hold >= 50 000
 * nodes (with the BVH the megakernel wins on every scene measured); f32 only -- the f64 parity gate always
 * runs the megakernel.                                                                  */
typedef enum rptb_engine { RPTB_ENGINE_AUTO = 0, RPTB_ENGINE_MEGAKERNEL = 1, RPTB_ENGINE_WAVEFRONT = 2 } rptb_engine;

typedef struct rptb_render_params {
    uint32_t width;
    uint32_t height;
    uint32_t iterations;
    uint32_t max_bounces;
    double exposure_value;
    uint64_t seed;
    uint64_t first_sample;
    uint32_t shard_index; /* this process renders pixel tiles t with      */
    uint32_t shard_count; /* t % shard_count == shard_index; others stay 0 */
    uint32_t precision;   /* rptb_precision */
    uint32_t collect_stats; /* 0 = segments / rays only; 1 = + traversal counters of the structure that rendered the image
                               (the f32 path's BVH -> bvh_node_visits / bvh_tri_tests; a kd-tree scene or the f64 gate ->
                               node_visits / tri_tests); 2 = a counting pass over the reference-shaped kd-trees whatever
                               the scene was created with (SURVEY 8d's algorithmic work) */
    uint32_t engine;      /* rptb_engine: 0 = pick by scene                   */
    uint32_t compact_out; /* rptb_render_samples_device only.  0 = out is the full row-major width*height*3 image, other
                             shards' pixels written as zero.  1 = out holds ONLY this shard's tiles, tile-major: owned tile
                             k (= tile shard_index + k*shard_count, tiles are 16x8 pixels numbered row-major) occupies
                             out[k*384 .. k*384+384), pixel j of the tile at (x0 + (j>>5&1)*8 + (j&7), y0 + (j>>6)*4 + (j>>3&3))
                             -- 1/shard_count of the bytes, so a multi-GPU host all-gathers shards instead of all-reducing
                             full images (rptb_tile_pixel gives the mapping)                                             */
} rptb_render_params;

typedef struct rptb_stats {
    uint64_t segments;    /* trace_ray invocations (src/renderer.rs:145)       */
    uint64_t rays;        /* get_closest_hit calls incl. shadow rays (:211)    */
    uint64_t node_visits; /* kd nodes visited (src/kdtree.rs:151) and Triangle::intersect calls (mesh.rs:49) on the      */
    uint64_t tri_tests;   /* reference-shaped trees, when those were walked (collect_stats above)                         */
    uint64_t mesh_hits;   /* closest hits that landed on a mesh                */
    uint64_t env_lookups; /* escaped paths that sampled an HDRI                */
    uint64_t object_tests;/* Shape::intersect dispatches (objects tested per ray, summed) */
    double gpu_ms;        /* device time of the render launch(es)              */
    uint32_t launches;    /* kernels launched by the call                      */
    uint32_t engine;      /* rptb_engine that rendered the call (1 or 2)       */
    uint64_t bvh_node_visits; /* 64-byte two-box nodes of the f32 path's BVH fetched, and triangles (48 B + 4 B id) tested  */
    uint64_t bvh_tri_tests;   /* in its leaves -- what the product path actually read when the scene has a BVH              */
} rptb_stats;

typedef struct rptb_scene rptb_scene; /* opaque */

/* Thread-local message of the last failing call. */
const char* rptb_last_error(void);

/* Library/device info: returns the CUDA device count (>=0) or a negative status. */
int rptb_device_count(void);

/* Replaces: construction of the borrowed `&Scene` the renderer walks
 * (src/renderer.rs:20, src/scene.rs:7-18).  Copies everything to `device`. */
int rptb_scene_create(const rptb_scene_desc* desc, int device, rptb_scene** out);
/* The same scene replicated on `ndevices` GPUs (devices[i], or 0..ndevices-1 when `devices` is NULL): flattened
 * once, uploaded once per device.  Replaces: the fan-out inside Renderer::sample (src/renderer.rs:117-129, rayon
 * over rows) -- rptb_render_samples on such a handle runs one host thread per GPU, GPU i renders the 16x8-pixel
 * tiles t with t % ndevices == i and copies exactly its own pixels into the caller's image, so there is nothing to
 * reduce and the image is bit-identical for any ndevices.  rptb_render_samples_device, rptb_closest_hit and
 * rptb_illuminate on it address replica 0 (the first is RPTB_ERR_UNSUPPORTED when ndevices > 1).          */
int rptb_scene_create_multi(const rptb_scene_desc* desc, const int* devices, int ndevices, rptb_scene** out);
int rptb_scene_device_count(const rptb_scene* scene);
void rptb_scene_destroy(rptb_scene* scene);
/* Bytes of flattened scene resident on the device (f32 layout). */
uint64_t rptb_scene_device_bytes(const rptb_scene* scene);

/* Replaces: Renderer::sample's `colors: Vec<Color>` (src/renderer.rs:117-129).
 * Writes width*height*3 doubles, row-major y*width+x, y = 0 top row: the mean
 * of `iterations` path samples per pixel times 2^exposure_value (:131-142).  */
int rptb_render_samples(rptb_scene* scene, const rptb_camera* camera,
                        const rptb_render_params* params, double* out_rgb,
                        rptb_stats* stats /* nullable */);

/* Same computation, result left in device memory as float[width*height*3] on
 * CUDA stream `stream` (a cudaStream_t; NULL = the library's own stream, and
 * the call then synchronises).  Used by multi-GPU hosts that all-reduce the
 * buffer with NCCL, and by bench.py's device-resident timing.  Pixels of
 * other shards are written as zero.                                          */
int rptb_render_samples_device(rptb_scene* scene, const rptb_camera* camera,
                               const rptb_render_params* params, float* out_rgb_device,
                               void* stream, rptb_stats* stats /* nullable, forces sync */);

/* Pixel index (y*width + x) of element j (0..127) of the k-th tile owned by shard_index of shard_count, or -1 when
 * that element lies outside a ragged image edge: the layout of compact_out = 1 and of the tile ownership of every
 * sharded render.  Host side.                                                                              */
int64_t rptb_tile_pixel(uint32_t width, uint32_t height, uint32_t shard_index, uint32_t shard_count, uint32_t k, uint32_t j);

/* Replaces: Renderer::get_closest_hit (src/renderer.rs:211-220) for `n` world
 * rays (n x 6 doubles: origin, dir).  out_t[i] = +inf and out_object[i] = -1
 * on a miss; out_normal is n x 3.  precision as in rptb_precision.           */
int rptb_closest_hit(rptb_scene* scene, const double* rays, uint64_t n, double t_min,
                     uint32_t precision, double* out_t, int32_t* out_object,
                     double* out_normal /* nullable */, rptb_stats* stats /* nullable */);

/* Point-wise Material::bsdf (src/material.rs:125-210) on the device:
 * `dirs` is n x 9 doubles (n, wo, wi); out is n x 3.                         */
int rptb_bsdf_eval(const rptb_material* material, const double* dirs, uint64_t n,
                   uint32_t precision, int device, double* out);

/* Material::sample_f (src/material.rs:224-313) on the device: `dirs` is n x 6
 * (n, wo); draw i uses Philox key (seed, i).  out_wi n x 3, out_pdf n;
 * pdf = -1 encodes `None`.                                                    */
int rptb_sample_f(const rptb_material* material, const double* dirs, uint64_t n, uint64_t seed,
                  uint32_t precision, int device, double* out_wi, double* out_pdf);

/* Point-wise Light::illuminate (src/light.rs:23-47) of scene.lights[light] at n world positions (n x 3
 * doubles), Shape::sample of an Object light included (src/shape/sphere.rs:52-64, src/shape.rs:139-150,
 * src/kdtree.rs:138-143, src/shape/mesh.rs:84-98, src/shape/cube.rs:74-87); draw i uses Philox key (seed, i).
 * out_intensity n x 3, out_wi n x 3 (direction to the light), out_dist n.                                   */
int rptb_illuminate(rptb_scene* scene, uint32_t light, const double* pos, uint64_t n, uint64_t seed,
                    uint32_t precision, double* out_intensity, double* out_wi, double* out_dist);

/* Replaces: KdTree::new -> construct (src/kdtree.rs:108-119,235-355).  Host
 * side; produces the reference-shaped tree for hosts that cannot hand theirs
 * over.  Free with rptb_free_kdtree.                                          */
typedef struct rptb_kdtree_out {
    rptb_kdnode* nodes;
    uint64_t nnodes;
    uint32_t* refs;
    uint64_t nrefs;
    uint32_t depth;
    uint32_t max_leaf;
} rptb_kdtree_out;
int rptb_build_kdtree(const double* tris, uint64_t ntris, rptb_kdtree_out* out);
/* The same `construct`, over arbitrary bounding boxes (6 doubles each: p_min, p_max): the tree of a
 * KdTree<Box<dyn Bounded>> (rptb_group).  Host side.                                          */
int rptb_build_kdtree_boxes(const double* boxes, uint64_t nboxes, rptb_kdtree_out* out);
void rptb_free_kdtree(rptb_kdtree_out* out);

/* Replaces: load_obj -> parse_obj_point / parse_obj_face (src/io.rs:27-73,151-200) on an in-memory
 * .OBJ text.  *out_tris receives ntris x 18 doubles (v1 v2 v3 n1 n2 n3), the input Mesh::new takes;
 * free with rptb_free_triangles.  Host side.                                              */
int rptb_parse_obj(const char* text, uint64_t len, double** out_tris, uint64_t* out_ntris);
void rptb_free_triangles(double* tris);

/* Replaces: load_obj_with_mtl + load_mtl (src/io.rs:83-149,202-258) on in-memory .OBJ and .MTL
 * texts.  The reference returns Vec<Object>, one Mesh per run of faces between `usemtl` switches;
 * here all triangles come back in file order (18 doubles each) and groups[g] names the run
 * [first_tri, first_tri + ntris) with the Material load_mtl derived for it (Material::default(),
 * src/material.rs:28-32, before the first `usemtl`).  Free with rptb_free_obj_groups.  Host side. */
typedef struct rptb_obj_group {
    rptb_material material;
    uint64_t first_tri;
    uint64_t ntris;
} rptb_obj_group;
typedef struct rptb_obj_groups_out {
    double* tris;
    uint64_t ntris;
    rptb_obj_group* groups;
    uint64_t ngroups;
} rptb_obj_groups_out;
int rptb_parse_obj_mtl(const char* obj_text, uint64_t obj_len, const char* mtl_text, uint64_t mtl_len,
                       rptb_obj_groups_out* out);
void rptb_free_obj_groups(rptb_obj_groups_out* out);

/* Replaces: load_stl -> load_stl_ascii / load_stl_binary (src/io.rs:260-360) on the bytes of an .STL
 * file: binary when len == 84 + 50 n (n = the u32 at byte 80), else ASCII when it starts with
 * "solid ".  Each facet's stored normal is used for all three corners, unnormalised, as the
 * reference does.  Unlike the reference's ASCII loop, a closing `endsolid` line is accepted.
 * Free with rptb_free_triangles.  Host side.                                              */
int rptb_parse_stl(const void* data, uint64_t len, double** out_tris, uint64_t* out_ntris);

/* Replaces: Buffer::variance (src/buffer.rs:59-73) for nbatches >= 2 equally weighted entries per
 * pixel: batches = nbatches x npixels x 3 doubles; the mean over pixels of the per-pixel sample
 * variance (n - 1 degrees of freedom) of the entries, summed over the three channels.   */
int rptb_film_variance(const double* batches, uint32_t nbatches, uint64_t npixels, int device, double* out);

/* Replaces: Buffer::image -> get_filtered_color -> color_bytes
 * (src/buffer.rs:43-56,75-93, src/color.rs:17-23) for a buffer holding
 * `nbatches` equally weighted entries per pixel (sums[] = per-pixel sum over
 * the entries, width*height*3 doubles).  out_rgb8 = width*height*3 bytes.    */
int rptb_film_resolve(const double* sums, uint32_t nbatches, uint32_t width, uint32_t height,
                      uint32_t box_radius, int device, uint8_t* out_rgb8);

#ifdef __cplusplus
}
#endif
#endif /* RPT_B200_H */
