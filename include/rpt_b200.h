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
 *   Buffer (device-resident) / add_samples     src/buffer.rs:6-40
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
 * rptb_illuminate on it address replica 0 (the first is RPTB_ERR_UNSUPPORTED when ndevices > 1).  A device listed
 * twice is RPTB_ERR_BAD_ARG unless the environment has RPTB_ALLOW_REPEATED_DEVICES=1 (a testing switch, read on
 * every call): then each listing is a replica of its own, as a distinct GPU would be, which is no faster.    */
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

/* ---- Buffer on the device: src/buffer.rs:6-93 -------------------------------------------------------------
 * Replaces: Buffer::new(width, height, Filter::Box(box_radius)) (src/buffer.rs:17-29), kept in device memory on
 * every replica of `scene`: per pixel the running sum of its entries in double, added in entry order (the
 * sequential sum np.sum(batches, axis=0) computes, bit for bit), and one streaming (Welford) M2 summed over the
 * three channels.  Replica i of n holds the 16x8 tiles t with t % n == i.  image / variance / sums gather the
 * replicas on the first device and cost O(width*height) however many entries were added; their results are the
 * same bits for any device count.  The buffer owns its memory: it and its scene may be destroyed in either order.
 * A buffer is used from one thread at a time (calls on it are serialised internally).                        */
typedef struct rptb_buffer rptb_buffer; /* opaque */
int rptb_buffer_create(rptb_scene* scene, uint32_t width, uint32_t height, uint32_t box_radius, rptb_buffer** out);
void rptb_buffer_destroy(rptb_buffer* buffer);
/* Replaces: Renderer::sample(iterations, &mut Buffer) (src/renderer.rs:117-129): renders params->iterations samples
 * and adds ONE entry per pixel -- the mean times 2^exposure_value, exactly what rptb_render_samples writes (the
 * f32 path's float widened to double) -- to `buffer`, on the device.  The render is not copied to the host; with
 * stats == NULL the call returns once the work is enqueued.  width/height must be the buffer's and `scene` must have
 * the device list of the scene the buffer was created on (else RPTB_ERR_BAD_ARG); shard_count > 1 is
 * RPTB_ERR_UNSUPPORTED on a whole buffer, and a shard buffer (rptb_buffer_create_shard) takes exactly its own
 * shard_index / shard_count (else RPTB_ERR_BAD_ARG); compact_out is ignored.                                  */
int rptb_sample_into(rptb_scene* scene, const rptb_camera* camera, const rptb_render_params* params,
                     rptb_buffer* buffer, rptb_stats* stats /* nullable, forces sync */);
/* Replaces: Buffer::add_samples (src/buffer.rs:32-40) of a host entry: width*height*3 doubles, row-major.      */
int rptb_buffer_add_samples(rptb_buffer* buffer, const double* rgb);
/* Replaces: Buffer::image (src/buffer.rs:43-56,75-93): width*height*3 bytes, the bytes rptb_film_resolve gives
 * for the same sums.  No entry yet: RPTB_ERR_BAD_ARG, "Pixel found with no samples" (src/buffer.rs:89).       */
int rptb_buffer_image(rptb_buffer* buffer, uint8_t* out_rgb8);
/* Replaces: Buffer::variance (src/buffer.rs:59-73): the mean over pixels of M2 / (entries - 1), reduced in a
 * fixed order.  NaN with fewer than two entries, as in the reference.                                        */
int rptb_buffer_variance(rptb_buffer* buffer, double* out);
/* The per-pixel sums (width*height*3 doubles, row-major) and the entry count (out_entries nullable): the largest
 * per-pixel count, which is every pixel's count in a buffer that never had an adaptive call.               */
int rptb_buffer_sums(rptb_buffer* buffer, double* out_sums, uint32_t* out_entries);

/* ---- Adaptive sampling on the device Buffer ---------------------------------------------------------------
 * The reference's Buffer keeps one list of entries per pixel (src/buffer.rs:24-29), so its pixels may hold
 * different numbers of entries: image() divides each window's sum by the entries in the window and variance()
 * each pixel's M2 by its own count - 1 (:59-93).  rptb_sample_into_adaptive adds an entry only to the pixels
 * that have not converged.  A pixel with n entries, sums S_c and M2 is active iff
 *     n < min_entries   or   NOT( M2 / ((n-1)*n*3) <= (rel_tol * (S_0+S_1+S_2)/(3n) + abs_tol)^2 ),
 * evaluated in double with every operation rounded on its own, in the order rpt_b200/csrc/adaptive.h documents:
 * the channel-mean variance of the pixel's mean against a relative-plus-absolute tolerance.  A NaN statistic
 * compares false and keeps the pixel active.  The decision is a pure function of the pixel's state, taken
 * before each render: the first call renders every pixel, a skipped pixel stays skipped under the same
 * criterion, and a changed criterion simply re-decides.  min_entries must be >= 2 and both tolerances finite
 * and >= 0 (else RPTB_ERR_BAD_ARG).
 * Known bias of variance-based stopping: a dark pixel whose first min_entries entries happen to agree stops
 * early.  min_entries and abs_tol are the guards.                                                            */
typedef struct rptb_adaptive {
    double rel_tol;
    double abs_tol;
    uint32_t min_entries;
    uint32_t _pad;
} rptb_adaptive;
/* Renders one entry of params->iterations samples for every ACTIVE pixel and adds it to `buffer`; inactive
 * pixels' sums, M2 and counts do not change.  An active pixel draws exactly the samples rptb_sample_into
 * would give it (Philox key (seed, pixel, first_sample + i)), so its entry is that call's entry for it.
 * Argument checks as rptb_sample_into; engine == RPTB_ENGINE_WAVEFRONT is RPTB_ERR_UNSUPPORTED: AUTO and
 * MEGAKERNEL are the slot megakernel (RPTB_VX is ignored), scheduled over the active 8x4 warp blocks only.
 * collect_stats 0, 1 and 2 are all supported.  out_active (nullable) receives the number of pixels that got
 * this entry.  With out_active and stats both NULL the call returns once the work is enqueued.  Once a buffer
 * has had an adaptive call, rptb_sample_into and rptb_buffer_add_samples keep adding one entry to every pixel
 * (Buffer::add_samples), on top of each pixel's own count.                                                   */
int rptb_sample_into_adaptive(rptb_scene* scene, const rptb_camera* camera, const rptb_render_params* params,
                              const rptb_adaptive* criterion, rptb_buffer* buffer,
                              uint64_t* out_active /* nullable, forces sync */, rptb_stats* stats /* nullable, forces sync */);
/* Per-pixel state, row-major, each pointer nullable: sums (width*height*3), M2 (width*height, summed over the
 * channels) and entry counts (width*height).                                                                 */
int rptb_buffer_pixel_stats(rptb_buffer* buffer, double* sums, double* m2, uint32_t* counts);

/* ---- Denoising the device Buffer ---------------------------------------------------------------------------
 * Not in the reference, which has one filter, Filter::Box(radius) (src/buffer.rs:75-108): it averages a square
 * window and blurs silhouettes and shadow edges as much as noise.  These stand beside it: a first-hit feature
 * pass, and the spatial part of SVGF (Schied et al., HPG 2017), an edge-avoiding a-trous wavelet filter
 * (Dammertz et al., HPG 2010) guided by the features and by each pixel's variance of the mean -- the statistic
 * rptb_adaptive tests.  Temporal reprojection across camera moves: rptb_buffer_reproject.
 *
 * Adds, for every pixel and every sample i in [first_sample, first_sample + iterations), the first hit of the
 * render's camera ray for Philox key (seed, pixel, i) -- the same draws in the same order, tmin 1e-12, in
 * params->precision -- to per-pixel double sums kept in the buffer: on a hit, the hit count, the shading normal
 * turned to face the ray, the distance t and the material's colour; on a miss, only the ray count.  The sums are
 * added in sample order; features may be added before, between or after entries and never touch them.  Argument
 * checks as rptb_sample_into.  The results are the same bits for any device count.  stats (nullable, forces
 * sync): rays, gpu_ms, launches.                                                                             */
int rptb_buffer_add_features(rptb_scene* scene, const rptb_camera* camera, const rptb_render_params* params,
                             rptb_buffer* buffer, rptb_stats* stats /* nullable, forces sync */);
/* The resolved features (AOVs), row-major, each pointer nullable: normal (width*height*3) = the normalised sum of
 * the hit normals, 0 where nothing was hit; depth (width*height) = the mean hit distance, +inf where nothing was
 * hit; albedo (width*height*3) = the mean material colour over all rays, a miss counting 1 (it sees the
 * environment); hit_fraction (width*height) = hits / rays.  No features yet: RPTB_ERR_BAD_ARG.              */
int rptb_buffer_features(rptb_buffer* buffer, double* normal, double* depth, double* albedo, double* hit_fraction);
/* The filter's parameters (rpt_b200/csrc/denoise.h gives every formula and its order of operations).
 * iterations: a-trous passes with steps 1, 2, 4, ... (0 = the mean itself, <= 12); sigma_normal: the exponent of
 * the normal weight; sigma_depth, sigma_luminance: the depth and luminance tolerances (finite, >= 0); albedo_eps:
 * added to the albedo before the colour is divided by it, finite and > 0 -- a pixel whose feature rays all hit a black
 * material has albedo 0, and with albedo_eps 0 its colour would be divided by 0 and come back NaN.  A positive
 * albedo_eps keeps every colour finite while mean / albedo_eps stays within the double range: a mean of 1e6 overflows
 * below albedo_eps ~ 1e-303.  Defaults 5, 128, 1, 4, 1e-3.                                                     */
typedef struct rptb_denoise {
    uint32_t iterations;
    uint32_t sigma_normal;
    double sigma_depth;
    double sigma_luminance;
    double albedo_eps;
} rptb_denoise;
/* Denoises the buffer's mean image on its first device, each pixel with its own entry count (adaptive buffers
 * included): out_rgb (nullable) = width*height*3 linear doubles; out_rgb8 (nullable) = their bytes through the
 * film resolve of Buffer::image with one entry and radius 0 (clamp, gamma 1/2.2, truncation) -- the buffer's box
 * radius does not apply to a denoised image.  RPTB_ERR_BAD_ARG: no entries ("Pixel found with no samples"), a
 * pixel with fewer than 2 entries (no variance), no features, iterations > 12, a sigma that is negative or not
 * finite, or an albedo_eps that is not finite and > 0.                                                        */
int rptb_buffer_denoise(rptb_buffer* buffer, const rptb_denoise* params, double* out_rgb /* nullable */,
                        uint8_t* out_rgb8 /* nullable */);
/* Stands beside rptb_buffer_denoise: the variance v' of each pixel's denoised value, the filter's own estimate carried
 * through its passes, v'_p = sum w^2 v_q / (sum w)^2 (rpt_b200/csrc/denoise.h) -- a per-pixel error map of the denoised
 * image, in the filter's radiance units.  With iterations == 0 it is each pixel's variance of the mean,
 * M2 / ((n-1) n 3).  The passes treat their inputs as independent, so after the first pass v' underestimates the true
 * variance (DESIGN.md section 6e measures by how much).  out_var: width*height doubles, row-major.  Refusals as
 * rptb_buffer_denoise.                                                                                        */
int rptb_buffer_denoise_variance(rptb_buffer* buffer, const rptb_denoise* params, double* out_var);

/* ---- Adaptive sampling guided by the denoiser --------------------------------------------------------------
 * Stands beside rptb_sample_into_adaptive: the same entry for the active pixels, but the test looks at the value the
 * denoiser will show instead of the raw mean.  Before rendering, the filter of rptb_buffer_denoise runs with `guide`
 * over the buffer, and a pixel with n entries is active iff
 *     n < min_entries   or   NOT( v' <= (rel_tol * m' + abs_tol)^2 ),
 * where c' is the pixel's denoised colour (rptb_buffer_denoise's output, bit for bit), m' = ((c'_0 + c'_1) + c'_2) / 3
 * and v' its variance after the last pass (rptb_buffer_denoise_variance), every operation a double rounded on its own
 * in the order rpt_b200/csrc/guided.h documents.  So flat regions, which the filter averages over many neighbours,
 * stop early, and pixels at edges, which it leaves almost alone, render on.  A pixel with 0 or 1 entries (after a
 * reprojection) has a NaN v' and stays active; it gives its neighbours no weight.  The decision is a pure function of
 * the gathered state: the same bits for any device count.
 * guide->iterations == 0 is rptb_sample_into_adaptive exactly and needs no features.  While no pixel can hold
 * min_entries (the buffer has had fewer calls), every pixel is active, and the filter is skipped (stats->launches
 * shows it).  The filter runs on the buffer's first device; only each other part's mask and flags (132 bytes a 16x8
 * tile) go to that part's device.  stats->gpu_ms times each part's select, render and accumulate, as
 * rptb_sample_into_adaptive's does; stats->launches counts the filter's kernels too.
 * RPTB_ERR_BAD_ARG: as rptb_sample_into_adaptive, as rptb_denoise's parameters in rptb_buffer_denoise, and, when
 * guide->iterations > 0, a buffer with no features, features not made through exactly `camera`, or entries made
 * through another camera, through several, or from the host (rptb_buffer_add_samples); a reprojected buffer's
 * entries count as its feature camera's.  RPTB_ERR_UNSUPPORTED: a shard buffer (gather the shards first), and the
 * wavefront engine.  out_active and stats as rptb_sample_into_adaptive.                                        */
int rptb_sample_into_guided(rptb_scene* scene, const rptb_camera* camera, const rptb_render_params* params,
                            const rptb_adaptive* criterion, const rptb_denoise* guide, rptb_buffer* buffer,
                            uint64_t* out_active /* nullable, forces sync */, rptb_stats* stats /* nullable, forces sync */);

/* ---- The denoised image's error from two half buffers ------------------------------------------------------
 * v' (rptb_buffer_denoise_variance) treats each pass's inputs as independent and underestimates the variance of the
 * denoised value.  A buffer with halves keeps one more plane, HALF: the sums of each pixel's odd entries (entry k,
 * k the pixel's count before the add, for odd k) -- 24 more bytes a pixel.  Every way an entry arrives (rptb_sample_into,
 * the adaptive and guided calls, rptb_buffer_add_samples) follows the rule, and everything else a buffer returns is
 * the same bits as a plain buffer's given the same calls, for any device count.
 * The filter runs over the scaled difference of the two halves' means with the weights it computes from the whole
 * buffer, and the square of the result, remodulated, averaged over the channels and smoothed over 3x3, is E: an
 * estimate of each pixel's variance of the denoised value that accounts for the correlation between passes.
 * rpt_b200/csrc/halves.h gives every formula and its order of operations.
 * A buffer with halves may be a reprojection's or merge's src or dst.  A dst with halves needs a src with halves
 * (RPTB_ERR_UNSUPPORTED from a plain src: its history has no halves), and then takes the history's HALF too (see
 * rptb_buffer_reproject).  It imports the blocks of shards with halves (rptb_buffer_create_shard_halves), whose
 * exchange blocks carry HALF, and only those.
 * Arguments and refusals of create as rptb_buffer_create.                                                      */
int rptb_buffer_create_halves(rptb_scene* scene, uint32_t width, uint32_t height, uint32_t box_radius, rptb_buffer** out);
/* The HALF plane: width*height*3 doubles, row-major.  RPTB_ERR_BAD_ARG: a buffer without halves;
 * RPTB_ERR_UNSUPPORTED: a shard buffer (gather the shards first).                                              */
int rptb_buffer_half_sums(rptb_buffer* buffer, double* out);
/* E, the error estimate of rptb_buffer_denoise(params)'s output, in the units of v': width*height doubles, row-major.
 * A pixel with fewer than 2 entries in either half's sense (n_B = 0) gives no difference and no weight; where no
 * finite tap is left, E is NaN.  Refusals as rptb_buffer_denoise, and RPTB_ERR_BAD_ARG: a buffer without halves,
 * params->iterations == 0 (there is no filter to estimate).                                                  */
int rptb_buffer_denoise_error(rptb_buffer* buffer, const rptb_denoise* params, double* out);
/* rptb_sample_into_guided with E in place of v': a pixel with n entries is active iff
 *     n < min_entries   or   NOT( E <= (rel_tol * m' + abs_tol)^2 ),
 * m' as in rptb_sample_into_guided.  The same flow, checks, refusals, plain mark while no pixel can hold min_entries,
 * out_active and stats.  Besides: RPTB_ERR_BAD_ARG: a buffer without halves, guide->iterations == 0;
 * RPTB_ERR_UNSUPPORTED: a shard buffer (rptb_sample_into_guided_error_shard takes it), the wavefront engine.      */
int rptb_sample_into_guided_error(rptb_scene* scene, const rptb_camera* camera, const rptb_render_params* params,
                                  const rptb_adaptive* criterion, const rptb_denoise* guide, rptb_buffer* buffer,
                                  uint64_t* out_active /* nullable, forces sync */, rptb_stats* stats /* nullable, forces sync */);
/* rptb_buffer_denoise with each pixel's number of passes chosen from a half-buffer estimate of each level's error.
 * Level k (0 .. params->iterations) is rptb_buffer_denoise's output with iterations = k.  Per pixel, m_k estimates
 * the squared error of level k (bias included) from the two halves, M_k smooths it over 5x5, and the level with the
 * least M_k is kept (level 0 unless a deeper one is strictly less); select.h gives every formula.  So every output pixel
 * is rptb_buffer_denoise(iterations = level) at that pixel, bit for bit.  out_rgb: width*height*3 doubles;
 * out_rgb8: its bytes as rptb_buffer_denoise writes them; out_level: width*height chosen levels; out_mse:
 * width*height M at the chosen level, in the units of v' (NaN where no finite tap was left).  Refusals as
 * rptb_buffer_denoise_error.  Allocates 9 doubles and 1 byte a pixel on first use (151 MB at 1920x1080), beside the
 * error estimate's.                                                                                          */
int rptb_buffer_denoise_select(rptb_buffer* buffer, const rptb_denoise* params, double* out_rgb /* nullable */,
                               uint8_t* out_rgb8 /* nullable */, uint8_t* out_level /* nullable */, double* out_mse /* nullable */);
/* A buffer with halves, denoised by cross-filtering with a smoothed selection map.  Each half is filtered through
 * params->iterations passes whose weights come from the other half's own chain of passes (not from its own entries),
 * giving level k = 0 .. iterations: level 0 is S / n, level k the count-weighted mean of the two cross-filtered halves,
 * remodulated.  Per pixel, m_k estimates the squared error of level k (bias included) from the halves, M_k smooths it
 * over 5x5, k* is the level with the least M_k (level 0 unless a deeper one is strictly less), and the output blends
 * the levels by the 5x5-smoothed share of each level among its neighbours' k*; a pixel whose 5x5 neighbourhood chose one
 * level gets that level bit for bit.  cross.h gives every formula.  out_rgb: width*height*3 doubles; out_rgb8: its bytes
 * as rptb_buffer_denoise writes them; out_level: width*height k*; out_mse: width*height M^, the blend of M_k with the
 * colour's weights, in the units of v' (NaN where a blended level had no finite tap).  Refusals as
 * rptb_buffer_denoise_select: RPTB_ERR_BAD_ARG for a buffer without halves or features, iterations == 0, or a pixel with
 * fewer than 2 entries; RPTB_ERR_UNSUPPORTED for a shard (gather it first).  Allocates 23 doubles and 1 byte a pixel on
 * first use (384 MB at 1920x1080), beside the error estimate's.                                                  */
int rptb_buffer_denoise_cross(rptb_buffer* buffer, const rptb_denoise* params, double* out_rgb /* nullable */,
                              uint8_t* out_rgb8 /* nullable */, uint8_t* out_level /* nullable */, double* out_mse /* nullable */);

/* ---- Reprojecting the device Buffer across a camera move ---------------------------------------------------
 * The temporal half of SVGF for a static scene: each pixel of `dst`'s view finds, through its own first-hit depth,
 * the world point it sees, projects it into `src`'s view and takes the history of the (up to four, bilinear) src
 * pixels there whose depth, normal and hit fraction agree with it -- their mean, their per-entry variance and at
 * most max_history entries.  A pixel with no consistent history (a disocclusion, the edge of the old view) gets
 * count 0, and an adaptive call renders it first.  rpt_b200/csrc/reproject.h gives every formula and its order of
 * operations.
 *
 * A buffer records the camera its entries were rendered through (rptb_sample_into, rptb_sample_into_adaptive) and
 * the camera of its features (rptb_buffer_add_features), compared bitwise; a second, different camera makes that
 * side "mixed", and rptb_buffer_add_samples makes the entries "unknown".  The recording changes no other call.
 *
 * RPTB_ERR_BAD_ARG: a null pointer or src == dst; params out of range; dst holding entries or no features; src
 * holding no entries or no features; entries or features of either buffer mixed or unknown, or src's entry camera
 * not its feature camera; buffers created on scenes with different device lists.  RPTB_ERR_UNSUPPORTED: an open
 * aperture on either camera (depth of field blurs the first hits: there is no one point to reproject).  The two
 * buffers may differ in size.  The results are the same bits for any device count.  Afterwards dst's entries count
 * as rendered through its feature camera.  A reprojected buffer may hold pixels with 0 or 1 entries: its image()
 * fails ("Pixel found with no samples") while a pixel has none, denoise() while a pixel has fewer than 2, and its
 * variance() is NaN while a pixel has fewer than 2.
 *
 * Halves (rptb_buffer_create_halves): a dst with halves takes history with halves from a src with halves -- each
 * pixel's HALF scaled so that the error estimate (rptb_buffer_denoise_error) sees the variance of the mean that the
 * capped count claims, not that of the taps' full counts -- and RPTB_ERR_UNSUPPORTED from a plain src.  A plain dst
 * ignores a src's halves.  The sums, M2 and counts are the plain dst's bits.                                    */
typedef struct rptb_reproject {
    double depth_tol;      /* relative depth tolerance, finite, >= 0                        */
    double normal_cos;     /* least N_p . N_q, in [-1, 1]                                  */
    uint32_t max_history;  /* entries a reprojected pixel keeps, >= 2                       */
    uint32_t _pad;
} rptb_reproject;
int rptb_buffer_reproject(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* params,
                          uint64_t* out_reused /* nullable, forces sync: pixels that got history */);

/* ---- Sharding the device Buffer across processes ---------------------------------------------------------
 * Stands beside rptb_render_samples_device's shards for hosts that run one process per GPU (torchrun): each process
 * keeps a buffer of its own tiles, samples, adapts and adds features into it with no exchange, and one all-gather of
 * the shards' blocks gives every process an ordinary whole buffer whose image, variance, pixel_stats, features and
 * denoise are the same bits as those of one whole buffer given the same calls -- same bits for any shard count.
 *
 * A buffer holding only the 16x8 tiles t with t % shard_count == shard_index (a shard may own none: its calls are then
 * no-ops), in one part on scene's device.  rptb_sample_into, rptb_sample_into_adaptive and rptb_buffer_add_features
 * take it when params->shard_index / shard_count are its own (else RPTB_ERR_BAD_ARG); out_active counts this shard's
 * pixels.  Its whole-image calls -- image, variance, sums, pixel_stats, features, denoise, reproject (as dst or src)
 * and add_samples -- are RPTB_ERR_UNSUPPORTED: gather the shards first.  It is reprojected into with
 * rptb_buffer_reproject_shard.  RPTB_ERR_BAD_ARG: shard_index >=
 * shard_count, and the checks of rptb_buffer_create; RPTB_ERR_UNSUPPORTED: a scene with more than one replica.   */
int rptb_buffer_create_shard(rptb_scene* scene, uint32_t width, uint32_t height, uint32_t box_radius, uint32_t shard_index,
                             uint32_t shard_count, rptb_buffer** out);
/* The size in bytes of the shard buffer's exchange block, the same for every shard of one image and shard count: a
 * 256-byte header, then the shard's planes, each padded to shard 0's pixel slots P = (its tiles) * 128 -- sums (3P
 * doubles), M2 (P doubles), with_features the feature sums (8P doubles: normal 3P, albedo 3P, hits P, depth P), then
 * counts (P uint32).  256 + 36 P bytes, 256 + 100 P with features; a shard with halves appends HALF (3P doubles):
 * 256 + 60 P, 256 + 124 P with features.  0 for NULL or a whole buffer.                                      */
uint64_t rptb_buffer_shard_bytes(const rptb_buffer* buffer, uint32_t with_features);
/* rptb_buffer_create_shard with halves: the shard also keeps HALF (rptb_buffer_create_halves) for its own tiles.  Every
 * entry, adaptive and guided call and feature pass takes it as it takes a plain shard, and entry k of a pixel (k its
 * count before the add) goes into HALF iff k is odd, so a shard's HALF is the whole buffer's for its tiles.  Its
 * exchange block appends HALF (3P doubles) after counts: 256 + 60 P bytes, 256 + 124 P with features, and its header's
 * flags say so.  Such blocks import into a whole buffer with halves only (RPTB_ERR_BAD_ARG into a plain one), and a
 * buffer with halves imports no plain blocks (RPTB_ERR_UNSUPPORTED).  It is a reprojection's or merge's dst
 * (rptb_buffer_reproject_shard, rptb_buffer_reproject_merge_shard) from a whole src with halves (RPTB_ERR_UNSUPPORTED
 * from a plain one), and afterwards its block's flags say reprojected and halves.  Its half_sums and denoise_error are
 * refused like every other whole-image read.  Arguments and refusals as rptb_buffer_create_shard.                                        */
int rptb_buffer_create_shard_halves(rptb_scene* scene, uint32_t width, uint32_t height, uint32_t box_radius, uint32_t shard_index,
                                    uint32_t shard_count, rptb_buffer** out);
/* Writes the shard buffer's block (rptb_buffer_shard_bytes) to dst_device, on `stream` (a cudaStream_t, behind the
 * buffer's earlier calls; NULL = the buffer's own stream, and the call then synchronises).  The header holds the
 * image size, shard_index, shard_count, with_features, the entry count, whether the shard was reprojected
 * (rptb_buffer_reproject_shard), the feature rays and the recorded entry and feature cameras; the planes are device-to-device copies of the shard's own.  Slots past the shard's own are not
 * written.  RPTB_ERR_BAD_ARG: a null pointer, a whole buffer, or with_features on a buffer holding no features.  */
int rptb_buffer_export_shard(rptb_buffer* buffer, void* dst_device, uint32_t with_features, void* stream);
/* Replaces the state of `dst`, a whole buffer, with the shards gathered in `gathered_device` on dst's first device:
 * shard_count blocks of rptb_buffer_shard_bytes each, shard 0 first -- what an all-gather of every shard's export
 * gives.  The bytes must be complete when the call is made; it returns once it has read them.  Afterwards dst holds
 * the shards' entries, counts and recorded cameras -- and their features with with_features, none without -- and is
 * indistinguishable from a whole buffer that received the same calls (it may be reprojected from or into; gathered
 * from reprojected shards, it is a reprojected buffer, whose image, variance and denoise check the least count).
 * RPTB_ERR_BAD_ARG: a null pointer or shard_count 0; dst a shard buffer; a block that is not an export, or was made
 * for another image size, shard count or with_features; shards out of order (block i must hold shard i); shards that
 * received different calls (entry counts, reprojection, feature rays or cameras differ); halves blocks into a plain
 * dst.  RPTB_ERR_UNSUPPORTED: plain blocks into a dst with halves.  A dst with halves takes its HALF from the blocks. */
int rptb_buffer_import_shards(rptb_buffer* dst, const void* gathered_device, uint32_t shard_count, uint32_t with_features);
/* rptb_buffer_reproject into a shard buffer: `dst`, a shard, takes the history of its own pixels from `src`, a whole
 * buffer on the shard's device -- in a frame loop, the previous frame's shards gathered with features.  Each pixel
 * gets the bits rptb_buffer_reproject gives it in a whole dst of the same size, features and camera, so the shards'
 * blocks, gathered, are that whole dst.  The checks and refusals are rptb_buffer_reproject's, and the two buffers may
 * differ in size; besides, RPTB_ERR_BAD_ARG: dst a whole buffer, or src's first device not the shard's;
 * RPTB_ERR_UNSUPPORTED: src a shard buffer (gather the shards first).  Afterwards dst is reprojected as by
 * rptb_buffer_reproject, and its block says so (rptb_buffer_export_shard).  A shard that owns no tile does no device
 * work and takes the same state.  out_reused counts this shard's pixels: summed over the shards, the whole call's. */
int rptb_buffer_reproject_shard(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* params,
                                uint64_t* out_reused /* nullable, forces sync: this shard's pixels that got history */);

/* ---- Testing reprojected history against fresh entries ----------------------------------------------------
 * rptb_buffer_reproject writes history into an empty buffer, and nothing checks that the new view agrees with it:
 * stale history (a view-dependent highlight, glass) looks converged to the adaptive criterion and to the denoiser.
 * rptb_buffer_reproject_merge instead takes a dst that already holds >= 2 fresh entry calls through its own feature
 * camera, and tests each pixel's history (the one rptb_buffer_reproject would give it) against that pixel's own fresh
 * mean and variance: with delta the difference of the two means, d2 = |delta|^2 and v the channel-summed variance of
 * that difference, history with d2 > gamma^2 v is rejected and the pixel keeps its bits; agreeing history is merged
 * by the parallel (Chan) combination, whose between-means term d2 n_f n_h / n goes into M2.  gamma = +inf accepts
 * every history, gamma = 0 rejects any whose mean differs.  rpt_b200/csrc/reproject.h gives every formula.  A pixel
 * with no history is left as it is and counted in neither total; out_reused + out_rejected is what out_reused of
 * rptb_buffer_reproject into a fresh buffer with the same features counts.
 *
 * The checks and refusals are rptb_buffer_reproject's for src, the parameters and the device lists; for dst,
 * RPTB_ERR_BAD_ARG: fewer than 2 entry calls, already reprojected, or entries whose camera is not exactly its feature
 * camera (or mixed or unknown); gamma NaN or negative.  Afterwards dst is reprojected, its entry count is its fresh
 * calls plus max_history (a bound), and its entry camera is unchanged, so the next frame can reproject from it.  A dst
 * with halves (from a src with halves) adds the accepted history's half that keeps "entry k goes into HALF iff k is
 * odd" true: its B half when the pixel's fresh count is even, its A half when odd.                               */
int rptb_buffer_reproject_merge(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* params, double gamma,
                                uint64_t* out_reused /* nullable, forces sync: pixels whose history was merged */,
                                uint64_t* out_rejected /* nullable, forces sync: pixels whose history was rejected */);
/* rptb_buffer_reproject_merge into a shard buffer, in place in its own tiles: what rptb_buffer_reproject_shard is to
 * rptb_buffer_reproject, with its extra refusals.  The counts are this shard's pixels; summed over the shards, the
 * whole call's.  A shard that owns no tile does no device work and takes the same state.                         */
int rptb_buffer_reproject_merge_shard(rptb_buffer* dst, rptb_buffer* src, const rptb_reproject* params, double gamma,
                                      uint64_t* out_reused /* nullable, forces sync */,
                                      uint64_t* out_rejected /* nullable, forces sync */);

/* ---- Guided adaptive sampling on shards: a gathered whole buffer kept current by deltas -------------------------
 * The guided criterion's filter reaches across other shards' tiles, so a shard decides from a whole buffer on its own
 * device that holds every shard's state: one full gather (rptb_buffer_export_shard with features, an all-gather,
 * rptb_buffer_import_shards), then, after each adaptive or guided call, one delta per shard carrying only the pixels
 * that call changed, imported in place.  The decisions, and so the shards' entries, are those of the whole buffer's
 * rptb_sample_into_guided, bit for bit, for any shard count.
 *
 * A delta block of capacity m (the same on every shard): a 256-byte header (the image size, shard_index, shard_count,
 * the entry count before and after the call, the reprojected flag, the feature rays, the recorded entry and feature
 * cameras, the pixel count n <= m and m), then sums (3m doubles), M2 (m doubles), counts (m uint32) and the slots (m
 * uint32: each pixel's compact slot in the shard, ascending).  256 + 40 m bytes; only n entries of each plane are
 * written.  No device needed.                                                                                    */
uint64_t rptb_delta_bytes(uint32_t capacity);
/* The delta block of a shard with halves (rptb_buffer_create_shard_halves): the block above, its header's flags saying
 * halves, then HALF (3m doubles) at 256 + 40 m.  256 + 64 m bytes.  No device needed.                            */
uint64_t rptb_delta_bytes_halves(uint32_t capacity);
/* Writes the shard buffer's delta block of `capacity` (rptb_delta_bytes, or rptb_delta_bytes_halves for a shard with
 * halves) to dst_device, on `stream` as
 * rptb_buffer_export_shard does; out_pixels (nullable) receives n.  It reads n, the call's active count, first (one
 * synchronising 8-byte copy).  A delta exists only when the shard's last call was rptb_sample_into_adaptive or
 * rptb_sample_into_guided_shard, that call came right after an export (full or delta), and it kept the shard's entry
 * camera (or made its first entry).  RPTB_ERR_BAD_ARG: a null pointer, a
 * whole buffer, no delta (any other call since the last export -- an entry of another kind, a feature pass, a
 * reprojection or merge, or two calls: gather the full block), or a capacity below n.  A shard with no tile exports
 * n = 0.                                                                                                         */
int rptb_buffer_export_delta(rptb_buffer* buffer, void* dst_device, uint32_t capacity, void* stream, uint32_t* out_pixels);
/* Applies shard_count delta blocks of `capacity`, shard 0 first (an all-gather of every shard's export), in place to
 * `dst`, on dst's device; the bytes must be complete when the call is made, and it returns once it has read them.
 * Afterwards dst holds the shards' state after the call, and its image, variance, pixel_stats, features, denoise and
 * later gathers are those of a full import of the same shards.  RPTB_ERR_BAD_ARG: a null pointer or shard_count 0; dst
 * a shard buffer; a block that is not a delta block, or was made for another image size, shard count or capacity;
 * shards out of order; shards that received different calls (entry counts, reprojection, feature rays or cameras);
 * n > capacity; and a dst that is not at the blocks' state before the call -- one not last written by an import (full
 * or delta) of shard_count shards, or at another entry count, reprojection, feature rays or cameras.
 * RPTB_ERR_UNSUPPORTED: a dst of more than one part.  A dst with halves takes halves blocks only, at the stride of
 * rptb_delta_bytes_halves (RPTB_ERR_UNSUPPORTED: plain blocks); a plain dst plain ones (RPTB_ERR_BAD_ARG: halves blocks). */
int rptb_buffer_import_deltas(rptb_buffer* dst, const void* gathered_device, uint32_t shard_count, uint32_t capacity);
/* rptb_sample_into_guided for a shard buffer: the filter runs over `whole`, a one-part whole buffer on the shard's
 * device holding the gathered state of every shard at the shard's current state, and the mark writes this shard's
 * pixels only.  Each shard renders exactly the pixels the whole buffer's call renders among its tiles; out_active
 * counts them, and summed over the shards it is the whole call's.  While the shard holds fewer than min_entries entry
 * calls the plain mark decides, as in the whole call, and `whole` may be NULL.  Refusals as rptb_sample_into_guided on
 * the shard (its features and entry camera included), and, once the filter runs, RPTB_ERR_BAD_ARG: `whole` NULL, a
 * shard buffer, on another device or of another size; the shard changed since its last export; `whole` not last
 * written by an import (full or delta) of shard_count shards, or not at the shard's entries, reprojection, feature
 * rays and cameras; `whole` failing rptb_sample_into_guided's feature and camera checks.  RPTB_ERR_UNSUPPORTED: a
 * `whole` of more than one part.  RPTB_ERR_BAD_ARG: `shard` a whole buffer.                                     */
int rptb_sample_into_guided_shard(rptb_scene* scene, const rptb_camera* camera, const rptb_render_params* params,
                                  const rptb_adaptive* criterion, const rptb_denoise* guide, rptb_buffer* shard,
                                  rptb_buffer* whole /* nullable while shard entries < min_entries */,
                                  uint64_t* out_active /* nullable, forces sync */, rptb_stats* stats /* nullable, forces sync */);
/* rptb_sample_into_guided_shard with E in place of v' (rptb_sample_into_guided_error): `shard` is a shard with halves
 * (rptb_buffer_create_shard_halves), and once the filter runs, the error estimate runs over `whole`, a whole buffer
 * with halves kept current by halves blocks, and the mark tests E for this shard's pixels.  Each shard renders exactly
 * the pixels rptb_sample_into_guided_error renders among its tiles on a whole buffer with halves.  `whole` may be NULL
 * while the shard holds fewer than min_entries entry calls.  Refusals as rptb_sample_into_guided_shard, and
 * RPTB_ERR_BAD_ARG: the shard or `whole` without halves, guide->iterations == 0.                                 */
int rptb_sample_into_guided_error_shard(rptb_scene* scene, const rptb_camera* camera, const rptb_render_params* params,
                                        const rptb_adaptive* criterion, const rptb_denoise* guide, rptb_buffer* shard,
                                        rptb_buffer* whole /* nullable while shard entries < min_entries */,
                                        uint64_t* out_active /* nullable, forces sync */, rptb_stats* stats /* nullable, forces sync */);

#ifdef __cplusplus
}
#endif
#endif /* RPT_B200_H */
