//! FFI mirror of `include/rpt_b200.h` (rpt-b200, C ABI version 100).  UNVERIFIED: never compiled, there is
//! no Rust toolchain in the image this was written in.  Every struct is field for field the C struct; the
//! sizes the C compiler reports (tests/test_capi.py) are asserted in `tests::layout`.
//!
//! | struct | bytes |   | struct | bytes |
//! |---|---|---|---|---|
//! | RptbMaterial | 64 | | RptbEnv | 48 |
//! | RptbKdNode | 32 | | RptbSceneDesc | 128 |
//! | RptbMesh | 48 | | RptbCamera | 96 |
//! | RptbObject | 192 | | RptbRenderParams | 64 |
//! | RptbGroup | 48 | | RptbStats | 88 |
//! | RptbLight | 248 | | RptbKdTreeOut | 40 |
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_void};

pub const RPTB_OK: c_int = 0;
pub const RPTB_ERR_BAD_ARG: c_int = -1;
pub const RPTB_ERR_CUDA: c_int = -2;
pub const RPTB_ERR_NO_DEVICE: c_int = -3;
pub const RPTB_ERR_OOM: c_int = -4;
pub const RPTB_ERR_UNSUPPORTED: c_int = -5;

pub const RPTB_SHAPE_SPHERE: u32 = 0;
pub const RPTB_SHAPE_PLANE: u32 = 1;
pub const RPTB_SHAPE_CUBE: u32 = 2;
pub const RPTB_SHAPE_MESH: u32 = 3;
pub const RPTB_SHAPE_MONOMIAL: u32 = 4;
pub const RPTB_SHAPE_GROUP: u32 = 5;

pub const RPTB_LIGHT_POINT: u32 = 0;
pub const RPTB_LIGHT_AMBIENT: u32 = 1;
pub const RPTB_LIGHT_DIRECTIONAL: u32 = 2;
pub const RPTB_LIGHT_OBJECT: u32 = 3;

pub const RPTB_ENV_COLOR: u32 = 0;
pub const RPTB_ENV_HDRI: u32 = 1;

pub const RPTB_ACCEL_AUTO: u32 = 0;
pub const RPTB_ACCEL_KDTREE: u32 = 1;
pub const RPTB_ACCEL_BVH: u32 = 2;

pub const RPTB_PRECISION_F32: u32 = 0;
pub const RPTB_PRECISION_F64: u32 = 1;

pub const RPTB_ENGINE_AUTO: u32 = 0;
pub const RPTB_ENGINE_MEGAKERNEL: u32 = 1;
pub const RPTB_ENGINE_WAVEFRONT: u32 = 2;

#[repr(C)]
#[derive(Copy, Clone, Debug, Default)]
pub struct RptbMaterial {
    pub color: [f64; 3],
    pub index: f64,
    pub roughness: f64,
    pub metallic: f64,
    pub emittance: f64,
    pub transparent: u32,
    pub _pad: u32,
}

#[repr(C)]
#[derive(Copy, Clone, Debug, Default)]
pub struct RptbKdNode {
    pub split: f64,
    pub kind: u32, // 0/1/2 = SplitX/Y/Z, 3 = Leaf
    pub left: u32,
    pub right: u32,
    pub first_ref: u32,
    pub num_refs: u32,
    pub _pad: u32,
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbMesh {
    pub tris: *const f64, // ntris x 18: v1 v2 v3 n1 n2 n3
    pub ntris: u64,
    pub nodes: *const RptbKdNode, // null: the library builds the reference-shaped tree
    pub nnodes: u64,
    pub refs: *const u32,
    pub nrefs: u64,
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbObject {
    pub kind: u32,
    pub material: u32,
    pub mesh: u32, // MESH: mesh index; GROUP: group index
    pub has_transform: u32,
    pub transform: [f64; 16], // column-major, as nalgebra stores DMat4
    pub plane_normal: [f64; 3],
    pub plane_value: f64,
    pub monomial_height: f64,
    pub monomial_exp: f64,
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbGroup {
    pub children: *const RptbObject,
    pub nchildren: u64,
    pub nodes: *const RptbKdNode,
    pub nnodes: u64,
    pub refs: *const u32,
    pub nrefs: u64,
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbLight {
    pub kind: u32,
    pub _pad: u32,
    pub color: [f64; 3],
    pub vec: [f64; 3],
    pub object: RptbObject,
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbEnv {
    pub kind: u32,
    pub width: u32,
    pub height: u32,
    pub _pad: u32,
    pub color: [f64; 3],
    pub texels: *const f64, // width * height * 3
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbSceneDesc {
    pub materials: *const RptbMaterial,
    pub nmaterials: u32,
    pub meshes: *const RptbMesh,
    pub nmeshes: u32,
    pub objects: *const RptbObject,
    pub nobjects: u32,
    pub lights: *const RptbLight,
    pub nlights: u32,
    pub environment: RptbEnv,
    pub groups: *const RptbGroup,
    pub ngroups: u32,
    pub accel: u32,
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbCamera {
    pub eye: [f64; 3],
    pub direction: [f64; 3],
    pub up: [f64; 3],
    pub fov: f64,
    pub aperture: f64,
    pub focal_distance: f64,
}

#[repr(C)]
#[derive(Copy, Clone, Debug, Default)]
pub struct RptbRenderParams {
    pub width: u32,
    pub height: u32,
    pub iterations: u32,
    pub max_bounces: u32,
    pub exposure_value: f64,
    pub seed: u64,
    pub first_sample: u64,
    pub shard_index: u32,
    pub shard_count: u32,
    pub precision: u32,
    pub collect_stats: u32,
    pub engine: u32,
    pub compact_out: u32,
}

#[repr(C)]
#[derive(Copy, Clone, Debug, Default)]
pub struct RptbStats {
    pub segments: u64,
    pub rays: u64,
    pub node_visits: u64,
    pub tri_tests: u64,
    pub mesh_hits: u64,
    pub env_lookups: u64,
    pub object_tests: u64,
    pub gpu_ms: f64,
    pub launches: u32,
    pub engine: u32,
    pub bvh_node_visits: u64,
    pub bvh_tri_tests: u64,
}

#[repr(C)]
#[derive(Copy, Clone, Debug)]
pub struct RptbKdTreeOut {
    pub nodes: *mut RptbKdNode,
    pub nnodes: u64,
    pub refs: *mut u32,
    pub nrefs: u64,
    pub depth: u32,
    pub max_leaf: u32,
}

/// Opaque `rptb_scene`.
#[repr(C)]
pub struct RptbScene {
    _private: [u8; 0],
}

/// Opaque `rptb_buffer`: `Buffer` (src/buffer.rs:6-93) kept in device memory.
#[repr(C)]
pub struct RptbBuffer {
    _private: [u8; 0],
}

extern "C" {
    pub fn rptb_last_error() -> *const c_char;
    pub fn rptb_device_count() -> c_int;
    pub fn rptb_scene_create(desc: *const RptbSceneDesc, device: c_int, out: *mut *mut RptbScene) -> c_int;
    /// The scene replicated on `ndevices` GPUs (`devices` null = 0..ndevices-1): `rptb_render_samples` then fans
    /// out over them -- the rayon loop of `Renderer::sample` (src/renderer.rs:117-129) behind the same call.
    pub fn rptb_scene_create_multi(desc: *const RptbSceneDesc, devices: *const c_int, ndevices: c_int, out: *mut *mut RptbScene) -> c_int;
    pub fn rptb_scene_device_count(scene: *const RptbScene) -> c_int;
    pub fn rptb_scene_destroy(scene: *mut RptbScene);
    pub fn rptb_scene_device_bytes(scene: *const RptbScene) -> u64;
    pub fn rptb_render_samples(
        scene: *mut RptbScene,
        camera: *const RptbCamera,
        params: *const RptbRenderParams,
        out_rgb: *mut f64, // width * height * 3, row-major, y = 0 top
        stats: *mut RptbStats, // nullable
    ) -> c_int;
    pub fn rptb_render_samples_device(
        scene: *mut RptbScene,
        camera: *const RptbCamera,
        params: *const RptbRenderParams,
        out_device: *mut f32,
        stream: *mut c_void, // cudaStream_t; null = the scene's own stream, synchronised
        stats: *mut RptbStats,
    ) -> c_int;
    pub fn rptb_closest_hit(
        scene: *mut RptbScene,
        rays: *const f64, // n x 6
        n: u64,
        t_min: f64,
        precision: u32,
        out_t: *mut f64,
        out_object: *mut i32,
        out_normal: *mut f64, // nullable, n x 3
        stats: *mut RptbStats,
    ) -> c_int;
    pub fn rptb_illuminate(
        scene: *mut RptbScene,
        light: u32,
        pos: *const f64, // n x 3
        n: u64,
        seed: u64,
        precision: u32,
        out_intensity: *mut f64, // n x 3
        out_wi: *mut f64,        // n x 3
        out_dist: *mut f64,      // n
    ) -> c_int;
    pub fn rptb_build_kdtree(tris: *const f64, ntris: u64, out: *mut RptbKdTreeOut) -> c_int;
    pub fn rptb_build_kdtree_boxes(boxes: *const f64, nboxes: u64, out: *mut RptbKdTreeOut) -> c_int;
    pub fn rptb_free_kdtree(out: *mut RptbKdTreeOut);
    pub fn rptb_film_resolve(
        sums: *const f64,
        nbatches: u32,
        width: u32,
        height: u32,
        box_radius: u32,
        device: c_int,
        out_rgb8: *mut u8,
    ) -> c_int;
    pub fn rptb_film_variance(batches: *const f64, nbatches: u32, npixels: u64, device: c_int, out: *mut f64) -> c_int;
    /// `Buffer::new(width, height, Filter::Box(box_radius))` on every GPU of `scene`; it may outlive the scene.
    pub fn rptb_buffer_create(scene: *mut RptbScene, width: u32, height: u32, box_radius: u32, out: *mut *mut RptbBuffer) -> c_int;
    pub fn rptb_buffer_destroy(buffer: *mut RptbBuffer);
    /// `Renderer::sample(iterations, &mut buffer)` (src/renderer.rs:117-129) with the entry added on the device;
    /// with `stats` null it returns once the work is enqueued.
    pub fn rptb_sample_into(
        scene: *mut RptbScene,
        camera: *const RptbCamera,
        params: *const RptbRenderParams,
        buffer: *mut RptbBuffer,
        stats: *mut RptbStats, // nullable
    ) -> c_int;
    pub fn rptb_buffer_add_samples(buffer: *mut RptbBuffer, rgb: *const f64) -> c_int; // width * height * 3, row-major
    pub fn rptb_buffer_image(buffer: *mut RptbBuffer, out_rgb8: *mut u8) -> c_int;
    pub fn rptb_buffer_variance(buffer: *mut RptbBuffer, out: *mut f64) -> c_int; // NaN below two entries
    pub fn rptb_buffer_sums(buffer: *mut RptbBuffer, out_sums: *mut f64, out_entries: *mut u32) -> c_int;
}

/// The thread-local message of the last failing call.
pub fn last_error() -> String {
    unsafe {
        let p = rptb_last_error();
        if p.is_null() {
            String::new()
        } else {
            std::ffi::CStr::from_ptr(p).to_string_lossy().into_owned()
        }
    }
}

#[cfg(test)]
mod tests {
    use super::*;
    use std::mem::size_of;

    #[test]
    fn layout() {
        // sizeof() of the C structs, printed by tests/test_capi.py::test_struct_layouts_match_header_sizes
        assert_eq!(size_of::<RptbMaterial>(), 64);
        assert_eq!(size_of::<RptbKdNode>(), 32);
        assert_eq!(size_of::<RptbMesh>(), 48);
        assert_eq!(size_of::<RptbObject>(), 192);
        assert_eq!(size_of::<RptbGroup>(), 48);
        assert_eq!(size_of::<RptbLight>(), 248);
        assert_eq!(size_of::<RptbEnv>(), 48);
        assert_eq!(size_of::<RptbSceneDesc>(), 128);
        assert_eq!(size_of::<RptbCamera>(), 96);
        assert_eq!(size_of::<RptbRenderParams>(), 64);
        assert_eq!(size_of::<RptbStats>(), 88);
        assert_eq!(size_of::<RptbKdTreeOut>(), 40);
    }
}
