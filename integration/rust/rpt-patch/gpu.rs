//! `rpt::gpu` -- puts librpt_b200.so behind `Renderer::sample`.  UNVERIFIED SOURCE (never
//! compiled); see ../README.md and the repository's INTEGRATION.md.
//!
//! The crate's shapes are type-erased (`Object.shape: Box<dyn Shape>`, src/object.rs:12), so the flattening
//! needs one addition to the `Shape` trait: `describe`, implemented by every shape of the crate
//! (CHANGES.md).  Everything else lives here.
#![allow(unsafe_code)]

use std::collections::HashMap;

use rpt_b200_sys as sys;

use crate::camera::Camera;
use crate::color::Color;
use crate::environment::Environment;
use crate::light::Light;
use crate::material::Material;
use crate::scene::Scene;
use crate::shape::Shape;

/// What a shape says about itself.  `Transformed<T>` wraps the description of `T`; chained transforms are
/// already composed into one matrix by `Transformed`'s own builder methods (src/shape.rs:234-284).
pub enum FlatShape {
    Sphere,
    Plane { normal: glm::DVec3, value: f64 },
    Cube,
    /// `KdTree<Triangle>`; `key` identifies the allocation (an `Arc<Mesh>` shared by many instances is
    /// described once): the address of the tree's `objects` buffer.
    Mesh { key: usize, mesh: MeshData },
    Monomial { height: f64, exp: f64 },
    /// `KdTree<T: Bounded>` over whole shapes: the children in `objects` order, and the tree.
    Group { children: Vec<FlatShape>, tree: TreeData },
    Transformed { inner: Box<FlatShape>, transform: glm::DMat4 },
}

/// Triangles as 18 doubles each (v1 v2 v3 n1 n2 n3) plus the kd-tree serialised in DFS pre-order.
pub struct MeshData {
    pub tris: Vec<f64>,
    pub tree: TreeData,
}

#[derive(Default)]
pub struct TreeData {
    pub nodes: Vec<sys::RptbKdNode>,
    pub refs: Vec<u32>,
}

/// The method `Shape` gains (default: not representable on the GPU path).
pub trait Describe {
    fn describe(&self) -> Option<FlatShape> {
        None
    }
}

/// Owns every array the `RptbSceneDesc` points into; must outlive `rptb_scene_create` only.
#[derive(Default)]
pub struct FlatScene {
    materials: Vec<sys::RptbMaterial>,
    meshes: Vec<sys::RptbMesh>,
    mesh_data: Vec<MeshData>,
    mesh_index: HashMap<usize, u32>,
    objects: Vec<sys::RptbObject>,
    lights: Vec<sys::RptbLight>,
    groups: Vec<sys::RptbGroup>,
    group_children: Vec<Vec<sys::RptbObject>>,
    group_trees: Vec<TreeData>,
    texels: Vec<f64>,
}

fn material_to_c(m: &Material) -> sys::RptbMaterial {
    sys::RptbMaterial {
        color: [m.color.x, m.color.y, m.color.z],
        index: m.index,
        roughness: m.roughness,
        metallic: m.metallic,
        emittance: m.emittance,
        transparent: m.transparent as u32,
        _pad: 0,
    }
}

fn identity16() -> [f64; 16] {
    let mut t = [0.0; 16];
    t[0] = 1.0;
    t[5] = 1.0;
    t[10] = 1.0;
    t[15] = 1.0;
    t
}

impl FlatScene {
    pub fn new(scene: &Scene) -> Result<Self, String> {
        let mut f = FlatScene::default();
        for (i, o) in scene.objects.iter().enumerate() {
            let shape = o.shape.describe().ok_or_else(|| format!("object {}: shape has no GPU description", i))?;
            let mut c = f.shape_to_c(shape)?;
            c.material = f.materials.len() as u32;
            f.materials.push(material_to_c(&o.material));
            f.objects.push(c);
        }
        for (i, l) in scene.lights.iter().enumerate() {
            let mut c = sys::RptbLight {
                kind: 0,
                _pad: 0,
                color: [0.0; 3],
                vec: [0.0; 3],
                object: sys::RptbObject {
                    kind: 0, material: 0, mesh: 0, has_transform: 0, transform: identity16(),
                    plane_normal: [0.0; 3], plane_value: 0.0, monomial_height: 0.0, monomial_exp: 0.0,
                },
            };
            match l {
                Light::Point(color, location) => {
                    c.kind = sys::RPTB_LIGHT_POINT;
                    c.color = [color.x, color.y, color.z];
                    c.vec = [location.x, location.y, location.z];
                }
                Light::Ambient(color) => {
                    c.kind = sys::RPTB_LIGHT_AMBIENT;
                    c.color = [color.x, color.y, color.z];
                }
                Light::Directional(color, dir) => {
                    c.kind = sys::RPTB_LIGHT_DIRECTIONAL;
                    c.color = [color.x, color.y, color.z];
                    c.vec = [dir.x, dir.y, dir.z];
                }
                Light::Object(o) => {
                    c.kind = sys::RPTB_LIGHT_OBJECT;
                    let shape = o.shape.describe().ok_or_else(|| format!("light {}: shape has no GPU description", i))?;
                    c.object = f.shape_to_c(shape)?;
                    c.object.material = f.materials.len() as u32;
                    f.materials.push(material_to_c(&o.material));
                }
            }
            f.lights.push(c);
        }
        if let Environment::Hdri(h) = &scene.environment {
            // Hdri { width, height, buf: Vec<Color> } (src/environment.rs:55-63; fields need pub(crate))
            f.texels = h.buf.iter().flat_map(|c: &Color| vec![c.x, c.y, c.z]).collect();
        }
        Ok(f)
    }

    fn shape_to_c(&mut self, shape: FlatShape) -> Result<sys::RptbObject, String> {
        let mut c = sys::RptbObject {
            kind: 0, material: 0, mesh: 0, has_transform: 0, transform: identity16(),
            plane_normal: [0.0; 3], plane_value: 0.0, monomial_height: 0.0, monomial_exp: 0.0,
        };
        let base = match shape {
            FlatShape::Transformed { inner, transform } => {
                c.has_transform = 1;
                // nalgebra matrices are column-major: as_slice() is exactly rptb_object.transform
                c.transform.copy_from_slice(transform.as_slice());
                *inner
            }
            other => other,
        };
        match base {
            FlatShape::Sphere => c.kind = sys::RPTB_SHAPE_SPHERE,
            FlatShape::Cube => c.kind = sys::RPTB_SHAPE_CUBE,
            FlatShape::Plane { normal, value } => {
                c.kind = sys::RPTB_SHAPE_PLANE;
                c.plane_normal = [normal.x, normal.y, normal.z];
                c.plane_value = value;
            }
            FlatShape::Monomial { height, exp } => {
                c.kind = sys::RPTB_SHAPE_MONOMIAL;
                c.monomial_height = height;
                c.monomial_exp = exp;
            }
            FlatShape::Mesh { key, mesh } => {
                c.kind = sys::RPTB_SHAPE_MESH;
                c.mesh = match self.mesh_index.get(&key) {
                    Some(&i) => i,
                    None => {
                        let i = self.mesh_data.len() as u32;
                        self.mesh_data.push(mesh);
                        self.mesh_index.insert(key, i);
                        i
                    }
                };
            }
            FlatShape::Group { children, tree } => {
                c.kind = sys::RPTB_SHAPE_GROUP;
                let mut kids = Vec::with_capacity(children.len());
                for child in children {
                    if matches!(child, FlatShape::Group { .. } | FlatShape::Plane { .. }) {
                        return Err("a kd-tree child must be a bounded, non-kd-tree shape".into());
                    }
                    kids.push(self.shape_to_c(child)?);
                }
                c.mesh = self.group_children.len() as u32;
                self.group_children.push(kids);
                self.group_trees.push(tree);
            }
            FlatShape::Transformed { .. } => return Err("nested Transformed: compose the matrices first".into()),
        }
        Ok(c)
    }

    /// Fills the pointer tables and returns the description; `self` must not move or change afterwards.
    pub fn desc(&mut self, scene: &Scene) -> sys::RptbSceneDesc {
        self.meshes = self
            .mesh_data
            .iter()
            .map(|m| sys::RptbMesh {
                tris: m.tris.as_ptr(),
                ntris: (m.tris.len() / 18) as u64,
                nodes: m.tree.nodes.as_ptr(),
                nnodes: m.tree.nodes.len() as u64,
                refs: m.tree.refs.as_ptr(),
                nrefs: m.tree.refs.len() as u64,
            })
            .collect();
        self.groups = self
            .group_children
            .iter()
            .zip(self.group_trees.iter())
            .map(|(kids, tree)| sys::RptbGroup {
                children: kids.as_ptr(),
                nchildren: kids.len() as u64,
                nodes: if tree.nodes.is_empty() { std::ptr::null() } else { tree.nodes.as_ptr() },
                nnodes: tree.nodes.len() as u64,
                refs: tree.refs.as_ptr(),
                nrefs: tree.refs.len() as u64,
            })
            .collect();
        let environment = match &scene.environment {
            Environment::Color(c) => sys::RptbEnv {
                kind: sys::RPTB_ENV_COLOR, width: 0, height: 0, _pad: 0, color: [c.x, c.y, c.z], texels: std::ptr::null(),
            },
            Environment::Hdri(h) => sys::RptbEnv {
                kind: sys::RPTB_ENV_HDRI, width: h.width, height: h.height, _pad: 0, color: [0.0; 3], texels: self.texels.as_ptr(),
            },
        };
        sys::RptbSceneDesc {
            materials: self.materials.as_ptr(),
            nmaterials: self.materials.len() as u32,
            meshes: self.meshes.as_ptr(),
            nmeshes: self.meshes.len() as u32,
            objects: self.objects.as_ptr(),
            nobjects: self.objects.len() as u32,
            lights: self.lights.as_ptr(),
            nlights: self.lights.len() as u32,
            environment,
            groups: self.groups.as_ptr(),
            ngroups: self.groups.len() as u32,
            accel: sys::RPTB_ACCEL_AUTO,
        }
    }
}

/// RAII owner of the device-resident scene.  Immutable after creation, like `&Scene` (`Send + Sync`).
pub struct GpuScene {
    handle: *mut sys::RptbScene,
}
unsafe impl Send for GpuScene {}
unsafe impl Sync for GpuScene {}

impl GpuScene {
    pub fn new(scene: &Scene, device: i32) -> Result<Self, String> {
        Self::on_devices(scene, &[device])
    }

    /// The scene replicated on every GPU of the box (`rptb_device_count`): what `Renderer::sample` wants by
    /// default -- its rayon loop over rows (src/renderer.rs:118-127) becomes one host thread per GPU inside
    /// `rptb_render_samples`, each GPU owning the pixel tiles `t % n == i`; same image for any `n`.
    pub fn on_all_gpus(scene: &Scene) -> Result<Self, String> {
        let n = unsafe { sys::rptb_device_count() };
        if n <= 0 {
            return Err(sys::last_error());
        }
        let devices: Vec<i32> = (0..n).collect();
        Self::on_devices(scene, &devices)
    }

    pub fn on_devices(scene: &Scene, devices: &[i32]) -> Result<Self, String> {
        let mut flat = FlatScene::new(scene)?;
        let desc = flat.desc(scene);
        let mut handle = std::ptr::null_mut();
        let rc = unsafe { sys::rptb_scene_create_multi(&desc, devices.as_ptr(), devices.len() as i32, &mut handle) };
        if rc != sys::RPTB_OK {
            return Err(sys::last_error());
        }
        Ok(GpuScene { handle }) // `flat` may die now: the library copied everything to the device(s)
    }

    pub fn device_count(&self) -> i32 {
        unsafe { sys::rptb_scene_device_count(self.handle) }
    }

    /// What `Renderer::get_color` returns for every pixel: mean of `iterations` samples x 2^EV,
    /// row-major, y = 0 is the top row (src/renderer.rs:131-142).
    #[allow(clippy::too_many_arguments)]
    pub fn render_samples(
        &self,
        camera: &Camera,
        width: u32,
        height: u32,
        iterations: u32,
        max_bounces: u32,
        exposure_value: f64,
        seed: u64,
        first_sample: u64,
    ) -> Vec<Color> {
        let cam = sys::RptbCamera {
            eye: [camera.eye.x, camera.eye.y, camera.eye.z],
            direction: [camera.direction.x, camera.direction.y, camera.direction.z],
            up: [camera.up.x, camera.up.y, camera.up.z],
            fov: camera.fov,
            aperture: camera.aperture,
            focal_distance: camera.focal_distance,
        };
        let params = sys::RptbRenderParams {
            width, height, iterations, max_bounces, exposure_value, seed, first_sample,
            shard_index: 0, shard_count: 1, precision: sys::RPTB_PRECISION_F32, collect_stats: 0,
            engine: sys::RPTB_ENGINE_AUTO, compact_out: 0,
        };
        let mut colors = vec![glm::vec3(0.0, 0.0, 0.0); (width * height) as usize];
        // a DVec3 is three contiguous f64: the Vec<Color> is the W*H*3 double buffer the library fills
        let rc = unsafe {
            sys::rptb_render_samples(self.handle, &cam, &params, colors.as_mut_ptr() as *mut f64, std::ptr::null_mut())
        };
        if rc != sys::RPTB_OK {
            // Renderer::render is infallible by signature and the crate panics on misuse (src/buffer.rs:26,33-36)
            panic!("rpt_b200: {}", sys::last_error());
        }
        colors
    }
}

impl Drop for GpuScene {
    fn drop(&mut self) {
        unsafe { sys::rptb_scene_destroy(self.handle) }
    }
}
