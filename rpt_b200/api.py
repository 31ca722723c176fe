"""Host-side mirror of rpt's public API for the path-tracing hot path.

Same names, argument meaning and error behaviour as the reference's builder
API, so scene scripts and tests read like the reference's examples:

    Scene / SceneAdd            src/scene.rs:7-41
    Object                      src/object.rs:10-32
    Material::{diffuse,...}     src/material.rs:28-106
    Light                       src/light.rs:7-19
    Environment / Hdri          src/environment.rs:4-23,55-70
    Camera::{look_at,focus}     src/camera.rs:8-61
    Transformable / Transformed src/shape.rs:99-125,179-284
    sphere/plane/cube/polygon   src/shape.rs:286-313
    load_obj                    src/io.rs:27-73,151-200
    Renderer                    src/renderer.rs:18-115
    Buffer / Filter             src/buffer.rs:6-108
    DeviceBuffer                src/buffer.rs:6-93, kept on the GPU (rptb_buffer)
    Adaptive                    not in the reference: which pixels an adaptive Renderer.sample renders
    Denoise                     not in the reference: the edge-avoiding filter of DeviceBuffer.denoise
    hex_color / color_bytes     src/color.rs:10-23

Everything below `Renderer.sample` (src/renderer.rs:117-129) is *not* here:
that is the hot path, and it runs in the CUDA library behind the C ABI of
include/rpt_b200.h.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from . import _capi as capi

SRGB_GAMMA = 2.2  # src/color.rs:4


def vec3(x: float, y: float, z: float) -> np.ndarray:
    return np.array([x, y, z], dtype=np.float64)


# ------------------------------------------------------------------ colour ----
def hex_color(x: int) -> np.ndarray:
    """src/color.rs:10-15 -- sRGB hex integer to linear intensities (gamma 2.2)."""
    r = ((x >> 16) & 0xFF) / 255.0
    g = ((x >> 8) & 0xFF) / 255.0
    b = (x & 0xFF) / 255.0
    return vec3(r**SRGB_GAMMA, g**SRGB_GAMMA, b**SRGB_GAMMA)


def color_bytes(color: Sequence[float]) -> List[int]:
    """src/color.rs:17-23 -- clamp, gamma-encode, truncate to u8."""
    return [int(min(max(float(c), 0.0), 1.0) ** (1.0 / SRGB_GAMMA) * 255.0) for c in color]


# ---------------------------------------------------------------- glm bits ----
def _translate(v) -> np.ndarray:
    m = np.eye(4)
    m[:3, 3] = v
    return m


def _scale(v) -> np.ndarray:
    return np.diag([v[0], v[1], v[2], 1.0])


def _rotate(angle: float, axis) -> np.ndarray:
    a = np.asarray(axis, dtype=np.float64)
    a = a / np.linalg.norm(a)  # glm::rotate normalises the axis
    c, s = math.cos(angle), math.sin(angle)
    x, y, z = a
    r = np.array(
        [
            [c + x * x * (1 - c), x * y * (1 - c) - z * s, x * z * (1 - c) + y * s],
            [y * x * (1 - c) + z * s, c + y * y * (1 - c), y * z * (1 - c) - x * s],
            [z * x * (1 - c) - y * s, z * y * (1 - c) + x * s, c + z * z * (1 - c)],
        ]
    )
    m = np.eye(4)
    m[:3, :3] = r
    return m


# ------------------------------------------------------------------ shapes ----
class Shape:
    """src/shape.rs:18-25.  `intersect`/`sample` live on the device; the host
    object only describes the geometry (the reference's Box<dyn Shape> is opaque,
    which is why the boundary makes the kind explicit)."""

    kind: int = -1

    # Transformable (src/shape.rs:202-230): first transform wraps the bare shape
    def translate(self, v) -> "Transformed":
        return Transformed(self, _translate(v))

    def scale(self, v) -> "Transformed":
        return Transformed(self, _scale(v))

    def rotate(self, angle: float, axis) -> "Transformed":
        return Transformed(self, _rotate(angle, axis))

    def rotate_x(self, angle: float) -> "Transformed":
        return Transformed(self, _rotate(angle, (1.0, 0.0, 0.0)))

    def rotate_y(self, angle: float) -> "Transformed":
        return Transformed(self, _rotate(angle, (0.0, 1.0, 0.0)))

    def rotate_z(self, angle: float) -> "Transformed":
        return Transformed(self, _rotate(angle, (0.0, 0.0, 1.0)))

    def transform(self, m) -> "Transformed":
        return Transformed(self, np.asarray(m, dtype=np.float64))


class Sphere(Shape):
    """Unit sphere at the origin, src/shape/sphere.rs:8-10."""

    kind = capi.SHAPE_SPHERE


class Cube(Shape):
    """Unit cube at the origin, src/shape/cube.rs:6-8."""

    kind = capi.SHAPE_CUBE


class Plane(Shape):
    """x . normal = value, src/shape/plane.rs:6-14."""

    kind = capi.SHAPE_PLANE

    def __init__(self, normal, value: float):
        self.normal = np.asarray(normal, dtype=np.float64)
        self.value = float(value)


class Triangle:
    """src/shape/mesh.rs:7-37 -- a row of 18 doubles v1,v2,v3,n1,n2,n3."""

    @staticmethod
    def from_vertices(v1, v2, v3) -> np.ndarray:
        v1, v2, v3 = (np.asarray(v, dtype=np.float64) for v in (v1, v2, v3))
        n = np.cross(v2 - v1, v3 - v1)
        n = n / np.linalg.norm(n)
        return np.concatenate([v1, v2, v3, n, n, n])


class Mesh(Shape):
    """Mesh = KdTree<Triangle> (src/shape/mesh.rs:102, src/kdtree.rs:99-119).

    The kd-tree is built at construction like `KdTree::new`, by the library's
    host-side restatement of `construct` (rptb_build_kdtree)."""

    kind = capi.SHAPE_MESH

    def __init__(self, triangles, build: bool = True):
        self.triangles = np.ascontiguousarray(np.asarray(triangles, dtype=np.float64).reshape(-1, 18))
        self.nodes = None  # ctypes array of KdNode
        self.refs = None  # np.uint32
        self.depth = 0
        self.max_leaf = 0
        if build:
            self._build()

    def _build(self) -> None:
        lib = capi.lib()
        out = capi.KdTreeOut()
        tris = self.triangles
        capi.check(
            lib.rptb_build_kdtree(tris.ctypes.data_as(capi.c_double_p), tris.shape[0], C.byref(out)),
            "rptb_build_kdtree",
        )
        try:
            n = int(out.nnodes)
            self.nodes = (capi.KdNode * n)()
            C.memmove(self.nodes, out.nodes, C.sizeof(capi.KdNode) * n)
            self.refs = np.ctypeslib.as_array(out.refs, shape=(int(out.nrefs),)).copy() if out.nrefs else np.zeros(0, np.uint32)
            self.depth, self.max_leaf = int(out.depth), int(out.max_leaf)
        finally:
            lib.rptb_free_kdtree(C.byref(out))

    def __len__(self) -> int:
        return self.triangles.shape[0]


class MonomialSurface(Shape):
    """y = height * (x^2 + z^2)^(exp/2) over the unit disc, src/shape/monomial_surface.rs:13-18.
    As in the reference, intersection and normals are only right for exp = 4."""

    kind = capi.SHAPE_MONOMIAL

    def __init__(self, height: float, exp: float = 4.0):
        self.height = float(height)
        self.exp = float(exp)


class KdTree(Shape):
    """KdTree::new(objects) over whole Bounded shapes (src/kdtree.rs:99-119): the kd-tree of
    kd-trees of examples/fractal_teapots.rs:53-59 and the sphere clouds of fractal_spheres.rs.
    `objects` are spheres, cubes, monomial surfaces and meshes, bare or transformed; a Mesh may
    appear many times (the reference shares it through Arc<Mesh>).  The tree over the children's
    bounding boxes is built by the library when the scene is created."""

    kind = capi.SHAPE_GROUP

    def __init__(self, objects):
        self.objects = list(objects)
        for o in self.objects:
            base = o.shape if isinstance(o, Transformed) else o
            if isinstance(base, Plane):
                raise TypeError("Plane is not Bounded (no bounding_box): it cannot go into a KdTree")
            if isinstance(base, KdTree):
                raise TypeError("a KdTree inside a KdTree is not supported by the device scene")
            if not isinstance(base, (Sphere, Cube, Mesh, MonomialSurface)):
                raise TypeError(f"not a Bounded shape: {type(base).__name__}")

    def __len__(self) -> int:
        return len(self.objects)


class Transformed(Shape):
    """src/shape.rs:99-125; chaining composes instead of nesting (:234-284)."""

    def __init__(self, shape: Shape, transform: np.ndarray):
        assert not isinstance(shape, Transformed)
        self.shape = shape
        self.matrix = np.asarray(transform, dtype=np.float64)

    @property
    def kind(self):  # type: ignore[override]
        return self.shape.kind

    def translate(self, v):
        return Transformed(self.shape, _translate(v) @ self.matrix)

    def scale(self, v):
        return Transformed(self.shape, _scale(v) @ self.matrix)

    def rotate(self, angle, axis):
        return Transformed(self.shape, _rotate(angle, axis) @ self.matrix)

    def rotate_x(self, angle):
        return Transformed(self.shape, _rotate(angle, (1.0, 0.0, 0.0)) @ self.matrix)

    def rotate_y(self, angle):
        return Transformed(self.shape, _rotate(angle, (0.0, 1.0, 0.0)) @ self.matrix)

    def rotate_z(self, angle):
        return Transformed(self.shape, _rotate(angle, (0.0, 0.0, 1.0)) @ self.matrix)

    def transform(self, m):
        return Transformed(self.shape, np.asarray(m, dtype=np.float64) @ self.matrix)


def sphere() -> Sphere:  # src/shape.rs:287-289
    return Sphere()


def plane(normal, value: float) -> Plane:  # :297-299
    return Plane(normal, value)


def cube() -> Cube:  # :302-304
    return Cube()


def monomial_surface(height: float, exp: float) -> MonomialSurface:  # :292-294
    return MonomialSurface(height, exp)


def polygon(verts) -> Mesh:  # :307-313 (triangle fan)
    verts = [np.asarray(v, dtype=np.float64) for v in verts]
    tris = [Triangle.from_vertices(verts[0], verts[i], verts[i + 1]) for i in range(1, len(verts) - 1)]
    return Mesh(np.stack(tris))


def parse_obj(lines) -> np.ndarray:
    """src/io.rs:27-73,151-200: v / vn / f with fan triangulation, `v//vn` and negative
    indices; vt, mtllib, usemtl are skipped.  Returns an (n, 18) triangle array."""
    vertices: List[np.ndarray] = []
    normals: List[np.ndarray] = []
    tris: List[np.ndarray] = []

    def parse_index(value: str, length: int) -> Optional[int]:
        try:
            index = int(value)
        except ValueError:
            return None
        return index - 1 if index > 0 else length + index

    for raw in lines:
        line = raw.strip()
        if not line or line.startswith("#"):
            continue
        tok = line.split()
        if tok[0] == "v":
            vertices.append(vec3(float(tok[1]), float(tok[2]), float(tok[3])))
        elif tok[0] == "vn":
            normals.append(vec3(float(tok[1]), float(tok[2]), float(tok[3])))
        elif tok[0] == "f":
            vi, vni = [], []
            for vert in tok[1:]:
                args = (vert.split("/") + ["", "", ""])[:3]
                idx = parse_index(args[0], len(vertices))
                if idx is None:
                    raise ValueError("Invalid vertex index")
                vi.append(idx)
                vni.append(parse_index(args[2], len(normals)))
            for i in range(1, len(vi) - 1):
                a, b, c = 0, i, i + 1
                v1, v2, v3 = vertices[vi[a]], vertices[vi[b]], vertices[vi[c]]
                if vni[a] is None or vni[b] is None or vni[c] is None:
                    tris.append(Triangle.from_vertices(v1, v2, v3))
                else:
                    tris.append(np.concatenate([v1, v2, v3, normals[vni[a]], normals[vni[b]], normals[vni[c]]]))
    return np.stack(tris) if tris else np.zeros((0, 18))


def parse_obj_native(text) -> np.ndarray:
    """The same parse through the library's C++ implementation (rptb_parse_obj): what load_obj uses."""
    data = text.encode() if isinstance(text, str) else bytes(text)
    lib = capi.lib()
    out = capi.c_double_p()
    n = C.c_uint64(0)
    capi.check(lib.rptb_parse_obj(data, len(data), C.byref(out), C.byref(n)), "rptb_parse_obj")
    try:
        if n.value == 0:
            return np.zeros((0, 18))
        return np.ctypeslib.as_array(out, shape=(int(n.value), 18)).copy()
    finally:
        lib.rptb_free_triangles(out)


def load_obj(path_or_file) -> Mesh:
    """src/io.rs:27-73."""
    if hasattr(path_or_file, "read"):
        return Mesh(parse_obj_native(path_or_file.read()))
    with open(path_or_file, "rb") as f:
        return Mesh(parse_obj_native(f.read()))


def _read_bytes(path_or_file) -> bytes:
    if hasattr(path_or_file, "read"):
        data = path_or_file.read()
        return data.encode() if isinstance(data, str) else bytes(data)
    with open(path_or_file, "rb") as f:
        return f.read()


def _take_triangles(out, n) -> np.ndarray:
    if n == 0:
        return np.zeros((0, 18))
    return np.ctypeslib.as_array(out, shape=(int(n), 18)).copy()


def load_mtl(path_or_file) -> dict:
    """src/io.rs:202-258: `newmtl` starts from Material.default(); Kd -> color, Ns -> roughness =
    (2/(Ns+2))^(1/4), Ni -> index = max(Ni, 1+1e-4), d < 0.8 -> transparent; everything else is
    ignored.  Pure-Python restatement (the native path is rptb_parse_obj_mtl); returns name -> Material."""
    materials: dict = {}
    current = None
    for raw in _read_bytes(path_or_file).decode().split("\n"):
        line = raw.strip()
        if not line or line.startswith("#"):
            continue
        tok = line.split()
        if tok[0] == "newmtl":
            current = tok[1]
            materials.setdefault(current, Material.default())
            continue
        if current is None:
            raise ValueError("Material was not specified with `newmtl` before properties were added")
        mat = materials[current]
        if tok[0] == "Kd":
            mat.color = vec3(float(tok[1]), float(tok[2]), float(tok[3]))
        elif tok[0] == "Ns":
            mat.roughness = math.sqrt(math.sqrt(2.0 / (float(tok[1]) + 2.0)))
        elif tok[0] == "Ni":
            mat.index = max(float(tok[1]), 1.0 + 1e-4)
        elif tok[0] == "d":
            if float(tok[1]) < 0.8:
                mat.transparent = True
    return materials


def parse_obj_with_mtl(lines, materials: dict):
    """Pure-Python restatement of the body of load_obj_with_mtl (src/io.rs:83-149), used to check
    the native parser: returns [(Material, (n, 18) triangles)] in file order."""
    groups = []
    # `replay` holds every v / vn record seen so far, in place, plus the faces of the open run only, so
    # parse_obj(replay) resolves relative indices exactly as the reference does at each face.
    replay: List[str] = []
    open_faces = 0
    current_material = Material.default()
    last_usemtl = None

    def flush():
        nonlocal replay, open_faces
        if open_faces:
            tris = parse_obj(replay)
            if len(tris):  # a run whose faces produced no triangle is not an Object
                groups.append((current_material, tris))
            replay = [ln for ln in replay if ln.split()[0] != "f"]
            open_faces = 0

    for raw in lines:
        line = raw.strip()
        if not line or line.startswith("#"):
            continue
        tok = line.split()
        if tok[0] in ("v", "vn"):
            replay.append(line)
        elif tok[0] == "f":
            replay.append(line)
            open_faces += 1
        elif tok[0] == "usemtl":
            if last_usemtl is None or last_usemtl != tok[1]:
                flush()
                if tok[1] not in materials:
                    raise ValueError(f"Could not found `usemtl {tok[1]}` in library")
                current_material = materials[tok[1]]
                last_usemtl = tok[1]
    flush()
    return groups


def load_obj_with_mtl(obj_file, mtl_file, build: bool = True) -> List["Object"]:
    """src/io.rs:83-149: one Object(Mesh) per run of faces between `usemtl` switches, each carrying
    the material load_mtl derived; `mtllib` lines are ignored (the .mtl is passed explicitly).
    Parsed by the library (rptb_parse_obj_mtl)."""
    obj, mtl = _read_bytes(obj_file), _read_bytes(mtl_file)
    lib = capi.lib()
    out = capi.ObjGroupsOut()
    capi.check(lib.rptb_parse_obj_mtl(obj, len(obj), mtl, len(mtl), C.byref(out)), "rptb_parse_obj_mtl")
    try:
        tris = _take_triangles(out.tris, out.ntris)
        objects = []
        for g in range(int(out.ngroups)):
            grp = out.groups[g]
            m = grp.material
            mat = Material(list(m.color), m.index, m.roughness, m.metallic, m.emittance, bool(m.transparent))
            first, n = int(grp.first_tri), int(grp.ntris)
            objects.append(Object(Mesh(tris[first:first + n], build=build)).material(mat))
        return objects
    finally:
        lib.rptb_free_obj_groups(C.byref(out))


def parse_stl_native(data: bytes) -> np.ndarray:
    """src/io.rs:260-360 through the library (rptb_parse_stl): (n, 18) triangles, every corner
    carrying its facet's stored normal."""
    lib = capi.lib()
    out = capi.c_double_p()
    n = C.c_uint64(0)
    capi.check(lib.rptb_parse_stl(data, len(data), C.byref(out), C.byref(n)), "rptb_parse_stl")
    try:
        return _take_triangles(out, n.value)
    finally:
        lib.rptb_free_triangles(out)


def load_stl(path_or_file) -> Mesh:
    """src/io.rs:260-287: binary or ASCII .STL -> Mesh."""
    return Mesh(parse_stl_native(_read_bytes(path_or_file)))


# ---------------------------------------------------------------- material ----
class Material:
    """src/material.rs:7-26."""

    def __init__(self, color, index: float, roughness: float, metallic: float, emittance: float, transparent: bool):
        self.color = np.asarray(color, dtype=np.float64)
        self.index = float(index)
        self.roughness = float(roughness)
        self.metallic = float(metallic)
        self.emittance = float(emittance)
        self.transparent = bool(transparent)

    @staticmethod
    def default() -> "Material":  # :28-32
        return Material.specular(hex_color(0xFF0000), 0.5)

    @staticmethod
    def diffuse(color) -> "Material":  # :36-45
        return Material(color, 1.5, 1.0, 0.0, 0.0, False)

    @staticmethod
    def specular(color, roughness: float) -> "Material":  # :48-57
        return Material(color, 1.5, roughness, 0.0, 0.0, False)

    @staticmethod
    def clear(index: float, roughness: float) -> "Material":  # :60-69
        return Material(vec3(1.0, 1.0, 1.0), index, roughness, 0.0, 0.0, True)

    @staticmethod
    def transparent_(color, index: float, roughness: float) -> "Material":  # :72-81 (`transparent`)
        return Material(color, index, roughness, 0.0, 0.0, True)

    @staticmethod
    def metallic_(color, roughness: float) -> "Material":  # :84-93 (`metallic`)
        return Material(color, 1.5, roughness, 1.0, 0.0, False)

    @staticmethod
    def light(color, emittance: float) -> "Material":  # :96-105
        return Material(color, 1.0, 1.0, 0.0, emittance, False)

    def to_c(self) -> capi.Material:
        m = capi.Material()
        m.color[:] = list(self.color)
        m.index, m.roughness, m.metallic, m.emittance = self.index, self.roughness, self.metallic, self.emittance
        m.transparent = 1 if self.transparent else 0
        return m


class Object:
    """src/object.rs:10-32: `Object::new(shape).material(m)`."""

    def __init__(self, shape: Shape):
        self.shape = shape
        self.mat = Material.default()

    def material(self, material: Material) -> "Object":
        self.mat = material
        return self


class Light:
    """src/light.rs:7-19."""

    def __init__(self, kind: int, color=None, vec=None, obj: Optional[Object] = None):
        self.kind = kind
        self.color = vec3(0, 0, 0) if color is None else np.asarray(color, dtype=np.float64)
        self.vec = vec3(0, 0, 0) if vec is None else np.asarray(vec, dtype=np.float64)
        self.object = obj

    @staticmethod
    def Point(color, location) -> "Light":
        return Light(capi.LIGHT_POINT, color, location)

    @staticmethod
    def Ambient(color) -> "Light":
        return Light(capi.LIGHT_AMBIENT, color)

    @staticmethod
    def Directional(color, direction) -> "Light":
        return Light(capi.LIGHT_DIRECTIONAL, color, direction)

    @staticmethod
    def Object(obj: Object) -> "Light":
        return Light(capi.LIGHT_OBJECT, obj=obj)


class Hdri:
    """src/environment.rs:4-23."""

    def __init__(self, width: int, height: int, buf):
        buf = np.ascontiguousarray(np.asarray(buf, dtype=np.float64).reshape(-1, 3))
        assert buf.shape[0] == width * height
        assert width > 0 and height > 0
        self.width, self.height, self.buf = int(width), int(height), buf


class Environment:
    """src/environment.rs:55-70."""

    def __init__(self, color=None, hdri: Optional[Hdri] = None):
        self.color = vec3(0, 0, 0) if color is None else np.asarray(color, dtype=np.float64)
        self.hdri = hdri

    @staticmethod
    def Color(color) -> "Environment":
        return Environment(color=color)

    @staticmethod
    def Hdri(hdri: Hdri) -> "Environment":
        return Environment(hdri=hdri)


class Scene:
    """src/scene.rs:7-41."""

    def __init__(self):
        self.objects: List[Object] = []
        self.lights: List[Light] = []
        self.environment = Environment()

    def add(self, node) -> None:  # SceneAdd<Object> / SceneAdd<Light>
        if isinstance(node, Object):
            self.objects.append(node)
        elif isinstance(node, Light):
            self.lights.append(node)
        else:
            raise TypeError("Scene.add takes an Object or a Light")


class Camera:
    """src/camera.rs:8-61."""

    def __init__(self, eye=None, direction=None, up=None, fov: float = math.pi / 6, aperture: float = 0.0,
                 focal_distance: float = 0.0):
        self.eye = vec3(0.0, 0.0, 10.0) if eye is None else np.asarray(eye, dtype=np.float64)
        self.direction = vec3(0.0, 0.0, -1.0) if direction is None else np.asarray(direction, dtype=np.float64)
        self.up = vec3(0.0, 1.0, 0.0) if up is None else np.asarray(up, dtype=np.float64)
        self.fov, self.aperture, self.focal_distance = float(fov), float(aperture), float(focal_distance)

    @staticmethod
    def default() -> "Camera":
        return Camera()

    @staticmethod
    def look_at(eye, center, up, fov: float) -> "Camera":  # :43-54
        eye, center, up = (np.asarray(v, dtype=np.float64) for v in (eye, center, up))
        direction = center - eye
        direction = direction / np.linalg.norm(direction)
        up = up - np.dot(up, direction) * direction
        up = up / np.linalg.norm(up)
        return Camera(eye, direction, up, fov)

    def focus(self, focal_point, aperture: float) -> "Camera":  # :57-61
        self.focal_distance = float(np.dot(np.asarray(focal_point, dtype=np.float64) - self.eye, self.direction))
        self.aperture = float(aperture)
        return self

    def to_c(self) -> capi.Camera:
        c = capi.Camera()
        c.eye[:] = list(self.eye)
        c.direction[:] = list(self.direction)
        c.up[:] = list(self.up)
        c.fov, c.aperture, c.focal_distance = self.fov, self.aperture, self.focal_distance
        return c


# ------------------------------------------------------ Scene -> rptb_scene_desc
class FlatScene:
    """Owns the ctypes arrays a rptb_scene_desc points into (caller-owned memory
    borrowed by rptb_scene_create for the duration of the call)."""

    def __init__(self, scene: Scene, accel: int = capi.ACCEL_AUTO):
        self._keep: list = []
        mats: List[capi.Material] = []
        meshes: List[capi.Mesh] = []
        mesh_index: dict = {}

        def add_material(m: Material) -> int:
            mats.append(m.to_c())
            return len(mats) - 1

        def add_mesh(mesh: Mesh) -> int:
            key = id(mesh)
            if key in mesh_index:
                return mesh_index[key]
            cm = capi.Mesh()
            cm.tris = mesh.triangles.ctypes.data_as(capi.c_double_p)
            cm.ntris = mesh.triangles.shape[0]
            if mesh.nodes is not None:
                cm.nodes = C.cast(mesh.nodes, C.POINTER(capi.KdNode))
                cm.nnodes = len(mesh.nodes)
                cm.refs = mesh.refs.ctypes.data_as(capi.c_u32_p)
                cm.nrefs = mesh.refs.shape[0]
            self._keep.append(mesh)
            meshes.append(cm)
            mesh_index[key] = len(meshes) - 1
            return mesh_index[key]

        groups: List[capi.Group] = []

        def add_group(tree: KdTree) -> int:
            children = (capi.Object * max(len(tree.objects), 1))(*[to_shape(c) for c in tree.objects])
            self._keep.append(children)
            g = capi.Group()
            g.children, g.nchildren = children, len(tree.objects)
            groups.append(g)  # nodes stay NULL: the library runs `construct` over the children's boxes
            return len(groups) - 1

        def to_shape(shape: Shape) -> capi.Object:
            co = capi.Object()
            if isinstance(shape, Transformed):
                co.has_transform = 1
                co.transform[:] = list(shape.matrix.T.reshape(-1))  # column-major
                shape = shape.shape
            else:
                co.has_transform = 0
                co.transform[:] = list(np.eye(4).reshape(-1))
            co.kind = shape.kind
            if isinstance(shape, Plane):
                co.plane_normal[:] = list(shape.normal)
                co.plane_value = shape.value
            if isinstance(shape, MonomialSurface):
                co.monomial_height, co.monomial_exp = shape.height, shape.exp
            if isinstance(shape, Mesh):
                co.mesh = add_mesh(shape)
            if isinstance(shape, KdTree):
                co.mesh = add_group(shape)
            return co

        def to_object(o: Object) -> capi.Object:
            co = to_shape(o.shape)
            co.material = add_material(o.mat)
            return co

        objs = [to_object(o) for o in scene.objects]
        lights = []
        for l in scene.lights:
            cl = capi.Light()
            cl.kind = l.kind
            cl.color[:] = list(l.color)
            cl.vec[:] = list(l.vec)
            if l.kind == capi.LIGHT_OBJECT:
                cl.object = to_object(l.object)
            lights.append(cl)

        self.materials = (capi.Material * max(len(mats), 1))(*mats)
        self.meshes = (capi.Mesh * max(len(meshes), 1))(*meshes)
        self.objects = (capi.Object * max(len(objs), 1))(*objs)
        self.lights = (capi.Light * max(len(lights), 1))(*lights)
        d = capi.SceneDesc()
        d.materials, d.nmaterials = self.materials, len(mats)
        d.meshes, d.nmeshes = self.meshes, len(meshes)
        self.groups = (capi.Group * max(len(groups), 1))(*groups)
        d.groups, d.ngroups = self.groups, len(groups)
        d.accel = int(accel)
        d.objects, d.nobjects = self.objects, len(objs)
        d.lights, d.nlights = self.lights, len(lights)
        env = scene.environment
        if env.hdri is not None:
            d.environment.kind = capi.ENV_HDRI
            d.environment.width, d.environment.height = env.hdri.width, env.hdri.height
            d.environment.texels = env.hdri.buf.ctypes.data_as(capi.c_double_p)
            self._keep.append(env.hdri)
        else:
            d.environment.kind = capi.ENV_COLOR
            d.environment.color[:] = list(env.color)
        self.desc = d

    def host_bytes(self) -> int:
        """Bytes rptb_scene_create reads from the host (the per-call H2D payload)."""
        n = C.sizeof(self.materials) + C.sizeof(self.objects) + C.sizeof(self.lights)
        for i in range(self.desc.nmeshes):
            m = self.meshes[i]
            n += m.ntris * 18 * 8 + m.nnodes * C.sizeof(capi.KdNode) + m.nrefs * 4
        for i in range(self.desc.ngroups):
            n += self.groups[i].nchildren * C.sizeof(capi.Object)
        if self.desc.environment.kind == capi.ENV_HDRI:
            n += self.desc.environment.width * self.desc.environment.height * 24
        return int(n)


class DeviceScene:
    """RAII wrapper of the opaque rptb_scene handle."""

    def __init__(self, scene_or_flat, device=0, accel: int = capi.ACCEL_AUTO):
        """`device`: one CUDA device index, or a sequence of them -> rptb_scene_create_multi (the scene replicated
        on every listed GPU; Renderer::sample then fans out over them inside rptb_render_samples)."""
        self.flat = scene_or_flat if isinstance(scene_or_flat, FlatScene) else FlatScene(scene_or_flat, accel)
        self.handle = C.c_void_p()
        if isinstance(device, (list, tuple)):
            self.devices = [int(d) for d in device]
            arr = (C.c_int * len(self.devices))(*self.devices)
            self.device = self.devices[0]
            capi.check(capi.lib().rptb_scene_create_multi(C.byref(self.flat.desc), arr, len(self.devices), C.byref(self.handle)),
                       "rptb_scene_create_multi")
        else:
            self.device = int(device)
            self.devices = [self.device]
            capi.check(capi.lib().rptb_scene_create(C.byref(self.flat.desc), self.device, C.byref(self.handle)),
                       "rptb_scene_create")

    def device_count(self) -> int:
        return int(capi.lib().rptb_scene_device_count(self.handle))

    # Light::illuminate of scene.lights[light] at a batch of positions (src/light.rs:23-47)
    def illuminate(self, light: int, pos: np.ndarray, seed: int = 0, precision: int = capi.PRECISION_F32):
        pos = np.ascontiguousarray(pos, dtype=np.float64).reshape(-1, 3)
        n = pos.shape[0]
        inten = np.empty((n, 3), np.float64)
        wi = np.empty((n, 3), np.float64)
        dist = np.empty(n, np.float64)
        capi.check(
            capi.lib().rptb_illuminate(self.handle, light, pos.ctypes.data_as(capi.c_double_p), n, seed, precision,
                                       inten.ctypes.data_as(capi.c_double_p), wi.ctypes.data_as(capi.c_double_p),
                                       dist.ctypes.data_as(capi.c_double_p)),
            "rptb_illuminate",
        )
        return inten, wi, dist

    def close(self) -> None:
        if self.handle:
            capi.lib().rptb_scene_destroy(self.handle)
            self.handle = C.c_void_p()

    def device_bytes(self) -> int:
        return int(capi.lib().rptb_scene_device_bytes(self.handle))

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # Renderer::get_closest_hit for a batch of rays (src/renderer.rs:211-220)
    def closest_hit(self, rays: np.ndarray, t_min: float = 1e-12, precision: int = capi.PRECISION_F32,
                    want_stats: bool = False):
        rays = np.ascontiguousarray(rays, dtype=np.float64).reshape(-1, 6)
        n = rays.shape[0]
        t = np.empty(n, np.float64)
        obj = np.empty(n, np.int32)
        nrm = np.empty((n, 3), np.float64)
        stats = capi.Stats()
        capi.check(
            capi.lib().rptb_closest_hit(self.handle, rays.ctypes.data_as(capi.c_double_p), n, t_min, precision,
                                        t.ctypes.data_as(capi.c_double_p), obj.ctypes.data_as(capi.c_i32_p),
                                        nrm.ctypes.data_as(capi.c_double_p), C.byref(stats) if want_stats else None),
            "rptb_closest_hit",
        )
        return (t, obj, nrm, stats.as_dict()) if want_stats else (t, obj, nrm)


# ------------------------------------------------------------------ buffer ----
class Filter:
    """src/buffer.rs:95-108."""

    def __init__(self, radius: int = 0):
        self.radius = int(radius)

    @staticmethod
    def Box(radius: int) -> "Filter":
        return Filter(radius)


class Adaptive:
    """The convergence criterion of adaptive sampling (rptb_adaptive): Renderer.sample(n, device_buffer, adaptive=...)
    renders only the pixels that are still active.  A pixel with n entries is active while n < min_entries, or while
    the channel-mean variance of its mean, M2 / ((n - 1) n 3), exceeds (rel_tol * mean + abs_tol)^2.  Defaults: stop
    at 2 % relative error of the mean or 1/1000 absolute, and never before 4 entries (the guard against a dark pixel
    whose first entries happen to agree).
    `guide` (a Denoise): test the value the denoiser will show instead of the raw mean (rptb_sample_into_guided).  Each
    call first runs the filter with those parameters over the buffer, and a pixel is active while n < min_entries, or
    while the variance of its denoised value, v' (DeviceBuffer.denoised_variance), exceeds (rel_tol * m' + abs_tol)^2,
    m' the channel mean of its denoised colour.  The buffer needs features (Renderer.sample_features) and entries made
    through the renderer's camera alone; guide.iterations == 0 is the plain criterion.  rpt_b200/csrc/guided.h gives
    every formula; DESIGN.md section 6e what it buys and where it loses.
    `estimate` (with a guide): which variance of the denoised value the test uses.  "filter" (the default) is v', the
    filter's own; "halves" is E (DeviceBuffer.denoised_error, rptb_sample_into_guided_error), estimated from two half
    buffers, which needs a buffer with halves (Renderer.device_buffer(halves=True)) and guide.iterations >= 1.  v'
    underestimates the variance 10-31x, E 4-7x; with E, rel_tol 0.05 is the recommended setting (DESIGN.md section 6g,
    BASELINE.md section 3.0h)."""

    ESTIMATES = ("filter", "halves")

    def __init__(self, rel_tol: float = 0.02, abs_tol: float = 1e-3, min_entries: int = 4, guide: Optional["Denoise"] = None,
                 estimate: str = "filter"):
        self.rel_tol, self.abs_tol, self.min_entries = float(rel_tol), float(abs_tol), int(min_entries)
        if guide is not None and not isinstance(guide, Denoise):
            raise TypeError(f"guide must be an api.Denoise, not {type(guide).__name__}")
        if estimate not in Adaptive.ESTIMATES:
            raise ValueError(f"estimate must be one of {Adaptive.ESTIMATES}, not {estimate!r}")
        if estimate == "halves" and guide is None:
            raise ValueError('estimate="halves" estimates the denoised value\'s error: it needs a guide (Denoise)')
        self.guide, self.estimate = guide, estimate

    def to_c(self) -> capi.Adaptive:
        return capi.Adaptive(self.rel_tol, self.abs_tol, self.min_entries, 0)

    def active(self, counts, sums, m2) -> np.ndarray:
        """The criterion in numpy on per-pixel (counts, sums (n, 3), M2): the same operations in the same order as the
        device (rpt_b200/csrc/adaptive.h), so the same decisions."""
        n = np.asarray(counts, dtype=np.float64)
        s = np.asarray(sums, dtype=np.float64).reshape(-1, 3)
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            err2 = np.asarray(m2, dtype=np.float64) / (((n - 1.0) * n) * 3.0)
            m = ((s[:, 0] + s[:, 1]) + s[:, 2]) / (3.0 * n)
            t = self.rel_tol * m + self.abs_tol
            converged = err2 <= t * t
        return (np.asarray(counts) < self.min_entries) | ~converged


class Denoise:
    """Parameters of DeviceBuffer.denoise (rptb_denoise), which stands beside the reference's Filter::Box: the spatial
    part of SVGF, an edge-avoiding a-trous wavelet filter guided by the buffer's first-hit features (normal, depth,
    albedo) and by each pixel's variance of the mean.  `iterations` passes (0 = the mean itself, at most 12);
    sigma_normal is the exponent of the normal weight, sigma_depth and sigma_luminance the depth and luminance
    tolerances, albedo_eps what is added to the albedo before the colour is divided by it.  albedo_eps must be finite and
    > 0: a pixel whose feature rays all hit a black surface has albedo 0, and dividing by it would make that pixel NaN
    even where its mean is 0.  A tiny albedo_eps still overflows once mean / albedo_eps leaves the double range (about
    1e-303 for a mean of 1e6).  rpt_b200/csrc/denoise.h gives every formula."""

    def __init__(self, iterations: int = 5, sigma_normal: int = 128, sigma_depth: float = 1.0, sigma_luminance: float = 4.0,
                 albedo_eps: float = 1e-3):
        self.iterations, self.sigma_normal = int(iterations), int(sigma_normal)
        self.sigma_depth, self.sigma_luminance, self.albedo_eps = float(sigma_depth), float(sigma_luminance), float(albedo_eps)

    def to_c(self) -> capi.Denoise:
        return capi.Denoise(self.iterations, self.sigma_normal, self.sigma_depth, self.sigma_luminance, self.albedo_eps)


class Reproject:
    """Parameters of DeviceBuffer.reproject_from (rptb_reproject): how a pixel of the new view decides which pixels of the
    old view saw the same surface.  depth_tol: the largest |z_q - l| / l between an old pixel's first-hit depth z_q and
    the distance l from the old eye to the new pixel's first hit; normal_cos: the least dot product of the two
    first-hit normals; max_history: the most entries a reprojected pixel keeps, which bounds how long a view-dependent
    highlight lags behind the camera.  Defaults 0.02, 0.9, 8: over 16-frame orbits of the sphere, Cornell, the teapot
    and glass they are the setting of tools/reproject_measure.py's sweep under which no scene's raw MSE loses to fresh
    frames, and the best for the denoised ones (DESIGN.md section 6c).  rpt_b200/csrc/reproject.h gives every formula."""

    def __init__(self, depth_tol: float = 0.02, normal_cos: float = 0.9, max_history: int = 8):
        self.depth_tol, self.normal_cos, self.max_history = float(depth_tol), float(normal_cos), int(max_history)

    def to_c(self) -> capi.Reproject:
        return capi.Reproject(self.depth_tol, self.normal_cos, self.max_history, 0)


class HistoryTest:
    """Testing reprojected history against fresh entries (DeviceBuffer.merge_history_from, rptb_buffer_reproject_merge;
    render_frames(history_test=...)).  A frame first renders `fresh_entries` plain entries (>= 2: a mean and a
    variance per pixel), then each pixel's history is merged in only where it agrees with them: it is rejected when
    the squared distance of the two means exceeds gamma^2 times the variance of their difference.  gamma = inf accepts
    every history, 0 rejects any that differs.  Default gamma 4: of tools/reproject_measure.py's sweep over gamma in
    {2, 3, 4, 6} on 16-frame orbits of the sphere, Cornell, the teapot and glass at 4 and 16 fresh spp, it gives the best
    geometric mean of the denoised gains over fresh frames (DESIGN.md section 6c).  rpt_b200/csrc/reproject.h gives
    every formula."""

    def __init__(self, gamma: float = 4.0, fresh_entries: int = 2):
        self.gamma, self.fresh_entries = float(gamma), int(fresh_entries)


class Buffer:
    """src/buffer.rs:6-93.  Holds one equally weighted entry per pixel per
    `add_samples` call, like the reference's Vec<Vec<Color>>."""

    def __init__(self, width: int, height: int, filter: Optional[Filter] = None, device: int = 0):
        self.width, self.height = int(width), int(height)
        self.filter = filter or Filter()
        self.batches: List[np.ndarray] = []
        self.device = device

    def add_samples(self, samples) -> None:  # :32-40
        samples = np.asarray(samples, dtype=np.float64).reshape(-1, 3)
        assert samples.shape[0] == self.width * self.height, "Invalid sample dimension"
        self.batches.append(samples)

    def image(self) -> np.ndarray:
        """:43-56 -> (height, width, 3) uint8, resolved on the device (rptb_film_resolve)."""
        assert self.batches, "Pixel found with no samples"
        sums = np.ascontiguousarray(np.sum(self.batches, axis=0))
        out = np.empty((self.height, self.width, 3), np.uint8)
        capi.check(
            capi.lib().rptb_film_resolve(sums.ctypes.data_as(capi.c_double_p), len(self.batches), self.width,
                                         self.height, self.filter.radius, self.device,
                                         out.ctypes.data_as(capi.c_u8_p)),
            "rptb_film_resolve",
        )
        return out

    def variance(self) -> float:
        """:59-73, on the device (rptb_film_variance).  With a single entry per pixel the reference
        divides by n - 1 = 0 and returns NaN; so does this."""
        if len(self.batches) < 2:
            return float("nan")
        b = np.ascontiguousarray(np.stack(self.batches))  # (nb, npix, 3)
        out = C.c_double(0.0)
        capi.check(capi.lib().rptb_film_variance(b.ctypes.data_as(capi.c_double_p), b.shape[0], b.shape[1],
                                                 self.device, C.byref(out)), "rptb_film_variance")
        return float(out.value)


class DeviceBuffer:
    """src/buffer.rs:6-93 kept in device memory (rptb_buffer): per pixel the running sum of its entries and a
    streaming variance, on every GPU of the scene it was made for.  Renderer.sample adds an entry without
    copying the render to the host, and image() / variance() cost O(width * height) however many entries it
    holds.  The numbers are those of the host Buffer over the same entries: sums() is np.sum(batches, axis=0)
    bit for bit, image() gives the same bytes, variance() agrees to rounding (Welford instead of two passes)."""

    shard: Optional[tuple] = None  # (shard_index, shard_count) of a distributed.ShardBuffer; None = the whole image

    def __init__(self, scene: DeviceScene, width: int, height: int, filter: Optional[Filter] = None, halves: bool = False):
        """`halves`: also keep the sums of each pixel's odd entries (rptb_buffer_create_halves, 24 more bytes a pixel),
        from which denoised_error() estimates the denoised image's error.  Everything else is the same bits either way."""
        self.width, self.height = int(width), int(height)
        self.filter = filter or Filter()
        self.devices = list(scene.devices)
        self.entries = 0  # the most entries any pixel holds (every pixel, without adaptive calls)
        self.feature_rays = 0  # camera rays per pixel in the features (Renderer.sample_features)
        self.halves = bool(halves)
        self.handle = C.c_void_p()
        create = capi.lib().rptb_buffer_create_halves if self.halves else capi.lib().rptb_buffer_create
        capi.check(create(scene.handle, self.width, self.height, self.filter.radius, C.byref(self.handle)),
                   "rptb_buffer_create_halves" if self.halves else "rptb_buffer_create")

    def add_samples(self, samples) -> None:  # :32-40
        samples = np.ascontiguousarray(np.asarray(samples, dtype=np.float64).reshape(-1, 3))
        assert samples.shape[0] == self.width * self.height, "Invalid sample dimension"
        capi.check(capi.lib().rptb_buffer_add_samples(self.handle, samples.ctypes.data_as(capi.c_double_p)),
                   "rptb_buffer_add_samples")
        self.entries += 1

    def sums(self) -> np.ndarray:
        """(width * height, 3) per-pixel sums over the entries, row-major."""
        out = np.empty((self.width * self.height, 3), np.float64)
        n = C.c_uint32(0)
        capi.check(capi.lib().rptb_buffer_sums(self.handle, out.ctypes.data_as(capi.c_double_p), C.byref(n)),
                   "rptb_buffer_sums")
        self.entries = int(n.value)
        return out

    def pixel_stats(self):
        """Per pixel, row-major: (sums (width * height, 3), M2 (width * height,) summed over the channels, entry counts
        (width * height,) uint32)."""
        npix = self.width * self.height
        sums, m2, counts = np.empty((npix, 3), np.float64), np.empty(npix, np.float64), np.empty(npix, np.uint32)
        capi.check(capi.lib().rptb_buffer_pixel_stats(self.handle, sums.ctypes.data_as(capi.c_double_p),
                                                      m2.ctypes.data_as(capi.c_double_p),
                                                      counts.ctypes.data_as(capi.c_u32_p)), "rptb_buffer_pixel_stats")
        return sums, m2, counts

    def counts(self) -> np.ndarray:
        """(height, width) entries per pixel."""
        out = np.empty(self.width * self.height, np.uint32)
        capi.check(capi.lib().rptb_buffer_pixel_stats(self.handle, None, None, out.ctypes.data_as(capi.c_u32_p)),
                   "rptb_buffer_pixel_stats")
        return out.reshape(self.height, self.width)

    def image(self) -> np.ndarray:
        """:43-56 -> (height, width, 3) uint8."""
        out = np.empty((self.height, self.width, 3), np.uint8)
        capi.check(capi.lib().rptb_buffer_image(self.handle, out.ctypes.data_as(capi.c_u8_p)), "rptb_buffer_image")
        return out

    def variance(self) -> float:
        """:59-73.  NaN with fewer than two entries, like the reference."""
        out = C.c_double(0.0)
        capi.check(capi.lib().rptb_buffer_variance(self.handle, C.byref(out)), "rptb_buffer_variance")
        return float(out.value)

    def features(self):
        """The first-hit features added by Renderer.sample_features, row-major: (normal (H, W, 3), 0 where nothing was
        hit; depth (H, W), +inf where nothing was hit; albedo (H, W, 3), a miss counting 1; hit fraction (H, W))."""
        h, w = self.height, self.width
        nrm, depth, alb, frac = np.empty((h, w, 3)), np.empty((h, w)), np.empty((h, w, 3)), np.empty((h, w))
        capi.check(capi.lib().rptb_buffer_features(self.handle, nrm.ctypes.data_as(capi.c_double_p), depth.ctypes.data_as(capi.c_double_p),
                                                   alb.ctypes.data_as(capi.c_double_p), frac.ctypes.data_as(capi.c_double_p)),
                   "rptb_buffer_features")
        return nrm, depth, alb, frac

    def denoise(self, d: Optional[Denoise] = None) -> np.ndarray:
        """The mean image through the edge-avoiding filter: (H, W, 3) float64, linear.  Needs features and at least two
        entries per pixel."""
        out = np.empty((self.height, self.width, 3))
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise(self.handle, C.byref(c), out.ctypes.data_as(capi.c_double_p), None),
                   "rptb_buffer_denoise")
        return out

    def denoised_variance(self, d: Optional[Denoise] = None) -> np.ndarray:
        """The variance of each pixel of denoise(d), as the filter estimates it (rptb_buffer_denoise_variance): (H, W)
        float64, in the filter's radiance units -- an error map of the denoised image.  It treats each pass's inputs as
        independent, so it underestimates the true variance (DESIGN.md section 6e).  Refusals as denoise()."""
        out = np.empty((self.height, self.width))
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise_variance(self.handle, C.byref(c), out.ctypes.data_as(capi.c_double_p)),
                   "rptb_buffer_denoise_variance")
        return out

    def half_sums(self) -> np.ndarray:
        """(width * height, 3) per-pixel sums of the odd entries (entry k, counted from 0, for odd k), row-major.  Needs
        a buffer with halves."""
        out = np.empty((self.width * self.height, 3), np.float64)
        capi.check(capi.lib().rptb_buffer_half_sums(self.handle, out.ctypes.data_as(capi.c_double_p)), "rptb_buffer_half_sums")
        return out

    def denoised_error(self, d: Optional[Denoise] = None) -> np.ndarray:
        """E, the variance of each pixel of denoise(d) estimated from two half buffers (rptb_buffer_denoise_error): (H, W)
        float64, in the units of denoised_variance().  Unlike v' it accounts for the correlation between the filter's
        passes (DESIGN.md section 6g).  Needs a buffer with halves and d.iterations >= 1; otherwise refusals as denoise()."""
        out = np.empty((self.height, self.width))
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise_error(self.handle, C.byref(c), out.ctypes.data_as(capi.c_double_p)),
                   "rptb_buffer_denoise_error")
        return out

    def denoised_image(self, d: Optional[Denoise] = None) -> np.ndarray:
        """denoise() through Buffer::image's clamp, gamma and cast (no box filter): (H, W, 3) uint8."""
        out = np.empty((self.height, self.width, 3), np.uint8)
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise(self.handle, C.byref(c), None, out.ctypes.data_as(capi.c_u8_p)),
                   "rptb_buffer_denoise")
        return out

    def denoise_select(self, d: Optional[Denoise] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """denoise(d) with each pixel's number of passes chosen by the estimated error of each level
        (rptb_buffer_denoise_select): level k is denoise(Denoise(iterations=k, ...)), and each pixel keeps the level
        whose error, estimated from the two half buffers and smoothed over 5x5, is least (DESIGN.md section 6h).
        Returns (rgb (H, W, 3) float64, level (H, W) uint8, mse (H, W) float64): every rgb pixel is that level's denoise
        output bit for bit, and mse is the estimated squared error (bias included) at the chosen level, in the units of
        denoised_variance().  Needs a buffer with halves and d.iterations >= 1; otherwise refusals as denoise()."""
        h, w = self.height, self.width
        rgb, level, mse = np.empty((h, w, 3)), np.empty((h, w), np.uint8), np.empty((h, w))
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise_select(self.handle, C.byref(c), rgb.ctypes.data_as(capi.c_double_p), None,
                                                         level.ctypes.data_as(capi.c_u8_p), mse.ctypes.data_as(capi.c_double_p)),
                   "rptb_buffer_denoise_select")
        return rgb, level, mse

    def selected_image(self, d: Optional[Denoise] = None) -> np.ndarray:
        """denoise_select()'s colour through Buffer::image's clamp, gamma and cast, as denoised_image(): (H, W, 3) uint8."""
        out = np.empty((self.height, self.width, 3), np.uint8)
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise_select(self.handle, C.byref(c), None, out.ctypes.data_as(capi.c_u8_p), None, None),
                   "rptb_buffer_denoise_select")
        return out

    def denoise_cross(self, d: Optional[Denoise] = None) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """The buffer denoised by cross-filtering with a smoothed selection map (rptb_buffer_denoise_cross): each half is
        filtered through d.iterations passes whose weights come from the other half's own passes, level k (0 ..
        d.iterations) is the count-weighted mean of the two filtered halves (level 0 the raw mean), and each pixel blends
        the levels by the 5x5-smoothed share of its neighbours whose estimated error is least at each level (DESIGN.md
        section 6i).  Returns (rgb (H, W, 3) float64, level (H, W) uint8, mse (H, W) float64): the blended colour, each
        pixel's own least-error level, and the estimated squared error (bias included) blended with the colour's weights,
        in the units of denoised_variance().  Needs a buffer with halves and d.iterations >= 1; otherwise refusals as
        denoise()."""
        h, w = self.height, self.width
        rgb, level, mse = np.empty((h, w, 3)), np.empty((h, w), np.uint8), np.empty((h, w))
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise_cross(self.handle, C.byref(c), rgb.ctypes.data_as(capi.c_double_p), None,
                                                        level.ctypes.data_as(capi.c_u8_p), mse.ctypes.data_as(capi.c_double_p)),
                   "rptb_buffer_denoise_cross")
        return rgb, level, mse

    def cross_image(self, d: Optional[Denoise] = None) -> np.ndarray:
        """denoise_cross()'s colour through Buffer::image's clamp, gamma and cast, as denoised_image(): (H, W, 3) uint8."""
        out = np.empty((self.height, self.width, 3), np.uint8)
        c = (d or Denoise()).to_c()
        capi.check(capi.lib().rptb_buffer_denoise_cross(self.handle, C.byref(c), None, out.ctypes.data_as(capi.c_u8_p), None, None),
                   "rptb_buffer_denoise_cross")
        return out

    def reproject_from(self, src: "DeviceBuffer", params: Optional[Reproject] = None) -> int:
        """Carries `src`'s entries over a camera move into this buffer, which must hold features (Renderer.sample_features
        through its camera) and no entries; `src` must hold entries and features made through one camera.  Each pixel
        takes the history of the old pixels that saw its first-hit point, or none (count 0: a disocclusion or the edge of
        the old view, which an adaptive sample() renders first).  Returns the number of pixels that got history.

        A buffer with halves takes history with halves from a `src` with halves: each pixel's HALF is scaled so that
        denoised_error and Adaptive(estimate="halves") see the variance of the mean its capped count claims
        (rpt_b200/csrc/reproject.h).  From a plain `src` it raises RptbError (RPTB_ERR_UNSUPPORTED).  A plain buffer
        ignores a `src`'s halves; the sums, M2 and counts are the same bits either way."""
        c = (params or Reproject()).to_c()
        n = C.c_uint64(0)
        capi.check(capi.lib().rptb_buffer_reproject(self.handle, src.handle, C.byref(c), C.byref(n)), "rptb_buffer_reproject")
        self.entries = int(self.counts().max())
        return int(n.value)

    def merge_history_from(self, src: "DeviceBuffer", reproject: Optional[Reproject] = None,
                           test: Optional[HistoryTest] = None) -> tuple:
        """Tests the history reproject_from would carry from `src` against this buffer's own fresh entries, and merges it
        only where they agree (rptb_buffer_reproject_merge).  This buffer must hold features and >= 2 entry calls, all
        through its feature camera, and must not be reprojected; `src` as for reproject_from.  A merged pixel holds both
        groups' entries, and the gap between their means goes into its variance; a rejected one keeps its fresh entries
        only.  Returns (reused, rejected) pixel counts; pixels with no history are in neither.  A buffer with halves needs
        a `src` with halves, as for reproject_from, and a merged pixel's HALF takes the history's half that keeps "entry
        k goes into HALF iff k is odd" true."""
        c = (reproject or Reproject()).to_c()
        gamma = (test or HistoryTest()).gamma
        n, j = C.c_uint64(0), C.c_uint64(0)
        capi.check(capi.lib().rptb_buffer_reproject_merge(self.handle, src.handle, C.byref(c), gamma, C.byref(n), C.byref(j)),
                   "rptb_buffer_reproject_merge")
        self.entries = int(self.counts().max())
        return int(n.value), int(j.value)

    def close(self) -> None:
        if self.handle:
            capi.lib().rptb_buffer_destroy(self.handle)
            self.handle = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---------------------------------------------------------------- renderer ----
class Renderer:
    """src/renderer.rs:18-115.  Builder methods carry the reference's names; the
    private `sample` (:117-129) is the seam where the CUDA library is called."""

    def __init__(self, scene: Scene, camera: Camera):
        self.scene = scene
        self.camera = camera
        self._width, self._height = 800, 600  # :46-57 defaults
        self._exposure_value = 0.0
        self._filter = Filter()
        self._max_bounces = 0
        self._num_samples = 1
        # not in the reference (its RNG is OS entropy): reproducible stream + device choice
        self._seed = 0
        self._device = 0
        self._precision = capi.PRECISION_F32
        self._engine = capi.ENGINE_AUTO
        self._accel = capi.ACCEL_AUTO
        self._dev_scene: Optional[DeviceScene] = None
        self._next_sample = 0
        self.last_stats: Optional[dict] = None

    def width(self, width: int) -> "Renderer":
        self._width = int(width)
        return self

    def height(self, height: int) -> "Renderer":
        self._height = int(height)
        return self

    def exposure_value(self, ev: float) -> "Renderer":
        self._exposure_value = float(ev)
        return self

    def filter(self, f: Filter) -> "Renderer":
        self._filter = f
        return self

    def max_bounces(self, n: int) -> "Renderer":
        self._max_bounces = int(n)
        return self

    def num_samples(self, n: int) -> "Renderer":
        self._num_samples = int(n)
        return self

    def seed(self, seed: int) -> "Renderer":
        self._seed = int(seed)
        return self

    def device(self, device) -> "Renderer":
        """One CUDA device index, or a list of them: Renderer::sample then fans out over those GPUs behind the
        same rptb_render_samples call (rptb_scene_create_multi)."""
        self._device = [int(d) for d in device] if isinstance(device, (list, tuple)) else int(device)
        return self

    def precision(self, precision: int) -> "Renderer":
        self._precision = int(precision)
        return self

    def engine(self, engine: int) -> "Renderer":
        self._engine = int(engine)
        return self

    def accel(self, accel: int) -> "Renderer":
        """rptb_accel: what the f32 path traverses meshes with (capi.ACCEL_KDTREE = the reference-shaped tree,
        capi.ACCEL_BVH = the library's own BVH).  Takes effect when the device scene is created."""
        self._accel = int(accel)
        return self

    def params(self, iterations: int, first_sample: int = 0, shard_index: int = 0, shard_count: int = 1,
               collect_stats: int = 0) -> capi.RenderParams:
        p = capi.RenderParams()
        p.width, p.height = self._width, self._height
        p.iterations, p.max_bounces = int(iterations), self._max_bounces
        p.exposure_value = self._exposure_value
        p.seed, p.first_sample = self._seed, int(first_sample)
        p.shard_index, p.shard_count = shard_index, shard_count
        p.precision = self._precision
        p.collect_stats = collect_stats
        p.engine = self._engine
        return p

    def _first_device(self) -> int:
        return self._device[0] if isinstance(self._device, list) else self._device

    def device_scene(self) -> DeviceScene:
        if self._dev_scene is None:
            self._dev_scene = DeviceScene(self.scene, self._device, self._accel)
        return self._dev_scene

    def close(self) -> None:
        if self._dev_scene is not None:
            self._dev_scene.close()
            self._dev_scene = None

    def device_buffer(self, halves: bool = False) -> DeviceBuffer:
        """A DeviceBuffer of this renderer's size and filter on the GPUs of its device scene; `halves`: one with halves
        (DeviceBuffer), which Adaptive(estimate="halves") needs."""
        return DeviceBuffer(self.device_scene(), self._width, self._height, self._filter, halves=halves)

    # ---- the seam: Renderer::sample (:117-129) ---------------------------------
    _NO_GUIDE_BUFFER = object()

    def sample(self, iterations: int, buffer, collect_stats: int = 0, want_stats: bool = True,
               adaptive: Optional[Adaptive] = None, guide_buffer=_NO_GUIDE_BUFFER) -> Optional[int]:
        """Adds one entry of `iterations` samples per pixel to `buffer`.  A host Buffer gets the image through
        host memory; a DeviceBuffer gets it on the device, and the call returns once the work is enqueued unless
        `want_stats` (then last_stats is filled, which waits for the render).
        `adaptive` (DeviceBuffer only): add the entry only to the pixels the criterion leaves active
        (rptb_sample_into_adaptive, or rptb_sample_into_guided with adaptive.guide, or rptb_sample_into_guided_error with
        estimate="halves"); returns how many pixels got it, which waits for the call.
        A distributed.ShardBuffer renders and adds its own shard's tiles only; `adaptive` then counts its pixels.
        `guide_buffer` (a ShardBuffer with a guided `adaptive`; rptb_sample_into_guided_shard): the whole DeviceBuffer the
        shard's filter runs over -- every shard gathered with features on this rank's device, at the shard's current state
        (ShardBuffer.gather, then ShardBuffer.gather_delta after each call).  None is allowed while the shard has fewer
        than adaptive.min_entries calls, when the plain mark decides.  With estimate="halves"
        (rptb_sample_into_guided_error_shard) the shard and guide_buffer both have halves."""
        ds = self.device_scene()
        shard = getattr(buffer, "shard", None) or (0, 1)
        p = self.params(iterations, self._next_sample, *shard, collect_stats=collect_stats)
        cam = self.camera.to_c()
        if adaptive is not None:
            if not isinstance(buffer, DeviceBuffer):
                raise TypeError("adaptive sampling needs a DeviceBuffer (Renderer.device_buffer())")
            stats, active, crit = capi.Stats(), C.c_uint64(0), adaptive.to_c()
            st = C.byref(stats) if want_stats else None
            if adaptive.estimate == "halves" and guide_buffer is not Renderer._NO_GUIDE_BUFFER:
                guide = adaptive.guide.to_c()
                capi.check(capi.lib().rptb_sample_into_guided_error_shard(
                    ds.handle, C.byref(cam), C.byref(p), C.byref(crit), C.byref(guide), buffer.handle,
                    guide_buffer.handle if guide_buffer is not None else None, C.byref(active), st), "rptb_sample_into_guided_error_shard")
            elif adaptive.estimate == "halves":
                guide = adaptive.guide.to_c()
                capi.check(capi.lib().rptb_sample_into_guided_error(ds.handle, C.byref(cam), C.byref(p), C.byref(crit), C.byref(guide),
                                                                    buffer.handle, C.byref(active), st), "rptb_sample_into_guided_error")
            elif adaptive.guide is not None and guide_buffer is not Renderer._NO_GUIDE_BUFFER:
                guide = adaptive.guide.to_c()
                capi.check(capi.lib().rptb_sample_into_guided_shard(ds.handle, C.byref(cam), C.byref(p), C.byref(crit), C.byref(guide),
                                                                    buffer.handle, guide_buffer.handle if guide_buffer is not None else None,
                                                                    C.byref(active), st), "rptb_sample_into_guided_shard")
            elif adaptive.guide is not None:
                guide = adaptive.guide.to_c()
                capi.check(capi.lib().rptb_sample_into_guided(ds.handle, C.byref(cam), C.byref(p), C.byref(crit), C.byref(guide),
                                                              buffer.handle, C.byref(active), st), "rptb_sample_into_guided")
            else:
                capi.check(capi.lib().rptb_sample_into_adaptive(ds.handle, C.byref(cam), C.byref(p), C.byref(crit), buffer.handle,
                                                                C.byref(active), st), "rptb_sample_into_adaptive")
            self._next_sample += int(iterations)
            if buffer.shard is not None:  # a shard's counts are read after the gather; the calls bound them
                buffer.entries += 1
            elif active.value:  # the largest per-pixel count, as rptb_buffer_sums reports it
                buffer.entries = int(buffer.counts().max())
            self.last_stats = stats.as_dict() if want_stats else None
            return int(active.value)
        if isinstance(buffer, DeviceBuffer):
            stats = capi.Stats()
            capi.check(capi.lib().rptb_sample_into(ds.handle, C.byref(cam), C.byref(p), buffer.handle,
                                                   C.byref(stats) if want_stats else None), "rptb_sample_into")
            self._next_sample += int(iterations)
            buffer.entries += 1
            self.last_stats = stats.as_dict() if want_stats else None
            return
        colors = np.empty((self._width * self._height, 3), np.float64)
        stats = capi.Stats()
        capi.check(
            capi.lib().rptb_render_samples(ds.handle, C.byref(cam), C.byref(p),
                                           colors.ctypes.data_as(capi.c_double_p), C.byref(stats)),
            "rptb_render_samples",
        )
        self._next_sample += int(iterations)
        self.last_stats = stats.as_dict()
        buffer.add_samples(colors)

    def sample_features(self, iterations: int, buffer: "DeviceBuffer", want_stats: bool = False) -> None:
        """Adds the first hits of `iterations` more camera rays per pixel to the buffer's features
        (rptb_buffer_add_features): the samples after those the buffer's features already hold (0 .. iterations - 1 on
        the first call, the camera rays of the first entries' samples) of this renderer's seed, in its precision,
        through its camera.  The entries of the buffer are not touched."""
        if not isinstance(buffer, DeviceBuffer):
            raise TypeError("features live in a DeviceBuffer (Renderer.device_buffer())")
        ds = self.device_scene()
        p = self.params(iterations, buffer.feature_rays, *(buffer.shard or (0, 1)))
        cam = self.camera.to_c()
        stats = capi.Stats()
        capi.check(capi.lib().rptb_buffer_add_features(ds.handle, C.byref(cam), C.byref(p), buffer.handle,
                                                       C.byref(stats) if want_stats else None), "rptb_buffer_add_features")
        buffer.feature_rays += int(iterations)
        self.last_stats = stats.as_dict() if want_stats else None

    def render(self, denoise: Optional[Denoise] = None, entries: int = 8, feature_samples: int = 16,
               select: bool = False, cross: bool = False) -> np.ndarray:  # :96-100
        """Renderer::render.  With `denoise`, num_samples are rendered as `entries` equal entries of a DeviceBuffer,
        `feature_samples` camera rays per pixel give it features, and the denoised bytes are returned.  With `select`
        as well, the buffer keeps halves and each pixel takes the number of passes (0 .. denoise.iterations) whose
        estimated error is least (DeviceBuffer.selected_image).  With `cross` in place of `select`, the buffer keeps
        halves and is cross-filtered with a smoothed selection map (DeviceBuffer.cross_image)."""
        if select and denoise is None:
            raise ValueError("select=True chooses each pixel's number of filter passes: it needs denoise (a Denoise)")
        if cross and denoise is None:
            raise ValueError("cross=True cross-filters the buffer's halves: it needs denoise (a Denoise)")
        if cross and select:
            raise ValueError("cross=True and select=True are two ways to choose the passes per pixel: pass one of them")
        if denoise is None:
            buffer = Buffer(self._width, self._height, self._filter, self._first_device())
            self.sample(self._num_samples, buffer)
            return buffer.image()
        if entries < 2 or self._num_samples % entries:
            # the entries are weighted equally: unequal ones would bias the mean
            raise ValueError(f"num_samples {self._num_samples} must be a multiple of entries {entries} (and entries >= 2)")
        with self.device_buffer(halves=select or cross) as buf:
            for _ in range(entries):
                self.sample(self._num_samples // entries, buf, want_stats=False)
            self.sample_features(feature_samples, buf)
            if cross:
                return buf.cross_image(denoise)
            return buf.selected_image(denoise) if select else buf.denoised_image(denoise)

    def _check_frames(self, entries: int, adaptive: Optional[Adaptive], denoise: Optional[Denoise],
                      reproject: Optional[Reproject] = None, history_test: Optional[HistoryTest] = None) -> None:
        """The arguments render_frames and distributed.render_frames_distributed refuse."""
        if entries < 1 or self._num_samples % entries:
            raise ValueError(f"num_samples {self._num_samples} must be a multiple of entries {entries} (and entries >= 1)")
        if denoise is not None and entries < 2 and adaptive is None:
            raise ValueError("a denoised frame needs entries >= 2 (or adaptive entries)")
        if adaptive is not None and adaptive.estimate == "halves":
            raise ValueError('estimate="halves" is not supported in frame loops: drive frames through reproject_from / '
                             'merge_history_from on buffers with halves')
        if history_test is not None:
            if history_test.fresh_entries < 2 or history_test.fresh_entries > entries:
                raise ValueError(f"history_test.fresh_entries {history_test.fresh_entries} must lie in [2, entries {entries}]")
            if reproject is None:
                raise ValueError("history_test tests reprojected history: it needs reproject")

    def _frame_entries(self, buf: DeviceBuffer, prev: Optional[DeviceBuffer], entries: int, reproject: Optional[Reproject],
                       adaptive: Optional[Adaptive], history_test: Optional[HistoryTest],
                       entry: Optional[Callable[[int], None]] = None) -> None:
        """A frame's entries after its feature pass, for render_frames and distributed.render_frames_distributed: the
        previous frame's history reprojected, then `entries` entries -- or, with `history_test`, its fresh_entries plain
        entries first, the history merged where they agree with it, then the other entries.  `entry(samples)`, when
        given, adds each of those last entries instead of sample()."""
        n, fresh = self._num_samples // entries, 0
        if history_test is not None:
            fresh = history_test.fresh_entries
            for _ in range(fresh):
                self.sample(n, buf, want_stats=False)
            if prev is not None:
                buf.merge_history_from(prev, reproject, history_test)
        elif prev is not None and reproject is not None:
            buf.reproject_from(prev, reproject)
        for _ in range(entries - fresh):
            if entry is None:
                self.sample(n, buf, want_stats=False, adaptive=adaptive)
            else:
                entry(n)

    def render_frames(self, cameras, entries: int = 8, feature_samples: int = 16, reproject: Optional[Reproject] = Reproject(),
                      adaptive: Optional[Adaptive] = None, denoise: Optional[Denoise] = None,
                      history_test: Optional[HistoryTest] = None):
        """Renders one frame per camera of a static scene and yields each as (height, width, 3) uint8.  Per frame: a new
        DeviceBuffer gets `feature_samples` feature rays through the frame's camera, the previous frame's buffer is
        reprojected into it (unless `reproject` is None), and `entries` entries of num_samples / entries samples each are
        added -- adaptive ones with `adaptive` -- continuing the renderer's sample streams; the frame is image(), or
        denoised_image(denoise).  The device scene is uploaded once for all frames.
        With `history_test` (which needs `reproject`), a frame renders history_test.fresh_entries plain entries before
        it takes the previous frame's history, merges that history only where it agrees with them
        (DeviceBuffer.merge_history_from), and then adds the other entries."""
        self._check_frames(entries, adaptive, denoise, reproject, history_test)
        own, prev = self.camera, None
        try:
            for cam in cameras:
                self.camera = cam
                buf = self.device_buffer()
                self.sample_features(feature_samples, buf)
                self._frame_entries(buf, prev, entries, reproject, adaptive, history_test)
                img = buf.image() if denoise is None else buf.denoised_image(denoise)
                if prev is not None:
                    prev.close()
                prev = buf
                yield img
        finally:
            self.camera = own
            if prev is not None:
                prev.close()

    def iterative_render(self, callback_interval: int, callback: Callable[[int, Buffer], None],
                         buffer: Optional[DeviceBuffer] = None, adaptive: Optional[Adaptive] = None,
                         feature_samples: int = 16) -> None:  # :103-115
        """`buffer`: a DeviceBuffer (Renderer.device_buffer()) to accumulate into on the device; None keeps a
        host Buffer.  The callback receives whichever it is.  `adaptive` (needs a DeviceBuffer): every batch renders
        only the pixels the criterion leaves active, and the render stops early after a batch that rendered none.  A
        guided criterion (adaptive.guide) needs features: a buffer that holds none first gets `feature_samples` feature
        rays per pixel through this renderer's camera.  With estimate="halves" and no buffer, the loop makes its own
        DeviceBuffer with halves (destroyed when it returns)."""
        own = None
        if buffer is None and adaptive is not None and adaptive.estimate == "halves":
            buffer = own = self.device_buffer(halves=True)
        try:
            self._iterate(callback_interval, callback, buffer, adaptive, feature_samples)
        finally:
            if own is not None:
                own.close()

    def _iterate(self, callback_interval, callback, buffer, adaptive, feature_samples) -> None:
        device = buffer is not None
        if adaptive is not None and not device:
            raise TypeError("adaptive sampling needs a DeviceBuffer (Renderer.device_buffer())")
        if buffer is None:
            buffer = Buffer(self._width, self._height, self._filter, self._first_device())
        elif adaptive is not None and adaptive.guide is not None and buffer.feature_rays == 0:
            self.sample_features(feature_samples, buffer)
        iteration = 0
        while iteration < self._num_samples:
            steps = min(self._num_samples - iteration, callback_interval)
            active = self.sample(steps, buffer, want_stats=not device, adaptive=adaptive)
            iteration += steps
            if adaptive is not None and active == 0:
                break
            callback(iteration, buffer)
