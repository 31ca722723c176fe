"""ctypes view of include/rpt_b200.h and loader of the CUDA library.

The product path has no CPU fallback: if ``librpt_b200.so`` is missing or does
not export every symbol of the header, importing ``lib()`` raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RPTB_LIB") or os.path.join(_HERE, "lib", "librpt_b200.so")  # RPTB_LIB: A/B builds only

# ---- enums (include/rpt_b200.h) ------------------------------------------------
OK = 0
ERR_BAD_ARG, ERR_CUDA, ERR_NO_DEVICE, ERR_OOM, ERR_UNSUPPORTED = -1, -2, -3, -4, -5
SHAPE_SPHERE, SHAPE_PLANE, SHAPE_CUBE, SHAPE_MESH, SHAPE_MONOMIAL, SHAPE_GROUP = 0, 1, 2, 3, 4, 5
LIGHT_POINT, LIGHT_AMBIENT, LIGHT_DIRECTIONAL, LIGHT_OBJECT = 0, 1, 2, 3
ENV_COLOR, ENV_HDRI = 0, 1
PRECISION_F32, PRECISION_F64 = 0, 1
ENGINE_AUTO, ENGINE_MEGAKERNEL, ENGINE_WAVEFRONT = 0, 1, 2
ACCEL_AUTO, ACCEL_KDTREE, ACCEL_BVH = 0, 1, 2

c_double_p = C.POINTER(C.c_double)
c_float_p = C.POINTER(C.c_float)
c_u32_p = C.POINTER(C.c_uint32)
c_i32_p = C.POINTER(C.c_int32)
c_u8_p = C.POINTER(C.c_uint8)


class Material(C.Structure):
    _fields_ = [
        ("color", C.c_double * 3),
        ("index", C.c_double),
        ("roughness", C.c_double),
        ("metallic", C.c_double),
        ("emittance", C.c_double),
        ("transparent", C.c_uint32),
        ("_pad", C.c_uint32),
    ]


class KdNode(C.Structure):
    _fields_ = [
        ("split", C.c_double),
        ("kind", C.c_uint32),
        ("left", C.c_uint32),
        ("right", C.c_uint32),
        ("first_ref", C.c_uint32),
        ("num_refs", C.c_uint32),
        ("_pad", C.c_uint32),
    ]


class Mesh(C.Structure):
    _fields_ = [
        ("tris", c_double_p),
        ("ntris", C.c_uint64),
        ("nodes", C.POINTER(KdNode)),
        ("nnodes", C.c_uint64),
        ("refs", c_u32_p),
        ("nrefs", C.c_uint64),
    ]


class Object(C.Structure):
    _fields_ = [
        ("kind", C.c_uint32),
        ("material", C.c_uint32),
        ("mesh", C.c_uint32),
        ("has_transform", C.c_uint32),
        ("transform", C.c_double * 16),
        ("plane_normal", C.c_double * 3),
        ("plane_value", C.c_double),
        ("monomial_height", C.c_double),
        ("monomial_exp", C.c_double),
    ]


class Group(C.Structure):
    _fields_ = [
        ("children", C.POINTER(Object)),
        ("nchildren", C.c_uint64),
        ("nodes", C.POINTER(KdNode)),
        ("nnodes", C.c_uint64),
        ("refs", c_u32_p),
        ("nrefs", C.c_uint64),
    ]


class Light(C.Structure):
    _fields_ = [
        ("kind", C.c_uint32),
        ("_pad", C.c_uint32),
        ("color", C.c_double * 3),
        ("vec", C.c_double * 3),
        ("object", Object),
    ]


class Env(C.Structure):
    _fields_ = [
        ("kind", C.c_uint32),
        ("width", C.c_uint32),
        ("height", C.c_uint32),
        ("_pad", C.c_uint32),
        ("color", C.c_double * 3),
        ("texels", c_double_p),
    ]


class SceneDesc(C.Structure):
    _fields_ = [
        ("materials", C.POINTER(Material)),
        ("nmaterials", C.c_uint32),
        ("meshes", C.POINTER(Mesh)),
        ("nmeshes", C.c_uint32),
        ("objects", C.POINTER(Object)),
        ("nobjects", C.c_uint32),
        ("lights", C.POINTER(Light)),
        ("nlights", C.c_uint32),
        ("environment", Env),
        ("groups", C.POINTER(Group)),
        ("ngroups", C.c_uint32),
        ("accel", C.c_uint32),
    ]


class Camera(C.Structure):
    _fields_ = [
        ("eye", C.c_double * 3),
        ("direction", C.c_double * 3),
        ("up", C.c_double * 3),
        ("fov", C.c_double),
        ("aperture", C.c_double),
        ("focal_distance", C.c_double),
    ]


class RenderParams(C.Structure):
    _fields_ = [
        ("width", C.c_uint32),
        ("height", C.c_uint32),
        ("iterations", C.c_uint32),
        ("max_bounces", C.c_uint32),
        ("exposure_value", C.c_double),
        ("seed", C.c_uint64),
        ("first_sample", C.c_uint64),
        ("shard_index", C.c_uint32),
        ("shard_count", C.c_uint32),
        ("precision", C.c_uint32),
        ("collect_stats", C.c_uint32),
        ("engine", C.c_uint32),
        ("compact_out", C.c_uint32),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("segments", C.c_uint64),
        ("rays", C.c_uint64),
        ("node_visits", C.c_uint64),
        ("tri_tests", C.c_uint64),
        ("mesh_hits", C.c_uint64),
        ("env_lookups", C.c_uint64),
        ("object_tests", C.c_uint64),
        ("gpu_ms", C.c_double),
        ("launches", C.c_uint32),
        ("engine", C.c_uint32),
        ("bvh_node_visits", C.c_uint64),
        ("bvh_tri_tests", C.c_uint64),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if not k.startswith("_")}


class Adaptive(C.Structure):
    """rptb_adaptive: the convergence criterion of rptb_sample_into_adaptive."""
    _fields_ = [
        ("rel_tol", C.c_double),
        ("abs_tol", C.c_double),
        ("min_entries", C.c_uint32),
        ("_pad", C.c_uint32),
    ]


class Denoise(C.Structure):
    """rptb_denoise: the parameters of rptb_buffer_denoise."""
    _fields_ = [
        ("iterations", C.c_uint32),
        ("sigma_normal", C.c_uint32),
        ("sigma_depth", C.c_double),
        ("sigma_luminance", C.c_double),
        ("albedo_eps", C.c_double),
    ]


class Reproject(C.Structure):
    """rptb_reproject: the parameters of rptb_buffer_reproject."""
    _fields_ = [
        ("depth_tol", C.c_double),
        ("normal_cos", C.c_double),
        ("max_history", C.c_uint32),
        ("_pad", C.c_uint32),
    ]


class KdTreeOut(C.Structure):
    _fields_ = [
        ("nodes", C.POINTER(KdNode)),
        ("nnodes", C.c_uint64),
        ("refs", c_u32_p),
        ("nrefs", C.c_uint64),
        ("depth", C.c_uint32),
        ("max_leaf", C.c_uint32),
    ]


class ObjGroup(C.Structure):
    _fields_ = [("material", Material), ("first_tri", C.c_uint64), ("ntris", C.c_uint64)]


class ObjGroupsOut(C.Structure):
    _fields_ = [
        ("tris", c_double_p),
        ("ntris", C.c_uint64),
        ("groups", C.POINTER(ObjGroup)),
        ("ngroups", C.c_uint64),
    ]


# Every symbol include/rpt_b200.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("rptb_last_error", C.c_char_p, []),
    ("rptb_device_count", C.c_int, []),
    ("rptb_scene_create", C.c_int, [C.POINTER(SceneDesc), C.c_int, C.POINTER(C.c_void_p)]),
    ("rptb_scene_create_multi", C.c_int, [C.POINTER(SceneDesc), C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_void_p)]),
    ("rptb_scene_device_count", C.c_int, [C.c_void_p]),
    ("rptb_scene_destroy", None, [C.c_void_p]),
    ("rptb_scene_device_bytes", C.c_uint64, [C.c_void_p]),
    ("rptb_render_samples", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), c_double_p, C.POINTER(Stats)]),
    ("rptb_render_samples_device", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.c_void_p, C.c_void_p, C.POINTER(Stats)]),
    ("rptb_tile_pixel", C.c_int64, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
    ("rptb_closest_hit", C.c_int,
     [C.c_void_p, c_double_p, C.c_uint64, C.c_double, C.c_uint32, c_double_p, c_i32_p, c_double_p,
      C.POINTER(Stats)]),
    ("rptb_bsdf_eval", C.c_int, [C.POINTER(Material), c_double_p, C.c_uint64, C.c_uint32, C.c_int, c_double_p]),
    ("rptb_sample_f", C.c_int,
     [C.POINTER(Material), c_double_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, c_double_p, c_double_p]),
    ("rptb_illuminate", C.c_int,
     [C.c_void_p, C.c_uint32, c_double_p, C.c_uint64, C.c_uint64, C.c_uint32, c_double_p, c_double_p, c_double_p]),
    ("rptb_build_kdtree", C.c_int, [c_double_p, C.c_uint64, C.POINTER(KdTreeOut)]),
    ("rptb_build_kdtree_boxes", C.c_int, [c_double_p, C.c_uint64, C.POINTER(KdTreeOut)]),
    ("rptb_free_kdtree", None, [C.POINTER(KdTreeOut)]),
    ("rptb_parse_obj", C.c_int, [C.c_char_p, C.c_uint64, C.POINTER(c_double_p), C.POINTER(C.c_uint64)]),
    ("rptb_free_triangles", None, [c_double_p]),
    ("rptb_parse_obj_mtl", C.c_int, [C.c_char_p, C.c_uint64, C.c_char_p, C.c_uint64, C.POINTER(ObjGroupsOut)]),
    ("rptb_free_obj_groups", None, [C.POINTER(ObjGroupsOut)]),
    ("rptb_parse_stl", C.c_int, [C.c_char_p, C.c_uint64, C.POINTER(c_double_p), C.POINTER(C.c_uint64)]),
    ("rptb_film_variance", C.c_int, [c_double_p, C.c_uint32, C.c_uint64, C.c_int, c_double_p]),
    ("rptb_film_resolve", C.c_int,
     [c_double_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, c_u8_p]),
    ("rptb_buffer_create", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]),
    ("rptb_buffer_destroy", None, [C.c_void_p]),
    ("rptb_sample_into", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.c_void_p, C.POINTER(Stats)]),
    ("rptb_buffer_add_samples", C.c_int, [C.c_void_p, c_double_p]),
    ("rptb_buffer_image", C.c_int, [C.c_void_p, c_u8_p]),
    ("rptb_buffer_variance", C.c_int, [C.c_void_p, c_double_p]),
    ("rptb_buffer_sums", C.c_int, [C.c_void_p, c_double_p, c_u32_p]),
    ("rptb_sample_into_adaptive", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.POINTER(Adaptive), C.c_void_p, C.POINTER(C.c_uint64),
      C.POINTER(Stats)]),
    ("rptb_buffer_pixel_stats", C.c_int, [C.c_void_p, c_double_p, c_double_p, c_u32_p]),
    ("rptb_buffer_add_features", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.c_void_p, C.POINTER(Stats)]),
    ("rptb_buffer_features", C.c_int, [C.c_void_p, c_double_p, c_double_p, c_double_p, c_double_p]),
    ("rptb_buffer_denoise", C.c_int, [C.c_void_p, C.POINTER(Denoise), c_double_p, c_u8_p]),
    ("rptb_buffer_denoise_variance", C.c_int, [C.c_void_p, C.POINTER(Denoise), c_double_p]),
    ("rptb_sample_into_guided", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.POINTER(Adaptive), C.POINTER(Denoise), C.c_void_p,
      C.POINTER(C.c_uint64), C.POINTER(Stats)]),
    ("rptb_buffer_reproject", C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(Reproject), C.POINTER(C.c_uint64)]),
    ("rptb_buffer_create_shard", C.c_int,
     [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]),
    ("rptb_buffer_shard_bytes", C.c_uint64, [C.c_void_p, C.c_uint32]),
    ("rptb_buffer_export_shard", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]),
    ("rptb_buffer_import_shards", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]),
    ("rptb_buffer_reproject_shard", C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(Reproject), C.POINTER(C.c_uint64)]),
    ("rptb_buffer_reproject_merge", C.c_int,
     [C.c_void_p, C.c_void_p, C.POINTER(Reproject), C.c_double, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("rptb_buffer_reproject_merge_shard", C.c_int,
     [C.c_void_p, C.c_void_p, C.POINTER(Reproject), C.c_double, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    ("rptb_delta_bytes", C.c_uint64, [C.c_uint32]),
    ("rptb_buffer_export_delta", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.POINTER(C.c_uint32)]),
    ("rptb_buffer_import_deltas", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]),
    ("rptb_sample_into_guided_shard", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.POINTER(Adaptive), C.POINTER(Denoise), C.c_void_p, C.c_void_p,
      C.POINTER(C.c_uint64), C.POINTER(Stats)]),
    ("rptb_buffer_create_halves", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]),
    ("rptb_buffer_half_sums", C.c_int, [C.c_void_p, c_double_p]),
    ("rptb_buffer_denoise_error", C.c_int, [C.c_void_p, C.POINTER(Denoise), c_double_p]),
    ("rptb_buffer_denoise_select", C.c_int, [C.c_void_p, C.POINTER(Denoise), c_double_p, c_u8_p, c_u8_p, c_double_p]),
    ("rptb_buffer_denoise_cross", C.c_int, [C.c_void_p, C.POINTER(Denoise), c_double_p, c_u8_p, c_u8_p, c_double_p]),
    ("rptb_sample_into_guided_error", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.POINTER(Adaptive), C.POINTER(Denoise), C.c_void_p,
      C.POINTER(C.c_uint64), C.POINTER(Stats)]),
    ("rptb_buffer_create_shard_halves", C.c_int,
     [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]),
    ("rptb_delta_bytes_halves", C.c_uint64, [C.c_uint32]),
    ("rptb_sample_into_guided_error_shard", C.c_int,
     [C.c_void_p, C.POINTER(Camera), C.POINTER(RenderParams), C.POINTER(Adaptive), C.POINTER(Denoise), C.c_void_p, C.c_void_p,
      C.POINTER(C.c_uint64), C.POINTER(Stats)]),
]

_lib = None


class RptbError(RuntimeError):
    """A C-ABI call returned a negative status (the reference would panic here)."""


def lib() -> C.CDLL:
    """Load librpt_b200.so and bind every declared symbol.  No fallback."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RptbError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make`).  rpt_b200 has no CPU fallback."
        )
    dll = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(dll, name)  # AttributeError if the symbol is not exported
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = dll
    return dll


def check(status: int, what: str) -> None:
    if status != OK:
        msg = lib().rptb_last_error()
        raise RptbError(f"{what} failed with status {status}: {msg.decode() if msg else ''}")
