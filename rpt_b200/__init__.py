"""rpt_b200 -- H100-native path-tracing core behind rpt's Renderer/Scene/Camera/Material API.

Host mirror of the reference API: rpt_b200.api (re-exported here).  The hot path --
everything under Renderer::sample (ekzhang/rpt src/renderer.rs:117-220) -- runs in
rpt_b200/lib/librpt_b200.so (CUDA, sm_90a) behind the C ABI of include/rpt_b200.h.
"""
from .api import (Buffer, Camera, Cube, DeviceScene, Environment, Filter, FlatScene, Hdri, KdTree, Light, Material, Mesh,
                  MonomialSurface, monomial_surface,
                  Object, Plane, Renderer, Scene, Shape, Sphere, Transformed, Triangle, color_bytes, cube, hex_color,
                  load_mtl, load_obj, load_obj_with_mtl, load_stl, parse_obj, plane, polygon, sphere, vec3)
from ._capi import PRECISION_F32, PRECISION_F64, RptbError

__all__ = [
    "Buffer", "Camera", "Cube", "DeviceScene", "Environment", "Filter", "FlatScene", "Hdri", "Light", "Material",
    "Mesh", "MonomialSurface", "KdTree", "monomial_surface", "Object", "Plane", "Renderer", "Scene", "Shape", "Sphere", "Transformed", "Triangle", "color_bytes",
    "cube", "hex_color", "load_mtl", "load_obj", "load_obj_with_mtl", "load_stl", "parse_obj", "plane", "polygon", "sphere", "vec3", "PRECISION_F32",
    "PRECISION_F64", "RptbError",
]
