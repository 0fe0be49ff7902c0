"""ctypes wrappers of the mesh depth pre-pass checkers (row f-9): the C restatement (libm2s_depth_oracle.so) and the
reference's own shaders in their GL environment (_ref/libm2s_refdepth.so, present only where it could be built)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from mesh2splat_b200 import _abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None
_ref = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_depth import build_depth_oracle
        L = C.CDLL(build_depth_oracle())
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.orc_depth_pvm.restype = None
        L.orc_depth_pvm.argtypes = [vp, vp, vp, vp]
        L.orc_depth_code.restype = C.c_int
        L.orc_depth_code.argtypes = [C.c_double, vp]
        L.orc_depth_poly.restype = C.c_int
        L.orc_depth_poly.argtypes = [vp, vp, vp]
        L.orc_depth_pairs.restype = u64
        L.orc_depth_pairs.argtypes = [vp, u64, vp, vp, u32, u32, vp]
        L.orc_mesh_depth.restype = None
        L.orc_mesh_depth.argtypes = [vp, u64, vp, vp, u32, u32, vp]
        L.orc_depth_vs.restype = None
        L.orc_depth_vs.argtypes = [vp, u64, vp, vp]
        L.orc_depth_test_mask.restype = None
        L.orc_depth_test_mask.argtypes = [vp, u64, vp, vp, vp, vp, u32, u32, u32, vp]
        _lib = L
    return _lib


def ref_lib():
    """The reference's depth shaders and prepass in their GL environment, or None if never built (no reference checkout)."""
    global _ref
    if _ref is None:
        path = os.path.join(_HERE, "_ref", "libm2s_refdepth.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        vp, u32 = C.c_void_p, C.c_uint32
        R.ref_depth_vs.restype = None
        R.ref_depth_vs.argtypes = [vp, u32, vp, vp, vp, vp]
        R.ref_depth_ps.restype = C.c_float
        R.ref_depth_ps.argtypes = [C.c_float]
        R.ref_depth_prepass.restype = u32
        R.ref_depth_prepass.argtypes = [vp, u32, vp, vp, vp, vp, vp, C.c_float, C.c_int, u32, vp, u32, u32, u32, vp, vp]
        R.ref_depth_keep.restype = None
        R.ref_depth_keep.argtypes = [vp, u32, vp, vp, vp, vp, vp, C.c_float, u32, vp, u32, u32, vp, vp]
        _ref = R
    return _ref


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, np.float32).ravel())


def pvm(world_to_view, view_to_clip, model_to_world) -> np.ndarray:
    """(P V) M as the pass builds it: 16 floats, column-major."""
    V, P, M, out = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world), np.zeros(16, np.float32)
    lib().orc_depth_pvm(V.ctypes.data, P.ctypes.data, M.ctypes.data, out.ctypes.data)
    return out


def code(z: float):
    """The D24 code of fp64 depth z, or None for NaN (no write)."""
    c = C.c_uint32(0)
    return int(c.value) if lib().orc_depth_code(float(z), C.byref(c)) else None


def poly(tri36, pvm16) -> np.ndarray:
    """The clipped polygon of one triangle (36 floats) in clip space: [n, 4] float32."""
    t, m, out = _f32(tri36), _f32(pvm16), np.zeros(9 * 4, np.float32)
    n = lib().orc_depth_poly(t.ctypes.data, m.ctypes.data, out.ctypes.data)
    return out[: 4 * n].reshape(n, 4)


def vs(pos3, pvm16) -> np.ndarray:
    """gl_Position of depthPrepassVS.glsl as the pass computes it: [n, 4]."""
    p, m = np.ascontiguousarray(np.asarray(pos3, np.float32).reshape(-1, 3)), _f32(pvm16)
    out = np.zeros((max(1, len(p)), 4), np.float32)
    lib().orc_depth_vs(p.ctypes.data, len(p), m.ctypes.data, out.ctypes.data)
    return out[: len(p)]


def ref_vs(pos3, world_to_view, view_to_clip, model_to_world) -> np.ndarray:
    p = np.ascontiguousarray(np.asarray(pos3, np.float32).reshape(-1, 3))
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    out = np.zeros((max(1, len(p)), 4), np.float32)
    ref_lib().ref_depth_vs(p.ctypes.data, len(p), V.ctypes.data, P.ctypes.data, M.ctypes.data, out.ctypes.data)
    return out[: len(p)]


def ref_prepass(g24, world_to_view, view_to_clip, model_to_world, resolution, near_far, std_dev, render_mode, fmt, depth_map):
    """The reference's prepass with u_depthTestMesh = 1 over the map: (quads [m, 24], depths [m]) in input order."""
    g = np.ascontiguousarray(g24, np.float32).reshape(-1, 24)
    d = np.ascontiguousarray(depth_map, np.float32)
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    r, nf = _f32(resolution), _f32(near_far)
    q, dd = np.zeros((max(1, len(g)), 24), np.float32), np.zeros(max(1, len(g)), np.float32)
    m = ref_lib().ref_depth_prepass(g.ctypes.data, len(g), V.ctypes.data, P.ctypes.data, M.ctypes.data, r.ctypes.data, nf.ctypes.data,
                                    float(std_dev), int(render_mode), int(fmt), d.ctypes.data, d.shape[1], d.shape[0], 1,
                                    q.ctypes.data, dd.ctypes.data)
    return q[:m].copy(), dd[:m].copy()


def ref_keep(g24, world_to_view, view_to_clip, model_to_world, resolution, near_far, std_dev, fmt, depth_map):
    """Per gaussian, from the reference run one gaussian at a time: (kept with the test on, kept with it off)."""
    g = np.ascontiguousarray(g24, np.float32).reshape(-1, 24)
    d = np.ascontiguousarray(depth_map, np.float32)
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    r, nf = _f32(resolution), _f32(near_far)
    on, off = np.zeros(max(1, len(g)), np.uint8), np.zeros(max(1, len(g)), np.uint8)
    ref_lib().ref_depth_keep(g.ctypes.data, len(g), V.ctypes.data, P.ctypes.data, M.ctypes.data, r.ctypes.data, nf.ctypes.data,
                             float(std_dev), int(fmt), d.ctypes.data, d.shape[1], d.shape[0], on.ctypes.data, off.ctypes.data)
    return on[: len(g)].astype(bool), off[: len(g)].astype(bool)


def opaque_mask(scene: _abi.Scene) -> np.ndarray:
    """Per triangle: 1 if its primitive's base colour factor alpha is exactly 1.0f (DepthPrepass.cpp:33)."""
    m = np.zeros(scene.triangle_count, np.uint8)
    for p in scene.primitives:
        m[p.first_triangle: p.first_triangle + p.triangle_count] = np.float32(p.base_color_factor[3]) == np.float32(1.0)
    return m


def _tris(scene_or_tris):
    if isinstance(scene_or_tris, _abi.Scene):
        return np.ascontiguousarray(scene_or_tris.triangles, np.float32).reshape(-1, 36), opaque_mask(scene_or_tris)
    t = np.ascontiguousarray(scene_or_tris, np.float32).reshape(-1, 36)
    return t, np.ones(len(t), np.uint8)


def pairs(scene_or_tris, pvm16, width: int, height: int):
    """(per-triangle pair counts, total) of the binning; a bare triangle array counts every triangle as opaque."""
    t, op = _tris(scene_or_tris)
    m = _f32(pvm16)
    c = np.zeros(max(1, len(t)), np.uint32)
    total = lib().orc_depth_pairs(t.ctypes.data, len(t), op.ctypes.data, m.ctypes.data, width, height, c.ctypes.data)
    return c[: len(t)], int(total)


def mesh_depth(scene_or_tris, pvm16, width: int, height: int, n: int | None = None) -> np.ndarray:
    """The depth map (height, width) float32 after the first n source triangles (default all)."""
    t, op = _tris(scene_or_tris)
    m = _f32(pvm16)
    out = np.zeros((height, width), np.float32)
    lib().orc_mesh_depth(t.ctypes.data if len(t) else None, len(t) if n is None else n, op.ctypes.data if len(op) else None,
                         m.ctypes.data, width, height, out.ctypes.data)
    return out


def test_mask(gaussians24, world_to_view, view_to_clip, model_to_world, depth_map, fmt: int = 0) -> np.ndarray:
    """Per REF96 gaussian: True if the prepass's mesh depth test keeps it (the frustum cull aside)."""
    g = np.ascontiguousarray(gaussians24, np.float32).reshape(-1, 24)
    d = np.ascontiguousarray(depth_map, np.float32)
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    keep = np.zeros(max(1, len(g)), np.uint8)
    lib().orc_depth_test_mask(g.ctypes.data, len(g), V.ctypes.data, P.ctypes.data, M.ctypes.data, d.ctypes.data, d.shape[1], d.shape[0],
                              fmt, keep.ctypes.data)
    return keep[: len(g)].astype(bool)
