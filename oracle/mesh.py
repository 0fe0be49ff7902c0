"""ctypes wrappers of the mesh G-buffer pass's checkers (SURVEY 8 row 14): the C restatement (libm2s_mesh_oracle.so) of
MeshRenderPass::execute and of the split-screen composite of the deferred lighting, and the reference's own mesh shaders
(_ref/libm2s_refmesh.so, present only where it could be built)."""
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
        from oracle.build_mesh import build_mesh_oracle
        L = C.CDLL(build_mesh_oracle())
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.orc_mesh_normal_matrix.restype = C.c_int
        L.orc_mesh_normal_matrix.argtypes = [vp, vp]
        L.orc_mesh_log2.restype = C.c_double
        L.orc_mesh_log2.argtypes = [C.c_double]
        L.orc_mesh_sin.restype = C.c_double
        L.orc_mesh_sin.argtypes = [C.c_double]
        L.orc_mesh_hash.restype = C.c_float
        L.orc_mesh_hash.argtypes = [C.c_float]
        L.orc_mesh_vs_one.restype = None
        L.orc_mesh_vs_one.argtypes = [vp, vp, vp, vp, vp, vp, vp]
        L.orc_mesh_level.restype = None
        L.orc_mesh_level.argtypes = [u32, u32, u32, C.c_float, C.c_float, C.c_float, C.c_float, vp, vp]
        L.orc_mesh_fs.restype = None
        L.orc_mesh_fs.argtypes = [vp, vp, u32, vp, vp, u32, u32, vp]
        L.orc_mesh_render.restype = C.c_int
        L.orc_mesh_render.argtypes = [vp, u64, u32, vp, vp, vp, vp, vp, vp, vp, vp, u32, vp, vp, vp, vp, vp, u32, u32, u32,
                                      vp, vp, vp, vp, vp]
        L.orc_mesh_pairs.restype = u64
        L.orc_mesh_pairs.argtypes = [vp, u64, vp, vp, vp, vp, u32, u32, vp]
        L.orc_mesh_split.restype = None
        L.orc_mesh_split.argtypes = [vp, vp, u32, u32, C.c_float, vp]
        _lib = L
    return _lib


def ref_lib():
    """The reference's mesh shaders in their GL environment, or None if never built (no reference checkout)."""
    global _ref
    if _ref is None:
        path = os.path.join(_HERE, "_ref", "libm2s_refmesh.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        vp, u32 = C.c_void_p, C.c_uint32
        R.ref_mesh_vs.restype = None
        R.ref_mesh_vs.argtypes = [vp, u32, vp, vp, vp, vp, vp]
        R.ref_mesh_ps.restype = None
        R.ref_mesh_ps.argtypes = [vp, vp, u32, vp, vp, C.c_int, C.c_int, vp]
        _ref = R
    return _ref


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a, np.float32).ravel())


def normal_matrix(model_to_world):
    """mat3(transpose(inverse(M))) as the pass builds it (9 floats, column-major), or None for a singular M."""
    M, N = _f32(model_to_world), np.zeros(9, np.float32)
    return N if lib().orc_mesh_normal_matrix(M.ctypes.data, N.ctypes.data) else None


def log2(x: float) -> float:
    return float(lib().orc_mesh_log2(float(x)))


def sin(x: float) -> float:
    return float(lib().orc_mesh_sin(float(x)))


def hash_(arg: float) -> float:
    """fract(sin(arg) * 43758.5453) of render mode 3, arg an fp32 value."""
    return float(lib().orc_mesh_hash(float(np.float32(arg))))


def level(w0: int, h0: int, nlevels: int, dudx, dvdx, dudy, dvdy):
    """(first level, blend fraction) the pass samples a w0 x h0 map of nlevels levels with for the quad's uv steps."""
    l0, f = C.c_int(0), C.c_float(0)
    lib().orc_mesh_level(w0, h0, nlevels, *(float(np.float32(x)) for x in (dudx, dvdx, dudy, dvdy)), C.byref(l0), C.byref(f))
    return int(l0.value), float(f.value)


def vs(tri36, world_to_view, view_to_clip, model_to_world):
    """meshRenderVS.glsl per vertex of the triangles: (clip [n, 3, 4], varyings [n, 3, 13]: worldPos, v_normal,
    v_tangent, v_uv, v_viewDepth)."""
    t = np.ascontiguousarray(np.asarray(tri36, np.float32).reshape(-1, 36))
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    N = normal_matrix(M)
    clip, vary = np.zeros((len(t), 3, 4), np.float32), np.zeros((len(t), 3, 13), np.float32)
    for i in range(len(t)):
        for k in range(3):
            v12 = np.ascontiguousarray(t[i, 12 * k: 12 * k + 12])
            c, o = np.zeros(4, np.float32), np.zeros(13, np.float32)
            lib().orc_mesh_vs_one(v12.ctypes.data, M.ctypes.data, V.ctypes.data, P.ctypes.data, N.ctypes.data, c.ctypes.data, o.ctypes.data)
            clip[i, k], vary[i, k] = c, o
    return clip, vary


def ref_vs(vtx12, world_to_view, view_to_clip, model_to_world):
    """The reference's meshRenderVS.glsl per vertex (n x 12 floats): (clip [n, 4], varyings [n, 13])."""
    v = np.ascontiguousarray(np.asarray(vtx12, np.float32).reshape(-1, 12))
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    clip, vary = np.zeros((max(1, len(v)), 4), np.float32), np.zeros((max(1, len(v)), 13), np.float32)
    ref_lib().ref_mesh_vs(v.ctypes.data, len(v), V.ctypes.data, P.ctypes.data, M.ctypes.data, clip.ctypes.data, vary.ctypes.data)
    return clip[: len(v)], vary[: len(v)]


def vs_vertices(vtx12, world_to_view, view_to_clip, model_to_world):
    """The pass's vertex stage per vertex (n x 12 floats), as ref_vs: (clip [n, 4], varyings [n, 13])."""
    v = np.ascontiguousarray(np.asarray(vtx12, np.float32).reshape(-1, 12))
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    N = normal_matrix(M)
    clip, vary = np.zeros((len(v), 4), np.float32), np.zeros((len(v), 13), np.float32)
    for i in range(len(v)):
        c, o = np.zeros(4, np.float32), np.zeros(13, np.float32)
        lib().orc_mesh_vs_one(np.ascontiguousarray(v[i]).ctypes.data, M.ctypes.data, V.ctypes.data, P.ctypes.data, N.ctypes.data,
                              c.ctypes.data, o.ctypes.data)
        clip[i], vary[i] = c, o
    return clip, vary


def _fs_call(fn, vary13, tex12, has, factor, near_far, mode, prim_id):
    v, t, f, nf = _f32(vary13), _f32(tex12), _f32(factor), _f32(near_far)
    out = np.zeros(20, np.float32)
    fn(v.ctypes.data, t.ctypes.data, int(has), f.ctypes.data, nf.ctypes.data, int(mode), int(prim_id), out.ctypes.data)
    return out


def fs(vary13, tex12, has, factor, near_far, mode, prim_id) -> np.ndarray:
    """The pass's fragment stage on given varyings and texels: the five targets' fp32 values (20 floats)."""
    return _fs_call(lib().orc_mesh_fs, vary13, tex12, has, factor, near_far, mode, prim_id)


def ref_fs(vary13, tex12, has, factor, near_far, mode, prim_id) -> np.ndarray:
    """The reference's meshRenderPS.glsl on given varyings and texels (texture() returns them): 20 floats."""
    return _fs_call(ref_lib().ref_mesh_ps, vary13, tex12, has, factor, near_far, mode, prim_id)


def mip_arena(textures):
    """The mip chains of the scene's textures as the upload builds them: (nlevels [T], off [T, 5], w [T, 5], h [T, 5],
    arena uint32 RGBA8 words)."""
    import oracle
    nt = max(1, len(textures))
    nl, off, w, h = np.zeros(nt, np.uint32), np.zeros((nt, 5), np.uint32), np.zeros((nt, 5), np.uint32), np.zeros((nt, 5), np.uint32)
    chunks, pos = [], 0
    for t, img in enumerate(textures):
        img = np.ascontiguousarray(img, np.uint8)
        n = oracle.mip_count(img.shape[1], img.shape[0])
        nl[t] = n
        for lvl in range(n):
            lv = img if lvl == 0 else oracle.mip_level(img, lvl)
            off[t, lvl], w[t, lvl], h[t, lvl] = pos, lv.shape[1], lv.shape[0]
            words = np.ascontiguousarray(lv).reshape(-1).view(np.uint32)
            chunks.append(words)
            pos += len(words)
    arena = np.concatenate(chunks) if chunks else np.zeros(1, np.uint32)
    return nl, off, w, h, arena


def mesh_render(scene: _abi.Scene, world_to_view, view_to_clip, model_to_world, width: int, height: int, near_far,
                render_mode: int = 0, n: int | None = None, arena=None) -> dict:
    """The mesh G-buffer after the first n source triangles (default all) as {target: (height, width, 4) array}, float16
    for position / normal / depth, uint8 for albedo / metallic_roughness.  arena: mip_arena(scene.textures), reused."""
    t = np.ascontiguousarray(scene.triangles, np.float32).reshape(-1, 36)
    prims = scene.primitives
    npr = max(1, len(prims))
    first, count = np.zeros(npr, np.uint32), np.zeros(npr, np.uint32)
    factor, tex = np.zeros((npr, 4), np.float32), np.full((npr, 3), -1, np.int32)
    for i, p in enumerate(prims):
        first[i], count[i] = p.first_triangle, p.triangle_count
        factor[i] = p.base_color_factor
        tex[i] = (p.albedo_texture, p.normal_texture, p.metallic_roughness_texture)
    nl, off, w, h, ar = arena if arena is not None else mip_arena(scene.textures)
    V, P, M, nf = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world), _f32(near_far)
    out = {name: np.zeros((height, width, 4), dt) for name, dt in _abi.GBUFFER_TARGETS}
    ok = lib().orc_mesh_render(t.ctypes.data if len(t) else None, len(t) if n is None else n, len(prims), first.ctypes.data,
                               count.ctypes.data, factor.ctypes.data, tex.ctypes.data, nl.ctypes.data, off.ctypes.data, w.ctypes.data,
                               h.ctypes.data, len(scene.textures), ar.ctypes.data, V.ctypes.data, P.ctypes.data, M.ctypes.data,
                               nf.ctypes.data, width, height, render_mode, out["position"].ctypes.data, out["normal"].ctypes.data,
                               out["albedo"].ctypes.data, out["depth"].ctypes.data, out["metallic_roughness"].ctypes.data)
    if not ok:
        raise ValueError("model_to_world is singular")
    return out


def drawn_mask(scene: _abi.Scene) -> np.ndarray:
    """Per triangle: 1 if a primitive holds it (every primitive is drawn, whatever its base colour alpha)."""
    m = np.zeros(scene.triangle_count, np.uint8)
    for p in scene.primitives:
        m[p.first_triangle: p.first_triangle + p.triangle_count] = 1
    return m


def pairs(scene: _abi.Scene, world_to_view, view_to_clip, model_to_world, width: int, height: int):
    """(per-triangle pair counts, total) of the binning."""
    t = np.ascontiguousarray(scene.triangles, np.float32).reshape(-1, 36)
    d = drawn_mask(scene)
    V, P, M = _f32(world_to_view), _f32(view_to_clip), _f32(model_to_world)
    c = np.zeros(max(1, len(t)), np.uint32)
    total = lib().orc_mesh_pairs(t.ctypes.data, len(t), d.ctypes.data, V.ctypes.data, P.ctypes.data, M.ctypes.data, width, height,
                                 c.ctypes.data)
    return c[: len(t)], int(total)


def split(left, right, position: float) -> np.ndarray:
    """The split composite of two RGBA8 images (height, width, 4): left = the mesh side's lighting."""
    lft, rgt = np.ascontiguousarray(left, np.uint8), np.ascontiguousarray(right, np.uint8)
    hgt, wdt = lft.shape[:2]
    out = np.zeros_like(lft)
    lib().orc_mesh_split(lft.ctypes.data, rgt.ctypes.data, wdt, hgt, float(np.float32(position)), out.ctypes.data)
    return out
