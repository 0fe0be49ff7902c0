"""ctypes wrappers of the shadow pass and deferred lighting checkers (rows f-7, f-8): the C restatement
(libm2s_light_oracle.so) and the reference's own shaders in their GL environment (_ref/libm2s_reflight.so, present only
where it could be built)."""
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
        from oracle.build_light import build_light_oracle
        L = C.CDLL(build_light_oracle())
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        for name in ("orc_light_log2", "orc_light_exp2"):
            getattr(L, name).restype = f32
            getattr(L, name).argtypes = [f32]
        L.orc_light_pow.restype = f32
        L.orc_light_pow.argtypes = [f32, f32]
        L.orc_light_face.restype = C.c_int
        L.orc_light_face.argtypes = [f32, f32, f32]
        L.orc_cube_texel.restype = None
        L.orc_cube_texel.argtypes = [f32, f32, f32, u32, vp, vp, vp]
        L.orc_d24.restype = C.c_int
        L.orc_d24.argtypes = [f32, vp]
        L.orc_light_uniforms.restype = None
        L.orc_light_uniforms.argtypes = [C.POINTER(_abi.m2s_shadow_params), vp, vp, vp, vp]
        L.orc_light_prepass.restype = None
        L.orc_light_prepass.argtypes = [vp, C.c_uint64, C.POINTER(_abi.m2s_shadow_params), vp]
        L.orc_cube_pairs.restype = C.c_uint64
        L.orc_cube_pairs.argtypes = [vp, u32, u32, vp]
        L.orc_cube_raster.restype = None
        L.orc_cube_raster.argtypes = [vp, u32, u32, vp]
        L.orc_deferred_fs.restype = None
        L.orc_deferred_fs.argtypes = [vp, vp, vp, vp, vp, C.POINTER(_abi.m2s_light_params), vp]
        L.orc_deferred_light.restype = None
        L.orc_deferred_light.argtypes = [vp, vp, vp, vp, vp, C.POINTER(_abi.m2s_light_params), vp]
        _lib = L
    return _lib


def ref_lib():
    """The reference's shaders in their GL environment, or None if never built (no reference checkout)."""
    global _ref
    if _ref is None:
        path = os.path.join(_HERE, "_ref", "libm2s_reflight.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        vp, u32 = C.c_void_p, C.c_uint32
        R.ref_light_prepass.restype = None
        R.ref_light_prepass.argtypes = [vp, u32, C.POINTER(_abi.m2s_shadow_params), u32, vp]
        R.ref_shadow_map.restype = None
        R.ref_shadow_map.argtypes = [vp, u32, C.POINTER(_abi.m2s_shadow_params), u32, u32, vp]
        R.ref_deferred_fs.restype = None
        R.ref_deferred_fs.argtypes = [vp, vp, vp, vp, vp, C.POINTER(_abi.m2s_light_params), vp]
        R.ref_deferred_light.restype = None
        R.ref_deferred_light.argtypes = [vp, vp, vp, vp, vp, C.POINTER(_abi.m2s_light_params), vp]
        _ref = R
    return _ref


def ref_prepass(gaussians: np.ndarray, p: _abi.m2s_shadow_params, u_format: int) -> np.ndarray:
    """The reference's light prepass (and its cube pixel shader's depth) as light records [n, 8], source order."""
    g = np.ascontiguousarray(gaussians, np.float32).reshape(-1, 24)
    out = np.zeros((max(len(g), 1), 8), np.float32)
    ref_lib().ref_light_prepass(g.ctypes.data, len(g), C.byref(p), u_format, out.ctypes.data)
    return out[: len(g)]


def ref_cube(gaussians: np.ndarray, p: _abi.m2s_shadow_params, u_format: int) -> np.ndarray:
    """The reference's whole shadow pass: the cube [6, S, S] float32."""
    g = np.ascontiguousarray(gaussians, np.float32).reshape(-1, 24)
    out = np.zeros((6, p.size, p.size), np.float32)
    ref_lib().ref_shadow_map(g.ctypes.data, len(g), C.byref(p), u_format, p.size, out.ctypes.data)
    return out


def deferred_fs(pos16, nrm16, alb8, mr8, cube_map, p: _abi.m2s_light_params, ref: bool = False) -> np.ndarray:
    """One invocation of the lighting pixel shader on the given texels (position / normal as float16 or their bits):
    FragColor (4 float32)."""
    bits = lambda v: np.ascontiguousarray(v).view(np.uint16) if np.asarray(v).dtype == np.float16 else np.ascontiguousarray(v, np.uint16)  # noqa: E731
    a = [bits(pos16), bits(nrm16), np.ascontiguousarray(alb8, np.uint8),
         np.ascontiguousarray(mr8, np.uint8), np.ascontiguousarray(cube_map, np.float32)]
    out = np.zeros(4, np.float32)
    fn = ref_lib().ref_deferred_fs if ref else lib().orc_deferred_fs
    fn(*[x.ctypes.data for x in a], C.byref(p), out.ctypes.data)
    return out


def ref_deferred_light(gbuffer: dict, cube_map, p: _abi.m2s_light_params) -> np.ndarray:
    keep = [np.ascontiguousarray(gbuffer[t]).view(dt) for t, dt in
            (("position", np.uint16), ("normal", np.uint16), ("albedo", np.uint8), ("metallic_roughness", np.uint8))]
    cm = np.ascontiguousarray(cube_map, np.float32)
    img = np.zeros((p.height, p.width, 4), np.uint8)
    ref_lib().ref_deferred_light(*[k.ctypes.data for k in keep], cm.ctypes.data, C.byref(p), img.ctypes.data)
    return img


def _f32(fn, x) -> np.ndarray:
    a = np.asarray(x, np.float32).ravel()
    return np.array([fn(float(v)) for v in a], np.float32)


def log2(x) -> np.ndarray:
    return _f32(lib().orc_light_log2, x)


def exp2(x) -> np.ndarray:
    return _f32(lib().orc_light_exp2, x)


def pow(x, y: float) -> np.ndarray:   # noqa: A001 (the GLSL name)
    L = lib()
    return np.array([L.orc_light_pow(float(v), float(y)) for v in np.asarray(x, np.float32).ravel()], np.float32)


def face(x: float, y: float, z: float) -> int:
    return int(lib().orc_light_face(x, y, z))


def cube_texel(d, size: int):
    """(face, i, j) the cube sampler reads for direction d in an S x S cube."""
    f, i, j = C.c_int(), C.c_int(), C.c_int()
    lib().orc_cube_texel(float(d[0]), float(d[1]), float(d[2]), size, C.byref(f), C.byref(i), C.byref(j))
    return f.value, i.value, j.value


def d24(d: float):
    """The D24 code of depth d, or None for NaN (no write)."""
    c = C.c_uint32(0)
    return int(c.value) if lib().orc_d24(float(d), C.byref(c)) else None


def uniforms(p: _abi.m2s_shadow_params):
    """(V [6, 16], P [16], inverse(mat3(M)) [9], modelScale^2 [3]) as the shadow pass builds them."""
    V, P, R, s = np.zeros((6, 16), np.float32), np.zeros(16, np.float32), np.zeros(9, np.float32), np.zeros(3, np.float32)
    lib().orc_light_uniforms(C.byref(p), V.ctypes.data, P.ctypes.data, R.ctypes.data, s.ctypes.data)
    return V, P, R, s


def prepass(records: np.ndarray, n: int, p: _abi.m2s_shadow_params) -> np.ndarray:
    """Light records [n, 8] float32 (word 7 is the face as uint32 bits)."""
    r = np.ascontiguousarray(records)
    out = np.zeros((max(n, 1), 8), np.float32)
    lib().orc_light_prepass(r.ctypes.data, n, C.byref(p), out.ctypes.data)
    return out[:n]


def pairs(light_records: np.ndarray, size: int):
    r = np.ascontiguousarray(light_records, np.float32).reshape(-1, 8)
    c = np.zeros(max(1, len(r)), np.uint32)
    total = lib().orc_cube_pairs(r.ctypes.data, len(r), size, c.ctypes.data)
    return c[: len(r)], int(total)


def cube(light_records: np.ndarray, size: int, n: int | None = None) -> np.ndarray:
    """The cube map [6, S, S] float32 after the face draws of the first n light records."""
    r = np.ascontiguousarray(light_records, np.float32).reshape(-1, 8)
    n = len(r) if n is None else n
    out = np.zeros((6, size, size), np.float32)
    lib().orc_cube_raster(r.ctypes.data, n, size, out.ctypes.data)
    return out


def deferred_light(gbuffer: dict, cube_map, p: _abi.m2s_light_params) -> np.ndarray:
    """The RGBA8 image [H, W, 4] of the lighting pass; gbuffer: {target: (H, W, 4) array} (fp16 / uint8), missing = 0."""
    keep = []

    def ptr(name, dt):
        if name not in gbuffer or gbuffer[name] is None:
            return None
        a = np.ascontiguousarray(gbuffer[name]).view(dt)
        keep.append(a)
        return a.ctypes.data
    cm = None if cube_map is None else np.ascontiguousarray(cube_map, np.float32)
    img = np.zeros((p.height, p.width, 4), np.uint8)
    lib().orc_deferred_light(ptr("position", np.uint16), ptr("normal", np.uint16), ptr("albedo", np.uint8),
                             ptr("metallic_roughness", np.uint8), None if cm is None else cm.ctypes.data, C.byref(p), img.ctypes.data)
    return img
