"""ctypes wrappers of the splat draw's checkers (row f-6): the C restatement (libm2s_splat_oracle.so) and the
reference's own shaders in their GL environment (_ref/libm2s_refsplat.so, present only where it could be built)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
TARGETS = (("position", np.float16), ("normal", np.float16), ("albedo", np.uint8), ("depth", np.float16),
           ("metallic_roughness", np.uint8))
_lib = None
_ref = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_splat import build_splat_oracle
        L = C.CDLL(build_splat_oracle())
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        L.orc_splat_exp.restype = f32
        L.orc_splat_exp.argtypes = [f32]
        L.orc_splat_vs.restype = None
        L.orc_splat_vs.argtypes = [vp, C.c_int, f32, f32, vp]
        L.orc_splat_fs.restype = None
        L.orc_splat_fs.argtypes = [vp, f32, f32, C.c_int, vp]
        L.orc_splat_coverage.restype = None
        L.orc_splat_coverage.argtypes = [vp, C.c_int, u32, u32, vp]
        L.orc_splat_pairs.restype = C.c_uint64
        L.orc_splat_pairs.argtypes = [vp, u32, u32, u32, vp]
        L.orc_splat_draw.restype = None
        L.orc_splat_draw.argtypes = [vp, u32, u32, u32, u32, vp, vp, vp, vp, vp]
        _lib = L
    return _lib


def ref_lib():
    """The reference's shaders in their GL environment, or None if never built (no reference checkout)."""
    global _ref
    if _ref is None:
        path = os.path.join(_HERE, "_ref", "libm2s_refsplat.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        R.ref_splat_vs.restype = None
        R.ref_splat_vs.argtypes = [vp, C.c_int, f32, f32, vp]
        R.ref_splat_fs.restype = None
        R.ref_splat_fs.argtypes = [vp, f32, f32, C.c_int, vp]
        R.ref_splat_draw.restype = None
        R.ref_splat_draw.argtypes = [vp, u32, u32, u32, C.c_int, vp, vp, vp, vp, vp]
        _ref = R
    return _ref


def exp(x) -> np.ndarray:
    """The exp of DESIGN §2, elementwise over float32 values."""
    L = lib()
    a = np.asarray(x, np.float32).ravel()
    return np.array([L.orc_splat_exp(float(v)) for v in a], np.float32)


def _quads(quads) -> np.ndarray:
    return np.ascontiguousarray(quads, np.float32).reshape(-1, 24)


def vs(quad, vertex: int, width: float, height: float, ref: bool = False) -> np.ndarray:
    """One vertex-shader invocation: gl_Position.xy + the 18 varyings (20 float32)."""
    q = _quads(quad)
    out = np.zeros(20, np.float32)
    getattr(ref_lib() if ref else lib(), "ref_splat_vs" if ref else "orc_splat_vs")(q.ctypes.data, int(vertex), float(width), float(height), out.ctypes.data)
    return out


def fs(varyings, frag_x: float, frag_y: float, mode: int, ref: bool = False) -> np.ndarray:
    """One fragment-shader invocation: the five outputs (20 float32)."""
    v = np.ascontiguousarray(varyings, np.float32)
    out = np.zeros(20, np.float32)
    getattr(ref_lib() if ref else lib(), "ref_splat_fs" if ref else "orc_splat_fs")(v.ctypes.data, float(frag_x), float(frag_y), int(mode), out.ctypes.data)
    return out


def coverage(quad, tri: int, width: int, height: int) -> np.ndarray:
    """Pixels triangle `tri` (0: V0 V1 V2, 1: V0 V2 V3) of the quad covers: bool (height, width)."""
    q = _quads(quad)
    m = np.zeros((height, width), np.uint8)
    lib().orc_splat_coverage(q.ctypes.data, tri, width, height, m.ctypes.data)
    return m.astype(bool)


def pairs(quads, width: int, height: int):
    """(per-quad (16 x 16 tile, quad) pair counts as the draw's tile pass makes them, total)."""
    q = _quads(quads)
    c = np.zeros(max(1, len(q)), np.uint32)
    total = lib().orc_splat_pairs(q.ctypes.data, len(q), width, height, c.ctypes.data)
    return c[: len(q)], int(total)


def draw(quads, width: int, height: int, mode: int = 0, n: int | None = None, targets=None, ref: bool = False) -> dict:
    """orc_splat_draw (or the reference's shaders with ref=True) of the first n quads: {target: (height, width, 4)}."""
    q = _quads(quads)
    n = len(q) if n is None else n
    targets = [t for t, _ in TARGETS] if targets is None else targets
    bufs = {t: np.zeros((height, width, 4), dt) for t, dt in TARGETS if t in targets}
    ptr = [bufs[t].ctypes.data if t in bufs else None for t, _ in TARGETS]
    if ref:
        ref_lib().ref_splat_draw(q.ctypes.data, n, width, height, mode, *ptr)
    else:
        lib().orc_splat_draw(q.ctypes.data, n, width, height, mode, *ptr)
    return bufs
