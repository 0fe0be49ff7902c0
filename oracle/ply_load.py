"""ctypes wrappers of the .ply loader's checkers (build_ply_load.py): the plain-C restatement of loadPlyFile's
per-vertex arithmetic and the reference's own loadPlyFile."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from mesh2splat_b200 import _abi

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None
_ref = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_ply_load import build_ply_oracle
        L = C.CDLL(build_ply_oracle())
        L.orc_ply_load.restype = None
        L.orc_ply_load.argtypes = [C.c_void_p, C.POINTER(_abi.m2s_ply_info), C.c_uint64, C.c_void_p]
        _lib = L
    return _lib


def ref_lib():
    """The reference's loadPlyFile (oracle/_ref/libm2s_refplyload.so), or None when it was not built."""
    global _ref
    if _ref is None:
        path = os.path.join(HERE, "_ref", "libm2s_refplyload.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        R.ref_load_ply.restype = C.c_int64
        R.ref_load_ply.argtypes = [C.c_char_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_int)]
        _ref = R
    return _ref


def load(rows, info: _abi.m2s_ply_info, count: int | None = None) -> np.ndarray:
    """orc_ply_load: raw vertex rows (bytes / uint8 array of count * row_stride bytes) -> [count, 24] float32 records."""
    r = np.frombuffer(bytes(rows), np.uint8) if not isinstance(rows, np.ndarray) else np.ascontiguousarray(rows, np.uint8).reshape(-1)
    if count is None:
        count = len(r) // info.row_stride
    out = np.zeros((max(count, 1), 24), np.float32)
    lib().orc_ply_load(r.ctypes.data if len(r) else None, C.byref(info), count, out.ctypes.data)
    return out[:count]


def load_file(path: str, info: _abi.m2s_ply_info) -> np.ndarray:
    """orc_ply_load on the vertex rows of a file whose header `info` describes."""
    with open(path, "rb") as f:
        f.seek(info.body_offset)
        rows = f.read(info.vertex_count * info.row_stride)
    return load(rows, info, info.vertex_count)


def ref_load(path: str):
    """The reference's loadPlyFile on a file: (records [n, 24] float32, has_pbr), or None when it rejected the file."""
    R = ref_lib()
    if R is None:
        raise RuntimeError("oracle/_ref/libm2s_refplyload.so is not built (python -m oracle.build_ply_load)")
    pbr = C.c_int(0)
    n = R.ref_load_ply(str(path).encode(), None, 0, C.byref(pbr))
    if n < 0:
        return None
    out = np.zeros((max(n, 1), 24), np.float32)
    R.ref_load_ply(str(path).encode(), out.ctypes.data, n, C.byref(pbr))
    return out[:n], int(pbr.value)


def light_params(p: _abi.m2s_shadow_params) -> _abi.m2s_shadow_params:
    """The light oracle's parameters for a shadow pass on M2S_VIEW_PLY* records: the records are REF96 and the scale
    multiplier of u_format 1 is 1 (gaussianPointShadowMappingCS.glsl:96), i.e. REF96 with std_dev 1 (x * 1.0f == x
    exactly, so the restatement's arithmetic is unchanged)."""
    q = _abi.m2s_shadow_params.from_buffer_copy(p)
    if q.layout in (_abi.VIEW_PLY, _abi.VIEW_PLY_PBR):
        q.layout, q.std_dev = _abi.LAYOUT_REF96, 1.0
    return q
