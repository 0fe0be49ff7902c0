"""ctypes wrappers of the prepass's view-dependent colour checker (build_sh.py, m2s_sh_oracle.c) and an fp64 numpy
statement of graphdeco's computeColorFromSH it is held against."""
from __future__ import annotations

import ctypes as C

import numpy as np

from mesh2splat_b200 import _abi

_lib = None
# graphdeco's constants (utils/sh_utils.py, cuda_rasterizer/forward.cu), in fp64
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
         -0.5900435899266435)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_sh import build_sh_oracle
        L = C.CDLL(build_sh_oracle())
        L.orc_sh_camera.restype = C.c_int
        L.orc_sh_camera.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.orc_sh_colours.restype = None
        L.orc_sh_colours.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        L.orc_prepass_sh.restype = C.c_uint32
        L.orc_prepass_sh.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int,
                                     C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _mat(m) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(m, np.float32).ravel())


def _sh(sh, n: int, buffer_degree: int) -> np.ndarray:
    a = np.ascontiguousarray(np.asarray(sh, np.float32).reshape(-1))
    assert a.size >= n * _abi.SH_FLOATS[buffer_degree], (a.size, n, buffer_degree)
    return a if a.size else np.zeros(1, np.float32)


def camera(world_to_view, model_to_world):
    """orc_sh_camera: the camera position in model space (float32 [3]), or None for a singular V M."""
    cam = np.zeros(3, np.float32)
    V, M = _mat(world_to_view), _mat(model_to_world)
    return cam if lib().orc_sh_camera(V.ctypes.data, M.ctypes.data, cam.ctypes.data) else None


def colours(gaussians24, sh, buffer_degree: int, sh_degree: int, cam) -> np.ndarray:
    """orc_sh_colours: [n, 3] float32, max(record colour + rest, 0) per channel."""
    g = np.ascontiguousarray(gaussians24, np.float32).reshape(-1, 24)
    s = _sh(sh, len(g), buffer_degree)
    c = np.ascontiguousarray(cam, np.float32)
    out = np.zeros((max(len(g), 1), 3), np.float32)
    lib().orc_sh_colours(g.ctypes.data, len(g), s.ctypes.data, buffer_degree, sh_degree, c.ctypes.data, out.ctypes.data)
    return out[: len(g)]


def prepass_sh(gaussians24, world_to_view, view_to_clip, model_to_world, resolution, near_far, std_dev, render_mode, ply_has_pbr, sh,
               buffer_degree: int, sh_degree: int):
    """orc_prepass_sh on loaded .ply records (u_format 1): (quads [m, 24], depths [m]) in input order of the survivors."""
    g = np.ascontiguousarray(gaussians24, np.float32).reshape(-1, 24)
    s = _sh(sh, len(g), buffer_degree)
    V, P, M = _mat(world_to_view), _mat(view_to_clip), _mat(model_to_world)
    res, nf = np.asarray(resolution, np.float32), np.asarray(near_far, np.float32)
    quads = np.zeros((max(len(g), 1), 24), np.float32)
    depths = np.zeros(max(len(g), 1), np.float32)
    n = lib().orc_prepass_sh(g.ctypes.data, len(g), V.ctypes.data, P.ctypes.data, M.ctypes.data, res.ctypes.data, nf.ctypes.data,
                             C.c_float(std_dev), int(render_mode), 1, int(ply_has_pbr), s.ctypes.data, buffer_degree, sh_degree,
                             quads.ctypes.data, depths.ctypes.data)
    assert n != 0xFFFFFFFF, "singular V M"
    return quads[:n].copy(), depths[:n].copy()


def reference_rgb(dirs, coeffs, dc_colour) -> np.ndarray:
    """graphdeco's computeColorFromSH in fp64: dirs [n, 3] (any length), coeffs [n, K, 3] (K = 3, 8 or 15: coefficients 1..K),
    dc_colour [n, 3] (SH_C0 f_dc + 0.5, the record colour) -> max(colour + rest, 0) [n, 3]."""
    d = np.asarray(dirs, np.float64)
    d = d / np.linalg.norm(d, axis=1, keepdims=True)
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    sh = np.asarray(coeffs, np.float64)
    K = sh.shape[1]
    r = np.asarray(dc_colour, np.float64).copy()
    r = r - SH_C1 * y * sh[:, 0] + SH_C1 * z * sh[:, 1] - SH_C1 * x * sh[:, 2]
    if K > 3:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        r = (r + SH_C2[0] * xy * sh[:, 3] + SH_C2[1] * yz * sh[:, 4] + SH_C2[2] * (2.0 * zz - xx - yy) * sh[:, 5]
             + SH_C2[3] * xz * sh[:, 6] + SH_C2[4] * (xx - yy) * sh[:, 7])
        if K > 8:
            r = (r + SH_C3[0] * y * (3.0 * xx - yy) * sh[:, 8] + SH_C3[1] * xy * z * sh[:, 9]
                 + SH_C3[2] * y * (4.0 * zz - xx - yy) * sh[:, 10] + SH_C3[3] * z * (2.0 * zz - 3.0 * xx - 3.0 * yy) * sh[:, 11]
                 + SH_C3[4] * x * (4.0 * zz - xx - yy) * sh[:, 12] + SH_C3[5] * z * (xx - yy) * sh[:, 13]
                 + SH_C3[6] * x * (xx - 3.0 * yy) * sh[:, 14])
    return np.maximum(r, 0.0)


def block_from_file_order(rest, degree: int) -> np.ndarray:
    """f_rest values in file order [n, 3K] (channel-major: coefficient k of channel c at c K + k - 1) -> the SH buffer
    [n, M2S_SH_FLOATS(degree)] (coefficient-major, zero padding), as m2s_ply_read_sh writes it; float32, bit for bit."""
    K = (degree + 1) ** 2 - 1
    r = np.ascontiguousarray(rest, np.float32).reshape(len(rest), 3, K)
    out = np.zeros((len(r), _abi.SH_FLOATS[degree]), np.float32)
    out[:, : 3 * K] = r.transpose(0, 2, 1).reshape(len(r), 3 * K)
    return out
