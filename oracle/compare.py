"""ctypes wrapper of the image comparison's checker (build_compare.py, m2s_compare_oracle.c) and an fp64 numpy/scipy
statement of Wang et al.'s valid-window SSIM it is held against."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from mesh2splat_b200 import _abi

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_compare import build_compare_oracle
        L = C.CDLL(build_compare_oracle())
        L.orc_compare_taps.restype = None
        L.orc_compare_taps.argtypes = [C.c_void_p]
        L.orc_compare_constants.restype = None
        L.orc_compare_constants.argtypes = [C.c_void_p]
        L.orc_ssim_value.restype = C.c_float
        L.orc_ssim_value.argtypes = [C.c_float] * 5
        L.orc_image_compare.restype = C.c_int
        L.orc_image_compare.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                        C.c_void_p, C.POINTER(_abi.m2s_compare_result)]
        _lib = L
    return _lib


def taps() -> np.ndarray:
    out = np.zeros(11, np.float32)
    lib().orc_compare_taps(out.ctypes.data)
    return out


def constants() -> np.ndarray:
    """(C1, C2) as the kernel uses them."""
    out = np.zeros(2, np.float32)
    lib().orc_compare_constants(out.ctypes.data)
    return out


def ssim_value(mx, my, exx, eyy, exy) -> np.float32:
    return np.float32(lib().orc_ssim_value(float(mx), float(my), float(exx), float(eyy), float(exy)))


def _img(x, w: int, h: int):
    if x is None:
        return None
    a = np.ascontiguousarray(x, np.uint8).reshape(-1)
    assert a.size == w * h * 4, (a.size, w, h)
    return a


def compare(a, b, width: int, height: int, cover_a=None, cover_b=None, cover_min: int = 128):
    """orc_image_compare: (result dict as Context.compare_images returns it, map (h - 10, w - 10) float32, per-channel
    values (3, h - 10, w - 10) float32).  Images: (h, w, 4) uint8 (or flat), row 0 = the bottom row."""
    A, B, CA, CB = (_img(x, width, height) for x in (a, b, cover_a, cover_b))
    nw = (width - 10) * (height - 10)
    m = np.zeros(max(nw, 1), np.float32)
    planes = np.zeros(max(3 * nw, 1), np.float32)
    r = _abi.m2s_compare_result()
    st = lib().orc_image_compare(A.ctypes.data, B.ctypes.data, CA.ctypes.data if CA is not None else None,
                                 CB.ctypes.data if CB is not None else None, width, height, cover_min, m.ctypes.data, planes.ctypes.data,
                                 C.byref(r))
    if st != 0:
        raise ValueError("orc_image_compare: size or cover_min out of range")
    return (_abi.compare_result_dict(r, width * height), m[:nw].reshape(height - 10, width - 10),
            planes[: 3 * nw].reshape(3, height - 10, width - 10))


def gaussian_window() -> np.ndarray:
    """The fp64 normalised Gaussian of the window (sigma 1.5, 11 taps)."""
    g = np.array([math.exp(-(i * i) / 4.5) for i in range(-5, 6)], np.float64)
    return g / math.fsum(g)


def reference_ssim(a, b) -> np.ndarray:
    """Wang et al.'s SSIM in fp64 over the valid windows (scipy separable correlation with the Gaussian window), the mean
    over R, G, B: (h - 10, w - 10).  a, b: (h, w, >= 3) uint8."""
    from scipy.ndimage import correlate1d
    w = gaussian_window()
    C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2

    def blur(x):
        x = correlate1d(correlate1d(x, w, axis=1, mode="constant"), w, axis=0, mode="constant")
        return x[5:-5, 5:-5]
    out = np.zeros((a.shape[0] - 10, a.shape[1] - 10), np.float64)
    for c in range(3):
        x, y = a[..., c].astype(np.float64), b[..., c].astype(np.float64)
        mx, my = blur(x), blur(y)
        vx, vy, cxy = blur(x * x) - mx * mx, blur(y * y) - my * my, blur(x * y) - mx * my
        out += ((2 * mx * my + C1) * (2 * cxy + C2)) / ((mx * mx + my * my + C1) * (vx + vy + C2))
    return out / 3.0
