"""ctypes wrapper of the codec checker (build_codec.py): the writer's and the loader's per-value formulas with glibc's
logf / expf, on float32 arrays."""
from __future__ import annotations

import ctypes as C

import numpy as np

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_codec import build_codec_oracle
        L = C.CDLL(build_codec_oracle())
        for name in ("orc_codec_sh0", "orc_codec_logit", "orc_codec_expf", "orc_codec_sigmoid"):
            getattr(L, name).restype = None
            getattr(L, name).argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        L.orc_codec_log_scale.restype = None
        L.orc_codec_log_scale.argtypes = [C.c_void_p, C.c_uint64, C.c_float, C.c_void_p]
        _lib = L
    return _lib


def _apply(name: str, x, *extra) -> np.ndarray:
    a = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(a)
    if a.size:
        fn = getattr(lib(), name)
        if extra:
            fn(a.ctypes.data, a.size, *extra, out.ctypes.data)
        else:
            fn(a.ctypes.data, a.size, out.ctypes.data)
    return out


def sh0(c) -> np.ndarray:
    """(c - 0.5f) / SH_COEFF0 (utils.cpp:47)."""
    return _apply("orc_codec_sh0", c)


def logit(a) -> np.ndarray:
    """utils::invSigmoid (utils.hpp:270)."""
    return _apply("orc_codec_logit", a)


def log_scale(s, mult: float) -> np.ndarray:
    """logf(s * mult) (parsers.cpp:497-499)."""
    return _apply("orc_codec_log_scale", s, C.c_float(mult))


def expf(x) -> np.ndarray:
    return _apply("orc_codec_expf", x)


def sigmoid(o) -> np.ndarray:
    """utils::sigmoid (utils.hpp:269): 1.0 / (1.0 + (double)expf(-o))."""
    return _apply("orc_codec_sigmoid", o)
