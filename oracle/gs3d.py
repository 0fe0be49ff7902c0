"""ctypes wrappers of the standard 3DGS render's checker (build_3dgs.py, m2s_3dgs_oracle.c) and an fp64 numpy statement of
graphdeco's forward pass in graphdeco's own convention (an OpenCV camera, row 0 at the top) that it is held against."""
from __future__ import annotations

import ctypes as C

import numpy as np

from mesh2splat_b200 import _abi

_lib = None
SH_C0 = 0.28209479177387814


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_3dgs import build_3dgs_oracle
        L = C.CDLL(build_3dgs_oracle())
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        L.orc_3dgs_preprocess.restype = u32
        L.orc_3dgs_preprocess.argtypes = [vp, u32, u32, vp, vp, vp, u32, u32, f32, f32, f32, vp, u32, u32, vp, vp]
        L.orc_3dgs_render.restype = C.c_int
        L.orc_3dgs_render.argtypes = [vp, u32, u32, vp, vp, vp, u32, u32, f32, f32, f32, vp, vp, u32, u32, C.c_uint64, vp, vp,
                                      C.POINTER(u32), C.POINTER(C.c_uint64)]
        _lib = L
    return _lib


def _mat(m) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(m, np.float32).ravel())


def _records(records, layout: int) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(records, np.float32).reshape(-1, 14 if layout == _abi.LAYOUT_PACKED56 else 24))


def _sh(sh, n: int, buffer_degree: int) -> np.ndarray:
    if sh is None:
        return np.zeros(1, np.float32)
    a = np.ascontiguousarray(np.asarray(sh, np.float32).reshape(-1))
    assert a.size >= n * _abi.SH_FLOATS[buffer_degree], (a.size, n, buffer_degree)
    return a if a.size else np.zeros(1, np.float32)


def preprocess(records, layout: int, world_to_view, view_to_clip, model_to_world, width: int, height: int, near: float = 0.2,
               std_dev: float = 1.0, scale_modifier: float = 1.0, sh=None, buffer_degree: int = 0, sh_degree: int = 0):
    """orc_3dgs_preprocess: (splat records [n, 12] float32, keys [n] uint32, survivors)."""
    g = _records(records, layout)
    n = len(g)
    s = _sh(sh, n, buffer_degree)
    V, P, M = _mat(world_to_view), _mat(view_to_clip), _mat(model_to_world)
    splats = np.zeros((max(n, 1), 12), np.float32)
    keys = np.zeros(max(n, 1), np.uint32)
    alive = lib().orc_3dgs_preprocess(g.ctypes.data, n, layout, V.ctypes.data, P.ctypes.data, M.ctypes.data, width, height, near, std_dev,
                                      scale_modifier, s.ctypes.data, buffer_degree, sh_degree, splats.ctypes.data, keys.ctypes.data)
    assert alive != 0xFFFFFFFF, "singular V M"
    return splats[:n].copy(), keys[:n].copy(), int(alive)


def render(records, layout: int, world_to_view, view_to_clip, model_to_world, width: int, height: int, near: float = 0.2,
           std_dev: float = 1.0, scale_modifier: float = 1.0, background=(0.0, 0.0, 0.0), sh=None, buffer_degree: int = 0,
           sh_degree: int = 0, max_pairs: int | None = None):
    """orc_3dgs_render: (rgba32f (H, W, 4) float32, rgba8 (H, W, 4) uint8, drawn, pairs); row 0 = the bottom row."""
    g = _records(records, layout)
    n = len(g)
    s = _sh(sh, n, buffer_degree)
    V, P, M = _mat(world_to_view), _mat(view_to_clip), _mat(model_to_world)
    bg = np.asarray(background, np.float32)
    f32 = np.zeros((height, width, 4), np.float32)
    u8 = np.zeros((height, width, 4), np.uint8)
    drawn, pairs = C.c_uint32(0), C.c_uint64(0)
    rc = lib().orc_3dgs_render(g.ctypes.data if n else None, n, layout, V.ctypes.data, P.ctypes.data, M.ctypes.data, width, height, near,
                               std_dev, scale_modifier, bg.ctypes.data, s.ctypes.data, buffer_degree, sh_degree,
                               (1 << 64) - 1 if max_pairs is None else int(max_pairs), f32.ctypes.data, u8.ctypes.data, C.byref(drawn),
                               C.byref(pairs))
    assert rc == 0, "singular V M or out of memory"
    return f32, u8, int(drawn.value), int(pairs.value)


# ---- graphdeco's forward pass in fp64, in its own convention -------------------------------------------------------------
def decode(records, layout: int, std_dev: float = 1.0):
    """(position [n, 3], scale [n, 3], rotation wxyz [n, 4], colour [n, 3], opacity [n]) in fp64; REF96 scale times std_dev."""
    g = np.asarray(records, np.float32).reshape(-1, 14 if layout == _abi.LAYOUT_PACKED56 else 24).astype(np.float64)
    if layout == _abi.LAYOUT_PACKED56:
        return (g[:, 0:3], np.exp(g[:, 7:10]), g[:, 3:7], g[:, 10:13] * SH_C0 + 0.5, 1.0 / (1.0 + np.exp(-g[:, 13])))
    mult = std_dev if layout == _abi.LAYOUT_REF96 else 1.0
    return g[:, 0:3], g[:, 8:11] * np.float64(np.float32(mult)), g[:, 16:20], g[:, 4:7], g[:, 7]


def graphdeco_forward(pos, scale, rot, colour, opacity, world_to_view, view_to_clip, width: int, height: int, near: float,
                      scale_modifier: float = 1.0, background=(0.0, 0.0, 0.0), model_to_world=None, power_err=None, mean_err=None,
                      render: bool = True):
    """preprocessCUDA + renderCUDA in fp64 with an OpenCV camera made from the GL one (the view matrix's y and z rows
    negated, y_ndc negated), row 0 at the top.  Returns (per gaussian: dict of u, v (GL pixel frame), conic, radius,
    depth, alive, rect), and the image (H, W, 4) flipped to row 0 at the bottom, plus per pixel the smallest margin of any
    alpha to 1/255, 0.99 and the 1e-4 stop, and whether the pixel's set of gaussians depends on the tile rectangles:
    whether a gaussian that reaches it (power <= 0, alpha >= 1/255) lies outside its rectangle in either convention's
    rows, OpenCV's (counted from the top, the ones composited here) or GL's (from the bottom, the checker's).

    For error bounds the dict also holds, per gaussian, cov (a, b, c: the dilated 2-D covariance, GL frame) and mag
    (|T|_F^2 (s_x^2 + s_y^2 + s_z^2) + 0.3: the size of the terms cov is summed from), and per pixel (flipped like the
    image) blended (the number of terms composited) and dalpha: the sum over those terms of T alpha (power_err |power| +
    mean_err |grad_mean power|), power_err and mean_err being per-gaussian relative and absolute (pixel) error bounds of
    the power's quadratic form and of the mean (default 0): to first order, the largest change of any output channel
    those errors can make, in units of max(colour, background).  render False: the per-gaussian dict alone (then the
    image, margin and rectangle flags are None and the dict has no per-pixel entries)."""
    V = np.asarray(world_to_view, np.float64).reshape(4, 4).T
    M = np.eye(4) if model_to_world is None else np.asarray(model_to_world, np.float64).reshape(4, 4).T
    P = np.asarray(view_to_clip, np.float64).reshape(4, 4).T
    flip = np.diag([1.0, -1.0, -1.0, 1.0])
    Vcv = flip @ V @ M                                    # OpenCV view: x right, y down, z forward
    n = len(pos)
    ph = np.c_[pos, np.ones(n)]
    t = ph @ Vcv.T                                        # camera-space (OpenCV)
    z = t[:, 2]
    alive = z > near
    tan_x, tan_y = 1.0 / P[0, 0], 1.0 / P[1, 1]
    fx, fy = width / (2.0 * tan_x), height / (2.0 * tan_y)
    tgl = ph @ (V @ M).T
    clip = tgl @ P.T
    pw = 1.0 / (clip[:, 3] + 1e-7)
    ndc_x, ndc_y = clip[:, 0] * pw, -clip[:, 1] * pw     # OpenCV ndc y points down
    u = ((ndc_x + 1.0) * width - 1.0) * 0.5
    vcv = ((ndc_y + 1.0) * height - 1.0) * 0.5
    q = np.asarray(rot, np.float64)
    q = q / np.maximum(np.linalg.norm(q, axis=1, keepdims=True), 1e-12)
    w, x, y, zq = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.stack([np.stack([1 - 2 * (y * y + zq * zq), 2 * (x * y - w * zq), 2 * (x * zq + w * y)], -1),
                  np.stack([2 * (x * y + w * zq), 1 - 2 * (x * x + zq * zq), 2 * (y * zq - w * x)], -1),
                  np.stack([2 * (x * zq - w * y), 2 * (y * zq + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    s = np.asarray(scale, np.float64) * scale_modifier
    Sig = R @ (s[:, :, None] ** 2 * np.transpose(R, (0, 2, 1)))
    lx, ly = 1.3 * tan_x, 1.3 * tan_y
    zs = np.where(alive, z, 1.0)
    txc = np.clip(t[:, 0] / zs, -lx, lx) * zs
    tyc = np.clip(t[:, 1] / zs, -ly, ly) * zs
    J = np.zeros((n, 2, 3))
    J[:, 0, 0], J[:, 0, 2] = fx / zs, -fx * txc / zs ** 2
    J[:, 1, 1], J[:, 1, 2] = fy / zs, -fy * tyc / zs ** 2
    Wv = Vcv[:3, :3]
    T = J @ Wv
    cov = T @ Sig @ np.transpose(T, (0, 2, 1))
    a, b, c = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a * c - b * b
    alive &= det != 0
    dets = np.where(det != 0, det, 1.0)
    conic = np.stack([c / dets, -b / dets, a / dets], -1)
    mid = 0.5 * (a + c)
    sq = np.sqrt(np.maximum(0.1, mid * mid - det))
    radius = np.ceil(3.0 * np.sqrt(np.maximum(mid + sq, mid - sq)))
    gx, gy = (width + 15) // 16, (height + 15) // 16
    rect = np.stack([np.clip(((u - radius) / 16).astype(np.int64), 0, gx), np.clip(((vcv - radius) / 16).astype(np.int64), 0, gy),
                     np.clip(((u + radius + 15) / 16).astype(np.int64), 0, gx), np.clip(((vcv + radius + 15) / 16).astype(np.int64), 0, gy)], -1)
    alive &= (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1]) != 0
    mag = (T ** 2).sum(axis=(1, 2)) * (s ** 2).sum(axis=1) + 0.3
    info = {"u": u, "v": height - 1.0 - vcv, "conic": conic * np.array([1.0, -1.0, 1.0]), "radius": radius, "depth": z, "alive": alive,
            "rect": rect, "cov": np.stack([a, -b, c], -1), "mag": mag}
    if not render:
        return info, None, None, None
    order = sorted(np.nonzero(alive)[0], key=lambda i: (z[i], i))
    col = np.maximum(np.asarray(colour, np.float64), 0.0)
    op = np.asarray(opacity, np.float64)
    img = np.zeros((height, width, 4))
    margin = np.full((height, width), np.inf)
    ys, xs = np.mgrid[0:height, 0:width].astype(np.float64)
    T_ = np.ones((height, width))
    C_ = np.zeros((height, width, 3))
    done = np.zeros((height, width), bool)
    rect_dep = np.zeros((height, width), bool)
    blended = np.zeros((height, width), np.int64)
    dalpha = np.zeros((height, width))
    perr = np.zeros(n) if power_err is None else np.broadcast_to(np.asarray(power_err, np.float64), (n,))
    merr = np.zeros(n) if mean_err is None else np.broadcast_to(np.asarray(mean_err, np.float64), (n,))
    tile_x, tile_y = (xs // 16).astype(np.int64), (ys // 16).astype(np.int64)
    # the rows of the rectangles in the GL frame the checker bins in (rows counted from the bottom)
    tile_gl = ((height - 1 - ys) // 16).astype(np.int64)
    vgl = height - 1.0 - vcv
    rect_gl = np.stack([np.clip(((vgl - radius) / 16).astype(np.int64), 0, gy), np.clip(((vgl + radius + 15) / 16).astype(np.int64), 0, gy)], -1)
    for i in order:
        dx, dy = u[i] - xs, vcv[i] - ys
        power = -0.5 * (conic[i, 0] * dx * dx + conic[i, 2] * dy * dy) - conic[i, 1] * dx * dy
        grad = np.hypot(conic[i, 0] * dx + conic[i, 1] * dy, conic[i, 1] * dx + conic[i, 2] * dy)
        al = np.minimum(0.99, op[i] * np.exp(power))
        in_rect = (tile_x >= rect[i, 0]) & (tile_x < rect[i, 2]) & (tile_y >= rect[i, 1]) & (tile_y < rect[i, 3])
        in_gl = (tile_x >= rect[i, 0]) & (tile_x < rect[i, 2]) & (tile_gl >= rect_gl[i, 0]) & (tile_gl < rect_gl[i, 1])
        use = (power <= 0) & (al >= 1.0 / 255.0)
        rect_dep |= use & ~(in_rect & in_gl) & ~done
        use &= in_rect & ~done
        tt = T_ * (1 - al)
        stop = use & (tt < 1e-4)
        live = ~done & in_rect & (power <= 0)
        m = np.minimum(np.abs(al - 1.0 / 255.0), np.abs(op[i] * np.exp(power) - 0.99))
        m = np.minimum(m, np.abs(tt - 1e-4) / np.maximum(T_, 1e-30))
        margin = np.where(live, np.minimum(margin, m), margin)
        done |= stop
        add = use & ~stop
        C_ += np.where(add[..., None], col[i] * (al * T_)[..., None], 0.0)
        blended += add
        dalpha += np.where(add, T_ * al * (perr[i] * np.abs(power) + merr[i] * grad), 0.0)
        T_ = np.where(add, tt, T_)
    img[..., :3] = C_ + T_[..., None] * np.asarray(background, np.float64)
    img[..., 3] = 1.0 - T_
    info.update(blended=blended[::-1].copy(), dalpha=dalpha[::-1].copy())
    return info, img[::-1].copy(), margin[::-1].copy(), rect_dep[::-1].copy()
