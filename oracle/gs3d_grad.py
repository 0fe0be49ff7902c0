"""ctypes wrapper of the standard 3DGS render's backward checker (build_3dgs_grad.py, m2s_3dgs_grad_oracle.c) and an fp64
torch-autograd statement of graphdeco's forward pass with graphdeco's gradient conventions that it is held against.

The torch statement is a dense port of gs3d.graphdeco_forward written directly in the project's GL frame (row 0 at the
bottom, the checker's tile rows), so its tile rectangles are the checker's: they and the depth order are taken from the
forward checker (gs3d.preprocess) and carry no gradient.  Conventions: the 0.99 alpha clamp passes the gradient as if
unclamped; a gaussian below 1/255 or past a pixel's stop contributes nothing; a view x or y clamped at 1.3 tan(fov / 2)
is held (no gradient to it, and J's dependence on the depth is taken with it held); a colour clamped at 0 gets nothing;
an infinite opacity logit gets 0 and a record with a NaN logit a row of zeros (torch_backward)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle import gs3d

_lib = None
SH_C0 = 0.28209479177387814


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        from oracle.build_3dgs_grad import build_3dgs_grad_oracle
        L = C.CDLL(build_3dgs_grad_oracle())
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        L.orc_3dgs_backward.restype = C.c_int
        L.orc_3dgs_backward.argtypes = [vp, u32, vp, vp, vp, u32, u32, f32, f32, vp, C.c_uint64, vp, vp, C.POINTER(u32)]
        _lib = L
    return _lib


def backward(records, world_to_view, view_to_clip, model_to_world, width: int, height: int, grad_rgba, near: float = 0.2,
             scale_modifier: float = 1.0, background=(0.0, 0.0, 0.0), max_pairs: int | None = None):
    """orc_3dgs_backward: (dL/dparams [n, 14] float32, drawn) for PACKED56 records and dL/d(image) (H, W, 4)."""
    g = np.ascontiguousarray(np.asarray(records, np.float32).reshape(-1, 14))
    n = len(g)
    V, P, M = (np.ascontiguousarray(np.asarray(m, np.float32).ravel()) for m in (world_to_view, view_to_clip, model_to_world))
    bg = np.asarray(background, np.float32)
    gi = np.ascontiguousarray(np.asarray(grad_rgba, np.float32).reshape(height, width, 4))
    out = np.zeros((max(n, 1), 14), np.float32)
    drawn = C.c_uint32(0)
    rc = lib().orc_3dgs_backward(g.ctypes.data if n else None, n, V.ctypes.data, P.ctypes.data, M.ctypes.data, width, height, near,
                                 scale_modifier, bg.ctypes.data, (1 << 64) - 1 if max_pairs is None else int(max_pairs), gi.ctypes.data,
                                 out.ctypes.data, C.byref(drawn))
    assert rc == 0, "singular V M or out of memory"
    return out[:n].copy(), int(drawn.value)


def torch_forward(params, world_to_view, view_to_clip, model_to_world, width: int, height: int, near: float = 0.2,
                  scale_modifier: float = 1.0, background=(0.0, 0.0, 0.0), records32=None, max_pairs: int | None = None):
    """The (H, W, 4) fp64 image of PACKED56 params (an (n, 14) float64 torch tensor, CPU) as a differentiable function;
    row 0 = the bottom row.  records32: the float32 records whose checker preprocess gives the rectangles, survivors and
    depth order (default: params rounded to float32); max_pairs: the drawn prefix as the render's budget cuts it."""
    import torch
    n = params.shape[0]
    rec32 = np.asarray(params.detach().numpy() if records32 is None else records32, np.float32).reshape(-1, 14)
    sp, keys, alive = gs3d.preprocess(rec32, 1, world_to_view, view_to_clip, model_to_world, width, height, near=near,
                                      scale_modifier=scale_modifier)
    order = sorted(range(n), key=lambda i: (int(keys[i]), i))[:alive]
    rects = sp[:, 9:11].copy().view(np.uint32)
    if max_pairs is not None:
        tot, keep = 0, []
        for i in order:
            rx, ry = rects[i]
            tot += ((rx >> 16) - (rx & 0xFFFF)) * ((ry >> 16) - (ry & 0xFFFF))
            if tot > max_pairs:
                break
            keep.append(i)
        order = keep
    f64 = torch.float64
    V = torch.tensor(np.asarray(world_to_view, np.float32).reshape(4, 4).T, dtype=f64)
    M = torch.tensor(np.asarray(model_to_world, np.float32).reshape(4, 4).T, dtype=f64)
    P = torch.tensor(np.asarray(view_to_clip, np.float32).reshape(4, 4).T, dtype=f64)
    MV = V @ M
    p, q, ls, sh0, logit = params[:, 0:3], params[:, 3:7], params[:, 7:10], params[:, 10:13], params[:, 13]
    t = p @ MV[:3, :3].T + MV[:3, 3]
    d = -t[:, 2]
    th = torch.cat([t, torch.ones(n, 1, dtype=f64)], 1)
    clip = th @ P.T
    pw = 1.0 / (clip[:, 3] + 1e-7)
    u = ((clip[:, 0] * pw + 1.0) * width - 1.0) * 0.5
    v = ((clip[:, 1] * pw + 1.0) * height - 1.0) * 0.5
    s = torch.exp(ls) * scale_modifier
    qn = q / torch.clamp(torch.linalg.norm(q, dim=1, keepdim=True), min=1e-12)
    w, x, y, z = qn[:, 0], qn[:, 1], qn[:, 2], qn[:, 3]
    R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    Sig = R @ torch.diag_embed(s * s) @ R.transpose(1, 2)
    fx, fy = P[0, 0] * width * 0.5, P[1, 1] * height * 0.5
    limx, limy = 1.3 / P[0, 0], 1.3 / P[1, 1]
    ds = torch.where(d > 0, d, torch.ones_like(d))
    txd, tyd = t[:, 0] / ds, t[:, 1] / ds
    txc = torch.where(txd.abs() > limx, (torch.clamp(txd, -limx, limx) * ds).detach(), t[:, 0])
    tyc = torch.where(tyd.abs() > limy, (torch.clamp(tyd, -limy, limy) * ds).detach(), t[:, 1])
    zero = torch.zeros_like(ds)
    J = torch.stack([torch.stack([fx / ds, zero, fx * txc / ds ** 2], -1), torch.stack([zero, fy / ds, fy * tyc / ds ** 2], -1)], 1)
    T = J @ MV[:3, :3]
    cov = T @ Sig @ T.transpose(1, 2)
    ca, cb, cc = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = ca * cc - cb * cb
    det = torch.where(det != 0, det, torch.ones_like(det))
    cA, cB, cC = cc / det, -cb / det, ca / det
    col = torch.clamp(sh0 * SH_C0 + 0.5, min=0.0)
    op = torch.sigmoid(logit)
    ys, xs = torch.meshgrid(torch.arange(height, dtype=f64), torch.arange(width, dtype=f64), indexing="ij")
    tile_x, tile_y = (xs // 16).long(), (ys // 16).long()
    Tr = torch.ones(height, width, dtype=f64)
    Cc = torch.zeros(height, width, 3, dtype=f64)
    done = torch.zeros(height, width, dtype=torch.bool)
    for i in order:
        rx, ry = rects[i]
        in_rect = (tile_x >= int(rx & 0xFFFF)) & (tile_x < int(rx >> 16)) & (tile_y >= int(ry & 0xFFFF)) & (tile_y < int(ry >> 16))
        dx, dy = u[i] - xs, v[i] - ys
        power = -0.5 * (cA[i] * dx * dx + cC[i] * dy * dy) - cB[i] * dx * dy
        aG = op[i] * torch.exp(power)
        alpha = aG + (torch.clamp(aG, max=0.99) - aG).detach()   # the 0.99 clamp, straight through
        use = in_rect & ~done & (power <= 0) & (alpha >= 1.0 / 255.0)
        tt = Tr * (1 - alpha)
        stop = use & (tt < 1e-4)
        add = use & ~stop
        Cc = Cc + torch.where(add[..., None], col[i] * (alpha * Tr)[..., None], torch.zeros((), dtype=f64))
        Tr = torch.where(add, tt, Tr)
        done = done | stop
    bg = torch.tensor(background, dtype=f64)
    return torch.cat([Cc + Tr[..., None] * bg, (1.0 - Tr)[..., None]], -1)


def torch_backward(records, world_to_view, view_to_clip, model_to_world, width: int, height: int, grad_rgba, near: float = 0.2,
                   scale_modifier: float = 1.0, background=(0.0, 0.0, 0.0), max_pairs: int | None = None) -> np.ndarray:
    """dL/dparams [n, 14] in fp64 of L = sum(grad_rgba * image) through torch_forward."""
    import torch
    rec = np.asarray(records, np.float32).reshape(-1, 14)
    prm = torch.tensor(rec.astype(np.float64), requires_grad=True)
    img = torch_forward(prm, world_to_view, view_to_clip, model_to_world, width, height, near, scale_modifier, background, rec, max_pairs)
    (img * torch.tensor(np.asarray(grad_rgba, np.float64).reshape(height, width, 4))).sum().backward()
    g = prm.grad.numpy().copy()
    g[~np.isfinite(rec[:, 13]), 13] = 0.0
    g[np.isnan(rec[:, 13])] = 0.0
    return g
