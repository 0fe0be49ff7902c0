"""The standard 3DGS render's checker (oracle/m2s_3dgs_oracle.c) against graphdeco's forward pass in fp64
(oracle/gs3d.py) where fp32 goes wrong: ill-conditioned covariances, the frustum clamp, means close to the camera,
large viewports, radii past the int32 range, per-pixel image bounds and the SH colour.  CPU only; the inputs are the
module's generators, which tests/test_gpu_3dgs_edges.py also runs on the GPU.

Notation: u = 2^-24 (fp32 unit roundoff).  Every bound below is per record or per pixel; each test also asserts that
the bound is not more than 100 x the largest error observed (it is tight enough to notice a subtle fault).

Records.  The checker rounds once per operation along the chain of DESIGN §2.
- The 2-D covariance (a, b, c) is sums of products of T = J W and Sigma = sum_k s_k^2 r_k r_k^T.  Each entry's
  absolute error is a few tens of u times the size of its terms, mag = |T|_F^2 (s_x^2 + s_y^2 + s_z^2) + 0.3
  (gs3d's info["mag"]), not times the entry itself: an end-on needle's cov is tiny next to the needle's length.
  So |d cov| <= 32 u mag.
- The conic is cov^-1: |d conic| <= |conic|^2 |d cov| = |d cov| / lambda_min^2, which relative to max|conic| =
  1/lambda_min is kappa = mag / lambda_min times 32 u.  For a well-scaled gaussian kappa is the condition number of
  cov, which is the (|a c| + b^2) / det amplification of det = a c - b^2 when it cancels (needles, flat discs).
  Bound: |d conic_j| <= 64 u kappa max|conic| (the inversion's own roundings double it).
- The mean: t = MV p is a 4-term dot product whose terms may cancel (|d t_r| <= 4 u |t_r|', |t_r|' = sum_j
  |MV_rj p_j| + |MV_r3|), ndc = clip_x / (clip_w + 1e-7) and u = ((ndc + 1) W - 1) / 2 add a few roundings of |u| + W,
  and fx = P00 W / 2 carries t's error to pixels: |d u| <= 16 u (|u| + W + (fx |t_x|' + |u - (W - 1) / 2| |t_z|') / d),
  likewise v with H, fy.  (fx can dwarf W: a 1 x 4096 viewport has P00 = 4096 cot(fov / 2).)
- The radius r = ceil(3 sqrt(lambda)), lambda = mid + sqrt(max(0.1, mid^2 - det)).  The argument of the square root
  cancels for round gaussians, so its error x_err = 2 mid d_mid + d_det + 2 u (mid^2 + |det|) reaches lambda as
  min(sqrt(x_err), x_err / (2 sq)) (sqrt is 1/2-Hoelder, max(0.1, .) 1-Lipschitz); d(3 sqrt(lambda)) = 1.5 d_lambda /
  sqrt(lambda).  The two radii are equal except where 3 sqrt(lambda) lies within that window of an integer, and differ
  by at most 1 there; those records are counted.
- Past ~1e19 px^2 (radii past ~1e10 px) a c, b^2 or mid^2 overflows fp32, as in graphdeco's own fp32 code: det is
  inf or NaN, the conic 0 or NaN, the radius 3 sqrt(mid).  There the radius is held to that, the conic not at all;
  the rectangle (the whole grid on a saturated axis) is compared as below.
- The tile rectangle is trunc_sat((u - r) / 16) etc., clamped to the grid: the checker's equals the same formula in
  fp64 (GL rows, from the fp64 u, v, r), except where an argument lies within its error of an integer (counted).  A
  record is culled in both or neither, except at those rectangle ties and where d lies within 8 u |t| of near.

Image.  A pixel's output is C + T bg with C = sum_i c_i alpha_i T_i.  Its derivative in alpha_i is T_i (c_i - rest),
rest a convex mix of the later colours and the background, so a change d alpha_i moves any channel by at most T_i
d alpha_i max(colour, background), and 1 - T by at most T_i d alpha_i.  Each alpha = min(0.99, o exp(power)) carries
relative error d power + 4 u (rn_exp within 2 ulp, the product, the clamp exact), and d power <= 64 u kappa |power| +
|grad power| |d mean| (the quadratic form's relative error is bounded by cov's condition, as for the conic; the mean
enters through the gradient).  gs3d accumulates sum_i T_i alpha_i (that |power| term + that gradient term) per pixel
(info["dalpha"]).  The fp32 blend adds 4 u per composited term (1 - alpha, the products, the sum).  So, per pixel with
k composited terms and 1 - T covered,
    |C32 - C64| <= cmax (dalpha + 4 u (1 - T)) + 4 u k + 2 u,   cmax = max(1, colours, background),
wherever no alpha lies within 2^-16 of 1/255 or 0.99 and no T within it (relative) of the 1e-4 stop (there the two
may take different branches: excluded, counted, required to be under 2 % of the pixels), and no tile-rectangle
difference between the conventions decides a gaussian.

SH.  The record colour of gs3d.preprocess with an SH buffer against graphdeco's computeColorFromSH in fp64
(oracle/sh.py): the bound of tests/test_ply_sh_host.py, 32 u (|c| + sum |B_k coeff_k|) plus the direction's error
term; the clamp at 0 is exact on both sides."""
import math

import numpy as np
import pytest

from mesh2splat_b200 import _abi
from oracle import gs3d
from oracle import sh as osh
from test_3dgs_host import look_at, perspective, ref96

U = 2.0 ** -24
EYE = np.eye(4, dtype=np.float32)
CAMERAS = {"front": ((0.3, 0.4, 3.0), (0.0, 0.0, 0.0)), "oblique": ((-2.2, 1.7, 1.4), (0.1, -0.2, 0.0)),
           "below": ((0.5, -2.5, -1.5), (0.0, 0.1, 0.2))}


def camera(w, h, name="front", fov=50.0):
    eye, tgt = CAMERAS[name]
    return look_at(eye, tgt), perspective(fov, w / h, 0.1, 100.0)


def random_quats(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


# ---- input classes (shared with the GPU file) ------------------------------------------------------------------------
def shaped_scene(kind: str, n: int, seed: int) -> np.ndarray:
    """Gaussians around the origin at many orientations: isotropic, needle (one axis 10^3 x the others) or flat (two
    axes 10^3 x the third)."""
    rng = np.random.default_rng(seed)
    pos = rng.uniform(-0.8, 0.8, (n, 3))
    base = np.exp(rng.uniform(-7.0, -4.0, n))[:, None]
    axes = {"iso": (1.0, 1.0, 1.0), "needle": (1e3, 1.0, 1.0), "flat": (1e3, 1e3, 1.0)}[kind]
    scale = base * np.asarray(axes)
    if kind == "iso":
        scale = scale * 100.0
    return ref96(pos, scale, random_quats(rng, n), rng.uniform(0, 1, (n, 3)), rng.uniform(0.05, 1.0, n))


def clamp_scene(w: int, h: int, P, seed: int) -> np.ndarray:
    """Means outside the 1.3 tan(fov) limit on each side whose 3-sigma rectangle still reaches the image, and means
    exactly on the limit (x / d == limx in fp32), for the camera at (0, 0, 4) looking down -z."""
    rng = np.random.default_rng(seed)
    limx, limy = np.float32(1.3) / P.ravel()[0], np.float32(1.3) / P.ravel()[5]
    recs = []
    for d in (np.float32(2.0), np.float32(4.0), np.float32(8.0)):   # powers of two: x = lim d is exact, x / d == lim
        z = np.float32(4.0) - d
        for sx, sy in ((1, 0), (-1, 0), (0, 1), (0, -1), (1, 1), (-1, -1)):
            for f in (1.0, 1.05, 1.3, 2.0):   # on the limit, then past it
                x, y = np.float32(sx * f) * limx * d, np.float32(sy * f) * limy * d
                if sx == 0:
                    x = np.float32(rng.uniform(-0.3, 0.3)) * d
                if sy == 0:
                    y = np.float32(rng.uniform(-0.3, 0.3)) * d
                s = float(d) * (0.15 + 0.3 * (f - 1.0))
                recs.append(ref96(np.array([[x, y, z]]), np.array([[s, s * rng.uniform(0.2, 1), s * 0.5]]), random_quats(rng, 1),
                                  rng.uniform(0, 1, (1, 3)), np.array([rng.uniform(0.3, 1.0)])))
    return np.concatenate(recs)


CLAMP_V = look_at((0.0, 0.0, 4.0), (0.0, 0.0, 0.0))


def near_scene(near: float, seed: int, n: int = 300) -> np.ndarray:
    """Depths from just above near to 10^3 near in front of a camera at (0, 0, 4) looking down -z, scales a fixed share
    of the depth or (every other record) fixed, so J = fx / d grows the radii to thousands of pixels, lateral offsets
    inside the view."""
    rng = np.random.default_rng(seed)
    f = np.concatenate([[1.0 + 2.0 ** -8, 1.0 + 2.0 ** -4, 1.5], np.exp(rng.uniform(0, math.log(1e3), n - 3))])
    d = near * f
    lat = rng.uniform(-0.5, 0.5, (n, 2)) * d[:, None]
    pos = np.c_[lat, 4.0 - d]
    scale = np.where(np.arange(n)[:, None] % 2 == 0, d[:, None], 1.0) * np.exp(rng.uniform(-6, -2, (n, 3)))
    return ref96(pos, scale, random_quats(rng, n), rng.uniform(0, 1, (n, 3)), rng.uniform(0.05, 1.0, n))


def huge_scene(seed: int) -> np.ndarray:
    """Gaussians whose u +- radius leaves the int32 range (radius up to ~10^12 pixels), on and off screen, and a few
    ordinary ones, for the camera at (0, 0, 4)."""
    rng = np.random.default_rng(seed)
    n = 40
    d = np.exp(rng.uniform(math.log(0.02), math.log(2.0), n))
    lat = rng.uniform(-3.0, 3.0, (n, 2)) * d[:, None]
    s = np.exp(rng.uniform(math.log(10.0), math.log(1e6), (n, 1))) * np.array([[1.0, 0.7, 0.4]])
    s[-8:] = 0.02
    pos = np.c_[lat, 4.0 - d]
    return ref96(pos, s, random_quats(rng, n), rng.uniform(0, 1, (n, 3)), rng.uniform(0.05, 1.0, n))


def image_scene(n: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    pos = rng.uniform(-1, 1, (n, 3))
    scale = np.exp(rng.uniform(-4.0, -1.5, (n, 3)))
    return ref96(pos, scale, random_quats(rng, n), rng.uniform(0, 1, (n, 3)), rng.uniform(0.05, 1.0, n))


# ---- the per-record comparison -----------------------------------------------------------------------------------------
def _gl_rect(u, v, r, w, h):
    """getRect in fp64 in the checker's GL rows: (x0, y0, x1, y1) and each edge's argument (for the tie test)."""
    gx, gy = (w + 15) // 16, (h + 15) // 16
    args = np.stack([(u - r) / 16, (v - r) / 16, (u + r + 15) / 16, (v + r + 15) / 16], -1)
    lim = np.array([gx, gy, gx, gy])
    with np.errstate(invalid="ignore"):
        t = np.trunc(np.clip(args, -2.0 ** 40, 2.0 ** 40))
    return np.clip(t, 0, lim).astype(np.int64), args


def record_errors(rec, V, P, w, h, near, M=EYE):
    """The checker's records against fp64 under the module's per-record bounds.  Returns a dict of the ratios error /
    bound (each <= 1 asserted here) and the counts of records at ties, for the callers' margin and share checks."""
    splats, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, M, w, h, near=near)
    info, *_ = gs3d.graphdeco_forward(*gs3d.decode(rec, _abi.VIEW_PLY), V, P, w, h, near, model_to_world=M, render=False)
    ok32 = keys != _abi.GS3D_CULLED
    assert alive == ok32.sum()
    a, b, c = info["cov"].T
    det = a * c - b * b
    mid = 0.5 * (a + c)
    sq = np.sqrt(np.maximum(0.1, mid * mid - det))
    lam = mid + sq
    lmin = np.maximum(det / np.where(lam > 0, lam, 1.0), 1e-300)
    mag = info["mag"]
    dcov = 32 * U * mag
    kappa = mag / lmin
    # the radius window
    dmid = dcov + U * mid
    ddet = (a + c + 2 * np.abs(b)) * dcov + 2 * U * (a * c + b * b)
    dx = 2 * mid * dmid + ddet + 2 * U * (mid * mid + np.abs(det))
    dlam = dmid + np.minimum(np.sqrt(dx), dx / (2 * sq)) + U * lam
    r64 = 3 * np.sqrt(lam)
    window = 1.5 * dlam / np.sqrt(lam) + 4 * U * r64
    # fp32 overflow of a c, b^2 or mid^2 (covariances past ~1e19 px^2): det is inf or NaN, the conic 0 or NaN and the
    # radius 3 sqrt(mid) (max(0.1, NaN) = 0.1), as in graphdeco's fp32 code; only the (saturated) rectangle is compared
    ovf = np.maximum(np.maximum(a * c, b * b), mid * mid) >= 0.5 * float(np.finfo(np.float32).max)
    r_ovf = 3 * np.sqrt(np.abs(mid))
    window = np.where(ovf, 4 * U * r_ovf + 1, window)
    r64 = np.where(ovf, r_ovf, r64)
    near_int = np.abs(r64 - np.rint(r64)) <= window
    # the rectangle in fp64 (GL rows) and its ties
    r_want = np.where(ovf, np.ceil(r64), info["radius"])
    rect64, args = _gl_rect(info["u"], info["v"], r_want, w, h)
    MV = (np.asarray(V, np.float64).reshape(4, 4).T @ np.asarray(M, np.float64).reshape(4, 4).T)[:3]
    size = np.abs(rec[:, 0:3]).astype(np.float64) @ np.abs(MV[:, :3]).T + np.abs(MV[:, 3])   # |t_r| before cancellation
    zs = np.where(info["depth"] > 0, info["depth"], 1.0)
    fx, fy = P.ravel()[0] * w / 2.0, P.ravel()[5] * h / 2.0
    du = 16 * U * (np.abs(info["u"]) + w + fx * (size[:, 0] + size[:, 2] * np.abs(info["u"] - (w - 1) / 2) / fx) / zs)
    dv = 16 * U * (np.abs(info["v"]) + h + fy * (size[:, 1] + size[:, 2] * np.abs(info["v"] - (h - 1) / 2) / fy) / zs)
    slack = (np.stack([du, dv, du, dv], -1) + r_want[:, None] * 4 * U) / 16 + 4 * U * np.abs(args)
    tie = (np.abs(args - np.rint(args)) <= slack).any(1) | near_int
    area64 = (rect64[:, 2] - rect64[:, 0]) * (rect64[:, 3] - rect64[:, 1])
    ok64 = (info["depth"] > near) & (det != 0) & (area64 > 0)
    at_near = np.abs(info["depth"] - near) <= 8 * U * (np.abs(info["depth"]) + np.abs(rec[:, 0:3]).sum(1) + 8)
    differ = ok32 != ok64
    assert not (differ & ~(tie | at_near)).any(), np.nonzero(differ & ~(tie | at_near))[0][:10]
    both = ok32 & ok64
    out = {"n": int(both.sum()), "ties": int((tie & both).sum()), "culled_at_ties": int(differ.sum()), "overflow": int((ovf & both).sum())}
    if not both.any():
        return out
    s = splats[both].astype(np.float64)
    # mean
    ru = np.abs(s[:, 0] - info["u"][both]) / du[both]
    rv = np.abs(s[:, 1] - info["v"][both]) / dv[both]
    # conic
    want = info["conic"][both]
    cb = 64 * U * kappa[both] * np.abs(want).max(1)
    rc = np.where(ovf[both], 0.0, np.abs(s[:, 2:5] - want).max(1) / cb)
    # radius and rectangle
    r32 = s[:, 11]
    rw = r_want[both]
    assert np.all(np.abs(r32 - rw) <= 1 + np.ceil(window[both]))
    assert np.all((r32 == rw) | near_int[both]), np.nonzero((r32 != rw) & ~near_int[both])[0][:10]
    rx, ry = splats[both, 9].view(np.uint32), splats[both, 10].view(np.uint32)
    rect32 = np.stack([rx & 0xFFFF, ry & 0xFFFF, rx >> 16, ry >> 16], -1).astype(np.int64)
    same = (rect32 == rect64[both]).all(1)
    assert np.all(same | tie[both]), np.nonzero(~same & ~tie[both])[0][:10]
    # depth key: d = -t_z, a 4-term dot product
    dk = keys[both].view(np.float32).astype(np.float64)
    rd = np.abs(dk - info["depth"][both]) / (8 * U * (np.abs(info["depth"][both]) + np.abs(rec[both, 0:3]).sum(1) + 8))
    for name, r in (("mean u", ru), ("mean v", rv), ("conic", rc), ("depth", rd)):
        assert np.all(r <= 1.0), (name, float(r.max()), int(np.argmax(r)))
    out.update(u=float(max(ru.max(), rv.max())), conic=float(rc.max()), depth=float(rd.max()), rect32=rect32, rect64=rect64[both],
               radius=r32, kappa=kappa[both])
    return out


def _margin(ratio, what):
    """The bound is not more than 100 x the largest observed error."""
    assert ratio >= 1e-2, f"{what}: the largest error is {ratio:.2e} of the bound: the bound is too loose to notice a fault"


# ---- records ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["iso", "needle", "flat"])
def test_records_within_conditioning_bounds(kind):
    w, h = 96, 64
    worst = {"u": 0.0, "conic": 0.0}
    ties = n = 0
    for name in CAMERAS:
        V, P = camera(w, h, name)
        r = record_errors(shaped_scene(kind, 1500, {"iso": 1, "needle": 2, "flat": 3}[kind]), V, P, w, h, 0.2)
        assert r["n"] > 900, r["n"]
        worst = {k: max(worst[k], r[k]) for k in worst}
        ties, n = ties + r["ties"], n + r["n"]
        if kind != "iso":
            assert r["kappa"].max() > 1e3   # the class reaches the ill-conditioned covariances it is for
    _margin(worst["u"], "mean")
    _margin(worst["conic"], "conic")
    # round gaussians: mid^2 - det cancels, so the radius window is widest there (about 8 % of them)
    assert ties <= 0.1 * n, (ties, n)


def test_frustum_clamp():
    w, h = 96, 64
    P = perspective(50.0, w / h, 0.1, 100.0)
    rec = clamp_scene(w, h, P, 4)
    r = record_errors(rec, CLAMP_V, P, w, h, 0.2)
    assert r["n"] >= 0.8 * len(rec), (r["n"], len(rec))
    rect = r["rect32"]   # most reach an edge of the grid: their means lie off screen
    assert ((rect[:, 0] == 0) | (rect[:, 2] == (w + 15) // 16) | (rect[:, 1] == 0) | (rect[:, 3] == (h + 15) // 16)).mean() > 0.5
    _margin(r["u"], "mean")
    _margin(r["conic"], "conic")


@pytest.mark.parametrize("near", [1e-3, 0.01, 0.2])
def test_close_to_the_camera(near):
    w, h = 96, 64
    P = perspective(60.0, w / h, 0.001, 100.0)
    near32 = float(np.float32(near))
    r = record_errors(near_scene(near32, int(near * 1e4)), CLAMP_V, P, w, h, near32)
    assert r["n"] > 250, r["n"]
    if near < 0.1:
        assert r["radius"].max() > 1e3   # J is large: the radii reach far past the image
    _margin(r["u"], "mean")
    _margin(r["conic"], "conic")


@pytest.mark.parametrize("wh", [(1920, 1080), (4096, 4096), (4096, 1), (1, 4096)])
def test_large_viewports(wh):
    w, h = wh
    V, P = camera(w, h)
    r = record_errors(image_scene(3000, 5), V, P, w, h, 0.2)
    assert r["n"] > 1000
    assert max(r["rect32"][:, 2].max(), r["rect32"][:, 3].max()) * 16 >= 0.4 * max(w, h)   # u or v reach thousands
    _margin(r["u"], "mean")
    _margin(r["conic"], "conic")


def test_huge_radii_saturate():
    w, h = 1920, 1080
    P = perspective(60.0, w / h, 0.01, 100.0)
    rec = huge_scene(6)
    r = record_errors(rec, CLAMP_V, P, w, h, 0.01)
    big = r["radius"] >= 2.0 ** 31
    assert big.sum() >= 5 and r["overflow"] >= 1, (big.sum(), r["overflow"])
    gx, gy = (w + 15) // 16, (h + 15) // 16
    # u +- r past the int32 range: trunc_sat saturates, the clamp then gives the whole grid on that axis
    full = big & (np.abs(r["rect64"][:, :2]).sum(1) == 0)
    assert np.all(r["rect32"][full] == [0, 0, gx, gy])
    assert np.array_equal(r["rect32"], r["rect64"])


# ---- the image: per-pixel bound from the pixel's own terms ------------------------------------------------------------
@pytest.mark.parametrize("wh", [(96, 64), (640, 360)])
@pytest.mark.parametrize("cam", list(CAMERAS))
@pytest.mark.parametrize("seed", [2, 3])
def test_image_within_per_pixel_bound(seed, cam, wh):
    w, h = wh
    V, P = camera(w, h, cam)
    bg = (0.1, 0.2, 0.3)
    rec = image_scene(150, seed)
    f32, u8, drawn, pairs = gs3d.render(rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2, background=bg)
    dec = gs3d.decode(rec, _abi.VIEW_PLY)
    pre, *_ = gs3d.graphdeco_forward(*dec, V, P, w, h, 0.2, render=False)
    a, b, c = pre["cov"].T
    lam = 0.5 * (a + c) + np.sqrt(np.maximum(0.25 * (a - c) ** 2 + b * b, 0))
    kappa = pre["mag"] / ((a * c - b * b) / lam)
    mean_err = 16 * U * (np.abs(pre["u"]) + np.abs(pre["v"]) + w + h)
    info, img, margin, rect_dep = gs3d.graphdeco_forward(*dec, V, P, w, h, 0.2, background=bg, power_err=64 * U * kappa, mean_err=mean_err)
    assert drawn > 80 and pairs >= drawn
    k = info["blended"]
    cover = img[..., 3]
    cmax = max(1.0, float(rec[:, 4:7].max()), max(bg))
    bound = cmax * (info["dalpha"] + 4 * U * cover) + 4 * U * k + 2 * U
    clean = (margin > 2.0 ** -16) & ~rect_dep
    excluded = 1.0 - clean.mean()
    assert excluded < 0.02, excluded
    err = np.abs(f32.astype(np.float64) - img)
    ratio = (err / bound[..., None])[clean]
    assert ratio.max() <= 1.0, (ratio.max(), np.argwhere(err / bound[..., None] * clean[..., None] > 1)[:5])
    _margin(float(ratio.max()), "image")
    assert (k[clean] >= 3).mean() > 0.1   # many pixels composite several terms
    assert np.array_equal(u8, np.rint(np.clip(np.nan_to_num(f32), 0, 1) * 255).astype(np.uint8))


# ---- SH through the record colour ------------------------------------------------------------------------------------
OCTANT_EYE = (0.0, 0.0, 0.0)


def sh_scene(n: int, seed: int, degree: int):
    """Gaussians in all eight octants around a camera at the origin, with a degree-`degree` SH buffer; a quarter of
    them with a colour that the rest term drives below 0 (the clamp)."""
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    sign = np.array([[(o >> 2) & 1, (o >> 1) & 1, o & 1] for o in range(8)]) * 2 - 1
    d = np.abs(d) * sign[np.arange(n) % 8]
    pos = d * rng.uniform(1.0, 3.0, (n, 1))
    col = rng.normal(size=(n, 3)) * 0.28209479177387814 + 0.5
    col[::4] = -0.2
    rec = ref96(pos, np.full((n, 3), 0.01), random_quats(rng, n), col, np.full(n, 0.5))
    sh = (rng.normal(size=(n, _abi.SH_FLOATS[degree])) * 0.4).astype(np.float32)
    return rec, sh


def octant_cameras():
    """Eight views from the origin, each looking into one octant (all directions of dir = pos - cam are seen)."""
    out = []
    for o in range(8):
        tgt = np.array([(o >> 2) & 1, (o >> 1) & 1, o & 1], np.float64) * 2 - 1
        up = (0.0, 1.0, 0.0) if abs(tgt[1]) < 0.99 * np.linalg.norm(tgt) else (1.0, 0.0, 0.0)
        out.append(look_at(OCTANT_EYE, tuple(tgt), up))
    return out


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_sh_colour_through_the_record(degree):
    w, h = 64, 64
    P = perspective(120.0, 1.0, 0.05, 100.0)
    rec, sh = sh_scene(4000, 20 + degree, degree)
    K = (degree + 1) ** 2 - 1
    worst, clamped, seen = 0.0, 0, np.zeros(8, bool)
    for V in octant_cameras():
        splats, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.05, sh=sh, buffer_degree=degree,
                                              sh_degree=degree)
        ok = keys != _abi.GS3D_CULLED
        assert alive > 300
        cam = osh.camera(V, EYE).astype(np.float64)
        d = rec[ok, 0:3].astype(np.float64) - cam
        coeffs = sh[ok, : 3 * K].reshape(-1, K, 3)
        want = osh.reference_rgb(d, coeffs, rec[ok, 4:7])
        got = splats[ok, 6:9].astype(np.float64)
        mag = np.abs(rec[ok, 4:7]).astype(np.float64) + 1.1 * np.abs(coeffs).astype(np.float64).sum(axis=1)
        dist = np.linalg.norm(d, axis=1, keepdims=True)
        bound = 32 * U * mag + 8 * U * (np.abs(cam).max() + np.abs(rec[ok, 0:3]).max(axis=1, keepdims=True)) / dist * mag
        err = np.abs(got - want)
        assert np.all(err <= bound), float((err / bound).max())
        worst = max(worst, float((err / bound).max()))
        assert np.all(got >= 0)
        neg = want == 0
        assert np.all(got[neg] <= bound[neg])
        clamped += int((got == 0).sum())
        seen[(np.sign(d) > 0) @ np.array([4, 2, 1])] = True
    assert seen.all() and clamped > 100
    _margin(worst, "SH colour")
