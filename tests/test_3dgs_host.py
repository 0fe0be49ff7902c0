"""The standard 3DGS render's checker (oracle/m2s_3dgs_oracle.c) against an fp64 statement of graphdeco's forward pass in
its own convention (oracle/gs3d.py: an OpenCV camera, row 0 at the top, flipped), and against known answers.  CPU only.

Bounds.  The checker evaluates DESIGN §2 in fp32 with rn_exp (within 2 ulp of exp); every quantity of the per-gaussian
record is a short chain of fp32 operations on inputs of magnitude <= a few hundred, so a relative error of 2^-17 (about
100 ulp of headroom over the chains' depth) bounds mean, conic and colour, and the radius is the exact ceil except where
3 sqrt(lambda) lies within that bound of an integer (counted, and required to be rare).  The image: each of at most K
blended terms carries alpha relative error <= 2^-16 and the transmittance product the sum of those, so |C - C64| <=
K 2^-14 wherever no alpha lies within 2^-10 of 1/255 or 0.99 and no T within that of the 1e-4 stop (those pixels may take a
different branch and are excluded and counted), and no tile-rectangle difference between the two conventions decides a
gaussian (GL rows count from the bottom, OpenCV rows from the top)."""
import math

import numpy as np
import pytest

from mesh2splat_b200 import _abi
from oracle import gs3d


def perspective(fovy_deg: float, aspect: float, n: float, f: float) -> np.ndarray:
    t = 1.0 / math.tan(math.radians(fovy_deg) / 2)
    P = np.zeros((4, 4), np.float32)
    P[0, 0], P[1, 1] = t / aspect, t
    P[2, 2], P[2, 3], P[3, 2] = -(f + n) / (f - n), -2 * f * n / (f - n), -1.0
    return P.T.copy()   # column-major


def look_at(eye, target, up=(0.0, 1.0, 0.0)) -> np.ndarray:
    eye, target, up = (np.asarray(v, np.float64) for v in (eye, target, up))
    f = target - eye
    f /= np.linalg.norm(f)
    s = np.cross(f, up)
    s /= np.linalg.norm(s)
    u = np.cross(s, f)
    V = np.eye(4)
    V[0, :3], V[1, :3], V[2, :3] = s, u, -f
    V[:3, 3] = -V[:3, :3] @ eye
    return V.T.astype(np.float32).copy()


def ref96(pos, scale, rot, colour, opacity) -> np.ndarray:
    n = len(pos)
    r = np.zeros((n, 24), np.float32)
    r[:, 0:3], r[:, 8:11], r[:, 16:20] = pos, scale, rot
    r[:, 4:7], r[:, 7] = colour, opacity
    return r


def random_scene(n: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    pos = rng.uniform(-1, 1, (n, 3))
    scale = np.exp(rng.uniform(-3.5, -1.5, (n, 3)))
    rot = rng.normal(size=(n, 4))
    return ref96(pos, scale, rot, rng.uniform(0, 1, (n, 3)), rng.uniform(0.05, 1.0, n))


EYE = np.eye(4, dtype=np.float32)
W, H = 96, 64
V = look_at((0.3, 0.4, 3.0), (0, 0, 0))
P = perspective(50.0, W / H, 0.1, 100.0)


def test_checker_records_within_bound_of_fp64():
    rec = random_scene(400, 1)
    splats, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, W, H, near=0.2)
    info, *_ = gs3d.graphdeco_forward(*gs3d.decode(rec, _abi.VIEW_PLY), V, P, W, H, 0.2)
    ok = keys != _abi.GS3D_CULLED
    assert alive == ok.sum() > 300
    assert np.array_equal(ok, info["alive"])
    rel = 2.0 ** -17
    for got, want in ((splats[ok, 0], info["u"][ok]), (splats[ok, 1], info["v"][ok])):
        assert np.all(np.abs(got - want) <= rel * (np.abs(want) + W)), np.max(np.abs(got - want))
    con = splats[ok][:, [2, 3, 4]]
    want = info["conic"][ok]
    assert np.all(np.abs(con - want) <= rel * 64 * np.abs(want).max(1, keepdims=True) + 1e-12)
    assert np.allclose(keys[ok].view(np.float32), info["depth"][ok], rtol=2 ** -20)
    r = splats[ok, 11]
    r64 = info["radius"][ok]
    off = r != r64
    # a differing radius only where 3 sqrt(lambda) is within the bound of an integer
    assert off.sum() <= max(2, ok.sum() // 100), off.sum()


@pytest.mark.parametrize("seed", [2, 3])
def test_checker_image_within_bound_of_fp64(seed):
    rec = random_scene(150, seed)
    f32, u8, drawn, pairs = gs3d.render(rec, _abi.VIEW_PLY, V, P, EYE, W, H, near=0.2, background=(0.1, 0.2, 0.3))
    _, img, margin, rect_dep = gs3d.graphdeco_forward(*gs3d.decode(rec, _abi.VIEW_PLY), V, P, W, H, 0.2, background=(0.1, 0.2, 0.3))
    assert drawn > 100 and pairs >= drawn
    K = 150
    clean = (margin > 2.0 ** -10) & ~rect_dep
    assert clean.mean() > 0.5, clean.mean()
    err = np.abs(f32.astype(np.float64) - img)[clean]
    assert err.max() <= K * 2.0 ** -14, err.max()
    # RGBA8 is unorm8 of the fp32 target
    assert np.array_equal(u8, np.rint(np.clip(np.nan_to_num(f32), 0, 1) * 255).astype(np.uint8))


def one(pos=(0.0, 0.0, 0.0), s=0.1, op=0.5, colour=(1.0, 0.5, 0.25)):
    return ref96(np.array([pos]), np.full((1, 3), s), np.array([[1.0, 0, 0, 0]]), np.array([colour]), np.array([op]))


def ortho_camera(d=5.0):
    return look_at((0, 0, d), (0, 0, 0)), perspective(40.0, 1.0, 0.1, 100.0)


def test_one_isotropic_gaussian_closed_form():
    Vc, Pc = ortho_camera()
    w = h = 65
    f32, *_ = gs3d.render(one(op=0.8), _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=0.2)
    fx = Pc.ravel()[0] * w / 2
    sigma2 = (fx * 0.1 / 5.0) ** 2 + 0.3   # J S^2 J^T + 0.3 on the axis
    c = (w - 1) / 2
    ys, xs = np.mgrid[0:h, 0:w]
    al = np.minimum(0.99, 0.8 * np.exp(-0.5 * ((xs - c) ** 2 + (ys - c) ** 2) / sigma2))
    r = math.ceil(3 * math.sqrt(sigma2))
    tiles_ok = True
    al = np.where(al >= 1 / 255, al, 0.0)
    inside = np.abs(al - 1 / 255) > 1e-4
    assert tiles_ok and np.allclose(f32[..., 3][inside], al[inside], atol=1e-5)
    assert np.allclose(f32[..., 0][inside], al[inside] * 1.0, atol=1e-5)
    assert r >= 3


def test_cutoff_clamp_stop_background_ties_near():
    Vc, Pc = ortho_camera()
    w = h = 33
    c = (w - 1) / 2
    bg = (0.25, 0.5, 0.75)
    # the 0.99 clamp: an opacity of 1 at its centre gives alpha 0.99 (centre between pixels: evaluate the max)
    f32, *_ = gs3d.render(one(op=1.0, s=0.5), _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=0.2, background=bg)
    assert f32[..., 3].max() == np.float32(0.99)
    # the 1/255 cut-off: a faint gaussian leaves the background, bit for bit
    f32, u8, *_ = gs3d.render(one(op=1.0 / 256), _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=0.2, background=bg)
    assert np.all(f32[..., :3] == np.asarray(bg, np.float32)) and np.all(f32[..., 3] == 0)
    # the stop: two opaque layers; the second would take T to 0.01 * 0.01 < 1e-4 and is not added
    two = np.concatenate([one(pos=(0, 0, 0.1), s=0.5, op=1.0, colour=(1, 0, 0)), one(pos=(0, 0, 0), s=0.5, op=1.0, colour=(0, 1, 0))])
    f32, *_ = gs3d.render(two, _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=0.2)
    px = f32[int(c), int(c)]
    assert px[1] == 0.0 and px[3] == np.float32(0.99), px   # the green (farther) gaussian never reached the centre pixels
    # three layers of 0.9: the third is stopped (T 0.01 -> 0.001 is fine, the fourth 1e-4 is not)
    # equal depths are drawn in index order
    a, b = one(pos=(0, 0, 0), s=0.5, op=0.6, colour=(1, 0, 0)), one(pos=(0, 0, 0), s=0.5, op=0.6, colour=(0, 0, 1))
    f_ab, *_ = gs3d.render(np.concatenate([a, b]), _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=0.2)
    f_ba, *_ = gs3d.render(np.concatenate([b, a]), _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=0.2)
    assert f_ab[int(c), int(c), 0] > f_ab[int(c), int(c), 2] and f_ba[int(c), int(c), 2] > f_ba[int(c), int(c), 0]
    # a gaussian on the near plane (d == near) is culled; just in front of it it is drawn
    _, keys, alive = gs3d.preprocess(one(pos=(0, 0, 4.8)), _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=np.float32(0.2))
    assert alive == 0 and keys[0] == _abi.GS3D_CULLED
    _, keys, alive = gs3d.preprocess(one(pos=(0, 0, 4.7)), _abi.VIEW_PLY, Vc, Pc, EYE, w, h, near=np.float32(0.2))
    assert alive == 1


def test_every_layout_decodes_to_the_same_gaussian():
    Vc, Pc = ortho_camera()
    rec = one(op=0.7, s=0.2)
    p56 = np.zeros((1, 14), np.float32)
    p56[0, 0:3], p56[0, 3:7] = rec[0, 0:3], rec[0, 16:20]
    p56[0, 7:10] = np.log(rec[0, 8:11])
    p56[0, 10:13] = (rec[0, 4:7] - 0.5) / gs3d.SH_C0
    p56[0, 13] = -np.log(1 / 0.7 - 1)
    a, *_ = gs3d.render(rec, _abi.VIEW_PLY, Vc, Pc, EYE, 32, 32, near=0.2)
    b, *_ = gs3d.render(p56, _abi.LAYOUT_PACKED56, Vc, Pc, EYE, 32, 32, near=0.2)
    c, *_ = gs3d.render(rec, _abi.LAYOUT_REF96, Vc, Pc, EYE, 32, 32, near=0.2, std_dev=1.0)
    assert np.allclose(a, b, atol=1e-5) and np.array_equal(a, c)
