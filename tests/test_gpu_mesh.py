"""The viewer's mesh G-buffer pass and the split-screen lighting on the GPU (SURVEY 8 row 14: m2s_mesh_render,
m2s_deferred_light_split).  All five targets are compared bit for bit with the C restatement (oracle/m2s_mesh_oracle.c)
through guarded buffers, so a pixel written outside a target or never written fails; the split image is compared with
m2s_deferred_light of each G-buffer and with the oracle's composite."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_REF96
from mesh2splat_b200._lib import M2SError, check, lib
from oracle import light, mesh
from util import GuardedDevice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

NAMES = [t for t, _ in _abi.GBUFFER_TARGETS]
EYE = np.eye(4, dtype=np.float32)
MIRROR = column_major(np.diag([-1.0, 1.0, 1.0, 1.0]).astype(np.float32))
NEAR_FAR = (0.01, 100.0)


def _camera(eye, target, aspect, near=0.01, far=100.0, fov=45.0):
    V = column_major(look_at(np.array(eye, np.float64), np.array(target, np.float64), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(fov), aspect, near, far))
    return V, P


OUTSIDE = ((0.0, 0.5, 3.2), (0.0, 0.0, 0.0))     # the whole helmet stand-in in view
INSIDE = ((0.05, 0.02, -0.03), (1.0, 0.3, 0.2))  # inside the displaced sphere (mirrored: its inner side faces the camera)


def _targets(w, h, names=NAMES):
    import torch
    return {t: GuardedDevice(w * h, 8 if dt == np.float16 else 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, what=t)
            for t, dt in _abi.GBUFFER_TARGETS if t in names}


def _render(gpu_ctx, ds, V, P, M, w, h, mode=0, max_pairs=None, names=NAMES):
    """The pass through guarded targets: (images, drawn, pairs, {name: device tensor})."""
    g = _targets(w, h, names)
    imgs, drawn, pairs = gpu_ctx.mesh_render(ds, V, P, M, w, h, NEAR_FAR, mode, targets=tuple(names), max_pairs=max_pairs,
                                             gbuffer={t: g[t].view for t in g})
    for t in g:
        g[t].check(w * h)
    return imgs, drawn, pairs, {t: g[t].view for t in g}


def _check(gpu_ctx, scene, ds, V, P, M, w, h, mode=0, arena=None, **kw):
    imgs, drawn, pairs, dev = _render(gpu_ctx, ds, V, P, M, w, h, mode, **kw)
    want = mesh.mesh_render(scene, V, P, M, w, h, NEAR_FAR, mode, n=drawn, arena=arena)
    for t in imgs:
        a, b = imgs[t].view(np.uint8), want[t].view(np.uint8)
        assert np.array_equal(a, b), f"{t}: {int((a != b).reshape(h, w, -1).any(axis=-1).sum())} pixels differ"
    return imgs, drawn, pairs, dev


@pytest.fixture(scope="module")
def helmet(gpu_ctx):
    scene = synth.helmet_standin(64)
    ds = gpu_ctx.upload(scene)
    yield scene, ds, mesh.mip_arena(scene.textures)
    ds.free()


@pytest.mark.parametrize("cam", ["outside", "inside"])
@pytest.mark.parametrize("wh", [(1, 1), (17, 15), (1920, 1080)])
def test_helmet_outside_and_inside(gpu_ctx, helmet, cam, wh):
    scene, ds, arena = helmet
    eye, tgt = OUTSIDE if cam == "outside" else INSIDE
    V, P = _camera(eye, tgt, wh[0] / wh[1])
    imgs, drawn, pairs, _ = _check(gpu_ctx, scene, ds, V, P, EYE if cam == "outside" else MIRROR, *wh, arena=arena)
    assert drawn == scene.triangle_count
    cov = imgs["albedo"][..., 3] == 255
    if cam == "inside":
        assert cov.all()   # surrounded by the mesh
    elif wh[0] > 1:
        assert cov.any() and not cov.all() and pairs > 0


@pytest.mark.parametrize("mode", range(7))
def test_every_render_mode(gpu_ctx, helmet, mode):
    scene, ds, arena = helmet
    V, P = _camera(*OUTSIDE, 160 / 120)
    imgs, _, _, _ = _check(gpu_ctx, scene, ds, V, P, EYE, 160, 120, mode, arena=arena)
    if mode == 3:
        assert len(np.unique(imgs["albedo"].reshape(-1, 4), axis=0)) > 100


def test_rotated_and_mirrored_model_matrices(gpu_ctx, helmet):
    scene, ds, arena = helmet
    V, P = _camera(*OUTSIDE, 1.0)
    c, s = np.cos(0.7), np.sin(0.7)
    R = column_major(np.array([[1.3 * c, 0, 1.3 * s, 0.1], [0, 0.8, 0, -0.2], [-1.3 * s, 0, 1.3 * c, 0.05], [0, 0, 0, 1]], np.float32))
    for M in (R, MIRROR):
        imgs, _, _, _ = _check(gpu_ctx, scene, ds, V, P, M, 128, 128, 2, arena=arena)
        assert (imgs["albedo"][..., 3] == 255).any()
    with pytest.raises(M2SError):
        _render(gpu_ctx, ds, V, P, column_major(np.diag([1.0, 0.0, 1.0, 1.0]).astype(np.float32)), 8, 8)


def test_sponza_standin_repeat_and_25_materials(gpu_ctx):
    scene = synth.sponza_standin(32, target_tris=40_000)
    ds = gpu_ctx.upload(scene)
    try:
        V, P = _camera((2.0, 3.0, 6.0), (20.0, 4.0, 6.0), 320 / 180, near=0.05, far=60.0, fov=70.0)
        for mode in (0, 2, 6):
            imgs, _, _, _ = _check(gpu_ctx, scene, ds, V, P, EYE, 320, 180, mode)
            assert (imgs["albedo"][..., 3] == 255).mean() > 0.05
    finally:
        ds.free()


def _quad(z, s, x0=0.0, y0=0.0):
    return [[(x0 - s, y0 - s, z), (x0 + s, y0 - s, z), (x0 + s, y0 + s, z)], [(x0 - s, y0 - s, z), (x0 + s, y0 + s, z), (x0 - s, y0 + s, z)]]


def _soup(pos, uv_scale):
    pos = np.asarray(pos, np.float32)
    t = np.zeros((len(pos), 36), np.float32)
    for k in range(3):
        t[:, 12 * k: 12 * k + 3] = pos[:, k]
        t[:, 12 * k + 3: 12 * k + 6] = (0.1, 0.2, 1.0)
        t[:, 12 * k + 6: 12 * k + 10] = (1.0, 0.1, 0.0, -1.0)
        t[:, 12 * k + 10: 12 * k + 12] = pos[:, k, :2] * uv_scale
    return t


def test_maps_npot_magnification_minification_no_maps_and_alpha(gpu_ctx):
    """Four primitives in front of the camera: an NPOT map set magnified (uv steps far below a texel), the same maps
    minified past level 4 (uv tiled thousands of times, REPEAT), a primitive with no maps, and one whose base colour
    alpha is below 1 (still drawn, unlike the depth pre-pass)."""
    texs = [synth.random_texture(37, 23, 1), synth.random_texture(37, 23, 2), synth.random_texture(37, 23, 3)]
    tris = np.concatenate([_soup(_quad(-3.0, 0.5, -0.6, 0.3), 0.05), _soup(_quad(-3.0, 0.5, 0.6, 0.3), 3000.0),
                           _soup(_quad(-3.0, 0.5, -0.6, -0.7), 1.0), _soup(_quad(-2.5, 0.5, 0.6, -0.7), 2.0)])
    prims = [_abi.Primitive(0, 2, (1.0, 1.0, 1.0, 1.0), 0, 1, 2), _abi.Primitive(2, 2, (0.9, 0.8, 0.7, 1.0), 0, 1, 2),
             _abi.Primitive(4, 2, (0.5, 0.25, 0.75, 1.0), -1, -1, -1), _abi.Primitive(6, 2, (0.3, 0.6, 0.9, 0.25), 2, -1, 0)]
    scene = _abi.Scene(tris, prims, texs)
    scene.compute_bboxes()
    ds = gpu_ctx.upload(scene)
    try:
        V, P = _camera((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), 1.0, near=0.1, far=10.0, fov=60.0)
        for mode in range(7):
            imgs, _, _, _ = _check(gpu_ctx, scene, ds, V, P, EYE, 96, 96, mode)
        assert (imgs["albedo"][..., 3] == 255).mean() > 0.3
    finally:
        ds.free()


def test_non_finite_rho_next_to_a_near_plane_clipped_edge(gpu_ctx):
    """Triangles through the camera plane (clipped at the near plane) whose uvs make the quads' rho non-finite: uvs of
    +-3e38 (the squared steps overflow: +inf, the last level) and an infinite uv (0 * inf in the interpolation: NaN,
    level 0), beside one with ordinary uvs; the five targets bit for bit against the oracle in modes 0 and 2."""
    texs = [synth.random_texture(37, 23, 7), synth.random_texture(16, 16, 8), synth.random_texture(64, 32, 9)]
    base = [[(-2.0, -1.0, 1.0), (2.0, -1.0, 1.0), (0.0, 0.6, -3.0)]]
    pos = np.array(base * 3, np.float32)
    pos[1, :, 0] += 0.3
    pos[2, :, 0] -= 0.3
    tris = _soup(pos, 1.0)
    for k, uv in enumerate([((0, 0), (8, 0), (4, 8)), ((3e38, 0), (-3e38, 1), (0, -3e38)), ((np.inf, 0), (0, 0), (0, 1))]):
        for j in range(3):
            tris[k, 12 * j + 10: 12 * j + 12] = uv[j]
    prims = [_abi.Primitive(k, 1, (1.0, 1.0, 1.0, 1.0), 0, 1, 2) for k in range(3)]
    scene = _abi.Scene(tris, prims, texs)
    scene.compute_bboxes()
    ds = gpu_ctx.upload(scene)
    try:
        V, P = _camera((0.0, 0.0, 0.0), (0.0, -0.2, -1.0), 1.0, near=0.1, far=10.0, fov=70.0)
        for mode in (0, 2):
            imgs, _, _, _ = _check(gpu_ctx, scene, ds, V, P, EYE, 64, 64, mode)
            assert (imgs["albedo"][..., 3] == 255).sum() > 100
    finally:
        ds.free()


def test_pair_budget_prefix_and_determinism(gpu_ctx, helmet):
    scene, ds, arena = helmet
    w, h = 256, 192
    V, P = _camera(*OUTSIDE, w / h)
    counts, total = mesh.pairs(scene, V, P, EYE, w, h)
    _, drawn, pairs, _ = _check(gpu_ctx, scene, ds, V, P, EYE, w, h, arena=arena, max_pairs=1 << 29)
    assert drawn == scene.triangle_count and pairs == total
    budget = total // 3
    _, drawn, pairs, _ = _check(gpu_ctx, scene, ds, V, P, EYE, w, h, arena=arena, max_pairs=budget)
    cum = np.cumsum(counts.astype(np.int64))
    assert pairs == total and drawn == int(np.searchsorted(cum, budget, side="right"))
    a, _, _, _ = _render(gpu_ctx, ds, V, P, EYE, w, h, 6)
    b, _, _, _ = _render(gpu_ctx, ds, V, P, EYE, w, h, 6)
    assert all(np.array_equal(a[t].view(np.uint8), b[t].view(np.uint8)) for t in NAMES)
    _, drawn, _, _ = _check(gpu_ctx, scene, ds, V, P, EYE, w, h, arena=arena, max_pairs=0)
    assert drawn == int(np.searchsorted(cum, 0, side="right"))


def test_size_4096_accepted_4097_rejected(gpu_ctx):
    tris = _soup(_quad(-3.0, 0.2, 0.3, 0.1) + [[(-0.2, -0.3, -2.0), (0.1, -0.3, -2.0), (-0.05, -0.1, -2.0)]], 1.0)
    scene = _abi.Scene(tris, [_abi.Primitive(0, len(tris), (0.5, 0.6, 0.7, 1.0), -1, -1, -1)], [])
    ds = gpu_ctx.upload(scene)
    try:
        V, P = _camera((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), 1.0, near=0.1, far=10.0)
        imgs, _, _, _ = _check(gpu_ctx, scene, ds, V, P, EYE, 4096, 4096, 1)
        assert (imgs["albedo"][..., 3] == 255).any()
        import torch
        t = torch.empty(8 * 4097 * 4, dtype=torch.int16, device="cuda")
        for w, h, mode in ((4097, 4, 0), (4, 4097, 0), (0, 4, 0), (4, 4, 7)):
            with pytest.raises(M2SError):
                gpu_ctx.mesh_render(ds, V, P, EYE, w, h, NEAR_FAR, mode, targets=("position",), gbuffer={"position": t})
        with pytest.raises(M2SError):   # misaligned target
            gpu_ctx.mesh_render(ds, V, P, EYE, 4, 4, NEAR_FAR, 0, targets=("position",), gbuffer={"position": t[1:]})
    finally:
        ds.free()


# ---- split screen -----------------------------------------------------------------------------------------------------
def _split(gpu_ctx, sgb, mgb, cube, lp, position):
    import torch
    w, h = lp.width, lp.height
    gi = GuardedDevice(w * h, 4, what="image")
    img = gpu_ctx.deferred_light_split(sgb, mgb, cube, w, h, position, lp.render_mode, tuple(lp.light_position), tuple(lp.light_color),
                                       lp.light_intensity, tuple(lp.cam_pos), lp.far_plane, lp.shadow_size, image=gi.view)
    gi.check(w * h)
    return img


@pytest.mark.parametrize("mode", [0, 5, 6])
def test_split_lighting_columns_and_divider(gpu_ctx, helmet, mode):
    import torch
    scene, ds, _ = helmet
    w, h = 200, 120
    V, P = _camera(*OUTSIDE, w / h)
    _, _, _, mdev = _render(gpu_ctx, ds, V, P, EYE, w, h, 6)
    V2, P2 = _camera((0.5, -0.3, 2.5), (0.0, 0.0, 0.0), w / h)
    _, _, _, sdev = _render(gpu_ctx, ds, V2, P2, MIRROR, w, h, 6)   # any second G-buffer stands in for the splats'
    S = 16
    cube = torch.from_numpy(np.random.default_rng(4).random(6 * S * S).astype(np.float32)).cuda()
    lp = _abi.make_light_params(w, h, mode, (1.5, 2.0, 2.5), (1.0, 0.9, 0.8), 10.0, (0.0, 0.5, 3.2), 100.0, S)
    cp = cube if mode == 6 else None
    full_m = gpu_ctx.deferred_light(mdev, cp, w, h, mode, (1.5, 2.0, 2.5), (1.0, 0.9, 0.8), 10.0, (0.0, 0.5, 3.2), 100.0, S)
    full_s = gpu_ctx.deferred_light(sdev, cp, w, h, mode, (1.5, 2.0, 2.5), (1.0, 0.9, 0.8), 10.0, (0.0, 0.5, 3.2), 100.0, S)
    for position in (0.0, 0.5, 1.0, np.float32(0.3), np.float32(0.75)):   # 0.75 * 200 lands on an integer
        img = _split(gpu_ctx, sdev, mdev, cp, lp, float(position))
        split = int(np.float32(position) * np.float32(w))
        d0 = max(0, split - 1)
        assert (img[:, d0: min(w, d0 + 2)] == 255).all()
        left = np.ones(w, bool)
        left[split:] = False
        keep = np.ones(w, bool)
        keep[d0: min(w, d0 + 2)] = False
        assert np.array_equal(img[:, left & keep], full_m[:, left & keep])
        assert np.array_equal(img[:, ~left & keep], full_s[:, ~left & keep])
        assert np.array_equal(img, mesh.split(full_m, full_s, float(position)))
    for bad in (-0.1, 1.5, float("nan")):
        with pytest.raises(M2SError):
            _split(gpu_ctx, sdev, mdev, cp, lp, bad)


# ---- the whole frame --------------------------------------------------------------------------------------------------
def test_convert_mesh_prepass_sort_draw_shadow_split_light_chain_on_one_stream(gpu_ctx):
    """convert -> mesh render -> prepass -> sort -> splat draw -> shadow -> split light enqueued on one non-default stream
    with no host synchronisation, on the bench scene (helmet stand-in, R = 512) at 1920 x 1080.  The mesh G-buffer equals
    the oracle's, and the image the oracle's composite of the oracle's lighting of both G-buffers with the drawn cube."""
    import torch
    scene = synth.helmet_standin(2048)
    ds = gpu_ctx.upload(scene)
    R, S = 512, 1024
    cap = 6 * R * R
    w, h = 1920, 1080
    V, P = _camera(*OUTSIDE, 16 / 9)
    M = column_major(EYE)
    lpos = (1.5, 2.0, 2.5)
    stream = torch.cuda.Stream()
    out = torch.empty(cap * _abi.STRIDES[LAYOUT_REF96], dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    quads = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    depths = torch.empty(cap, dtype=torch.float32, device="cuda")
    valid = torch.zeros(1, dtype=torch.int32, device="cuda")
    sq = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    draw = torch.zeros(5, dtype=torch.int32, device="cuda")
    alloc = lambda: {t: torch.empty(w * h * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda")
                     for t, dt in _abi.GBUFFER_TARGETS}
    sbuf, mbuf = alloc(), alloc()
    gs = _abi.m2s_gbuffer(*[sbuf[t].data_ptr() for t in NAMES])
    gm = _abi.m2s_gbuffer(*[mbuf[t].data_ptr() for t in NAMES])
    gc = GuardedDevice(6 * S * S, 4, what="cube")
    gi = GuardedDevice(w * h, 4, what="image")
    res = torch.zeros(12, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    p = _abi.make_params(R, LAYOUT_REF96, 0.65, 0, FLAG_UNCAPPED)
    mp = _abi.make_mesh_render_params(V, P, M, w, h, NEAR_FAR, 6)
    pp = _abi.make_prepass_params(V, P, M, (w, h), NEAR_FAR, 0.65 / R, 6, LAYOUT_REF96)
    sp = _abi.m2s_splat_params(w, h, 6)
    shp = _abi.make_shadow_params(M, lpos, NEAR_FAR, (w, h), 0.65 / R, LAYOUT_REF96, S)
    lp = _abi.make_light_params(w, h, 6, lpos, (1.0, 1.0, 1.0), 10.0, OUTSIDE[0], 100.0, S)
    L, hs = lib(), stream.cuda_stream
    check(L.m2s_convert_enqueue(gpu_ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), hs))
    check(L.m2s_mesh_render_enqueue(gpu_ctx.handle, ds.handle, C.byref(mp), C.byref(gm), 60_000_000, res[8:].data_ptr(),
                                    res[10:].data_ptr(), hs))
    check(L.m2s_prepass_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                depths.data_ptr(), valid.data_ptr(), hs))
    check(L.m2s_depth_sort_enqueue(gpu_ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(), sq.data_ptr(),
                                   None, draw.data_ptr(), hs))
    check(L.m2s_splat_draw_enqueue(gpu_ctx.handle, sq.data_ptr(), cap, draw.data_ptr(), C.byref(sp), C.byref(gs),
                                   60_000_000, res.data_ptr(), res[2:].data_ptr(), hs))
    check(L.m2s_shadow_map_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(shp), gc.view.data_ptr(),
                                   None, 60_000_000, res[4:].data_ptr(), res[6:].data_ptr(), hs))
    check(L.m2s_deferred_light_split_enqueue(gpu_ctx.handle, C.byref(gs), C.byref(gm), gc.view.data_ptr(), C.byref(lp), 0.5,
                                             gi.view.data_ptr(), hs))
    stream.synchronize()
    o = res.cpu().numpy()
    assert int(o[10]) == scene.triangle_count, "the budget holds every mesh pair"
    gc.check(6 * S * S)
    gi.check(w * h)
    read = lambda buf: {t: buf[t].view(torch.uint8)[: w * h * 4 * np.dtype(dt).itemsize].cpu().numpy().view(dt).reshape(h, w, 4)
                        for t, dt in _abi.GBUFFER_TARGETS}
    mgb, sgb = read(mbuf), read(sbuf)
    want_m = mesh.mesh_render(scene, V, P, M, w, h, NEAR_FAR, 6)
    for t in NAMES:
        assert np.array_equal(mgb[t].view(np.uint8), want_m[t].view(np.uint8)), t
    cube = gc.view[: 6 * S * S * 4].cpu().numpy().view(np.float32).reshape(6, S, S)
    img = gi.view[: w * h * 4].cpu().numpy().reshape(h, w, 4)
    want = mesh.split(light.deferred_light(want_m, cube, lp), light.deferred_light(sgb, cube, lp), 0.5)
    assert np.array_equal(img, want), int((img != want).any(axis=-1).sum())
    assert (img[:, : w // 2 - 1, :3] > 0).any() and (img[:, w // 2 + 1:, :3] > 0).any()
    ds.free()
