"""The viewer's shadow pass and deferred lighting on the GPU (rows f-7, f-8: m2s_shadow_map, m2s_deferred_light). Every
case compares bit for bit with the C restatement (oracle/m2s_light_oracle.c) and writes through guarded buffers, so a
record, texel or pixel written outside its buffer or never written fails: the light records against orc_light_prepass,
the cube of the GPU's own light records against orc_cube_raster, the image against orc_deferred_light."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_REF96
from mesh2splat_b200._lib import M2SError, check, lib
from oracle import light, splat
from util import GuardedDevice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
PREPASS = os.path.join(HERE, "golden", "ref_prepass_vectors.npz")
SPLAT = os.path.join(HERE, "golden", "ref_splat_vectors.npz")
NAMES = [t for t, _ in _abi.GBUFFER_TARGETS]
# light positions for the golden prepass cases: outside the cloud, inside its box (all six faces), on a diagonal
LIGHTS = [(3.0, 4.0, 2.5), (0.05, 0.02, -0.03), (2.0, 2.0, 2.0)]


def _upload(a: np.ndarray, min_bytes: int = 16):
    import torch
    b = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return torch.from_numpy(b.copy() if len(b) else np.zeros(min_bytes, np.uint8)).cuda()


def _golden_case(i: int):
    z = np.load(PREPASS)
    g = z[f"g{i}"].copy()
    prm = z[f"params{i}"]
    return g, z[f"model{i}"], (float(prm[0]), float(prm[1])), (float(prm[2]), float(prm[3])), float(prm[4])


def _same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def _same_records(a, b):
    """Light records bit for bit, NaN as NaN (the device's NaN pattern is not the host's); the face words exactly."""
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    both_nan = np.isnan(a[:, :7]) & np.isnan(b[:, :7])
    same = (a[:, :7].view(np.uint32) == b[:, :7].view(np.uint32)) | both_nan
    return bool(same.all()) and np.array_equal(a[:, 7].view(np.uint32), b[:, 7].view(np.uint32))


def _shadow(gpu_ctx, records, count, layout, M, lightp, near_far, res, sd, size, max_pairs=None, d_count=None, n_written=None):
    """The shadow pass through guarded cube and light-record buffers; returns (cube, light records, drawn, pairs)."""
    gc = GuardedDevice(6 * size * size, 4, what="cube")
    gl = GuardedDevice(max(count, 1), 32, what="light records")
    cube, lq, drawn, pairs = gpu_ctx.shadow_map(records, count, layout, M, lightp, near_far, res, sd, size, max_pairs=max_pairs,
                                                d_count=d_count, cube=gc.view.view(__import__("torch").float32), light_quads=gl.view)
    gc.check(6 * size * size)
    gl.check(count if n_written is None else n_written)
    return cube, lq, drawn, pairs


def _check_shadow(gpu_ctx, g, count, layout, M, lightp, near_far, res, sd, size, **kw):
    dr = _upload(g)
    cube, lq, drawn, pairs = _shadow(gpu_ctx, dr, count, layout, M, lightp, near_far, res, sd, size, **kw)
    p = _abi.make_shadow_params(M, lightp, near_far, res, sd, layout, size)
    n = kw.get("n_written", count)
    want = light.prepass(g, n, p)
    assert _same_records(lq[:n], want), f"{int((lq[:n].view(np.uint32) != want.view(np.uint32)).any(axis=1).sum())} light records differ"
    wc = light.cube(lq[:n], size, n=drawn)
    assert _same_bits(cube, wc), f"{int((cube != wc).sum())} texels differ"
    return cube, lq, drawn, pairs


@pytest.mark.parametrize("case", range(5))
def test_light_records_and_cube_on_the_golden_cases(gpu_ctx, case):
    g, M, res, nf, sd = _golden_case(case)
    lights = list(LIGHTS)
    if case == 0:   # identity model: a light exactly at a gaussian, and gaussians on the light's diagonals (face ties)
        lights.append(tuple(float(v) for v in g[3, :3]))
        g[10:20, :3] = np.array(LIGHTS[2], np.float32) + np.linspace(0.1, 1.0, 10, dtype=np.float32)[:, None] * [1, -1, 1]
        g[20:30, :3] = np.array(LIGHTS[2], np.float32) + np.linspace(0.1, 1.0, 10, dtype=np.float32)[:, None] * [0, -1, 1]
    faces = set()
    for lp in lights:
        _, lq, drawn, _ = _check_shadow(gpu_ctx, g, len(g), LAYOUT_REF96, M, lp, nf, res, sd, 64)
        assert drawn == len(g)
        f = lq[:, 7].view(np.uint32)
        faces |= set(f[f < 6].tolist())
    assert faces == set(range(6))


@pytest.mark.parametrize("size", [1, 17, 1024])
def test_cube_sizes(gpu_ctx, size):
    g, M, res, nf, sd = _golden_case(1)
    cube, _, _, _ = _check_shadow(gpu_ctx, g, len(g), LAYOUT_REF96, M, LIGHTS[1], nf, res, sd, size)
    assert (cube < 1.0).any()


def test_no_records_gives_the_clear(gpu_ctx):
    cube, _, drawn, pairs = _check_shadow(gpu_ctx, np.zeros((0, 24), np.float32), 0, LAYOUT_REF96, np.eye(4, dtype=np.float32), LIGHTS[0],
                                          (0.01, 100.0), (1280, 720), 0.01, 33)
    assert drawn == 0 and pairs == 0 and (cube == 1.0).all()


def _crafted(n_extra=0):
    """Gaussians in front of the +Z face of a light at the origin: quads of chosen size and depth."""
    g = np.zeros((8 + n_extra, 24), np.float32)
    g[:, 16] = 1.0
    g[:, 2] = np.linspace(1.0, 3.0, len(g))
    g[:, 8:11] = 200.0
    return g


def test_face_filling_quads_past_the_guard_band_degenerate_and_overlapping(gpu_ctx):
    """Huge splats (axes at the 1024-pixel cap: they fill the face), splats past the guard band, degenerate ones (zero
    and NaN scales, NaN positions) and overlapping splats in both orders."""
    M, nf = np.eye(4, dtype=np.float32), (0.01, 100.0)
    g = _crafted(40)
    g[0, 8:11] = 1e6                          # axes capped at 1024 pixels of the 1920 x 1080 renderer: fills the face
    g[1:6, 0] = [50.0, -80.0, 1e6, np.inf, np.nan]   # far off-axis, past the guard band, non-finite
    g[6:10, 8:11] = 0.0                       # zero scale
    g[10:12, 8:11] = np.nan
    g[12:14, 16:20] = np.nan                  # NaN rotation
    for size in (64, 1024):
        a, _, _, _ = _check_shadow(gpu_ctx, g, len(g), LAYOUT_REF96, M, (0.0, 0.0, 0.0), nf, (1920, 1080), 0.01, size)
        b, _, _, _ = _check_shadow(gpu_ctx, g[::-1].copy(), len(g), LAYOUT_REF96, M, (0.0, 0.0, 0.0), nf, (1920, 1080), 0.01, size)
        assert np.array_equal(a, b)   # LESS on a per-quad constant: order does not matter
        assert (a[4] < 1.0).mean() > 0.99


def test_pair_cut_and_device_count(gpu_ctx):
    import torch
    g, M, res, nf, sd = _golden_case(4)
    p = _abi.make_shadow_params(M, LIGHTS[1], nf, res, sd, LAYOUT_REF96, 256)
    recs = light.prepass(g, len(g), p)
    counts, total = light.pairs(recs, 256)
    incl = np.cumsum(counts.astype(np.int64))
    k = int(np.searchsorted(incl, total // 2))
    for budget in sorted({0, 1, int(incl[k]), int(incl[k]) - 1, total - 1, total}):
        _, _, drawn, pairs = _check_shadow(gpu_ctx, g, len(g), LAYOUT_REF96, M, LIGHTS[1], nf, res, sd, 256, max_pairs=budget)
        assert pairs == total and drawn == int(np.searchsorted(incl, budget, side="right")), (budget, drawn)
    for n in (0, 1, 137):
        d = torch.tensor([n], dtype=torch.int64, device="cuda")
        _, _, drawn, pairs = _check_shadow(gpu_ctx, g, len(g), LAYOUT_REF96, M, LIGHTS[1], nf, res, sd, 256, max_pairs=total + 10,
                                           d_count=d, n_written=n)
        assert drawn == n and pairs == int(counts[:n].sum())


def test_deterministic_and_size_1025_rejected(gpu_ctx):
    rng = np.random.default_rng(5)
    g = np.zeros((50000, 24), np.float32)
    g[:, :3] = rng.uniform(-1, 1, (50000, 3))
    g[:, 8:11] = rng.uniform(1, 8, (50000, 3))
    g[:, 16:20] = rng.normal(0, 1, (50000, 4))
    dr = _upload(g)
    a = _shadow(gpu_ctx, dr, len(g), LAYOUT_REF96, np.eye(4), (0.1, 0.0, 0.0), (0.01, 100.0), (1920, 1080), 0.65 / 512, 512)
    b = _shadow(gpu_ctx, dr, len(g), LAYOUT_REF96, np.eye(4), (0.1, 0.0, 0.0), (0.01, 100.0), (1920, 1080), 0.65 / 512, 512)
    assert _same_bits(a[0], b[0]) and _same_bits(a[1], b[1])   # the same device: NaN patterns too
    with pytest.raises(M2SError):
        gpu_ctx.shadow_map(dr, len(g), LAYOUT_REF96, np.eye(4), (0, 0, 0), (0.01, 100.0), (1920, 1080), 0.01, 1025)


# ---- lighting -------------------------------------------------------------------------------------------------------
def _light(gpu_ctx, gb: dict, cube, lp: _abi.m2s_light_params, names=NAMES):
    """The lighting pass through a guarded image; gb: {name: numpy (H, W, 4)}; cube numpy or None."""
    import torch
    w, h = lp.width, lp.height
    dev = {t: _upload(gb[t]) for t in names if t in gb}
    dc = torch.from_numpy(np.ascontiguousarray(cube, np.float32).reshape(-1)).cuda() if cube is not None else None
    gi = GuardedDevice(w * h, 4, what="image")
    img = gpu_ctx.deferred_light(dev, dc, w, h, lp.render_mode, tuple(lp.light_position), tuple(lp.light_color), lp.light_intensity,
                                 tuple(lp.cam_pos), lp.far_plane, lp.shadow_size, image=gi.view)
    gi.check(w * h)
    want = light.deferred_light({t: gb[t] for t in names if t in gb}, cube, lp)
    assert np.array_equal(img, want), f"{int((img != want).any(axis=-1).sum())} pixels differ"
    return img


def _golden_cube(size=64):
    g, M, res, nf, sd = _golden_case(0)
    p = _abi.make_shadow_params(M, LIGHTS[0], nf, res, sd, LAYOUT_REF96, size)
    return light.cube(light.prepass(g, len(g), p), size)


@pytest.mark.parametrize("mode", range(7))
def test_lighting_all_modes_on_the_golden_gbuffers(gpu_ctx, mode):
    z = np.load(SPLAT)
    w, h = (int(v) for v in z["img_size"])
    cube = _golden_cube()
    for case in range(5):
        gb = {t: z[f"img{case}_{t}"] for t in NAMES}
        lp = _abi.make_light_params(w, h, mode, LIGHTS[0], (1.0, 0.9, 0.8), 25.0, (3.0, 2.0, 4.0), 100.0, 64)
        img = _light(gpu_ctx, gb, cube if mode == 6 else None, lp)
        if mode == 6:
            assert len(np.unique(img.reshape(-1, 4), axis=0)) > 20


def _random_gbuffer(rng, w, h):
    pos = rng.normal(0, 2, (h, w, 4)).astype(np.float16)
    nrm = rng.random((h, w, 4)).astype(np.float16)
    alb = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    mr = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    for a in (pos, nrm):
        flat = a.reshape(-1)
        k = min(len(flat), 40)
        idx = rng.choice(len(flat), k, replace=False)
        flat[idx[: k // 4]] = np.inf
        flat[idx[k // 4: k // 2]] = -np.inf
        flat[idx[k // 2: 3 * k // 4]] = np.nan
        flat[idx[3 * k // 4:]] = 0.0
    nrm.reshape(-1, 4)[: max(1, w * h // 10), :3] = -nrm.reshape(-1, 4)[: max(1, w * h // 10), :3]   # negative normals
    return {"position": pos, "normal": nrm, "albedo": alb, "depth": np.zeros((h, w, 4), np.float16), "metallic_roughness": mr}


@pytest.mark.parametrize("wh", [(1, 1), (17, 15), (1921, 1081), (4096, 4096)])
def test_lighting_sizes_with_inf_and_nan_texels(gpu_ctx, wh):
    rng = np.random.default_rng(wh[0])
    gb = _random_gbuffer(rng, *wh)
    cube = _golden_cube(17)
    for mode in (6, 5, 0):
        _light(gpu_ctx, gb, cube if mode == 6 else None, _abi.make_light_params(wh[0], wh[1], mode, (0.3, 0.2, 0.1), (1, 1, 1), 8.0,
                                                                                   (0.0, 0.0, 4.0), 10.0, 17))


def test_lighting_size_4097_and_null_targets(gpu_ctx):
    import torch
    t = torch.zeros(64 * 4, dtype=torch.uint8, device="cuda")
    h16 = torch.zeros(64 * 4, dtype=torch.int16, device="cuda")
    cube = torch.ones(6, dtype=torch.float32, device="cuda")
    with pytest.raises(M2SError):
        gpu_ctx.deferred_light({"albedo": t}, None, 4097, 1, 0)
    full = {"position": h16, "normal": h16, "albedo": t, "metallic_roughness": t}
    for drop in full:
        with pytest.raises(M2SError):
            gpu_ctx.deferred_light({k: v for k, v in full.items() if k != drop}, cube, 8, 8, 6, shadow_size=1)
    with pytest.raises(M2SError):
        gpu_ctx.deferred_light(full, None, 8, 8, 6, shadow_size=1)
    rng = np.random.default_rng(9)
    gb = _random_gbuffer(rng, 8, 8)
    for mode in range(6):   # NULL cube and only the needed targets accepted in modes 0-5
        _light(gpu_ctx, gb, None, _abi.make_light_params(8, 8, mode), names=["albedo", "metallic_roughness"] if mode == 5 else ["albedo"])


def test_lighting_light_at_a_pixel_and_on_the_tie_rule(gpu_ctx):
    """The light placed exactly at a pixel's world position (zero light direction: NaN taps), and pixels whose PCF taps
    land on the cube's face ties (|x| = |y| directions) and on the 0.05 bias threshold."""
    rng = np.random.default_rng(11)
    w, h = 32, 16
    gb = _random_gbuffer(rng, w, h)
    pos = gb["position"].astype(np.float32)
    lp_at = tuple(float(v) for v in pos[3, 5, :3])
    gb["position"][4, :, :3] = (np.array(lp_at, np.float32) + np.array([1, 1, 0.5], np.float32) * np.linspace(0.5, 2, w)[:, None]).astype(np.float16)
    cube = _golden_cube(64)
    _light(gpu_ctx, gb, cube, _abi.make_light_params(w, h, 6, lp_at, (1, 1, 1), 3.0, (1.0, 1.0, 5.0), 100.0, 64))
    # threshold: a cube of one constant depth c, pixels at distance c * far + 0.05 (and neighbours) from the light
    c = np.float32(0.25)
    flat = np.full((6, 8, 8), c, np.float32)
    d = np.float32(c * np.float32(20.0)) + np.float32(0.05)
    dirs = rng.normal(0, 1, (h, w, 3))
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    radius = d + np.array([-1e-3, 0.0, 1e-3], np.float32)[rng.integers(0, 3, (h, w))]
    gb["position"][..., :3] = (dirs * radius[..., None]).astype(np.float16)
    img = _light(gpu_ctx, gb, flat, _abi.make_light_params(w, h, 6, (0.0, 0.0, 0.0), (1, 1, 1), 3.0, (1.0, 1.0, 5.0), 20.0, 8))
    assert img[..., 3].min() == 255


# ---- the whole frame --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_convert_prepass_sort_draw_shadow_light_chain_on_one_stream(gpu_ctx, layout):
    """convert -> prepass -> sort -> draw -> shadow -> light enqueued on one non-default stream with no host
    synchronisation, on the bench scene (helmet stand-in, R = 512) with the chain test's camera at 1920 x 1080.  The light
    records equal the oracle's light prepass of the converted records, the cube the oracle's raster of those records,
    and the image the oracle's lighting of the drawn G-buffer and that cube."""
    import torch
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_prepass import column_major, look_at, perspective
    scene = synth.helmet_standin(2048)
    ds = gpu_ctx.upload(scene)
    R, S = 512, 1024
    cap = 6 * R * R
    V = column_major(look_at(np.array([0.0, 0.5, 3.2]), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(45.0), 16 / 9, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    lpos = (1.5, 2.0, 2.5)
    stream = torch.cuda.Stream()
    out = torch.empty(cap * _abi.STRIDES[layout], dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    quads = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    depths = torch.empty(cap, dtype=torch.float32, device="cuda")
    valid = torch.zeros(1, dtype=torch.int32, device="cuda")
    sq = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    draw = torch.zeros(5, dtype=torch.int32, device="cuda")
    w, h = 1920, 1080
    gbuf = {t: torch.empty(w * h * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda") for t, dt in _abi.GBUFFER_TARGETS}
    g = _abi.m2s_gbuffer(*[gbuf[t].data_ptr() for t in NAMES])
    gc = GuardedDevice(6 * S * S, 4, what="cube")
    gl = GuardedDevice(cap, 32, what="light records")
    gi = GuardedDevice(w * h, 4, what="image")
    res = torch.zeros(8, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    p = _abi.make_params(R, layout, 0.65, 0, FLAG_UNCAPPED)
    pp = _abi.make_prepass_params(V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 6, layout)
    sp = _abi.m2s_splat_params(w, h, 6)
    shp = _abi.make_shadow_params(M, lpos, (0.01, 100.0), (w, h), 0.65 / R, layout, S)
    lp = _abi.make_light_params(w, h, 6, lpos, (1.0, 1.0, 1.0), 10.0, (0.0, 0.5, 3.2), 100.0, S)
    L, hs = lib(), stream.cuda_stream
    check(L.m2s_convert_enqueue(gpu_ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), hs))
    check(L.m2s_prepass_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                depths.data_ptr(), valid.data_ptr(), hs))
    check(L.m2s_depth_sort_enqueue(gpu_ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(), sq.data_ptr(),
                                   None, draw.data_ptr(), hs))
    check(L.m2s_splat_draw_enqueue(gpu_ctx.handle, sq.data_ptr(), cap, draw.data_ptr(), C.byref(sp), C.byref(g),
                                   60_000_000, res.data_ptr(), res[2:].data_ptr(), hs))
    check(L.m2s_shadow_map_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(shp), gc.view.data_ptr(),
                                   gl.view.data_ptr(), 60_000_000, res[4:].data_ptr(), res[6:].data_ptr(), hs))
    check(L.m2s_deferred_light_enqueue(gpu_ctx.handle, C.byref(g), gc.view.data_ptr(), C.byref(lp), gi.view.data_ptr(), hs))
    stream.synchronize()
    n = int(total.item())
    o = res.cpu().numpy()
    assert n > 0 and int(o[6]) == n, "the budget holds every pair"
    gc.check(6 * S * S)
    gl.check(n)
    gi.check(w * h)
    recs = out[: n * _abi.STRIDES[layout]].cpu().numpy()
    lq = gl.view[: n * 32].cpu().numpy().view(np.float32).reshape(n, 8)
    assert _same_records(lq, light.prepass(recs, n, shp))
    cube = gc.view[: 6 * S * S * 4].cpu().numpy().view(np.float32).reshape(6, S, S)
    assert _same_bits(cube, light.cube(lq, S))
    assert int(o[4:6].view(np.uint64)[0]) == light.pairs(lq, S)[1]
    gb = {t: gbuf[t].view(torch.uint8)[: w * h * 4 * np.dtype(dt).itemsize].cpu().numpy().view(dt).reshape(h, w, 4)
          for t, dt in _abi.GBUFFER_TARGETS}
    img = gi.view[: w * h * 4].cpu().numpy().reshape(h, w, 4)
    want = light.deferred_light(gb, cube, lp)
    assert np.array_equal(img, want), int((img != want).any(axis=-1).sum())
    assert (img[..., :3] > 0).any()
    ds.free()
