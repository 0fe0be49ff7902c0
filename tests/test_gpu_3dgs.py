"""The standard 3DGS render on the GPU (m2s_3dgs_render): both targets bit for bit against the C restatement
(oracle/m2s_3dgs_oracle.c) through guarded buffers, across layouts, SH degrees, sizes, culling, deep stacks, ties, model
matrices, d_count, the pair budget and NULL targets; the preprocessed colour against m2s_prepass_sh's; the bench scene
end to end; the .ply export round trip within the codec's rounding; and the argument checks."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._lib import M2SError, lib
from oracle import gs3d
from util import GuardedDevice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

EYE = column_major(np.eye(4, dtype=np.float32))


def camera(w, h, eye=(0.3, 0.4, 3.0), tgt=(0.0, 0.0, 0.0), fov=50.0):
    V = column_major(look_at(np.array(eye, np.float64), np.array(tgt, np.float64), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(fov), w / h, 0.01, 100.0))
    return V, P


def ref96(n, seed, spread=1.0, log_s=(-3.5, -1.5)):
    rng = np.random.default_rng(seed)
    r = np.zeros((n, 24), np.float32)
    r[:, 0:3] = rng.uniform(-spread, spread, (n, 3))
    r[:, 8:11] = np.exp(rng.uniform(*log_s, (n, 3)))
    r[:, 16:20] = rng.normal(size=(n, 4))
    r[:, 4:7] = rng.uniform(-0.1, 1.1, (n, 3))
    r[:, 7] = rng.uniform(0.05, 1.0, n)
    r[:, 12:15] = rng.normal(size=(n, 3))
    return r


def packed56(n, seed):
    rng = np.random.default_rng(seed)
    r = np.zeros((n, 14), np.float32)
    r[:, 0:3] = rng.uniform(-1, 1, (n, 3))
    r[:, 3:7] = rng.normal(size=(n, 4))
    r[:, 7:10] = rng.uniform(-3.5, -1.5, (n, 3))
    r[:, 10:13] = rng.normal(size=(n, 3))
    r[:, 13] = rng.normal(size=n) * 2
    return r


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).reshape(-1).view(np.uint8)).cuda()


def render_guarded(ctx, rec, layout, V, P, M, w, h, targets=("rgba8", "rgba32f"), **kw):
    """ctx.render_3dgs into guarded targets; (rgba32f (h, w, 4) or None, rgba8 (h, w, 4) or None, drawn, pairs)."""
    import torch
    n = kw.pop("count", len(rec))
    gb = {}
    if "rgba8" in targets:
        gb["rgba8"] = GuardedDevice(w * h, 4, what="rgba8")
    if "rgba32f" in targets:
        gb["rgba32f"] = GuardedDevice(w * h, 16, dtype=torch.float32, what="rgba32f")
    records = _dev(rec) if len(rec) else torch.zeros(16, dtype=torch.uint8, device="cuda")
    imgs, drawn, pairs = ctx.render_3dgs(records, n, layout, V, P, M, w, h, targets=targets, images={k: g.view for k, g in gb.items()}, **kw)
    for g in gb.values():
        g.check(w * h)
    f32 = imgs["rgba32f"].cpu().numpy().reshape(h, w, 4) if "rgba32f" in imgs else None
    u8 = imgs["rgba8"].cpu().numpy().reshape(h, w, 4) if "rgba8" in imgs else None
    return f32, u8, drawn, pairs


def check_against_oracle(ctx, rec, layout, V, P, M, w, h, sh=None, buffer_degree=0, sh_degree=0, **kw):
    import torch
    shd = torch.from_numpy(np.ascontiguousarray(sh, np.float32)).cuda() if sh is not None else None
    f32, u8, drawn, pairs = render_guarded(ctx, rec, layout, V, P, M, w, h, sh=shd, sh_degree=sh_degree, **kw)
    kw.pop("max_pairs", None)
    kw.pop("d_count", None)
    wf, wu, wdrawn, wpairs = gs3d.render(rec, layout, V, P, M, w, h, sh=sh, buffer_degree=buffer_degree, sh_degree=sh_degree, **kw)
    assert f32.tobytes() == wf.tobytes(), np.argwhere(f32.view(np.uint32) != wf.view(np.uint32))[:5]
    assert u8.tobytes() == wu.tobytes()
    assert pairs == wpairs
    return f32, u8, pairs


@pytest.mark.parametrize("layout", [_abi.LAYOUT_REF96, _abi.LAYOUT_PACKED56, _abi.VIEW_PLY, _abi.VIEW_PLY_PBR])
def test_every_layout_bit_for_bit(gpu_ctx, layout):
    w, h = 200, 120
    V, P = camera(w, h)
    rec = packed56(3000, 1) if layout == _abi.LAYOUT_PACKED56 else ref96(3000, 1)
    check_against_oracle(gpu_ctx, rec, layout, V, P, EYE, w, h, near=0.2, std_dev=0.8, background=(0.1, 0.2, 0.3))


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_sh_degrees_bit_for_bit(gpu_ctx, degree):
    w, h = 160, 96
    V, P = camera(w, h)
    rec = ref96(2000, 2)
    rng = np.random.default_rng(3)
    sh = (rng.normal(size=(len(rec), _abi.SH_FLOATS[3])) * 0.3).astype(np.float32)
    check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, sh=sh, buffer_degree=3, sh_degree=degree, near=0.2)


@pytest.mark.parametrize("wh", [(1, 1), (16, 16), (17, 33), (250, 7), (4096, 4096)])
def test_sizes(gpu_ctx, wh):
    w, h = wh
    V, P = camera(w, h)
    n = 20000 if w == 4096 else 1500
    check_against_oracle(gpu_ctx, ref96(n, 4, log_s=(-4.5, -2.5)), _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)


def test_empty_culled_and_covering(gpu_ctx):
    w, h = 70, 50
    V, P = camera(w, h)
    f32, u8, pairs = check_against_oracle(gpu_ctx, np.zeros((0, 24), np.float32), _abi.VIEW_PLY, V, P, EYE, w, h, background=(0.5, 0.25, 1.0))
    assert pairs == 0 and np.all(f32[..., 3] == 0) and np.all(f32[..., 0] == 0.5)
    behind = ref96(500, 5)
    behind[:, 2] += 10.0   # behind the camera at z = 3
    _, _, pairs = check_against_oracle(gpu_ctx, behind, _abi.VIEW_PLY, V, P, EYE, w, h)
    assert pairs == 0
    big = ref96(1, 6)
    big[0, 0:3], big[0, 8:11], big[0, 7] = 0.0, 5.0, 0.9
    _, _, pairs = check_against_oracle(gpu_ctx, big, _abi.VIEW_PLY, V, P, EYE, w, h)
    assert pairs == 5 * 4


def test_deep_stacks_and_ties(gpu_ctx):
    w, h = 64, 64
    V, P = camera(w, h, eye=(0, 0, 3))
    rec = ref96(4000, 7, spread=0.2, log_s=(-2.5, -1.5))
    rec[:, 7] = 0.9
    rec[::2, 2] = rec[1::2, 2]           # pairs at equal depth
    rec[2000:, 0:3] = rec[:2000, 0:3]    # exact duplicates: equal depths, drawn in index order
    rec[2000:, 4:7] = 1.0 - rec[:2000, 4:7]
    f32, _, _ = check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h)
    assert np.mean(f32[..., 3] > 0.999) > 0.1   # the stacked centre stopped early


@pytest.mark.parametrize("which", ["rotated", "scaled", "mirrored"])
def test_model_matrices(gpu_ctx, which):
    w, h = 96, 80
    V, P = camera(w, h)
    c, s = np.cos(0.7), np.sin(0.7)
    M = {"rotated": np.array([[c, 0, s, 0.1], [0, 1, 0, -0.2], [-s, 0, c, 0.3], [0, 0, 0, 1]]),
         "scaled": np.diag([1.5, 0.5, 2.0, 1.0]),
         "mirrored": np.diag([-1.0, 1.0, 1.0, 1.0])}[which]
    check_against_oracle(gpu_ctx, ref96(1500, 8), _abi.LAYOUT_REF96, V, P, column_major(M.astype(np.float32)), w, h, std_dev=0.7)


def test_d_count_budget_and_null_target(gpu_ctx):
    import torch
    w, h = 128, 96
    V, P = camera(w, h)
    rec = ref96(3000, 9)
    d_count = torch.tensor([1200], dtype=torch.int64, device="cuda")
    f32, u8, drawn, pairs = render_guarded(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, max_pairs=(1 << 30) - 1, d_count=d_count)
    wf, wu, wdrawn, wpairs = gs3d.render(rec[:1200], _abi.VIEW_PLY, V, P, EYE, w, h)
    assert f32.tobytes() == wf.tobytes() and u8.tobytes() == wu.tobytes() and (drawn, pairs) == (wdrawn, wpairs)
    budget = wpairs // 3
    f32, u8, drawn, pairs = render_guarded(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, max_pairs=budget)
    wf, wu, wdrawn, wpairs = gs3d.render(rec, _abi.VIEW_PLY, V, P, EYE, w, h, max_pairs=budget)
    assert 0 < drawn == wdrawn and pairs == wpairs and f32.tobytes() == wf.tobytes() and u8.tobytes() == wu.tobytes()
    only8 = render_guarded(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, targets=("rgba8",))
    only32 = render_guarded(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, targets=("rgba32f",))
    full = gs3d.render(rec, _abi.VIEW_PLY, V, P, EYE, w, h)
    assert only8[0] is None and only8[1].tobytes() == full[1].tobytes()
    assert only32[1] is None and only32[0].tobytes() == full[0].tobytes()
    again = render_guarded(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h)
    assert again[0].tobytes() == full[0].tobytes()


def test_preprocess_records_and_sh_colour_match_prepass(gpu_ctx):
    import torch
    w, h = 160, 96
    V, P = camera(w, h)
    rec = ref96(2000, 10)
    rng = np.random.default_rng(11)
    sh = torch.from_numpy((rng.normal(size=(len(rec), 48)) * 0.3).astype(np.float32)).cuda()
    recd = _dev(rec)
    splats, keys, alive = gpu_ctx.gs3d_preprocess(recd, len(rec), _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2, sh=sh)
    ws, wk, walive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2, sh=sh.cpu().numpy(), buffer_degree=3, sh_degree=3)
    assert alive == walive and splats.tobytes() == ws.tobytes() and keys.tobytes() == wk.tobytes()
    quads, _ = gpu_ctx.prepass(recd, len(rec), _abi.VIEW_PLY, V, P, EYE, (w, h), (0.01, 100.0), 1.0, 0, sh=sh)
    # the prepass's survivors in arrival order: match them by world position (q[5].xyz) to records
    by_pos = {tuple(r[0:3].tolist()): i for i, r in enumerate(rec)}
    matched = 0
    for q in quads:
        i = by_pos[tuple(q[20:23].tolist())]
        if keys[i] == _abi.GS3D_CULLED or np.any(q[8:11] < 0):
            continue
        assert splats[i, 6:9].tobytes() == q[8:11].tobytes()
        matched += 1
    assert matched > 500


@pytest.mark.parametrize("view", ["outside", "inside"])
def test_bench_scene_end_to_end(gpu_ctx, view):
    scene = synth.helmet_standin(2048)
    ds = gpu_ctx.upload(scene)
    try:
        out = gpu_ctx.convert(ds, 512, _abi.LAYOUT_REF96, 0.65, flags=_abi.FLAG_UNCAPPED)
        n = out.written
        w, h = 480, 270
        eye = (0.0, 0.5, 3.2) if view == "outside" else (0.0, 0.0, 0.1)
        V, P = camera(w, h, eye=eye, tgt=(0.0, 0.0, 0.0) if view == "outside" else (0.0, 0.0, -1.0), fov=60.0)
        imgs, drawn, pairs = gpu_ctx.render_3dgs(out.data, n, _abi.LAYOUT_REF96, V, P, EYE, w, h, near=0.01, std_dev=0.65 / 512)
        rec = out.data[: n * 96].cpu().numpy().view(np.float32).reshape(n, 24)
        wf, wu, _, wpairs = gs3d.render(rec, _abi.LAYOUT_REF96, V, P, EYE, w, h, near=0.01, std_dev=0.65 / 512)
        assert imgs["rgba32f"].cpu().numpy().tobytes() == wf.tobytes() and imgs["rgba8"].cpu().numpy().tobytes() == wu.tobytes()
        assert pairs == wpairs > 0
        res = gpu_ctx.compare_images(imgs["rgba8"], imgs["rgba8"], w, h)
        assert res["ssim"] == 1.0
    finally:
        ds.free()


def test_export_round_trip(gpu_ctx, tmp_path):
    """REF96 records rendered, then written to a .ply and read back (VIEW_PLY) and rendered: the two images agree within
    the codec's roundings (log/exp of the scale, logit/sigmoid of the opacity, SH0 of the colour: each a few ulp relative,
    which moves a pixel's value by far less than 2^-12 except where an alpha crosses 1/255 or a T the 1e-4 stop)."""
    import torch
    from mesh2splat_b200 import api
    w, h = 128, 96
    V, P = camera(w, h)
    rec = ref96(1500, 12)
    rec[:, 4:7] = np.clip(rec[:, 4:7], 0.02, 0.98)
    rec[:, 16:20] /= np.linalg.norm(rec[:, 16:20], axis=1, keepdims=True)
    a, *_ = gpu_ctx.render_3dgs(_dev(rec), len(rec), _abi.LAYOUT_REF96, V, P, EYE, w, h, std_dev=1.0)
    path = str(tmp_path / "rt.ply")
    api.ply_write(path, rec, 0, 1.0)
    loaded, n, _ = gpu_ctx.ply_read(path)
    b, *_ = gpu_ctx.render_3dgs(loaded, n, _abi.VIEW_PLY, V, P, EYE, w, h)
    fa = a["rgba32f"].cpu().numpy().reshape(h, w, 4)
    fb = b["rgba32f"].cpu().numpy().reshape(h, w, 4)
    close = np.abs(fa - fb) <= 2.0 ** -12
    assert close.mean() > 0.99, close.mean()


def test_argument_checks(gpu_ctx):
    import torch
    w, h = 32, 32
    V, P = camera(w, h)
    rec = _dev(ref96(10, 13))
    img = torch.full((w * h * 4,), 7, dtype=torch.uint8, device="cuda")
    f32 = torch.full((w * h * 4,), 7.0, dtype=torch.float32, device="cuda")

    def call(count=10, records=rec, rgba32f=f32, rgba8=img, sh=None, bd=0, sd=0, **over):
        kw = dict(world_to_view=V, view_to_clip=P, model_to_world=EYE, width=w, height=h, near=0.2, std_dev=1.0, scale_modifier=1.0,
                  background=(0, 0, 0), layout=_abi.VIEW_PLY)
        kw.update(over)
        p = _abi.make_3dgs_params(**kw)
        ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
        return lib().m2s_3dgs_render(gpu_ctx.handle, ptr(records), count, C.byref(p), ptr(sh), bd, sd, ptr(rgba32f), ptr(rgba8), None)

    bad_P = P.copy()
    bad_P.ravel()[0] = -1.0
    nan_V = V.copy()
    nan_V.ravel()[3] = np.nan
    sh = torch.zeros(10 * 12, dtype=torch.float32, device="cuda")
    cases = [dict(width=0), dict(height=4097), dict(layout=2), dict(rgba32f=None, rgba8=None), dict(rgba8=img[1:]),
             dict(rgba32f=f32[1:]), dict(records=rec[4:]), dict(layout=_abi.LAYOUT_REF96, sh=sh, bd=1, sd=1), dict(sh=sh, bd=1, sd=2),
             dict(sh=None, bd=1, sd=1), dict(near=0.0), dict(near=float("nan")), dict(view_to_clip=bad_P), dict(world_to_view=nan_V),
             dict(model_to_world=np.zeros(16, np.float32)), dict(count=1 << 30)]
    for c in cases:
        assert call(**c) == _abi.M2S_E_INVALID, c
    torch.cuda.synchronize()
    assert torch.all(img == 7) and torch.all(f32 == 7.0)
    assert call() == _abi.M2S_OK
