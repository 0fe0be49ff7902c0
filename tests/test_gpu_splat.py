"""The viewer's splat draw on the GPU (row f-6, GaussianSplattingPass::execute -> m2s_splat_draw): every case compares
all five G-buffer targets bit for bit with orc_splat_draw (NaN as NaN: both store 0x7FFF) and writes through guarded
buffers, so a pixel written outside the W x H x 4 target or never written fails."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_REF96, Primitive, Scene
from mesh2splat_b200._lib import check, lib
from oracle import splat
from test_splat_host import prepass_quads_sorted
from util import GuardedDevice

pytestmark = pytest.mark.gpu
NAMES = [t for t, _ in _abi.GBUFFER_TARGETS]


def _upload(quads: np.ndarray):
    import torch
    q = np.ascontiguousarray(quads, np.float32).reshape(-1, 24)
    return torch.from_numpy(q.view(np.uint8).reshape(-1).copy() if len(q) else np.zeros(96, np.uint8)).cuda()


def _draw(gpu_ctx, quads, w, h, mode=0, targets=NAMES, max_pairs=None, d_draw=None, count=None, dq=None):
    """Draws on the GPU through guarded targets; returns (images, drawn, pairs) after checking the guards."""
    count = len(quads) if count is None else count
    dq = _upload(quads) if dq is None else dq
    guards = {t: GuardedDevice(w * h, 8 if dt == np.float16 else 4, what=t) for t, dt in _abi.GBUFFER_TARGETS if t in targets}
    imgs, drawn, pairs = gpu_ctx.splat_draw(dq, count, w, h, mode, d_draw=d_draw, targets=targets, max_pairs=max_pairs,
                                            gbuffer={t: g.view for t, g in guards.items()})
    for g in guards.values():
        g.check(w * h)
    return imgs, drawn, pairs


def _check(gpu_ctx, quads, w, h, mode=0, targets=NAMES, **kw):
    imgs, drawn, pairs = _draw(gpu_ctx, quads, w, h, mode, targets, **kw)
    want = splat.draw(quads, w, h, mode, n=drawn, targets=targets)
    for t in targets:
        a, b = imgs[t].view(np.uint8), want[t].view(np.uint8)
        assert np.array_equal(a, b), f"{t}: {int((a != b).any(axis=-1).sum())} pixels differ"
    return imgs, drawn, pairs


@pytest.mark.parametrize("mode", range(7))
def test_golden_prepass_quads_all_modes(gpu_ctx, mode):
    for case in range(5):
        imgs, drawn, pairs = _check(gpu_ctx, prepass_quads_sorted(case), 1280, 720, mode)
        assert drawn == len(prepass_quads_sorted(case)) and pairs == splat.pairs(prepass_quads_sorted(case), 1280, 720)[1]


def _random_quads(n, seed, spread=1.2, size=0.05):
    rng = np.random.default_rng(seed)
    q = np.zeros((n, 24), np.float32)
    q[:, 0:2] = rng.uniform(-spread, spread, (n, 2))
    q[:, 4:8] = rng.normal(0, size, (n, 4))
    q[:, 8:12] = rng.random((n, 4))
    q[:, 12:15] = rng.random((n, 3)) * [200, 50, 200]      # conic in pixels^-2
    q[:, 15] = rng.uniform(0.1, 50, n)                   # depth
    q[:, 16:24] = rng.normal(0, 1, (n, 8))
    return q


@pytest.mark.parametrize("wh", [(1, 1), (17, 15), (1921, 1081), (4096, 4096)])
def test_sizes(gpu_ctx, wh):
    q = _random_quads(300, seed=wh[0], size=0.2)
    q[:, 12:15] *= 1e-4 if wh[0] > 1000 else 1.0
    _check(gpu_ctx, q, wh[0], wh[1], 0)


def test_size_4097_rejected(gpu_ctx):
    from mesh2splat_b200._lib import M2SError
    with pytest.raises(M2SError):
        gpu_ctx.splat_draw(_upload(_random_quads(3, 1)), 3, 4097, 16)


def test_no_quads_gives_the_clear(gpu_ctx):
    imgs, drawn, pairs = _check(gpu_ctx, np.zeros((0, 24), np.float32), 100, 60)
    assert drawn == 0 and pairs == 0 and all(not imgs[t].view(np.uint8).any() for t in NAMES)


def test_screen_filling_quad_at_the_axis_cap(gpu_ctx):
    """One quad whose axes are 1024 pixels long in a 1024 x 1024 viewport, plus a 2048-pixel one (past the edges)."""
    q = _random_quads(2, 5)
    q[:, 0:2] = 0.0
    q[0, 4:8] = [1.0, 0.0, 0.0, 1.0]
    q[1, 4:8] = [1.4, 1.4, -1.4, 1.4]
    q[:, 12:15] = [1e-5, 0.0, 1e-5]
    _check(gpu_ctx, q, 1024, 1024, 0)
    _check(gpu_ctx, q[::-1].copy(), 1024, 1024, 4)


def test_past_the_edges_and_the_guard_band(gpu_ctx):
    q = _random_quads(400, 6, spread=3.0, size=0.5)
    q[:10, 0] = np.array([30.0, -30.0, 63.0, -64.5, 100.0, np.inf, np.nan, 1e30, -1e30, 64.0], np.float32)
    q[10:20, 4:8] = 50.0
    _check(gpu_ctx, q, 256, 256, 0)


def test_degenerate_quads(gpu_ctx):
    q = _random_quads(50, 8)
    q[:10, 4:8] = 0.0                  # a point
    q[10:20, 6:8] = q[10:20, 4:6]      # a segment: both axes equal
    q[20:25, 4:8] = 1e-7
    q[25:30, 4:8] = np.nan
    q[30:35, 12:15] = np.nan           # NaN exponent
    q[35:40, 12:15] = [-1e4, 0.0, -1e4]   # exp overflows to inf
    _check(gpu_ctx, q, 64, 48, 0)
    _check(gpu_ctx, q, 64, 48, 4)


def test_overlapping_snapped_triangles_blend_twice(gpu_ctx):
    rng = np.random.default_rng(0)
    for _ in range(100000):
        q = np.zeros(24, np.float32)
        q[0:2] = rng.uniform(-0.5, 0.5, 2)
        a = rng.normal(0, 0.2, 2); d = rng.normal(0, 1e-4, 2)
        q[4:6] = a; q[6:8] = a + d; q[8:12] = [0.6, 0.5, 0.4, 0.7]; q[12:15] = [0.01, 0.0, 0.01]; q[16:24] = 0.5
        if (splat.coverage(q, 0, 64, 48) & splat.coverage(q, 1, 64, 48)).any():
            break
    else:
        pytest.fail("no overlapping quad found")
    single = splat.draw(q[None], 64, 48, 0)
    imgs, _, _ = _check(gpu_ctx, q[None], 64, 48, 0)
    ov = splat.coverage(q, 0, 64, 48) & splat.coverage(q, 1, 64, 48)
    y, x = np.argwhere(ov)[0]
    assert imgs["albedo"][y, x, 3] > 0 and np.array_equal(imgs["albedo"], single["albedo"])


def test_two_overlapping_quads_in_both_orders(gpu_ctx):
    q = _random_quads(2, 9)
    q[:, 0:2] = [[0.0, 0.0], [0.05, 0.0]]
    q[:, 4:8] = [0.3, 0.0, 0.0, 0.3]
    q[:, 12:15] = [0.002, 0.0, 0.002]
    q[:, 8:12] = [[1.0, 0.0, 0.0, 0.8], [0.0, 1.0, 0.0, 0.6]]
    a, _, _ = _check(gpu_ctx, q, 128, 96, 0)
    b, _, _ = _check(gpu_ctx, q[::-1].copy(), 128, 96, 0)
    assert not np.array_equal(a["albedo"], b["albedo"])


def test_rgba8_clamp_saturates(gpu_ctx):
    q = _random_quads(30, 10, spread=0.3, size=0.3)
    q[:, 8:12] = [3.0, -2.0, 40.0, 1.5]     # colour * alpha out of [0, 1]
    q[:, 12:15] = [0.01, 0.0, 0.01]         # wide gaussians: g near 1 around the mean
    q[:, 16:24] = [5.0, 0, 0, -7.0, 0, 0, 0, 9.0]
    imgs, _, _ = _check(gpu_ctx, q, 64, 64, 0)
    assert (imgs["albedo"] == 255).any() and (imgs["metallic_roughness"] == 255).any()
    _check(gpu_ctx, q, 64, 64, 4)


def test_null_targets_leave_the_others_unchanged(gpu_ctx):
    q = prepass_quads_sorted(1)
    full, _, _ = _check(gpu_ctx, q, 320, 180, 0)
    for keep in (["albedo"], ["position", "metallic_roughness"], ["normal", "depth"]):
        part, _, _ = _check(gpu_ctx, q, 320, 180, 0, targets=keep)
        for t in keep:
            assert np.array_equal(part[t].view(np.uint8), full[t].view(np.uint8))


def test_pair_cut(gpu_ctx):
    q = prepass_quads_sorted(4)
    w, h = 1280, 720
    counts, total = splat.pairs(q, w, h)
    incl = np.cumsum(counts.astype(np.int64))
    k = int(np.searchsorted(incl, total // 2))      # a prefix boundary: incl[k] pairs draw exactly k + 1 quads
    for budget in sorted({0, 1, int(incl[k]), int(incl[k]) - 1, total - 1, total}):
        imgs, drawn, pairs = _check(gpu_ctx, q, w, h, 0, max_pairs=budget)
        assert pairs == total
        assert drawn == int(np.searchsorted(incl, budget, side="right")), (budget, drawn)


def test_draw_command_from_the_sort(gpu_ctx):
    import torch
    q = prepass_quads_sorted(0)
    dq = _upload(q)
    for instances in (len(q), len(q) - 7, 1, 0, len(q) + 50):
        d = torch.tensor([6, instances, 0, 0, 0], dtype=torch.int32, device="cuda")
        imgs, drawn, _ = _check(gpu_ctx, q, 400, 300, 0, max_pairs=500_000, d_draw=d, dq=dq)
        assert drawn == min(len(q), instances)


def test_deterministic(gpu_ctx):
    q = _random_quads(20000, 11, size=0.03)
    a, _, _ = _draw(gpu_ctx, q, 800, 600, 0)
    b, _, _ = _draw(gpu_ctx, q, 800, 600, 0)
    for t in NAMES:
        assert np.array_equal(a[t].view(np.uint8), b[t].view(np.uint8))


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_convert_prepass_sort_draw_chain_on_one_stream(gpu_ctx, layout):
    """convert -> prepass -> sort -> draw enqueued on one non-default stream with no host synchronisation: the bench
    scene (helmet stand-in, R = 512) through the sort bench's camera at 1920 x 1080 equals the oracle's draw of the
    sorted quads."""
    import torch
    import sys, os
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden_prepass import column_major, look_at, perspective
    scene = synth.helmet_standin(2048)
    ds = gpu_ctx.upload(scene)
    R = 512
    cap = 6 * R * R
    V = column_major(look_at(np.array([0.0, 0.5, 3.2]), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(45.0), 16 / 9, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    stream = torch.cuda.Stream()
    out = torch.empty(cap * _abi.STRIDES[layout], dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    quads = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    depths = torch.empty(cap, dtype=torch.float32, device="cuda")
    valid = torch.zeros(1, dtype=torch.int32, device="cuda")
    sq = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    draw = torch.zeros(5, dtype=torch.int32, device="cuda")
    w, h = 1920, 1080
    guards = {t: GuardedDevice(w * h, 8 if dt == np.float16 else 4, what=t) for t, dt in _abi.GBUFFER_TARGETS}
    g = _abi.m2s_gbuffer(*[guards[t].view.data_ptr() for t in NAMES])
    res = torch.zeros(4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    p = _abi.make_params(R, layout, 0.65, 0, FLAG_UNCAPPED)
    pp = _abi.make_prepass_params(V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 0, layout)
    sp = _abi.m2s_splat_params(w, h, 0)
    L, hs = lib(), stream.cuda_stream
    check(L.m2s_convert_enqueue(gpu_ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), hs))
    check(L.m2s_prepass_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                depths.data_ptr(), valid.data_ptr(), hs))
    check(L.m2s_depth_sort_enqueue(gpu_ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(), sq.data_ptr(),
                                   None, draw.data_ptr(), hs))
    check(L.m2s_splat_draw_enqueue(gpu_ctx.handle, sq.data_ptr(), cap, draw.data_ptr(), C.byref(sp), C.byref(g),
                                   60_000_000, res.data_ptr(), res[2:].data_ptr(), hs))
    stream.synchronize()
    n = int(valid.item())
    assert n > 0 and int(draw[1].item()) == n
    o = res.cpu().numpy()
    assert int(o[2]) == n, "the budget holds every pair"
    q = sq[: n * 96].cpu().numpy().view(np.float32).reshape(n, 24)
    want = splat.draw(q, w, h, 0)
    for t, dt in _abi.GBUFFER_TARGETS:
        guards[t].check(w * h)
        got = guards[t].view[: w * h * (8 if dt == np.float16 else 4)].cpu().numpy()
        assert np.array_equal(got, want[t].view(np.uint8).reshape(-1)), t
    assert int(o[:2].view(np.uint64)[0]) == splat.pairs(q, w, h)[1]
    ds.free()
