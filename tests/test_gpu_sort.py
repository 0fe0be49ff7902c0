"""The viewer's depth sort on the GPU (SURVEY 8 f-5, RadixSortPass::execute -> m2s_depth_sort): every case compares the
sorted quads, the order and the draw command bit for bit with numpy's stable argsort of the depth bits plus the gather.
Every output goes through a guarded buffer (no write past n, no hole below n) and every input is checked byte-unchanged."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_REF96, Primitive, Scene
from mesh2splat_b200._lib import check, lib
from mesh2splat_b200.api import depth_sort_tile
from test_sort_host import KEY_SETS, expected_sort, make_depths, make_quads
from util import GuardedDevice

pytestmark = pytest.mark.gpu


def _sort_and_check(gpu_ctx, depths: np.ndarray, quads: np.ndarray | None = None, count: int | None = None,
                    device_count: int | None = None):
    """Sorts `count` (default: all) quads, with *d_count = device_count if given, and checks everything against the
    stable argsort of the first n depths.  Returns the outputs."""
    import torch
    count = len(depths) if count is None else count
    quads = make_quads(count) if quads is None else quads
    dq = torch.from_numpy(np.ascontiguousarray(quads).view(np.uint8).reshape(-1)).cuda()
    dd = torch.from_numpy(np.ascontiguousarray(depths, np.float32)).cuda()
    gs = GuardedDevice(count, _abi.QUAD_BYTES, what="sorted quads")
    go = GuardedDevice(count, 4, torch.int32, what="order")
    gd = GuardedDevice(5, 4, torch.int32, what="draw")
    dc = None if device_count is None else torch.tensor([device_count], dtype=torch.int32, device="cuda")
    got_q, got_o, got_d = gpu_ctx.depth_sort(dq, dd, count, d_count=dc, sorted_quads=gs.view, order=go.view, draw=gd.view)
    n = count if device_count is None else min(count, device_count)
    want_q, want_o, want_d = expected_sort(quads[:n], depths[:n])
    assert np.array_equal(got_d, want_d), (got_d, want_d)
    assert np.array_equal(got_o, want_o), f"order differs at {np.flatnonzero(got_o != want_o)[:8]}"
    assert np.array_equal(got_q.view(np.uint32), want_q.view(np.uint32))
    gs.check(n)
    go.check(n)
    gd.check(5)
    assert np.array_equal(dq.cpu().numpy(), np.ascontiguousarray(quads).view(np.uint8).reshape(-1)), "quads changed"
    assert np.array_equal(dd.cpu().numpy().view(np.uint32), np.ascontiguousarray(depths, np.float32).view(np.uint32)), "depths changed"
    return got_q, got_o, got_d


@pytest.mark.parametrize("kind", KEY_SETS)
def test_key_sets(gpu_ctx, kind):
    """Each key set over 100 000 keys (25 tiles, the last one partial): uniform negative depths, 16 distinct values
    (stability), all keys equal (the identity), sorted and reverse sorted, one varying byte per pass, and the special
    bit patterns (+-0, denormals, positive z, +-inf, NaNs)."""
    _, order, _ = _sort_and_check(gpu_ctx, make_depths(kind, 100_000, seed=3))
    if kind == "all_equal":
        assert np.array_equal(order, np.arange(100_000, dtype=np.uint32))


def _sizes():
    t = depth_sort_tile()
    return [0, 1, 2, 31, 32, 33, t - 1, t, t + 1, 3 * t - 1, 3 * t + 1, (1 << 24) + 1, 7_000_000]


@pytest.mark.parametrize("n", _sizes())
def test_sizes(gpu_ctx, n):
    """Sizes around a warp, around one and three tiles (the tile size read from the library), 2^24 + 1 and the reference's
    MAX_GAUSSIANS_TO_SORT (7 000 000)."""
    _sort_and_check(gpu_ctx, make_depths("uniform", n, seed=n))


@pytest.mark.parametrize("kind", ["sixteen_values", "specials", "byte3"])
def test_key_sets_over_many_tiles(gpu_ctx, kind):
    """Stability and the special keys over 2^24 + 1 keys (4097 tiles: long look-back chains across the grid)."""
    _sort_and_check(gpu_ctx, make_depths(kind, (1 << 24) + 1, seed=11))


@pytest.mark.parametrize("device_count", [0, 1, 33, 4097, 49_999, 50_000, 80_000])
def test_device_side_count(gpu_ctx, device_count):
    """count = the capacity (50 000), n = min(count, *d_count): nothing is written past n and draw[1] == n."""
    _, _, draw = _sort_and_check(gpu_ctx, make_depths("sixteen_values", 50_000, seed=5), device_count=device_count)
    assert draw[1] == min(50_000, device_count)


def test_count_zero_writes_only_the_draw_command(gpu_ctx):
    """n = 0: the draw command becomes {6, 0, 0, 0, 0} (the reference dispatches nothing and leaves the previous frame's
    instanceCount; DESIGN §6), and nothing else is written."""
    _, _, draw = _sort_and_check(gpu_ctx, np.zeros(0, np.float32))
    assert draw.tolist() == [6, 0, 0, 0, 0]


def test_deterministic(gpu_ctx):
    d = make_depths("sixteen_values", 1_000_000, seed=9)
    a = _sort_and_check(gpu_ctx, d)
    b = _sort_and_check(gpu_ctx, d)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_convert_prepass_sort_chain_on_one_stream(gpu_ctx, layout):
    """convert -> m2s_prepass_enqueue -> m2s_depth_sort_enqueue on one non-default stream with no host synchronisation in
    between: the conversion's device counter feeds the prepass and the prepass's valid counter feeds the sort.  After the
    final synchronise the sorted quads equal the stable sort of what the prepass wrote, and conic.w (= -z) is
    non-decreasing over the visible quads (z < 0), which come after any with z >= 0."""
    import torch
    from test_gpu_parity import _prepass_cases
    tri = synth.displaced_sphere(96, 48, seed=5)
    s = Scene(tri, [Primitive(0, len(tri), (1.0, 0.9, 0.8, 0.7), 0, 1, 2)], synth.make_material_textures(128, 9))
    s.compute_bboxes()
    ds = gpu_ctx.upload(s)
    R = 200
    cap = 6 * R * R
    stride = _abi.STRIDES[layout]
    stream = torch.cuda.Stream()
    for c in _prepass_cases():
        out = torch.empty(cap * stride, dtype=torch.uint8, device="cuda")
        total = torch.zeros(1, dtype=torch.int64, device="cuda")
        quads = torch.empty(cap * _abi.QUAD_BYTES, dtype=torch.uint8, device="cuda")
        depths = torch.empty(cap, dtype=torch.float32, device="cuda")
        valid = torch.zeros(1, dtype=torch.int32, device="cuda")
        gs = GuardedDevice(cap, _abi.QUAD_BYTES, what="sorted quads")
        go = GuardedDevice(cap, 4, torch.int32, what="order")
        draw = torch.zeros(5, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        p = _abi.make_params(R, layout, 0.65, 0, FLAG_UNCAPPED)
        pp = _abi.make_prepass_params(c["view"], c["proj"], c["model"], c["resolution"], c["near_far"], 0.65 / R, 0, layout)
        L, h = lib(), stream.cuda_stream
        check(L.m2s_convert_enqueue(gpu_ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), h))
        check(L.m2s_prepass_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                    depths.data_ptr(), valid.data_ptr(), h))
        check(L.m2s_depth_sort_enqueue(gpu_ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(),
                                       gs.view.data_ptr(), go.view.data_ptr(), draw.data_ptr(), h))
        stream.synchronize()
        n = int(valid.item())
        assert 0 < n <= int(total.item()) <= cap
        q = quads[: n * _abi.QUAD_BYTES].cpu().numpy().view(np.float32).reshape(n, 24)
        d = depths[:n].cpu().numpy()
        want_q, want_o, want_d = expected_sort(q, d)
        assert draw.cpu().numpy().view(np.uint32).tolist() == want_d.tolist()
        got_o = go.view[:n].cpu().numpy().view(np.uint32)
        got_q = gs.view[: n * _abi.QUAD_BYTES].cpu().numpy().view(np.float32).reshape(n, 24)
        assert np.array_equal(got_o, want_o)
        assert np.array_equal(got_q.view(np.uint32), want_q.view(np.uint32))
        gs.check(n)
        go.check(n)
        w = got_q[:, 15]                     # conic.w = -z
        vis = np.ascontiguousarray(d[want_o]).view(np.uint32) >= np.uint32(0x80000000)   # sign bit: z < 0 (or -0)
        if vis.any():
            first = int(np.argmax(vis))
            assert vis[first:].all(), "a quad with z >= 0 sorted after a visible one"
            assert np.all(np.diff(w[first:].astype(np.float64)) >= 0), "conic.w decreases along the sorted quads"
    ds.free()
