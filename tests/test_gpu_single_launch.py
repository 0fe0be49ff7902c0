"""Conversions that end in the raster kernel (ConvertPlan::single_launch): PACKED56 launches on the direct path where no
work item can be queued, because every triangle's candidate box is small at the density (the scene's r_small_max) and
units beyond M2S_DIRECT_MAX are shaded in rounds.  The raster kernel's last CTA publishes the count; no fragment kernel
follows.

Each case converts on the single launch and again with the route switched off (Context.single_launch_off: the fragment
kernel is launched as well and shades the heavy units), and both must give the same count and the same multiset of
records, bit for bit.  The route checks read the plan of launches that must keep two kernels.  All marked gpu.
"""
from __future__ import annotations

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56, STRIDES
from mesh2splat_b200.api import Context

pytestmark = pytest.mark.gpu

L = LAYOUT_PACKED56
R = 512
N_HEAVY = 70_000   # enough triangles for several units per raster warp on an H100 (the direct path's launches)
CAP = 12 * R * R   # records: above every count here (the heavy scene's is 36 N_HEAVY)


def rows_sorted(rec: np.ndarray) -> np.ndarray:
    words = np.ascontiguousarray(rec).view(np.uint8).reshape(len(rec), STRIDES[L]).view(np.uint64)
    return words[np.lexsort(words.T[::-1])]


def heavy_scene(big: bool = False) -> _abi.Scene:
    """N_HEAVY right triangles of 7.85 x 7.85 pixels at R, each covering 36 pixel centres of an 8 x 8 box (small): a unit of
    16 holds 576 fragments (beyond M2S_DIRECT_MAX), a paired pass 1152 (more than one round of the direct list).  The
    triangles overlap on a 64 x 64 grid of cells.  big: triangle 0 spans 40 x 40 pixels instead (not small)."""
    t = np.arange(N_HEAVY)
    i0 = (t % 64) * 8.0
    j0 = ((t // 64) % 64) * 8.0
    x = np.stack([i0 + 0.1, i0 + 7.95, i0 + 0.1], axis=1)
    y = np.stack([j0 + 0.1, j0 + 0.1, j0 + 7.95], axis=1)
    if big:
        x[0] = [0.1, 40.1, 0.1]
        y[0] = [0.1, 0.1, 40.1]
    v = np.zeros((N_HEAVY, 3, 12), np.float32)
    v[:, :, 0] = x / R
    v[:, :, 1] = y / R
    v[:, :, 5] = 1.0                               # normal (0, 0, 1)
    v[:, :, 6] = 1.0; v[:, :, 9] = 1.0             # tangent (1, 0, 0, 1)
    v[:, :, 10] = v[:, :, 0]; v[:, :, 11] = v[:, :, 1]
    prim = _abi.Primitive(0, N_HEAVY, (0.9, 1.0, 0.8, 1.0), 0, -1, -1, bbox_min=(0.0, 0.0, 0.0), bbox_max=(1.0, 1.0, 0.0))
    return _abi.Scene(v.reshape(N_HEAVY, 36), [prim], synth.make_material_textures(256, 6)[:1])


def convert(ctx, ds, single: bool, capacity: int, max_gaussians: int = 0, want_keys: bool = False):
    """One conversion on the single launch (single) or on the two-kernel route; the route is checked in the plan."""
    flags = 0 if max_gaussians else FLAG_UNCAPPED
    if single:
        assert ctx.convert_plan(ds, R, L, capacity=capacity, max_gaussians=max_gaussians, flags=flags).single_launch
        return ctx.convert(ds, R, L, capacity=capacity, max_gaussians=max_gaussians, flags=flags, want_keys=want_keys)
    with Context.single_launch_off():
        plan = ctx.convert_plan(ds, R, L, capacity=capacity, max_gaussians=max_gaussians, flags=flags)
        assert plan.direct_ok and not plan.single_launch
        return ctx.convert(ds, R, L, capacity=capacity, max_gaussians=max_gaussians, flags=flags, want_keys=want_keys)


def assert_same(got, ref, want_keys: bool = False):
    assert got.total == ref.total and got.written == ref.written
    a, b = got.numpy(), ref.numpy()
    if want_keys:
        ak, bk = got.keys_numpy(), ref.keys_numpy()
        oa, ob = np.argsort(ak, kind="stable"), np.argsort(bk, kind="stable")
        assert np.array_equal(ak[oa], bk[ob]), "the fragment identities differ"
        assert a[oa].tobytes() == b[ob].tobytes(), "single launch and two-kernel route disagree"
    else:
        assert np.array_equal(rows_sorted(a), rows_sorted(b)), "single launch and two-kernel route disagree"


@pytest.fixture(scope="module")
def bench(gpu_ctx):
    ds = gpu_ctx.upload(synth.helmet_standin(2048))
    yield ds
    ds.free()


@pytest.fixture(scope="module")
def heavy(gpu_ctx):
    ds = gpu_ctx.upload(heavy_scene())
    yield ds
    ds.free()


@pytest.mark.parametrize("want_keys", [False, True], ids=["no_keys", "keys"])
def test_bench_scene(gpu_ctx, bench, want_keys):
    """The benchmark's conversion (helmet stand-in, R = 512) is a single launch, with the two-kernel route's records."""
    assert bench.r_small_max() >= R
    got = convert(gpu_ctx, bench, True, CAP, want_keys=want_keys)
    ref = convert(gpu_ctx, bench, False, CAP, want_keys=want_keys)
    assert got.total > 0
    assert_same(got, ref, want_keys)


@pytest.mark.parametrize("want_keys", [False, True], ids=["no_keys", "keys"])
def test_heavy_units_in_rounds(gpu_ctx, heavy, want_keys):
    """Units of 576 small-triangle fragments: the two-kernel route queues them for the fragment kernel, the single launch
    shades them in the raster kernel, a paired pass of 1152 in two rounds."""
    plan = gpu_ctx.convert_plan(heavy, R, L, capacity=CAP, flags=FLAG_UNCAPPED)
    assert plan.pair_first and plan.unit_tris == 16 and plan.direct_max < 16 * 36
    got = convert(gpu_ctx, heavy, True, CAP, want_keys=want_keys)
    ref = convert(gpu_ctx, heavy, False, CAP, want_keys=want_keys)
    assert got.total == 36 * N_HEAVY
    assert_same(got, ref, want_keys)


@pytest.mark.parametrize("scene", ["bench", "heavy"])
def test_capacity_cut(gpu_ctx, bench, heavy, scene):
    """A cap below the count: the count stays uncapped, the records stop at the cap, and every stored record is one of
    the uncut conversion's."""
    ds = bench if scene == "bench" else heavy
    full = convert(gpu_ctx, ds, True, CAP)
    cap = full.total * 2 // 3
    got = convert(gpu_ctx, ds, True, CAP, max_gaussians=cap)
    ref = convert(gpu_ctx, ds, False, CAP, max_gaussians=cap)
    assert got.overflow and ref.overflow
    assert got.total == ref.total == full.total and got.written == ref.written == cap
    every = {r.tobytes() for r in rows_sorted(full.numpy())}
    assert all(r.tobytes() in every for r in rows_sorted(got.numpy()))


def test_routes_alternate_on_one_context(bench):
    """single -> two -> single -> two on a fresh context (its first launch clears both scheduler sets), then the same
    after the host pipeline and the timed form (two kernels each) have used the sets: every conversion has the first
    one's count and records.  Each launch re-arms the other set as it starts, whichever route it takes."""
    scene = synth.helmet_standin(2048)
    with Context(0) as ctx:
        ds = ctx.upload(scene)
        first = convert(ctx, ds, True, CAP)
        for single in (False, True, False):
            assert_same(convert(ctx, ds, single, CAP), first)
        ctx.convert_host(scene, R, L, flags=FLAG_UNCAPPED, capacity=CAP)
        out = first.data.clone()
        ctx.convert_timed(ds, _abi.make_params(R, L, 0.65, 0, FLAG_UNCAPPED), out, CAP)
        for single in (True, False, True):
            assert_same(convert(ctx, ds, single, CAP), first)
        ds.free()


def test_route_one_large_triangle(gpu_ctx):
    """One triangle whose box is not small keeps the whole scene on two kernels."""
    ds = gpu_ctx.upload(heavy_scene(big=True))
    try:
        assert ds.r_small_max() < R
        plan = gpu_ctx.convert_plan(ds, R, L, capacity=CAP, flags=FLAG_UNCAPPED)
        assert plan.direct_ok and not plan.single_launch
        out = gpu_ctx.convert(ds, R, L, capacity=CAP, flags=FLAG_UNCAPPED)
        assert out.total > 36 * (N_HEAVY - 1)
    finally:
        ds.free()


def test_route_density_just_above_the_bound(gpu_ctx, bench):
    """R = floor(r_small_max) is a single launch, R + 1 takes two kernels."""
    r = int(np.floor(bench.r_small_max()))
    assert gpu_ctx.convert_plan(bench, r, L, capacity=CAP, flags=FLAG_UNCAPPED).single_launch
    plan = gpu_ctx.convert_plan(bench, r + 1, L, capacity=CAP, flags=FLAG_UNCAPPED)
    assert plan.direct_ok and not plan.single_launch


def test_route_upload_range(gpu_ctx):
    """A shard uploaded with m2s_scene_upload_range has no slim stream and no bound: two kernels."""
    scene = synth.helmet_standin(256)
    ds = gpu_ctx.upload_range(scene, L, 0, scene.triangle_count)
    try:
        assert ds.r_small_max() == 0.0
        plan = gpu_ctx.convert_plan(ds, R, L, capacity=CAP, flags=FLAG_UNCAPPED)
        assert plan.direct_ok and not plan.single_launch
    finally:
        ds.free()


def test_r_small_max_matches_the_host_bound(bench):
    """The device's bound is the host restatement's (tests/test_single_launch_host.py), over the oracle's uv."""
    from test_single_launch_host import scene_r_small_max
    want = scene_r_small_max(synth.helmet_standin(16))
    assert bench.r_small_max() == pytest.approx(want, rel=1e-5)
