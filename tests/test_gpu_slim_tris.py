"""The raster pass of PACKED56 from the 64-byte position/uv stream (m2s_dscene::d_tris_slim).

A scene uploaded whole carries its triangles' positions and uvs repacked into 4 float4 per triangle, {P0 u0} {P1 u1}
{P2 u2} {v0 v1 v2 0}, and a PACKED56 conversion stages those 64 bytes per triangle instead of the 144-byte AoS.  The
stream only repacks fp32 bits, so every record must be the one the 144-byte route (m2s_debug_set_slim_off) makes, bit for
bit, with the same count and the same fragment identities.  The cases cover the routes of the raster kernel: paired
direct passes, many units per warp, several primitives, larger triangles counted in row blocks, the capacity cut,
triangle sub-ranges and row bands, and a partially uploaded scene, which has no stream and takes the 144-byte route.
All marked gpu.
"""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager

import numpy as np
import pytest

from mesh2splat_b200 import _abi, _lib, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56

pytestmark = pytest.mark.gpu

L = LAYOUT_PACKED56


@contextmanager
def slim_off():
    _lib.lib().m2s_debug_set_slim_off(1)
    try:
        yield
    finally:
        _lib.lib().m2s_debug_set_slim_off(0)


def slim_stream(ctx, ds) -> np.ndarray | None:
    """The scene's 64-byte stream as (n, 16) uint32, or None when the scene has none."""
    fn = _lib.lib().m2s_debug_scene_slim_tris
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    buf = np.zeros((max(1, ds.triangle_count), 16), np.uint32)
    st = fn(ctx.handle, ds.handle, buf.ctypes.data)
    if st == _abi.M2S_E_INVALID:
        return None
    _lib.check(st)
    return buf[: ds.triangle_count]


def repack(tris: np.ndarray) -> np.ndarray:
    """numpy statement of the stream: the same bits, moved."""
    t = np.ascontiguousarray(tris, np.float32).view(np.uint32).reshape(-1, 3, 12)   # vertex: pos3 nrm3 tan4 uv2
    out = np.zeros((len(t), 4, 4), np.uint32)
    out[:, :3, :3] = t[:, :, 0:3]
    out[:, :3, 3] = t[:, :, 10]
    out[:, 3, :3] = t[:, :, 11]
    return out.reshape(-1, 16)


def by_key(o):
    k = o.keys_numpy()
    order = np.argsort(k, kind="stable")
    return k[order], o.numpy()[order]


def total_of(ctx, ds, R, **kw):
    return ctx.convert(ds, R, L, flags=FLAG_UNCAPPED, capacity=1, **kw).total


def convert_both(ctx, ds, R, capacity=None, **kw):
    """The same conversion on the slim route and on the 144-byte route; capacity None: the uncapped total."""
    cap = capacity if capacity is not None else max(1, total_of(ctx, ds, R, **kw))
    got = ctx.convert(ds, R, L, flags=FLAG_UNCAPPED, capacity=cap, want_keys=True, **kw)
    with slim_off():
        ref = ctx.convert(ds, R, L, flags=FLAG_UNCAPPED, capacity=cap, want_keys=True, **kw)
    assert got.total == ref.total and got.written == ref.written
    return got, ref


def assert_same(got, ref):
    gk, gr = by_key(got)
    rk, rr = by_key(ref)
    assert len(np.unique(gk)) == len(gk), "duplicate fragment identities"
    assert np.array_equal(gk, rk), "the slim route's fragment identities differ"
    assert gr.tobytes() == rr.tobytes(), "the slim route's records differ from the 144-byte route's"


def check_scene(ctx, scene, R, **kw):
    ds = ctx.upload(scene)
    try:
        s = slim_stream(ctx, ds)
        assert s is not None, "a scene uploaded whole has the slim stream"
        got, ref = convert_both(ctx, ds, R, **kw)
        assert got.total > 0 and not got.overflow
        assert_same(got, ref)
    finally:
        ds.free()
    return got


@pytest.fixture(scope="module")
def helmet():
    return synth.helmet_standin(2048)


@pytest.fixture(scope="module")
def sponza():
    return synth.sponza_standin(1024)


def test_stream_is_the_repacked_triangles(gpu_ctx, sponza):
    """The uploaded stream holds exactly the position and uv bits of the 144-byte triangles."""
    ds = gpu_ctx.upload(sponza)
    try:
        s = slim_stream(gpu_ctx, ds)
        assert s is not None and s.shape == (sponza.triangle_count, 16)
        assert np.array_equal(s, repack(sponza.triangles))
    finally:
        ds.free()


def test_bench_scene(gpu_ctx, helmet):
    """The benchmark's scene (helmet stand-in, R = 512): paired direct passes, late claims."""
    ds = gpu_ctx.upload(helmet)
    plan = gpu_ctx.convert_plan(ds, 512, L, flags=FLAG_UNCAPPED)
    ds.free()
    assert plan.direct_ok and plan.pair_first and plan.claim_late
    check_scene(gpu_ctx, helmet, 512)


def test_sphere_1m(gpu_ctx):
    """A million triangles at R = 256: many units per warp, claimed up front."""
    scene = synth.sphere_1m(2048)
    ds = gpu_ctx.upload(scene)
    plan = gpu_ctx.convert_plan(ds, 256, L, flags=FLAG_UNCAPPED)
    ds.free()
    assert plan.multi_round and not plan.claim_late and not plan.pair_first
    check_scene(gpu_ctx, scene, 256)


def test_sponza_many_primitives(gpu_ctx, sponza):
    """The sponza stand-in: many primitives (the set-up's primitive search) and large textured walls."""
    check_scene(gpu_ctx, sponza, 256)


@pytest.mark.parametrize("make", [synth.unit_quad, synth.box], ids=["quad", "box"])
def test_row_block_triangles(gpu_ctx, make):
    """Triangles far larger than the small-triangle box: counted in row blocks, shaded by the fragment kernel."""
    check_scene(gpu_ctx, make(), 512)


def test_capacity_cut(gpu_ctx, helmet):
    """Capped runs: both routes count the same total and store the same number of records, and every stored record is
    the uncapped route's record of the same fragment, bit for bit."""
    ds = gpu_ctx.upload(helmet)
    try:
        got, ref = convert_both(gpu_ctx, ds, 512)
        rk, rr = by_key(ref)
        total = got.total
        for cap in (total // 3, total - 777):
            for o in convert_both(gpu_ctx, ds, 512, capacity=cap):
                assert o.total == total and o.written == cap and o.overflow
                k = o.keys_numpy()
                assert len(np.unique(k)) == len(k)
                pos = np.minimum(np.searchsorted(rk, k), len(rk) - 1)
                assert np.array_equal(rk[pos], k), "a stored key is not a fragment of the uncapped result"
                assert o.numpy().tobytes() == rr[pos].tobytes()
    finally:
        ds.free()


@pytest.mark.parametrize("first,count,rows", [(1000, 20000, (0, 0)), (33333, 0, (0, 0)), (0, 0, (100, 300)),
                                              (517, 31000, (64, 80))],
                         ids=["range", "tail", "band", "range_band"])
def test_sub_ranges_and_bands(gpu_ctx, helmet, first, count, rows):
    """first_triangle / triangle_count and row bands (the shard parameters of a multi-GPU conversion): the shard's
    triangles are read at their global index in the stream."""
    check_scene(gpu_ctx, helmet, 512, first_triangle=first, triangle_count=count, row_begin=rows[0], row_end=rows[1])


def test_sponza_range_across_primitives(gpu_ctx, sponza):
    n = sponza.triangle_count
    check_scene(gpu_ctx, sponza, 256, first_triangle=n // 5, triangle_count=n // 2)


def test_partial_upload_falls_back(gpu_ctx, helmet):
    """A shard uploaded on its own (m2s_scene_upload_range) has no stream: its conversion takes the 144-byte route and
    makes the records the whole scene's slim route makes for the same triangles."""
    first, count = 4096, 30000
    part = gpu_ctx.upload_range(helmet, L, first, count)
    whole = gpu_ctx.upload(helmet)
    try:
        assert slim_stream(gpu_ctx, part) is None
        cap = max(1, total_of(gpu_ctx, whole, 512, first_triangle=first, triangle_count=count))
        a = gpu_ctx.convert(part, 512, L, flags=FLAG_UNCAPPED, capacity=cap, want_keys=True, first_triangle=first, triangle_count=count)
        b = gpu_ctx.convert(whole, 512, L, flags=FLAG_UNCAPPED, capacity=cap, want_keys=True, first_triangle=first, triangle_count=count)
        assert a.total == b.total > 0 and not a.overflow
        assert_same(a, b)
    finally:
        part.free()
        whole.free()


def test_other_layouts_unchanged_by_switch(gpu_ctx, helmet):
    """REF96 never reads the stream: the switch changes nothing there."""
    ds = gpu_ctx.upload(helmet)
    try:
        a = gpu_ctx.convert(ds, 256, _abi.LAYOUT_REF96, flags=FLAG_UNCAPPED, capacity=6 * 256 * 256, want_keys=True)
        with slim_off():
            b = gpu_ctx.convert(ds, 256, _abi.LAYOUT_REF96, flags=FLAG_UNCAPPED, capacity=6 * 256 * 256, want_keys=True)
        assert a.total == b.total > 0
        ka, ra = by_key(a)
        kb, rb = by_key(b)
        assert np.array_equal(ka, kb) and ra.tobytes() == rb.tobytes()
    finally:
        ds.free()
