"""Where the kernels write: the capacity cut on every write route, the output bounds of every call, and the resolution
limits.  All marked gpu.

Every conversion here writes into guarded buffers (util.GuardedDevice / GuardedHost): the bytes before the buffer and
everything from `written` records on must still hold the fill pattern afterwards, and no record below `written` may
still be entirely the pattern.  The scenes are stacked watertight tilings (util.layered_tiling) whose total, k R^2, is
known without the oracle.  Each case reads the launch plan (Context.convert_plan, the function the launch itself uses)
and asserts that it takes the route it is meant to test, whatever the SM count of the GPU.
"""
from __future__ import annotations

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import (FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_PLY_COMPRESSED, LAYOUT_PLY_PBR, LAYOUT_PLY_STANDARD,
                                  LAYOUT_REF96, M2S_E_CAPACITY, M2S_E_INVALID, STRIDES)
from util import GuardedDevice, GuardedHost, assert_records_match, layered_tiling

pytestmark = pytest.mark.gpu

K = 7   # layers: with one primitive the reference's own cap, 6 R^2, stores 6 of them


def caps_for(total: int):
    mid = total // 2 - (total // 2) % 32 + 17   # = 17 mod 32: the cut falls inside a warp's 32-record span
    return sorted({0, 1, 33, mid, total - 1, total, total + 1})


def _warps(ctx, layout):
    ds = ctx.upload(synth.unit_quad())
    w = int(ctx.convert_plan(ds, 64, layout).raster_warps)
    ds.free()
    return w


def _subset(keys, wkeys_sorted):
    """Indices into the sorted uncapped oracle keys of every key (asserting each is there)."""
    pos = np.minimum(np.searchsorted(wkeys_sorted, keys), len(wkeys_sorted) - 1)
    assert np.array_equal(wkeys_sorted[pos], keys), "a stored key is not a fragment of the uncapped result"
    return pos


def convert_guarded(ctx, ds, R, layout, cap, **kw):
    import torch
    out = GuardedDevice(cap, STRIDES[layout], what="records")
    keys = GuardedDevice(cap, 8, torch.int64, what="keys")
    o = ctx.convert(ds, R, layout, flags=FLAG_UNCAPPED, capacity=cap, out=out.view, keys=keys.view, want_keys=True, **kw)
    out.check(o.written)
    keys.check(o.written)
    return o


def cut_everywhere(ctx, scene, R, layout, want_total=None, ds=None, caps=None, **kw):
    """Converts at every cap of caps_for(total) and checks each result against ONE uncapped oracle run."""
    own = ds is None
    if own:
        ds = ctx.upload(scene)
    want, wkeys, total = oracle.convert(scene, R, layout, flags=FLAG_UNCAPPED, capacity=K * R * R + 64, **kw)
    assert total > 0
    assert len(want) == total
    if want_total is not None:
        assert total == want_total, (total, want_total)
    order = np.argsort(wkeys)
    ws, wk = want[order], wkeys[order]
    for cap in (caps or caps_for(total)):
        o = convert_guarded(ctx, ds, R, layout, cap, **kw)
        assert o.total == total, (cap, o.total, total)
        assert o.overflow == (total > cap), cap
        assert o.written == min(total, cap), (cap, o.written)
        k = o.keys_numpy()
        assert len(np.unique(k)) == len(k), f"cap {cap}: duplicate fragment identities"
        if len(k):
            pos = _subset(k, wk)
            assert_records_match(scene, layout, o.numpy(), k, ws[pos], k)
    if own:
        ds.free()
    return want, wkeys, total


def _unit_weights(wkeys, unit_tris, n_units):
    """Fragments per work unit (units of `unit_tris` triangles from triangle 0)."""
    tri = (wkeys >> np.uint64(24)).astype(np.int64)
    return np.bincount(tri // unit_tris, minlength=n_units)


# ---- the cut on every route ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("claim", ["late", "up_front"])
def test_cut_direct_route(gpu_ctx, claim):
    """PACKED56 with several units per warp: the raster kernel shades light units itself (direct_run), claiming its
    next unit late (< 3 units per warp) or up front."""
    w = _warps(gpu_ctx, LAYOUT_PACKED56)
    # triangles per raster warp: 65 = 3 rounds of 22-triangle units, 2.95 units per warp (late); 110 = 4 rounds (up front)
    per_warp = 65 if claim == "late" else 110
    n = per_warp * w // (2 * K)                         # Delaunay: ~2 n triangles per layer
    s = layered_tiling(K, 512, "delaunay", n=n, seed=3)
    ds = gpu_ctx.upload(s)
    plan = gpu_ctx.convert_plan(ds, 512, LAYOUT_PACKED56, capacity=K * 512 * 512)
    assert plan.multi_round and plan.direct_ok
    assert bool(plan.claim_late) == (claim == "late"), (s.triangle_count, w, plan.n_units)
    want, wkeys, total = cut_everywhere(gpu_ctx, s, 512, LAYOUT_PACKED56, K * 512 * 512, ds=ds)
    wt = _unit_weights(wkeys, int(plan.unit_tris), int(plan.n_units))
    assert len(wt) == plan.n_units
    direct = np.count_nonzero((wt >= 1) & (wt <= plan.direct_max))
    assert direct >= 0.9 * plan.n_units, f"only {direct} of {plan.n_units} units are light enough for the direct path"
    ds.free()


def test_cut_queue_route_unit_items(gpu_ctx):
    """The direct-path triangles in a single-round range (<= 32 triangles per raster warp): every unit's small triangles
    become one unit item for the fragment kernel."""
    w = _warps(gpu_ctx, LAYOUT_PACKED56)
    s = layered_tiling(K, 512, "delaunay", n=65 * w // (2 * K), seed=3)
    ds = gpu_ctx.upload(s)
    count = 32 * w
    plan = gpu_ctx.convert_plan(ds, 512, LAYOUT_PACKED56, capacity=K * 512 * 512, triangle_count=count)
    assert not plan.multi_round and not plan.direct_ok and plan.unit_tris == 32
    want, wkeys, _ = cut_everywhere(gpu_ctx, s, 512, LAYOUT_PACKED56, ds=ds, triangle_count=count)
    wt = _unit_weights(wkeys, int(plan.unit_tris), int(plan.n_units))
    assert np.count_nonzero(wt > 32) >= 0.9 * len(wt)   # unit items, not micro items
    ds.free()


def test_cut_micro_items(gpu_ctx):
    """A sub-pixel tiling at R = 64 (REF96): most units emit <= 32 fragments and are queued as micro items."""
    s = layered_tiling(K, 64, "delaunay", n=3000, seed=5)
    ds = gpu_ctx.upload(s)
    plan = gpu_ctx.convert_plan(ds, 64, LAYOUT_REF96, capacity=K * 64 * 64)
    assert not plan.direct_ok
    want, wkeys, _ = cut_everywhere(gpu_ctx, s, 64, LAYOUT_REF96, K * 64 * 64, ds=ds)
    wt = _unit_weights(wkeys, int(plan.unit_tris), int(plan.n_units))
    assert np.count_nonzero((wt >= 1) & (wt <= 32)) >= 0.5 * plan.n_units
    ds.free()


def test_cut_block_split_and_help_queue_items(gpu_ctx):
    """Full-height strips at R = 512: every triangle is counted in row blocks; 8 strips are 32 pixels wide (blocks of
    more fragments than a work item: split items); at >= 2 triangles of 16 blocks per unit, every unit posts to its CTA's
    help queue and every CTA posts more entries than the queue holds (the poster keeps the overflow)."""
    w = _warps(gpu_ctx, LAYOUT_REF96)
    n = max(300, -(-2 * w // K))   # strips per layer: 2 K n triangles >= 4 warps
    s = layered_tiling(K, 512, "strips", n=n, wide=8)
    ds = gpu_ctx.upload(s)
    plan = gpu_ctx.convert_plan(ds, 512, LAYOUT_REF96, capacity=K * 512 * 512)
    assert plan.unit_tris >= 2 and not plan.direct_ok
    assert plan.item_max < 32 * 31   # a 32-row block at the wide end of a 32-pixel strip is cut into several items
    cut_everywhere(gpu_ctx, s, 512, LAYOUT_REF96, K * 512 * 512, ds=ds)
    ds.free()


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56, LAYOUT_PLY_STANDARD, LAYOUT_PLY_PBR, LAYOUT_PLY_COMPRESSED],
                         ids=["ref96", "packed56", "ply_standard", "ply_pbr", "ply_compressed"])
def test_cut_every_layout_queue_route(gpu_ctx, layout):
    """Every record layout (strides 96, 56, 248, 76, 48: 16-byte, 8-byte head/tail and 4-byte-piece span copies) on the
    fragment kernel's route, with a few wide strips for split items."""
    s = layered_tiling(K, 128, "strips", n=600, wide=2)
    ds = gpu_ctx.upload(s)
    assert not gpu_ctx.convert_plan(ds, 128, layout, capacity=K * 128 * 128).direct_ok
    cut_everywhere(gpu_ctx, s, 128, layout, K * 128 * 128, ds=ds)
    ds.free()


# ---- route edges -----------------------------------------------------------------------------------------------------
def test_route_edges(gpu_ctx):
    """Triangle ranges of one layered scene that land on the edges of the raster kernel's route predicates: the largest
    single-round count, the first multi-round one, the last late-claim one and the first up-front one.  Each range at a
    mid cap and uncapped against the oracle's conversion of the same range."""
    w = _warps(gpu_ctx, LAYOUT_PACKED56)
    s = layered_tiling(K, 256, "delaunay", n=80 * w // (2 * K), seed=6)
    ds = gpu_ctx.upload(s)
    R, L = 256, LAYOUT_PACKED56

    def plan(c):
        return gpu_ctx.convert_plan(ds, R, L, capacity=K * R * R, triangle_count=c)
    single = 32 * w
    assert not plan(single).multi_round and plan(single + 1).multi_round
    assert plan(single + 1).claim_late
    c = single + 1
    while plan(c).claim_late:
        c += 1
        assert c <= s.triangle_count, "no up-front count in the scene"
    up = c
    assert plan(up).multi_round and plan(up).direct_ok and not plan(up).claim_late and plan(up - 1).claim_late
    for count in (single, single + 1, up - 1, up):
        want, wkeys, total = oracle.convert(s, R, L, flags=FLAG_UNCAPPED, capacity=K * R * R, triangle_count=count)
        order = np.argsort(wkeys)
        for cap in (total // 2 - (total // 2) % 32 + 17, total + 1):
            o = convert_guarded(gpu_ctx, ds, R, L, cap, triangle_count=count)
            assert o.total == total and o.written == min(cap, total) and o.overflow == (total > cap)
            k = o.keys_numpy()
            assert len(np.unique(k)) == len(k)
            pos = _subset(k, wkeys[order])
            assert_records_match(s, L, o.numpy(), k, want[order][pos], k)
    ds.free()


# ---- appended chunks (m2s_convert_host) with the direct path ----------------------------------------------------------
def test_convert_host_chunks_direct_path_capacity(gpu_ctx):
    """m2s_convert_host cuts a mesh of >= 65 536 triangles into 4 appended chunks; here every chunk is a multi-round
    launch with the direct path, whose cap is room = cap - (records of the earlier chunks).  Cuts inside chunk 1, on
    the boundary between chunks 1 and 2 and on the last record; guarded host buffers."""
    L, R = LAYOUT_PACKED56, 256
    w = _warps(gpu_ctx, L)
    n = (4 * (32 * w + 1)) // (2 * K) + 200
    s = layered_tiling(K, R, "delaunay", n=n, seed=8)
    T = s.triangle_count
    assert T >= 4 * (32 * w + 1) and T >= 65536
    per = -(-T // 4)
    ds = gpu_ctx.upload(s)
    for c in range(4):
        p = gpu_ctx.convert_plan(ds, R, L, capacity=K * R * R, first_triangle=c * per, triangle_count=min(per, T - c * per))
        assert p.multi_round and p.direct_ok, c
    ds.free()
    want, wkeys, total = oracle.convert(s, R, L, flags=FLAG_UNCAPPED, capacity=K * R * R)
    assert total == K * R * R
    tri = (wkeys >> np.uint64(24)).astype(np.int64)
    ends = [int(np.count_nonzero(tri < min(T, (c + 1) * per))) for c in range(4)]
    inside = ends[0] + (ends[1] - ends[0]) // 2 + 1
    order = np.argsort(wkeys)
    for cap in (inside, ends[1], total - 1, total):
        out = GuardedHost(cap, STRIDES[L], what="records")
        keys = GuardedHost(cap, 8, np.uint64, what="keys")
        rec, k, res = gpu_ctx.convert_host(s, R, L, flags=FLAG_UNCAPPED, capacity=cap, want_keys=True, out=out.view, keys=keys.view)
        assert res.total == total and res.written == min(cap, total) == len(rec)
        out.check(res.written)
        keys.check(res.written)
        k = np.asarray(k)
        assert len(np.unique(k)) == len(k)
        pos = _subset(k, wkeys[order])
        assert_records_match(s, L, rec, k, want[order][pos], k)


# ---- m2s_convert_file at overflow ------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_convert_file_overflow(gpu_ctx, tmp_path, fmt):
    """A 7-layer .glb at R = 64: the reference's cap (6 R^2 for one mesh) stores 6 of 7 layers.  The file holds exactly
    `cap` rows (header count and length), each a row of the oracle's uncapped file; status M2S_E_CAPACITY."""
    from mesh2splat_b200.gltf import load_glb
    from test_gpu_parity import match_ply_rows
    from util import write_soup_glb
    R, std = 64, 0.65
    glb, ply = tmp_path / "layers.glb", tmp_path / f"layers{fmt}.ply"
    write_soup_glb(str(glb), layered_tiling(K, R, "delaunay", n=300, seed=9).triangles, texture=synth.random_texture(32, 32, 4))
    import ctypes as C
    from mesh2splat_b200._lib import lib
    res = _abi.m2s_result()
    st = lib().m2s_convert_file(gpu_ctx.handle, str(glb).encode(), R, std, fmt, str(ply).encode(), C.byref(res))
    cap = 6 * R * R
    assert st == M2S_E_CAPACITY
    assert res.total == K * R * R and res.cap == cap and res.written == cap
    s = load_glb(str(glb))
    want, _, total = oracle.convert(s, R, LAYOUT_REF96, flags=FLAG_UNCAPPED, capacity=K * R * R)
    assert total == K * R * R
    ref = oracle.ply_bytes(want, fmt, float(np.float32(std) / np.float32(R)))
    got = ply.read_bytes()
    hdr = oracle.ply_header(fmt, cap)
    stride = {0: 248, 1: 76, 2: 48}[fmt]
    assert got[: len(hdr)] == hdr and len(got) == len(hdr) + cap * stride
    whdr = oracle.ply_header(fmt, total)
    match_ply_rows(got[len(hdr):], ref[len(whdr):], fmt, subset=True)


# ---- resolution limits -----------------------------------------------------------------------------------------------
def test_resolution_4097_is_rejected(gpu_ctx):
    from mesh2splat_b200._lib import M2SError
    ds = gpu_ctx.upload(synth.unit_quad())
    with pytest.raises(M2SError) as e:
        gpu_ctx.convert(ds, 4097, flags=FLAG_UNCAPPED, capacity=16)
    assert e.value.status == M2S_E_INVALID
    ds.free()


def test_resolution_4096_bands_match_the_oracle(gpu_ctx):
    """R = 4096, the width the 12-bit key coordinates, TriRec box origins and block rows are packed for: every band of
    512 rows of a Delaunay tiling against the oracle's band, guarded."""
    from util import planar_triangulation
    s = planar_triangulation(30000, seed=7)
    R = 4096
    ds = gpu_ctx.upload(s)
    seen = 0
    for r0 in range(0, R, 512):
        want, wkeys, total = oracle.convert(s, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=512 * R + 64,
                                            row_begin=r0, row_end=r0 + 512)
        assert total == 512 * R
        o = convert_guarded(gpu_ctx, ds, R, LAYOUT_PACKED56, 512 * R + 33, row_begin=r0, row_end=r0 + 512)
        assert o.total == total and o.written == total and not o.overflow
        k = o.keys_numpy()
        rows = (k >> np.uint64(12)) & np.uint64(0xFFF)
        assert rows.min() == r0 and rows.max() == r0 + 511
        assert_records_match(s, LAYOUT_PACKED56, o.numpy(), k, want, wkeys)
        seen += total
    assert seen == R * R
    ds.free()


# ---- prepass bounds --------------------------------------------------------------------------------------------------
def test_prepass_count_zero(gpu_ctx):
    import torch
    from test_gpu_parity import _prepass_cases
    c = list(_prepass_cases())[0]
    q = GuardedDevice(4, _abi.QUAD_BYTES, what="quads")
    d = GuardedDevice(4, 4, torch.float32, what="depths")
    rec = torch.zeros(96, dtype=torch.uint8, device="cuda")
    quads, depths = gpu_ctx.prepass(rec, 0, LAYOUT_REF96, c["view"], c["proj"], c["model"], c["resolution"], c["near_far"],
                                    c["std_dev"], 0, quads=q.view, depths=d.view)
    assert len(quads) == 0 and len(depths) == 0
    q.check(0)
    d.check(0)
