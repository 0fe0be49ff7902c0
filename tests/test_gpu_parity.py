"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same inputs.

All marked gpu; they run on an H100.  They read only files of this repository (golden vectors under tests/golden).
"""
from __future__ import annotations

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import (FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_PLY_COMPRESSED, LAYOUT_PLY_PBR,
                                  LAYOUT_PLY_STANDARD, LAYOUT_REF96, Primitive, Scene)
from util import assert_records_match

pytestmark = pytest.mark.gpu


def run_both(ctx, scene, R, layout=LAYOUT_REF96, **kw):
    ds = ctx.upload(scene)
    out = ctx.convert(ds, R, layout, want_keys=True, **kw)
    okw = {k: v for k, v in kw.items() if k != "capacity"}
    rec, keys, total = oracle.convert(scene, R, layout, want_keys=True, capacity=out.cap if out.cap else 1, **okw)
    ds.free()
    return out, rec, keys, total


def check(ctx, scene, R, layout=LAYOUT_REF96, **kw):
    out, rec, keys, total = run_both(ctx, scene, R, layout, **kw)
    assert out.total == total, f"total {out.total} != oracle {total}"
    assert out.written == len(rec)
    assert_records_match(scene, layout, out.numpy(), out.keys_numpy(), rec, keys)
    return out


# ---- KATs (SURVEY 8c) ------------------------------------------------------------------------------
def test_unit_quad_kat(gpu_ctx):
    """The unit quad at R = 64: 4096 = 2080 + 2016 records, one per pixel centre (the diagonal's belong to triangle 0)."""
    _unit_quad_kat(gpu_ctx, 64)


@pytest.mark.parametrize("R", [1, 2, 3])
def test_unit_quad_kat_smallest_grids(gpu_ctx, R):
    """The same KAT at the smallest resolutions: at R = 1 the single centre lies on the diagonal and belongs to
    triangle 0."""
    _unit_quad_kat(gpu_ctx, R)


def _unit_quad_kat(gpu_ctx, R):
    """R^2 records, one per pixel centre; the R of them on the diagonal belong to triangle 0 (left edge)."""
    s = synth.unit_quad()
    out = check(gpu_ctx, s, R)
    n = R * R
    assert out.total == n and out.written == n and not out.overflow
    rec, keys = out.numpy(), out.keys_numpy()
    tri = (keys >> np.uint64(24)).astype(np.int64)
    n0, n1 = R * (R + 1) // 2, R * (R - 1) // 2
    assert np.bincount(tri, minlength=2).tolist() == [n0, n1]  # diagonal centres belong to triangle 0 (left edge)
    px = (keys & np.uint64(0xfff)).astype(np.float32)
    py = ((keys >> np.uint64(12)) & np.uint64(0xfff)).astype(np.float32)
    assert len(np.unique(keys & np.uint64(0xffffff))) == n and px.max() < R and py.max() < R
    np.testing.assert_allclose(rec["position"][:, 0], (px + 0.5) / R, atol=1e-6)
    np.testing.assert_allclose(rec["position"][:, 1], (py + 0.5) / R, atol=1e-6)
    assert np.all(rec["position"][:, 2] == 0)
    if R == 64:
        np.testing.assert_allclose(rec["scale"], np.tile(np.array([1, 1, 1e-7, 0], np.float32), (n, 1)), rtol=1e-6)
    q0 = np.array([0, 0.9238795, 0.38268343, 0], np.float32)
    q1 = np.array([0.9238795, 0, 0, 0.38268343], np.float32)
    np.testing.assert_allclose(rec["rotation"][tri == 0], np.tile(q0, (n0, 1)), atol=1e-6)
    np.testing.assert_allclose(rec["rotation"][tri == 1], np.tile(q1, (n1, 1)), atol=1e-6)
    assert np.all(rec["color"] == 1.0)
    np.testing.assert_allclose(rec["pbr"], np.tile(np.array([0.1, 0.5, 0, 1], np.float32), (n, 1)))
    np.testing.assert_allclose(rec["normal"], np.tile(np.array([0, 0, 1, 0], np.float32), (n, 1)), atol=1e-6)


def test_unit_quad_textured(gpu_ctx):
    s = synth.unit_quad()
    s.textures = [synth.random_texture(256, 256, 7)]
    s.primitives[0].albedo_texture = 0
    s.primitives[0].base_color_factor = (0.5, 0.25, 1.0, 0.8)
    check(gpu_ctx, s, 64)
    check(gpu_ctx, s, 300)   # magnification
    check(gpu_ctx, s, 16)    # lambda at the level-4 clamp


def test_box_axis_selection(gpu_ctx):
    s = synth.box((1.0, 2.0, 3.0))
    out = check(gpu_ctx, s, 96)
    assert out.total > 0
    s2 = synth.box((2.0, 2.0, 2.0), origin=(-1, -1, -1))  # |nx| == |ny| style ties on a cube
    check(gpu_ctx, s2, 50)


@pytest.mark.parametrize("R", [33, 128, 256])
def test_textured_sphere(gpu_ctx, R):
    tri = synth.displaced_sphere(48, 24, seed=3, amplitude=0.1)
    tex = synth.make_material_textures(256, 11)
    s = Scene(tri, [Primitive(0, len(tri), (0.9, 0.8, 0.7, 1.0), 0, 1, 2)], tex)
    s.compute_bboxes()
    check(gpu_ctx, s, R)


def test_npot_textures_and_repeat(gpu_ctx):
    tri = synth.random_soup(600, seed=5, tri_size=0.3)
    tex = [synth.random_texture(100, 37, 1), synth.random_texture(17, 129, 2), synth.random_texture(1, 1, 3),
           synth.random_texture(5, 3, 4)]
    prims = [Primitive(0, 200, (1, 1, 1, 1), 0, 1, 2), Primitive(200, 200, (0.3, 0.6, 0.9, 0.5), 3, -1, 0),
             Primitive(400, 200, (1, 1, 1, 1), -1, 2, -1)]
    s = Scene(tri, prims, tex)
    s.compute_bboxes(cumulative=True)
    check(gpu_ctx, s, 200, flags=FLAG_UNCAPPED)


def test_multi_primitive_cumulative_bbox(gpu_ctx):
    a = synth.displaced_sphere(24, 12, seed=1, center=(0, 0, 0))
    b = synth.displaced_sphere(24, 12, seed=2, center=(3, 1, 0), radius=0.5)
    c = synth.box((1, 1, 1), origin=(-3, 0, 0)).triangles
    tri = np.concatenate([a, b, c])
    prims = [Primitive(0, len(a)), Primitive(len(a), len(b)), Primitive(len(a) + len(b), len(c))]
    s = Scene(tri, prims, [])
    s.compute_bboxes(cumulative=True)
    check(gpu_ctx, s, 128)
    s.compute_bboxes(cumulative=False)
    check(gpu_ctx, s, 128)


def test_big_triangles_are_deferred_and_split(gpu_ctx):
    s = synth.unit_quad()
    s.textures = synth.make_material_textures(128, 21)
    p = s.primitives[0]
    p.albedo_texture, p.normal_texture, p.metallic_roughness_texture = 0, 1, 2
    out = check(gpu_ctx, s, 512, flags=FLAG_UNCAPPED)
    assert out.total == 512 * 512
    out = check(gpu_ctx, s, 1024, flags=FLAG_UNCAPPED)
    assert out.total == 1024 * 1024


def test_mixed_big_and_small(gpu_ctx):
    room = synth.sponza_standin(tex_size=64, n_prims=12, n_materials=3, target_tris=6000)
    check(gpu_ctx, room, 256, flags=FLAG_UNCAPPED)


def test_degenerate_and_empty(gpu_ctx):
    # zero-area, collinear, NaN and sub-pixel triangles; plus an empty scene
    t = synth.random_soup(64, seed=9, tri_size=0.5)
    v = t.reshape(-1, 3, 12)
    v[0, 1, :3] = v[0, 0, :3]; v[0, 2, :3] = v[0, 0, :3]            # point
    v[1, 2, :3] = 2 * v[1, 1, :3] - v[1, 0, :3]                      # collinear
    v[2, 0, 0] = np.nan
    v[3, :, :3] = v[3, 0, :3] + np.random.default_rng(0).random((3, 3)).astype(np.float32) * 1e-6
    s = Scene(v.reshape(-1, 36))
    s.compute_bboxes()
    s.primitives[0].bbox_min = (0.0, 0.0, 0.0)   # NaN vertex must not poison the box
    s.primitives[0].bbox_max = (1.5, 1.5, 1.5)
    check(gpu_ctx, s, 64)
    empty = Scene(np.zeros((0, 36), np.float32))
    out = gpu_ctx.convert(gpu_ctx.upload(empty), 64)
    assert out.total == 0 and out.written == 0


def test_capacity_overflow(gpu_ctx):
    s = synth.unit_quad()
    ds = gpu_ctx.upload(s)
    out = gpu_ctx.convert(ds, 64, max_gaussians=1000, want_keys=True)
    assert out.overflow and out.total == 4096 and out.written == 1000 and out.cap == 1000
    rec, keys = out.numpy(), out.keys_numpy()
    assert len(np.unique(keys)) == 1000           # 1000 distinct, valid fragments survive
    full, fkeys, _ = oracle.convert(s, 64, want_keys=True)
    lut = {int(k): i for i, k in enumerate(fkeys)}
    idx = np.array([lut[int(k)] for k in keys])
    np.testing.assert_allclose(rec["position"], full["position"][idx], atol=1e-6)
    # reference rule: min(6 R^2 meshCount, 7e6)
    out = gpu_ctx.convert(ds, 64)
    assert out.cap == 6 * 64 * 64
    ds.free()


def test_shard_ranges_partition_the_output(gpu_ctx):
    tri = synth.displaced_sphere(40, 20, seed=8)
    s = Scene(tri, [Primitive(0, len(tri), (1, 1, 1, 1), 0, -1, -1)], [synth.random_texture(64, 64, 3)])
    s.compute_bboxes()
    ds = gpu_ctx.upload(s)
    whole = gpu_ctx.convert(ds, 128, want_keys=True)
    parts, n = [], len(tri)
    cuts = [0, 137, 138, 900, n]
    for a, b in zip(cuts[:-1], cuts[1:]):
        o = gpu_ctx.convert(ds, 128, first_triangle=a, triangle_count=b - a, want_keys=True)
        k = o.keys_numpy()
        assert np.all((k >> np.uint64(24)) >= a) and np.all((k >> np.uint64(24)) < b)
        rec, keys, total = oracle.convert(s, 128, first_triangle=a, triangle_count=b - a)
        assert o.total == total
        assert_records_match(s, LAYOUT_REF96, o.numpy(), k, rec, keys)
        parts.append(k)
    assert np.array_equal(np.sort(np.concatenate(parts)), np.sort(whole.keys_numpy()))
    ds.free()


def test_row_bands_partition_the_output(gpu_ctx):
    """m2s_params.row_begin/row_end: bands of pixel rows of the same triangles (huge and small) partition the
    whole result; each band equals the oracle's band."""
    a = synth.unit_quad()                       # 2 huge triangles (deferred, chunked) ...
    b = synth.displaced_sphere(30, 16, seed=4)  # ... plus ~900 small ones
    tri = np.vstack([a.triangles, b * np.float32(0.45) + np.float32(0.5)])
    s = Scene(tri, [Primitive(0, len(tri), (1, 1, 1, 1), 0, -1, -1)], [synth.random_texture(64, 64, 3)])
    s.compute_bboxes()
    ds = gpu_ctx.upload(s)
    R = 600
    whole = gpu_ctx.convert(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, want_keys=True)
    parts = []
    for r0, r1 in [(0, 1), (1, 77), (77, 300), (300, 599), (599, 0)]:
        o = gpu_ctx.convert(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, want_keys=True, row_begin=r0, row_end=r1)
        k = o.keys_numpy()
        rows = (k >> np.uint64(12)) & np.uint64(0xFFF)
        assert rows.min() >= r0 and rows.max() < (r1 or R)
        rec, keys, total = oracle.convert(s, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, row_begin=r0, row_end=r1)
        assert o.total == total
        assert_records_match(s, LAYOUT_PACKED56, o.numpy(), k, rec, keys)
        parts.append(k)
    assert np.array_equal(np.sort(np.concatenate(parts)), np.sort(whole.keys_numpy()))
    ds.free()


@pytest.mark.parametrize("layout", [LAYOUT_PACKED56, LAYOUT_PLY_STANDARD, LAYOUT_PLY_PBR, LAYOUT_PLY_COMPRESSED])
def test_other_layouts(gpu_ctx, layout):
    tri = synth.displaced_sphere(32, 16, seed=4)
    s = Scene(tri, [Primitive(0, len(tri), (0.9, 1.0, 0.8, 0.9), 0, 1, 2)], synth.make_material_textures(128, 5))
    s.compute_bboxes()
    check(gpu_ctx, s, 96, layout, gaussian_std=0.65)
    check(gpu_ctx, s, 64, layout, gaussian_std=1.3)


def test_mip_chain_bit_exact(gpu_ctx):
    imgs = [synth.random_texture(256, 256, 1), synth.random_texture(100, 37, 2), synth.random_texture(3, 1, 3),
            synth.random_texture(1, 1, 4), synth.random_texture(33, 64, 5)]
    s = synth.unit_quad()
    s.textures = imgs
    ds = gpu_ctx.upload(s)
    for t, img in enumerate(imgs):
        n = oracle.mip_count(img.shape[1], img.shape[0])
        for l in range(n):
            assert np.array_equal(ds.read_mip(t, l), oracle.mip_level(img, l)), f"texture {t} level {l}"
    ds.free()


def test_convert_host_matches_resident(gpu_ctx):
    tri = synth.displaced_sphere(32, 16, seed=6)
    s = Scene(tri, [Primitive(0, len(tri), (1, 1, 1, 1), 0, 1, 2)], synth.make_material_textures(64, 9))
    s.compute_bboxes()
    rec, keys, res = gpu_ctx.convert_host(s, 100, want_keys=True)
    want, wkeys, total = oracle.convert(s, 100)
    assert res.total == total
    assert_records_match(s, LAYOUT_REF96, rec, keys, want, wkeys)


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_convert_host_pipelined_chunks(gpu_ctx, layout):
    """Meshes of >= 16384 triangles go through m2s_convert_host in appended triangle chunks (H2D, kernels and
    D2H overlapped): the result must be the same multiset as the oracle's single pass, keys included."""
    tri = synth.displaced_sphere(101, 83, seed=11, amplitude=0.07)  # 16 766 triangles, odd chunk record offsets
    s = Scene(tri, [Primitive(0, len(tri), (0.9, 0.8, 1.0, 1.0), 0, 1, 2)], synth.make_material_textures(256, 5))
    s.compute_bboxes()
    rec, keys, res = gpu_ctx.convert_host(s, 200, layout, flags=FLAG_UNCAPPED, want_keys=True)
    want, wkeys, total = oracle.convert(s, 200, layout, flags=FLAG_UNCAPPED)
    assert res.total == total and res.written == total
    assert_records_match(s, layout, rec, keys, want, wkeys)


def test_convert_host_pipelined_chunks_through_the_direct_path(gpu_ctx):
    """A mesh big enough that every chunk of the host pipeline is a launch in which the warps take several units each
    (4 chunks of 90 000 triangles; asserted from the launch plan of each chunk's range): the raster kernel shades the
    small triangles itself (direct path) and appends after the earlier chunks' records.  Same multiset of records and
    keys as one device-resident conversion, bit for bit."""
    tri = synth.displaced_sphere(600, 300, seed=4, amplitude=0.05)   # 360 000 triangles
    s = Scene(tri, [Primitive(0, len(tri), (1.0, 0.8, 0.9, 1.0), 0, -1, -1)], synth.make_material_textures(256, 8)[:1])
    s.compute_bboxes()
    R = 300
    ds = gpu_ctx.upload(s)
    per = -(-s.triangle_count // 4)
    for c in range(4):
        p = gpu_ctx.convert_plan(ds, R, LAYOUT_PACKED56, capacity=6 * R * R, flags=FLAG_UNCAPPED, first_triangle=c * per,
                                 triangle_count=min(per, s.triangle_count - c * per))
        assert p.multi_round and p.direct_ok, c
    ds.free()
    rec, keys, res = gpu_ctx.convert_host(s, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, want_keys=True)
    ds = gpu_ctx.upload(s)
    whole = gpu_ctx.convert(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=6 * R * R, want_keys=True)
    ds.free()
    assert res.total == whole.total == res.written and res.total > 100_000
    a, ak = np.ascontiguousarray(rec), np.asarray(keys)
    b, bk = whole.numpy(), whole.keys_numpy()
    oa, ob = np.argsort(ak, kind="stable"), np.argsort(bk, kind="stable")
    assert np.array_equal(ak[oa], bk[ob]) and len(np.unique(ak)) == len(ak)
    assert a[oa].tobytes() == b[ob].tobytes()


def test_convert_host_pipelined_capacity(gpu_ctx):
    """The cap applies to the running index across chunks: exactly `cap` records come back, the total keeps
    counting (converterFS.glsl:46-51), status M2S_E_CAPACITY."""
    tri = synth.displaced_sphere(101, 83, seed=11, amplitude=0.07)
    s = Scene(tri, [Primitive(0, len(tri), (1, 1, 1, 1), 0, 1, 2)], synth.make_material_textures(64, 5))
    s.compute_bboxes()
    _, _, full = gpu_ctx.convert_host(s, 160, LAYOUT_PACKED56, flags=FLAG_UNCAPPED)
    cap = full.total * 5 // 8 + 1  # ends inside the second chunk
    rec, keys, res = gpu_ctx.convert_host(s, 160, LAYOUT_PACKED56, max_gaussians=cap, want_keys=True)
    assert res.total == full.total and res.written == cap and len(rec) == cap
    assert len(np.unique(keys)) == cap  # every stored record is a distinct fragment
    want, wkeys, _ = oracle.convert(s, 160, LAYOUT_PACKED56, flags=FLAG_UNCAPPED)
    order = np.argsort(wkeys)
    pos = np.minimum(np.searchsorted(wkeys[order], keys), len(wkeys) - 1)
    assert np.array_equal(wkeys[order][pos], keys)  # a subset of the uncapped result
    assert_records_match(s, LAYOUT_PACKED56, rec, keys, want[order][pos], keys)


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_convert_file_glb_to_ply(gpu_ctx, tmp_path, fmt):
    """m2s_convert_file = loadModel -> ConversionPass::execute -> exportPly: the file must be the oracle's file
    (same header bytes, same rows as a multiset; rows are ordered by atomic arrival in both)."""
    from util import write_quad_glb
    from mesh2splat_b200.gltf import load_glb
    glb, ply = tmp_path / "m.glb", tmp_path / f"m{fmt}.ply"
    write_quad_glb(str(glb), two_prims=True)
    R, std = 96, 0.65
    res = gpu_ctx.convert_file(str(glb), R, str(ply), std, fmt)
    s = load_glb(str(glb))
    want, wkeys, total = oracle.convert(s, R, LAYOUT_REF96)
    assert res.total == total and res.written == len(want) and total > 1000
    ref = oracle.ply_bytes(want, fmt, float(np.float32(std) / np.float32(R)))
    got = ply.read_bytes()
    hdr = oracle.ply_header(fmt, len(want))
    assert got[: len(hdr)] == hdr and len(got) == len(ref)
    match_ply_rows(got[len(hdr):], ref[len(hdr):], fmt)


def match_ply_rows(got_body: bytes, want_body: bytes, fmt: int, subset: bool = False) -> None:
    """.ply bodies as multisets of rows (both are in atomic arrival order): every row of `got_body` must be a row of
    `want_body`, equal within the encoding's tolerances; with subset = False the two have the same rows."""
    stride = {0: 248, 1: 76, 2: 48}[fmt]
    g = np.frombuffer(got_body, np.uint8).reshape(-1, stride)
    w = np.frombuffer(want_body, np.uint8).reshape(-1, stride)
    assert subset or len(g) == len(w)
    # identify rows by position (first 12 bytes: three floats, distinct per fragment within a primitive plane)
    gp, wp = g[:, :12].copy().view(np.float32), w[:, :12].copy().view(np.float32)
    go, wo = np.lexsort(np.round(gp * 4096).T), np.lexsort(np.round(wp * 4096).T)
    if subset:   # the rows of `want` with the same rounded position, one per row of `got`
        gk = np.round(gp.astype(np.float64) * 4096).astype(np.int64)
        wk = np.round(wp.astype(np.float64) * 4096).astype(np.int64)
        wmap = {tuple(r): i for i, r in enumerate(wk)}
        assert len(wmap) == len(wk), "positions do not identify the rows"
        idx = np.array([wmap.get(tuple(r), -1) for r in gk], np.int64)
        assert (idx >= 0).all(), f"{np.count_nonzero(idx < 0)} rows are not rows of the expected file"
        assert len(np.unique(idx)) == len(idx), "a row is written twice"
        go, wo = np.arange(len(g)), idx
    assert np.allclose(gp[go], wp[wo], atol=2e-5)
    G, W = g[go], w[wo]
    if fmt == 2:  # pos f32x3 | rgba u8x4 | quat f32x4 | log-scale f32x3 | octahedral normal u8x2 | roughness, metallic u8
        fcols = np.r_[0:12, 16:44]
        bcols = np.r_[12:16, 44:48]
        assert np.abs(G[:, bcols].astype(np.int16) - W[:, bcols].astype(np.int16)).max() <= 1  # one count of rounding slack
    else:
        fcols = np.r_[0:stride]
    gf, wf = np.ascontiguousarray(G[:, fcols]).view(np.float32), np.ascontiguousarray(W[:, fcols]).view(np.float32)
    fin = np.isfinite(wf)
    assert np.array_equal(fin, np.isfinite(gf))
    assert np.allclose(gf[fin], wf[fin], rtol=2e-4, atol=2e-4)
    assert np.array_equal(gf[~fin], wf[~fin])  # opacity = +inf for alpha = 1


def test_watertight_tiling_full_size(gpu_ctx):
    """The watertight tiling at R = 2048 (4 194 304 pixel centres); see _watertight_tiling."""
    _watertight_tiling(gpu_ctx, 2048)


def test_watertight_tiling_max_resolution(gpu_ctx):
    """The watertight tiling at the largest grid, R = 4096: the width the 12-bit key coordinates, box origins and block
    rows are packed for."""
    _watertight_tiling(gpu_ctx, 4096)


def _watertight_tiling(gpu_ctx, R):
    """Size-independent coverage property: a Delaunay tiling of the unit square (~60 k triangles of every shape, sub-pixel slivers to
    100-pixel triangles) emits each of the R^2 pixel centres exactly once, into guarded buffers, and a second run
    produces bit-identical records (as a set).  Compared on the device."""
    import torch
    from util import GuardedDevice, planar_triangulation
    s = planar_triangulation(30000, seed=7)
    ds = gpu_ctx.upload(s)
    n = R * R

    def run():
        out, keys = GuardedDevice(n + 64, 56, what="records"), GuardedDevice(n + 64, 8, torch.int64, what="keys")
        o = gpu_ctx.convert(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=n + 64, out=out.view, keys=keys.view, want_keys=True)
        assert o.total == n and o.written == n
        out.check(n)
        keys.check(n)
        k, order = torch.sort(keys.view[:n])
        return k, out.view[: n * 56].view(n, 56)[order]
    ka, ra = run()
    assert torch.unique(ka & 0xFFFFFF).numel() == n
    assert bool(((ka & 0xFFF) < R).all()) and bool((((ka >> 12) & 0xFFF) < R).all())
    kb, rb = run()
    assert torch.equal(ka, kb)
    assert torch.equal(ra, rb)
    ds.free()


def test_repeated_launches_rearm_the_scheduler(gpu_ctx):
    s = synth.unit_quad()
    ds = gpu_ctx.upload(s)
    for R in (64, 700, 32, 64, 513):
        out = gpu_ctx.convert(ds, R, flags=FLAG_UNCAPPED)
        assert out.total == R * R
    ds.free()


def test_reference_shaped_interface(tmp_path):
    from mesh2splat_b200.api import ConversionPass, RenderContext, SceneManager
    rc = RenderContext(0)
    sm = SceneManager(rc)
    s = synth.unit_quad()
    assert sm.setScene(s)
    rc.resolutionTarget = 64
    p = ConversionPass()
    p.setIsEnabled(True)
    assert p.isEnabled()
    p.execute(rc)
    assert rc.numberOfGaussians == 4096
    path = tmp_path / "quad.ply"
    sm.exportPly(str(path), 0)
    data = path.read_bytes()
    want_rec, _, _ = oracle.convert(s, 64, want_keys=False)
    hdr = oracle.ply_header(0, 4096)
    assert data[: len(hdr)] == hdr and len(data) == len(hdr) + 4096 * 248
    body = np.frombuffer(data[len(hdr):], np.float32).reshape(4096, 62)
    np.testing.assert_allclose(body[:, 55], np.log(np.float32(1.0) * np.float32(0.65) / np.float32(64)), rtol=1e-6)
    assert np.all(np.isposinf(body[:, 54]))  # alpha == 1 -> opacity = +inf (utils.hpp:270)
    rc.ctx.close()


# ---- full-size properties (BASELINE config 2 stand-in) -------------------------------------------------
def test_helmet_standin_density_512_full_parity(gpu_ctx):
    """BASELINE config 2 exactly as bench.py runs it: 70 074 triangles, three 2048^2 maps, density 512 — every record of
    both layouts against the oracle.  Premise (asserted from the launch plan): the PACKED56 launch gives the raster warps
    more than one unit each but fewer than three, so it takes the direct path with the late claim."""
    s = synth.helmet_standin(2048)
    ds = gpu_ctx.upload(s)
    plan = gpu_ctx.convert_plan(ds, 512, LAYOUT_PACKED56)
    ds.free()
    assert plan.multi_round and plan.direct_ok and plan.claim_late
    out = check(gpu_ctx, s, 512, LAYOUT_REF96)
    assert 0.4e6 < out.total < 1.2e6
    out2 = check(gpu_ctx, s, 512, LAYOUT_PACKED56)
    assert out2.total == out.total


# ---- CUDA per-triangle stage vs the REFERENCE's geometry shader (committed golden vectors) -------------
def test_cuda_matches_reference_gs_golden_vectors(gpu_ctx):
    """tests/golden/ref_shader_vectors.npz holds converterGS.glsl's own outputs (made by
    tests/golden/make_golden.py from /root/reference).  One primitive per golden triangle with the golden
    bbox; every gaussian the CUDA path emits for it must carry the reference's Scale and Quaternion bit for
    bit, and the number of gaussians must equal the oracle's coverage for gl_Position = reference."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_shader_vectors.npz"))
    tris = g["gs_tris"]
    n = len(tris)
    prims = [Primitive(i, 1, (1, 1, 1, 1), -1, -1, -1, tuple(float(v) for v in g["gs_bmin"][i]),
                       tuple(float(v) for v in g["gs_bmax"][i])) for i in range(n)]
    s = Scene(tris, prims, [])
    R = 48
    out, rec, keys, total = run_both(gpu_ctx, s, R, LAYOUT_REF96, flags=FLAG_UNCAPPED, capacity=n * R * R)
    assert out.total == total
    got, gk = out.numpy(), out.keys_numpy()
    tri = (gk >> np.uint64(24)).astype(np.int64)
    checked = 0
    for i in np.unique(tri):
        m = tri == i
        sc = got["scale"][m][:, :3]
        qt = got["rotation"][m]
        assert np.array_equal(sc.view(np.uint32), np.tile(g["gs_scale"][i].view(np.uint32), (m.sum(), 1))), f"Scale, triangle {i}"
        assert np.array_equal(qt.view(np.uint32), np.tile(g["gs_quat"][i].view(np.uint32), (m.sum(), 1))), f"Quaternion, triangle {i}"
        checked += 1
    assert checked >= n // 2, f"only {checked} of {n} golden triangles produced fragments"
    assert_records_match(s, LAYOUT_REF96, got, gk, rec, keys)


# ---- the other BASELINE configurations at full size: size-independent properties ------------------------
def _keys_unique_and_in_range(keys, scene, R):
    assert len(np.unique(keys)) == len(keys)
    tri = keys >> np.uint64(24)
    assert tri.max(initial=0) < scene.triangle_count
    assert ((keys & np.uint64(0xfff)) < R).all() and (((keys >> np.uint64(12)) & np.uint64(0xfff)) < R).all()


def test_config3_sponza_standin_reference_cap_and_uncapped(gpu_ctx):
    """BASELINE config 3: multi-material, R=1024.  With the reference rule the 7 M cap is hit (count keeps
    counting); uncapped, the total equals the oracle's and every fragment identity is unique."""
    s = synth.sponza_standin(256)       # same geometry/primitives as the bench stand-in, smaller textures
    ds = gpu_ctx.upload(s)
    capped = gpu_ctx.convert(ds, 1024, LAYOUT_PACKED56)
    assert capped.cap == 7_000_000
    prep = oracle.Prepared(s)
    _, total, _ = prep.convert(1024, LAYOUT_PACKED56, capacity=1)
    assert capped.total == total
    assert capped.overflow == (total > 7_000_000) and capped.written == min(total, 7_000_000)
    un = gpu_ctx.convert(ds, 1024, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=total + 16, want_keys=True)
    assert un.total == total and un.written == total and not un.overflow
    _keys_unique_and_in_range(un.keys_numpy(), s, 1024)
    # every primitive contributes exactly what the oracle says (per-primitive coverage, bit-exact)
    tri = (un.keys_numpy() >> np.uint64(24)).astype(np.int64)
    firsts = np.array([p.first_triangle for p in s.primitives] + [s.triangle_count])
    got = np.histogram(tri, bins=firsts)[0]
    orec, okeys, _ = oracle.convert(s, 1024, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=total + 16)
    want = np.histogram((okeys >> np.uint64(24)).astype(np.int64), bins=firsts)[0]
    assert np.array_equal(got, want)
    assert np.array_equal(np.sort(un.keys_numpy()), np.sort(okeys))
    assert_records_match(s, LAYOUT_PACKED56, un.numpy(), un.keys_numpy(), orec, okeys)  # every record value, not only the keys
    # the capped run stores exactly 7 M distinct fragments of the uncapped set (which ones is atomic-order dependent)
    if capped.overflow:
        ck = gpu_ctx.convert(ds, 1024, LAYOUT_PACKED56, want_keys=True).keys_numpy()
        assert len(ck) == 7_000_000 and len(np.unique(ck)) == len(ck) and np.isin(ck, okeys).all()
    ds.free()


def test_config4_million_triangle_sphere(gpu_ctx):
    """BASELINE config 4: 1 000 000 triangles, R=256 (most triangles are sub-pixel).  Total and the whole
    fragment-identity set equal the oracle's; 8 contiguous shards partition it."""
    s = synth.sphere_1m(256)
    ds = gpu_ctx.upload(s)
    out = gpu_ctx.convert(ds, 256, LAYOUT_PACKED56, want_keys=True)
    orec, okeys, total = oracle.convert(s, 256, LAYOUT_PACKED56)
    assert out.total == total and 50_000 < total < 400_000
    assert np.array_equal(np.sort(out.keys_numpy()), np.sort(okeys))
    assert_records_match(s, LAYOUT_PACKED56, out.numpy(), out.keys_numpy(), orec, okeys)
    from mesh2splat_b200.shard import plan_shards
    parts = []
    for first, count in plan_shards(s.triangle_count, 8):
        o = gpu_ctx.convert(ds, 256, LAYOUT_PACKED56, first_triangle=first, triangle_count=count, want_keys=True)
        parts.append(o.keys_numpy())
    assert np.array_equal(np.sort(np.concatenate(parts)), np.sort(okeys))
    ds.free()


def test_direct_path_and_queue_path_write_the_same_records(gpu_ctx):
    """PACKED56 has two routes for the small triangles of a light work unit: in a launch where the warps take several
    units each (here: 200 000 triangles in one call) the raster kernel shades them itself (direct path); with at most one
    unit per warp (here: the same triangles in ranges of 25 000) they are queued for the fragment kernel.  The launch
    plan asserts both premises.  Both run the
    same shading code on the same per-triangle records: the two results must be the same multiset of records, bit for
    bit, with the same fragment identities — and the whole thing must agree with the oracle."""
    tri = synth.displaced_sphere(500, 200, seed=11, amplitude=0.04)
    s = Scene(tri, [Primitive(0, len(tri), (0.9, 1.0, 0.8, 1.0), 0, -1, -1)], synth.make_material_textures(256, 6)[:1])
    s.compute_bboxes()
    R = 384
    ds = gpu_ctx.upload(s)
    plan = gpu_ctx.convert_plan(ds, R, LAYOUT_PACKED56, capacity=6 * R * R, flags=FLAG_UNCAPPED)
    assert plan.multi_round and plan.direct_ok
    whole = gpu_ctx.convert(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=6 * R * R, want_keys=True)
    a, ak = whole.numpy().copy(), whole.keys_numpy().copy()
    parts, pk = [], []
    step = 25_000
    for first in range(0, s.triangle_count, step):
        assert not gpu_ctx.convert_plan(ds, R, LAYOUT_PACKED56, capacity=6 * R * R, flags=FLAG_UNCAPPED, first_triangle=first,
                                        triangle_count=min(step, s.triangle_count - first)).multi_round
        o = gpu_ctx.convert(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=6 * R * R, want_keys=True, first_triangle=first,
                            triangle_count=min(step, s.triangle_count - first))
        parts.append(o.numpy().copy()); pk.append(o.keys_numpy().copy())
    ds.free()
    b, bk = np.concatenate(parts), np.concatenate(pk)
    assert len(a) == len(b) > 100_000
    oa, ob = np.argsort(ak, kind="stable"), np.argsort(bk, kind="stable")
    assert np.array_equal(ak[oa], bk[ob])
    assert a[oa].tobytes() == b[ob].tobytes(), "direct path and fragment-kernel path disagree"
    rec, keys, total = oracle.convert(s, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=6 * R * R, want_keys=True)
    assert total == len(a)
    assert_records_match(s, LAYOUT_PACKED56, a, ak, rec, keys)


# ---- BASELINE config 5: density sweep on the DamagedHelmet stand-in ---------------------------------------------
@pytest.mark.parametrize("R", [64, 128, 256, 512, 1024, 2048])
def test_config5_damaged_helmet_density_sweep(gpu_ctx, R):
    """BASELINE.json configs[4]: density 64 -> 2048 on the DamagedHelmet stand-in (15 488 triangles, three 2048^2 maps),
    the scene bench.py --workload damaged_helmet_standin runs.  Every record against the oracle at every density
    (R = 2048: 9.8 M gaussians, 24 x the box of a small triangle — the row-span path), plus the size-independent
    properties: fragment identities unique and inside the R x R grid, and the reference cap (7 M) applied to the
    running index."""
    s = _dh_scene()
    out = check(gpu_ctx, s, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, capacity=6 * R * R)
    _keys_unique_and_in_range(out.keys_numpy(), s, R)
    assert 2.0 * R * R < out.total < 2.8 * R * R
    if R == 2048:  # the reference's own capacity rule clamps this one
        ds = gpu_ctx.upload(s)
        capped = gpu_ctx.convert(ds, R, LAYOUT_PACKED56, want_keys=True)
        assert capped.cap == 7_000_000 and capped.overflow and capped.total == out.total and capped.written == 7_000_000
        ck = capped.keys_numpy()
        assert len(np.unique(ck)) == 7_000_000 and np.isin(ck, out.keys_numpy()).all()
        ds.free()


_DH = {}


def _dh_scene():
    if "s" not in _DH:
        _DH["s"] = synth.damaged_helmet_standin(2048)
    return _DH["s"]


# ---- shard upload: triangles of a range + only the texture rows they sample ---------------------------------------
@pytest.mark.parametrize("tex_hw", [(256, 256), (300, 64), (37, 100)])
def test_upload_range_brings_every_texel_the_shard_samples(gpu_ctx, tex_hw):
    """m2s_scene_upload_range copies a triangle range and, per 16-row group, only the texture rows (and their mip rows)
    that range can sample.  Converting each of 5 shards from its own partial upload must give exactly the records of the
    oracle's single pass — a missing row group would show up as a wrong colour.  Non-power-of-two and tall textures
    exercise the group/mip-row arithmetic, the REPEAT wrap at v = 0/1 the wrap-around groups."""
    h, w = tex_hw
    tri = synth.displaced_sphere(48, 40, seed=21, amplitude=0.06)
    tex = [synth.random_texture(w, h, 31), synth.random_texture(w, h, 32), synth.random_texture(w, h, 33)]
    s = Scene(tri, [Primitive(0, len(tri), (1.0, 0.9, 0.8, 1.0), 0, 1, 2)], tex)
    s.compute_bboxes()
    R = 160
    want, wkeys, total = oracle.convert(s, R, LAYOUT_REF96, flags=FLAG_UNCAPPED, capacity=6 * R * R)
    from mesh2splat_b200.shard import plan_shards
    recs, keys, h2d = [], [], []
    for first, count in plan_shards(s.triangle_count, 5):
        ds = gpu_ctx.upload_range(s, LAYOUT_REF96, first, count)
        h2d.append(ds.h2d_bytes())
        o = gpu_ctx.convert(ds, R, LAYOUT_REF96, flags=FLAG_UNCAPPED, capacity=6 * R * R, first_triangle=first,
                            triangle_count=count, want_keys=True)
        recs.append(o.numpy().copy()); keys.append(o.keys_numpy().copy())
        ds.free()
    got, gk = np.concatenate(recs), np.concatenate(keys)
    assert len(got) == total
    assert_records_match(s, LAYOUT_REF96, got, gk, want, wkeys)
    if h >= 256:  # the sphere's rows are latitude bands: a shard needs a fraction of the image
        full = s.triangles.nbytes + sum(t.nbytes for t in tex)
        assert max(h2d) < 0.75 * full, (h2d, full)


# ---- the viewer prepass (SURVEY 8 f-4): GaussiansPrepass::execute + gaussianSplattingPrepassCS.glsl ------------------
def _prepass_cases():
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_prepass_vectors.npz"))
    for i in range(int(g["ncases"])):
        p = g[f"params{i}"]
        yield dict(gaussians=g[f"g{i}"], view=g[f"view{i}"], proj=g[f"proj{i}"], model=g[f"model{i}"], resolution=(float(p[0]), float(p[1])),
                   near_far=(float(p[2]), float(p[3])), std_dev=float(p[4]), render_mode=int(p[5]), fmt=int(p[6]), quads=g[f"quads{i}"], depths=g[f"depths{i}"])


def _as_packed56(g24: np.ndarray) -> np.ndarray:
    """GaussianVertex values -> the PACKED56 record that decodes to them (what savePlyVector + loadPlyFile do to a gaussian)."""
    f = np.zeros((len(g24), 14), np.float32)
    f[:, 0:3] = g24[:, 0:3]; f[:, 3:7] = g24[:, 16:20]
    f[:, 7:10] = np.log(g24[:, 8:11].astype(np.float64)).astype(np.float32)
    f[:, 10:13] = ((g24[:, 4:7].astype(np.float64) - 0.5) / 0.28209479177387814).astype(np.float32)
    a = np.clip(g24[:, 7].astype(np.float64), 1e-6, 1 - 1e-6)
    f[:, 13] = np.log(a / (1 - a)).astype(np.float32)
    return f


def test_prepass_matches_reference_shader_golden_vectors(gpu_ctx):
    """The CUDA prepass against gaussianSplattingPrepassCS.glsl's own outputs (tests/golden/ref_prepass_vectors.npz, made
    from /root/reference by tests/golden/make_golden_prepass.py): the same survivors, values as util.assert_prepass_match
    states.  u_format 0 cases go in as REF96 records, u_format 1 cases as the PACKED56 records that decode to them."""
    import torch
    from util import assert_prepass_match
    for c in _prepass_cases():
        if c["fmt"] == 0:
            rec, layout, want_q, want_d = c["gaussians"], LAYOUT_REF96, c["quads"], c["depths"]
        else:   # the record round trip (log / exp, logit / sigmoid) is part of this input: the expected values come from the oracle on the decoded records
            rec, layout = _as_packed56(c["gaussians"]), LAYOUT_PACKED56
            want_q, want_d = oracle.prepass(oracle.packed56_as_gaussian_vertex(rec), c["view"], c["proj"], c["model"], c["resolution"], c["near_far"],
                                            c["std_dev"], c["render_mode"], 1, 0)
            assert len(want_q) == len(c["quads"])   # ... and are the reference's survivors
        d = torch.from_numpy(np.ascontiguousarray(rec).view(np.uint8).reshape(-1)).cuda()
        quads, depths = gpu_ctx.prepass(d, len(rec), layout, c["view"], c["proj"], c["model"], c["resolution"], c["near_far"], c["std_dev"], c["render_mode"])
        assert_prepass_match(quads, depths, want_q, want_d, c["resolution"], ordered=False)


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_prepass_on_the_conversion_output(gpu_ctx, layout):
    """convert -> prepass without leaving the device, both record layouts, against the oracle's prepass on the same records
    (100 k gaussians: every warp-append and the span copies are exercised; three render modes)."""
    from util import assert_prepass_match
    tri = synth.displaced_sphere(96, 48, seed=5)
    s = Scene(tri, [Primitive(0, len(tri), (1.0, 0.9, 0.8, 0.7), 0, 1, 2)], synth.make_material_textures(128, 9))
    s.compute_bboxes()
    ds = gpu_ctx.upload(s)
    R = 200
    out = gpu_ctx.convert(ds, R, layout, flags=FLAG_UNCAPPED, capacity=6 * R * R)
    ds.free()
    rec = out.numpy()
    raw = np.ascontiguousarray(rec).view(np.uint8).reshape(len(rec), -1)
    g24 = raw.view(np.float32).reshape(len(rec), 24) if layout == LAYOUT_REF96 else oracle.packed56_as_gaussian_vertex(raw)
    cases = list(_prepass_cases())
    for mode in (0, 1, 2):
        c = cases[1]   # a rotated, scaled model matrix and an oblique camera
        std = 0.65 / R
        quads, depths = gpu_ctx.prepass(out.data, out.written, layout, c["view"], c["proj"], c["model"], c["resolution"], c["near_far"], std, mode)
        want_q, want_d = oracle.prepass(g24, c["view"], c["proj"], c["model"], c["resolution"], c["near_far"], std, mode, 0 if layout == LAYOUT_REF96 else 1, 0)
        assert 0.2 * len(g24) < len(want_q) <= len(g24)
        assert_prepass_match(quads, depths, want_q, want_d, c["resolution"], ordered=False)


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_prepass_large_input_path(gpu_ctx, layout):
    """From 2 M (2 << 20) records on the kernel fetches a warp's records as one contiguous span through shared memory
    (another code path than the small-input one): 2 100 001 records (an odd count: the PACKED56 span of the last warp
    ends on an 8-byte tail) against the oracle, with guarded quad and depth buffers."""
    _prepass_bounds(gpu_ctx, layout, 2_100_001)


@pytest.mark.parametrize("count", [1, 31, 33, (1 << 21) - 1, 1 << 21])
@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_prepass_counts_around_the_thresholds(gpu_ctx, layout, count):
    """Counts around a warp and around the staged-fetch threshold (2 << 20: the last count of the small-input path and
    the first of the staged one) against the oracle, with guarded quad and depth buffers."""
    _prepass_bounds(gpu_ctx, layout, count)


def _prepass_bounds(gpu_ctx, layout, count):
    """`count` records against the oracle; guarded quads and depths: nothing is written beyond the survivors and no
    survivor's slot is left unwritten."""
    import torch
    from util import GuardedDevice, assert_prepass_match
    c = list(_prepass_cases())[0 if layout == LAYOUT_REF96 else 3]   # gaussians whose scales suit the format (u_format 1: no std_dev factor)
    base = c["gaussians"]
    reps = count // len(base) + 1
    g = np.tile(base, (reps, 1))[:count].copy()
    g[:, 0] += (np.arange(len(g)) // len(base)).astype(np.float32) * np.float32(2e-4)   # distinct positions per copy
    rec = g if layout == LAYOUT_REF96 else _as_packed56(g)
    g24 = g if layout == LAYOUT_REF96 else oracle.packed56_as_gaussian_vertex(rec)
    d = torch.from_numpy(np.ascontiguousarray(rec).view(np.uint8).reshape(-1)).cuda()
    fmt = 0 if layout == LAYOUT_REF96 else 1
    gq, gd = GuardedDevice(count, _abi.QUAD_BYTES, what="quads"), GuardedDevice(count, 4, torch.float32, what="depths")
    quads, depths = gpu_ctx.prepass(d, len(rec), layout, c["view"], c["proj"], c["model"], c["resolution"], c["near_far"], c["std_dev"], 0,
                                    quads=gq.view, depths=gd.view)
    gq.check(len(quads))
    gd.check(len(depths))
    want_q, want_d = oracle.prepass(g24, c["view"], c["proj"], c["model"], c["resolution"], c["near_far"], c["std_dev"], 0, fmt, 0)
    if count > 1_000_000:
        assert len(want_q) > 1_000_000
    assert_prepass_match(quads, depths, want_q, want_d, c["resolution"], ordered=False)
