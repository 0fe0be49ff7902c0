"""The viewer's mesh depth pre-pass and the prepass's mesh depth test on the GPU (row f-9: m2s_mesh_depth,
m2s_prepass_mesh_depth).  The map is compared bit for bit with the C restatement (oracle/m2s_depth_oracle.c) through a
guarded buffer, so a texel written outside the map or never written fails; the prepass with the test is compared with
orc_prepass applied to the records the oracle's depth-test mask keeps."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_REF96
from mesh2splat_b200._lib import M2SError, check, lib
import oracle
from oracle import depth, light
from util import GuardedDevice, assert_prepass_match

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

NAMES = [t for t, _ in _abi.GBUFFER_TARGETS]
EYE = np.eye(4, dtype=np.float32)


def _camera(eye, target, aspect, near=0.01, far=100.0, fov=45.0):
    V = column_major(look_at(np.array(eye, np.float64), np.array(target, np.float64), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(fov), aspect, near, far))
    return V, P


OUTSIDE = ((0.0, 0.5, 3.2), (0.0, 0.0, 0.0))   # the chain test's camera: the whole helmet stand-in in view
INSIDE = ((0.05, 0.02, -0.03), (1.0, 0.3, 0.2))  # inside the displaced sphere: triangles on every side and behind


def _depth(gpu_ctx, ds, V, P, M, w, h, max_pairs=None):
    """The map through a guarded buffer; returns (map, drawn, pairs)."""
    import torch
    g = GuardedDevice(w * h, 4, what="depth map")
    m, drawn, pairs = gpu_ctx.mesh_depth(ds, V, P, M, w, h, max_pairs=max_pairs, depth=g.view.view(torch.float32))
    g.check(w * h)
    return m, drawn, pairs


def _check(gpu_ctx, scene, ds, V, P, M, w, h, **kw):
    m, drawn, pairs = _depth(gpu_ctx, ds, V, P, M, w, h, **kw)
    pvm = depth.pvm(V, P, M)
    want = depth.mesh_depth(scene, pvm, w, h, n=drawn)
    assert np.array_equal(m.view(np.uint32), want.view(np.uint32)), f"{int((m != want).sum())} texels differ"
    return m, drawn, pairs


@pytest.fixture(scope="module")
def helmet(gpu_ctx):
    scene = synth.helmet_standin(64)
    ds = gpu_ctx.upload(scene)
    yield scene, ds
    ds.free()


@pytest.mark.parametrize("cam", ["outside", "inside"])
@pytest.mark.parametrize("wh", [(1, 1), (17, 15), (1920, 1080)])
def test_bench_scene_outside_and_inside(gpu_ctx, helmet, cam, wh):
    scene, ds = helmet
    eye, tgt = OUTSIDE if cam == "outside" else INSIDE
    V, P = _camera(eye, tgt, wh[0] / wh[1])
    m, drawn, pairs = _check(gpu_ctx, scene, ds, V, P, EYE, *wh)
    assert drawn == scene.triangle_count
    if wh[0] > 1 and cam == "inside":
        assert (m < 1.0).all()   # surrounded by the mesh: every texel covered
    if wh[0] > 1:
        assert (m < 1.0).any() and pairs > 0


def test_size_4096_rotated_model_and_4097_rejected(gpu_ctx, helmet):
    scene, ds = helmet
    V, P = _camera(OUTSIDE[0], OUTSIDE[1], 1.0)
    c, s = np.cos(0.7), np.sin(0.7)
    M = column_major(np.array([[1.3 * c, 0, 1.3 * s, 0.1], [0, 0.8, 0, -0.2], [-1.3 * s, 0, 1.3 * c, 0.05], [0, 0, 0, 1]], np.float32))
    m, _, _ = _check(gpu_ctx, scene, ds, V, P, M, 4096, 4096)
    assert (m < 1.0).mean() > 0.2
    import torch
    d = torch.empty(4097 * 4, dtype=torch.float32, device="cuda")
    for w, h in ((4097, 4), (4, 4097), (0, 4)):
        with pytest.raises(M2SError):
            gpu_ctx.mesh_depth(ds, V, P, M, w, h, depth=d)


def _soup(tris):
    """(T, 36) triangles from (T, 3, 3) positions; normals, tangents and uvs are irrelevant to the pass."""
    t = np.zeros((len(tris), 36), np.float32)
    for k in range(3):
        t[:, 12 * k: 12 * k + 3] = np.asarray(tris, np.float32)[:, k]
        t[:, 12 * k + 5] = 1.0
        t[:, 12 * k + 6] = 1.0
        t[:, 12 * k + 9] = 1.0
    return t


def _crafted():
    """Camera at the origin looking down -z (near 0.1, far 10): triangles behind the camera, across the near and the far
    plane, far past the guard band, around the camera, degenerate ones and non-finite ones, in both windings."""
    rng = np.random.default_rng(3)
    T = [
        [(-1, -1, 2), (1, -1, 2), (0, 1, 2)],            # behind the camera
        [(-1, -1, 1), (1, -1, -3), (0, 1, -3)],           # across the near plane
        [(-1, -1, -5), (1, -1, -15), (0, 1, -15)],        # across the far plane
        [(-500, -400, -2), (600, -300, -2.5), (0, 900, -3)],   # past the guard band in x and y
        [(-1e5, -1e5, -0.5), (1e5, -1e5, -9.0), (0, 1e5, 5.0)],  # past everything
        [(0, 0, -1), (1, 1, -1), (2, 2, -1)],             # degenerate: collinear
        [(0.3, 0.3, -2), (0.3, 0.3, -2), (0.5, 0.1, -2)],  # degenerate: repeated vertex
        [(np.nan, 0, -2), (1, 0, -2), (0, 1, -2)],        # NaN vertex
        [(np.inf, 0, -2), (1, 0, -2), (0, 1, -2)],
        [(0, 0, -4), (0, 1, -4), (1, 0, -4)],             # clockwise
        [(0, 0, -4.5), (1, 0, -4.5), (0, 1, -4.5)],       # counter-clockwise, behind it
        [(-3, -3, -0.1), (3, -3, -0.1), (0, 3, -0.1)],    # on the near plane exactly
    ]
    T += list(rng.uniform(-3, 3, (60, 3, 3)) + np.array([0, 0, -3.0]))   # random, many across the planes
    return _soup(T)


def test_clipping_degenerate_and_non_finite_triangles(gpu_ctx):
    tris = _crafted()
    scene = _abi.Scene(tris, [_abi.Primitive(0, len(tris), (1.0, 1.0, 1.0, 1.0), -1, -1, -1)], [])
    scene.compute_bboxes()
    ds = gpu_ctx.upload(scene)
    V = column_major(np.eye(4, dtype=np.float32))
    P = column_major(perspective(np.radians(60.0), 4 / 3, 0.1, 10.0))
    for wh in ((64, 48), (640, 480), (4096, 3072)):
        m, _, _ = _check(gpu_ctx, scene, ds, V, P, EYE, *wh)
        assert (m < 1.0).any()
    ds.free()


def test_only_the_factor_alpha_decides_what_is_drawn(gpu_ctx):
    """Three primitives: factor alpha 0.99 (skipped), factor alpha 1.0 with an albedo map whose alpha is below 1 (drawn:
    only the factor counts), factor alpha 0.0 (skipped).  A scene without an opaque primitive gives the cleared map."""
    V, P = _camera(OUTSIDE[0], OUTSIDE[1], 16 / 9)
    tri = synth.displaced_sphere(40, 20, seed=2)
    n = len(tri) // 3
    tex = synth.make_material_textures(32, 5)
    tex[0][..., 3] = 100
    prims = [_abi.Primitive(0, n, (1.0, 1.0, 1.0, 0.99), 0, 1, 2), _abi.Primitive(n, n, (0.5, 0.5, 0.5, 1.0), 0, 1, 2),
             _abi.Primitive(2 * n, len(tri) - 2 * n, (1.0, 1.0, 1.0, 0.0), 0, 1, 2)]
    scene = _abi.Scene(tri, prims, tex)
    scene.compute_bboxes()
    ds = gpu_ctx.upload(scene)
    m, _, pairs = _check(gpu_ctx, scene, ds, V, P, EYE, 320, 180)
    alone = _abi.Scene(tri[n: 2 * n], [_abi.Primitive(0, n, (0.5, 0.5, 0.5, 1.0), 0, 1, 2)], tex)
    assert np.array_equal(m, depth.mesh_depth(alone, depth.pvm(V, P, EYE), 320, 180))
    ds.free()
    for p in prims:
        p.base_color_factor = (1.0, 1.0, 1.0, 0.5)
    clear = _abi.Scene(tri, prims, tex)
    clear.compute_bboxes()
    ds = gpu_ctx.upload(clear)
    m, drawn, pairs = _check(gpu_ctx, clear, ds, V, P, EYE, 320, 180)
    assert (m == 1.0).all() and pairs == 0
    ds.free()


def test_pair_cut_and_determinism(gpu_ctx, helmet):
    scene, ds = helmet
    V, P = _camera(INSIDE[0], INSIDE[1], 16 / 9)
    w, h = 480, 270
    counts, total = depth.pairs(scene, depth.pvm(V, P, EYE), w, h)
    incl = np.cumsum(counts.astype(np.int64))
    k = int(np.searchsorted(incl, total // 2))
    for budget in sorted({0, 1, int(incl[k]), int(incl[k]) - 1, total - 1, total, total + 100}):
        _, drawn, pairs = _check(gpu_ctx, scene, ds, V, P, EYE, w, h, max_pairs=budget)
        assert pairs == total and drawn == int(np.searchsorted(incl, budget, side="right")), (budget, drawn)
    a = _depth(gpu_ctx, ds, V, P, EYE, 1920, 1080)[0]
    b = _depth(gpu_ctx, ds, V, P, EYE, 1920, 1080)[0]
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ---- the prepass's depth test --------------------------------------------------------------------------------------------
def _prepass_pair(gpu_ctx, records, n, layout, V, P, M, res, nf, sd, dmap):
    """(test on, test off) GPU prepass outputs of the same records."""
    import torch
    d = torch.from_numpy(np.ascontiguousarray(dmap, np.float32)).cuda()
    on = gpu_ctx.prepass(records, n, layout, V, P, M, res, nf, sd, 0, mesh_depth=d)
    off = gpu_ctx.prepass(records, n, layout, V, P, M, res, nf, sd, 0)
    return on, off


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56])
def test_prepass_with_the_test_against_the_oracle(gpu_ctx, helmet, layout):
    scene, ds = helmet
    R, w, h = 256, 960, 540
    out = gpu_ctx.convert(ds, R, layout, flags=FLAG_UNCAPPED)
    n = out.total
    raw = out.numpy()
    g24 = raw.view(np.float32).reshape(n, 24) if layout == LAYOUT_REF96 else oracle.packed56_as_gaussian_vertex(raw)
    for cam, (eye, tgt) in (("outside", OUTSIDE), ("inside", INSIDE)):
        V, P = _camera(eye, tgt, w / h)
        dmap = _check(gpu_ctx, scene, ds, V, P, EYE, w, h)[0]
        (q, dq), (q0, dq0) = _prepass_pair(gpu_ctx, out.data, n, layout, V, P, EYE, (w, h), (0.01, 100.0), 0.65 / R, dmap)
        keep = depth.test_mask(g24, V, P, EYE, dmap, 0 if layout == LAYOUT_REF96 else 1)
        want_q, want_d = oracle.prepass(g24[keep], V, P, EYE, (w, h), (0.01, 100.0), 0.65 / R, 0, 0 if layout == LAYOUT_REF96 else 1, 0)
        assert len(q) == len(want_q)
        assert_prepass_match(q, dq, want_q, want_d, (w, h), ordered=False)
        if layout == LAYOUT_PACKED56:   # u_format 1: the map is never read
            assert keep.all()
            o, o0 = np.lexsort(q.T[::-1]), np.lexsort(q0.T[::-1])
            assert np.array_equal(q[o].view(np.uint32), q0[o0].view(np.uint32))
        elif cam == "outside":
            assert len(q) < 0.8 * len(q0)   # a closed mesh seen from outside: about its back half is behind its front
        else:
            assert len(q) <= len(q0)   # from inside a star-shaped mesh every surface point is the nearest on its ray


def test_prepass_test_at_the_thresholds(gpu_ctx):
    """REF96 records placed on the decision boundaries over a constant map: myDepth at depth + eps and one ulp either
    side, alpha at 0.95 and the next float up, uv at 0, 1 and outside [0, 1], and w = 0 (a NaN uv)."""
    import torch
    V = column_major(np.eye(4, dtype=np.float32))
    P = column_major(perspective(np.radians(60.0), 1.0, 0.1, 10.0))
    pvm = np.asarray(P, np.float32).reshape(4, 4).T   # row-major P (V = M = I)
    rng = np.random.default_rng(8)
    dmap = rng.uniform(0.9, 0.999, (37, 53)).astype(np.float32)
    g = np.zeros((400, 24), np.float32)
    g[:, 7] = 1.0
    g[:, 16] = 1.0
    g[:, 8:11] = 0.01
    # depths from the near to the far plane along rays at random uv, some beyond [0, 1]
    uv = rng.uniform(-0.2, 1.2, (400, 2))
    z = -rng.uniform(0.2, 9.0, 400)
    g[:, 0] = (uv[:, 0] * 2 - 1) * -z * np.tan(np.radians(30.0))
    g[:, 1] = (uv[:, 1] * 2 - 1) * -z * np.tan(np.radians(30.0))
    g[:, 2] = z
    g[:100, 0] = 0.0   # uv exactly 0.5 ... and the edges
    g[100:110, :2] = np.array([[-1, -1], [1, 1], [-1, 1], [1, -1], [0, 1], [1, 0], [-1, 0], [0, -1], [0, 0], [0.5, 0.5]]) * (-g[100:110, 2:3]) * np.tan(np.radians(30.0))
    g[110:120, 7] = 0.95
    g[120:130, 7] = np.nextafter(np.float32(0.95), np.float32(1))
    g[130:140, 2] = 0.0   # w = 0: the gaussian at the eye
    g[130:140, :2] = 0.0
    # myDepth exactly at the texel's depth + eps and one ulp either side: solve for view z per gaussian
    for k in range(140, 200):
        u, v = uv[k % 40 + 200]
        u, v = min(max(u, 0.01), 0.99), min(max(v, 0.01), 0.99)
        i, j = int(np.floor(np.float32(u) * np.float32(53))), int(np.floor(np.float32(v) * np.float32(37)))
        target = np.float32(np.float32(dmap[j, i]) + np.float32(0.00002))
        target = [np.nextafter(target, np.float32(0)), target, np.nextafter(target, np.float32(2))][k % 3]
        ndc = np.float64(target) * 2 - 1
        A, B = pvm[2, 2], pvm[2, 3]   # z_ndc = (A z + B) / -z
        zz = -B / (ndc + A)
        g[k, :3] = [(u * 2 - 1) * -zz * np.tan(np.radians(30.0)), (v * 2 - 1) * -zz * np.tan(np.radians(30.0)), zz]
    dr = torch.from_numpy(g.view(np.uint8).reshape(-1).copy()).cuda()
    (q, dq), (q0, _) = _prepass_pair(gpu_ctx, dr, len(g), LAYOUT_REF96, V, P, EYE, (64, 64), (0.1, 10.0), 0.01, dmap)
    keep = depth.test_mask(g, V, P, EYE, dmap)
    want_q, want_d = oracle.prepass(g[keep], V, P, EYE, (64, 64), (0.1, 10.0), 0.01, 0, 0, 0)
    assert len(q) == len(want_q) and 0 < len(q) < len(q0)
    assert_prepass_match(q, dq, want_q, want_d, (64, 64), ordered=False)
    assert not keep[140:200].all() and keep[140:200].any()


def test_prepass_test_on_the_reference_golden_cases(gpu_ctx):
    """The records of tests/golden/ref_depth_vectors.npz (the boundary scans, uv at 0, 1 and outside, alpha at 0.95 and
    the next float, w = 0 at the eye with a NaN uv) over their maps: the GPU keeps exactly the gaussians the reference's
    own prepass keeps with u_depthTestMesh = 1, and its quads match the reference's."""
    import torch
    z = np.load(os.path.join(HERE, "golden", "ref_depth_vectors.npz"))
    for k in range(int(z["ncases"])):
        g, dmap, p = z[f"g{k}"], z[f"map{k}"], z[f"params{k}"]
        res, nf = (float(p[0]), float(p[1])), (float(p[2]), float(p[3]))
        dr = torch.from_numpy(np.ascontiguousarray(g).view(np.uint8).reshape(-1).copy()).cuda()
        q, dq = gpu_ctx.prepass(dr, len(g), LAYOUT_REF96, z[f"view{k}"], z[f"proj{k}"], z[f"model{k}"], res, nf, float(p[4]), 0,
                                mesh_depth=torch.from_numpy(np.ascontiguousarray(dmap)).cuda())
        assert len(q) == int(z[f"keep{k}_f0"].sum()) == len(z[f"quads{k}"]), k
        if len(q):
            assert_prepass_match(q, dq, z[f"quads{k}"], z[f"depths{k}"], res, ordered=False)


def test_sphere_behind_an_opaque_quad_is_culled(gpu_ctx):
    """Gaussians converted from a sphere behind a quad that covers it: all culled where the quad is opaque (factor alpha
    1.0); with the quad's alpha at 0.99 the map is the clear and nothing is culled."""
    import torch
    sphere = _abi.Scene(synth.displaced_sphere(48, 24, seed=4, amplitude=0.0, radius=0.5, center=(0.0, 0.0, -3.0)),
                        [], [])
    sphere.primitives = [_abi.Primitive(0, sphere.triangle_count, (0.8, 0.6, 0.4, 1.0), -1, -1, -1)]
    sphere.compute_bboxes()
    dss = gpu_ctx.upload(sphere)
    out = gpu_ctx.convert(dss, 64, LAYOUT_REF96, flags=FLAG_UNCAPPED)
    n = out.total
    V = column_major(np.eye(4, dtype=np.float32))
    P = column_major(perspective(np.radians(60.0), 1.0, 0.1, 10.0))
    quad = _soup([[(-2, -2, -1), (2, -2, -1), (2, 2, -1)], [(-2, -2, -1), (2, 2, -1), (-2, 2, -1)]])
    base = len(gpu_ctx.prepass(out.data, n, LAYOUT_REF96, V, P, EYE, (256, 256), (0.1, 10.0), 0.65 / 64)[0])
    assert base > 100
    for alpha, survivors in ((1.0, 0), (0.99, base)):
        qs = _abi.Scene(quad, [_abi.Primitive(0, 2, (1.0, 1.0, 1.0, alpha), -1, -1, -1)], [])
        qs.compute_bboxes()
        dsq = gpu_ctx.upload(qs)
        dmap = _check(gpu_ctx, qs, dsq, V, P, EYE, 256, 256)[0]
        q, _ = gpu_ctx.prepass(out.data, n, LAYOUT_REF96, V, P, EYE, (256, 256), (0.1, 10.0), 0.65 / 64,
                               mesh_depth=torch.from_numpy(dmap).cuda())
        assert len(q) == survivors, (alpha, len(q), base)
        dsq.free()
    dss.free()


# ---- the whole frame --------------------------------------------------------------------------------------------------
def test_convert_depth_prepass_sort_draw_shadow_light_chain_on_one_stream(gpu_ctx, helmet):
    """convert -> mesh depth -> prepass (test on) -> sort -> draw -> shadow -> light enqueued on one non-default stream
    with no host synchronisation, on the bench scene (R = 512) with the camera outside at 1920 x 1080.  The map equals the
    oracle's, the survivors the oracle's prepass of the records its mask keeps, the sort's count the survivors, and the
    image the oracle's lighting of the drawn G-buffer and the cube."""
    import torch
    scene, ds = helmet
    R, S, layout = 512, 256, LAYOUT_REF96
    cap = 6 * R * R
    w, h = 1920, 1080
    V, P = _camera(OUTSIDE[0], OUTSIDE[1], w / h)
    M = column_major(EYE)
    lpos = (1.5, 2.0, 2.5)
    stream = torch.cuda.Stream()
    out = torch.empty(cap * _abi.STRIDES[layout], dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    gd = GuardedDevice(w * h, 4, what="depth map")
    quads = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    depths = torch.empty(cap, dtype=torch.float32, device="cuda")
    valid = torch.zeros(1, dtype=torch.int32, device="cuda")
    sq = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    draw = torch.zeros(5, dtype=torch.int32, device="cuda")
    gbuf = {t: torch.empty(w * h * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda") for t, dt in _abi.GBUFFER_TARGETS}
    g = _abi.m2s_gbuffer(*[gbuf[t].data_ptr() for t in NAMES])
    cube = torch.empty(6 * S * S, dtype=torch.float32, device="cuda")
    image = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
    res = torch.zeros(12, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    p = _abi.make_params(R, layout, 0.65, 0, FLAG_UNCAPPED)
    dp = _abi.make_mesh_depth_params(V, P, M, w, h)
    pp = _abi.make_prepass_params(V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 6, layout)
    sp = _abi.m2s_splat_params(w, h, 6)
    shp = _abi.make_shadow_params(M, lpos, (0.01, 100.0), (w, h), 0.65 / R, layout, S)
    lp = _abi.make_light_params(w, h, 6, lpos, (1.0, 1.0, 1.0), 10.0, OUTSIDE[0], 100.0, S)
    L, hs = lib(), stream.cuda_stream
    check(L.m2s_convert_enqueue(gpu_ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), hs))
    check(L.m2s_mesh_depth_enqueue(gpu_ctx.handle, ds.handle, C.byref(dp), gd.view.data_ptr(), 20_000_000, res[8:].data_ptr(),
                                   res[10:].data_ptr(), hs))
    check(L.m2s_prepass_mesh_depth_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), gd.view.data_ptr(), w, h,
                                           quads.data_ptr(), depths.data_ptr(), valid.data_ptr(), hs))
    check(L.m2s_depth_sort_enqueue(gpu_ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(), sq.data_ptr(),
                                   None, draw.data_ptr(), hs))
    check(L.m2s_splat_draw_enqueue(gpu_ctx.handle, sq.data_ptr(), cap, draw.data_ptr(), C.byref(sp), C.byref(g),
                                   60_000_000, res.data_ptr(), res[2:].data_ptr(), hs))
    check(L.m2s_shadow_map_enqueue(gpu_ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(shp), cube.data_ptr(),
                                   None, 60_000_000, res[4:].data_ptr(), res[6:].data_ptr(), hs))
    check(L.m2s_deferred_light_enqueue(gpu_ctx.handle, C.byref(g), cube.data_ptr(), C.byref(lp), image.data_ptr(), hs))
    stream.synchronize()
    n = int(total.item())
    o = res.cpu().numpy()
    gd.check(w * h)
    assert int(o[10]) == scene.triangle_count, "the budget holds every depth pair"
    dmap = gd.view[: w * h * 4].cpu().numpy().view(np.float32).reshape(h, w)
    assert np.array_equal(dmap.view(np.uint32), depth.mesh_depth(scene, depth.pvm(V, P, M), w, h).view(np.uint32))
    g24 = out[: n * 96].cpu().numpy().view(np.float32).reshape(n, 24)
    keep = depth.test_mask(g24, V, P, M, dmap)
    want_q, want_d = oracle.prepass(g24[keep], V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 6, 0, 0)
    m = int(valid.item())
    assert m == len(want_q) and int(draw[1].item()) == m and int(o[2]) == m
    assert_prepass_match(quads[: m * 96].cpu().numpy().view(np.float32).reshape(m, 24), depths[:m].cpu().numpy(), want_q, want_d,
                         (w, h), ordered=False)
    gb = {t: gbuf[t].view(torch.uint8)[: w * h * 4 * np.dtype(dt).itemsize].cpu().numpy().view(dt).reshape(h, w, 4)
          for t, dt in _abi.GBUFFER_TARGETS}
    img = image.cpu().numpy().reshape(h, w, 4)
    want = light.deferred_light(gb, cube.cpu().numpy().reshape(6, S, S), lp)
    assert np.array_equal(img, want), int((img != want).any(axis=-1).sum())
    assert (img[..., :3] > 0).any()
