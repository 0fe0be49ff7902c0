"""The mesh depth pre-pass checker (row f-9) on the CPU: the oracle's D24 codes against fp64, its raster against an
independent fp64 ray cast on random triangles (near, far and guard-band crossings included), its clipping and PVM
product, and the C ABI's argument checks (which run before any CUDA call)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

from mesh2splat_b200 import _abi, _lib
from oracle import depth

F32 = np.float32


def test_d24_codes_at_code_boundaries():
    rng = np.random.default_rng(1)
    codes = np.concatenate([[0, 1, 2, 8388607, 8388608, 16777213, 16777214], rng.integers(0, 16777215, 2000)])
    for c in codes:
        mid = (float(c) + 0.5) / 16777215.0   # the boundary between codes c and c + 1
        for z in (np.nextafter(mid, 0.0), np.nextafter(mid, 1.0), float(c) / 16777215.0):
            want = int(np.rint(np.float64(z) * 16777215.0))
            assert depth.code(z) == want, (c, z)
        assert abs(depth.code(mid) - (c + 0.5)) == 0.5
    assert depth.code(-1.0) == 0 and depth.code(2.0) == 16777215 and depth.code(float("nan")) is None
    assert depth.code(float("inf")) == 16777215 and depth.code(float("-inf")) == 0


def test_pvm_is_glm_left_to_right():
    rng = np.random.default_rng(2)
    V, P, M = (rng.normal(0, 1, 16).astype(F32) for _ in range(3))
    m = lambda a: a.reshape(4, 4).T   # noqa: E731 (column-major -> row-major)
    got = m(depth.pvm(V, P, M))
    want = (m(P).astype(np.float64) @ m(V).astype(np.float64)).astype(F32).astype(np.float64) @ m(M).astype(np.float64)
    assert np.allclose(got, want, rtol=1e-5, atol=1e-5)
    # exact GLM operation order for one element, in fp32
    pm, vm = m(P), m(V)
    pv = np.array([[F32(F32(F32(pm[r, 0] * vm[0, c]) + F32(pm[r, 1] * vm[1, c])) + F32(pm[r, 2] * vm[2, c])) + F32(pm[r, 3] * vm[3, c])
                    for c in range(4)] for r in range(4)], F32)
    assert np.array_equal(m(depth.pvm(V, P, np.eye(4, dtype=F32).ravel())), pv)


def _tri36(pos):
    t = np.zeros(36, F32)
    for k in range(3):
        t[12 * k: 12 * k + 3] = pos[k]
    return t


def test_clipping_keeps_the_visible_part():
    eye = np.eye(4, dtype=F32).ravel()   # clip = position, w = 1
    assert len(depth.poly(_tri36([(0, 0, 0.5), (0.5, 0, 0.5), (0, 0.5, 0.5)]), eye)) == 3
    # two vertices before the far plane z = w, one past it: a quadrilateral inside
    p = depth.poly(_tri36([(0, 0, 0), (0.5, 0, 0), (0, 0.5, 2)]), eye)
    assert len(p) == 4 and (p[:, 2] <= p[:, 3]).all() and (p[:, 2] >= -p[:, 3]).all()
    # past the guard band in x: cut at x = 2 w
    p = depth.poly(_tri36([(0, 0, 0), (10, 0, 0), (0, 1, 0)]), eye)
    assert len(p) == 4 and np.isclose(p[:, 0].max(), 2.0)
    assert len(depth.poly(_tri36([(0, 0, 2), (1, 0, 2), (0, 1, 2)]), eye)) == 0   # wholly past the far plane
    assert len(depth.poly(_tri36([(np.nan, 0, 0), (1, 0, 0), (0, 1, 0)]), eye)) == 0
    # a triangle around the eye crossing near plane and guard band: every clipped vertex inside all six planes
    P = np.zeros((4, 4), F32)
    P[0, 0], P[1, 1], P[2, 2], P[2, 3], P[3, 2] = 1, 1, -1.02, -0.202, -1
    p = depth.poly(_tri36([(-50, -50, 1), (50, -50, -1), (0, 60, -3)]), P.T.ravel())
    assert 3 <= len(p) <= 9
    w = p[:, 3]
    assert (w > 0).all() and (np.abs(p[:, 2]) <= w * (1 + 1e-6)).all() and (np.abs(p[:, :2]) <= 2 * w[:, None] * (1 + 1e-6)).all()


def _ray_hits(tri_clip, X, Y):
    """fp64 intersection of the rays through NDC points (X, Y) with the clip-space triangle: barycentrics [.., 3], w, z."""
    x, y, z, w = (tri_clip[:, k] for k in range(4))
    r1 = x[None, :] - X[:, None] * w[None, :]
    r2 = y[None, :] - Y[:, None] * w[None, :]
    b = np.cross(r1, r2)
    s = b.sum(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        b = b / s[:, None]
    return b, b @ w, b @ z


@pytest.mark.parametrize("seed", range(4))
def test_raster_against_an_fp64_ray_cast(seed):
    """2 500 random triangles per seed (10 000 in all), many across the near or far plane or past the guard band, each
    drawn alone into a 32 x 24 map.  Every covered pixel: the fp64 ray through a point within 1/64 pixel of its centre
    hits the triangle in front of the eye between the near and far planes, and the code is within 2 of the fp64 depth at
    the centre, plus the depth change over the 1/256-pixel snap and the rounding bound of the fp32 vertex stage.  Every pixel whose centre neighbourhood lies wholly
    inside the triangle and the depth range is covered."""
    rng = np.random.default_rng(100 + seed)
    W, H = 32, 24
    P = np.zeros((4, 4), np.float64)
    n, f = 0.5, 20.0
    P[0, 0], P[1, 1], P[2, 2], P[2, 3], P[3, 2] = 1.2, 1.6, -(f + n) / (f - n), -2 * f * n / (f - n), -1.0
    pvm = P.T.astype(F32).ravel()
    ii, jj = np.meshgrid(np.arange(W), np.arange(H))
    Xc = ((ii.ravel() + 0.5) / W) * 2 - 1
    Yc = ((jj.ravel() + 0.5) / H) * 2 - 1
    off = np.array([(dx, dy) for dx in (-1, 0, 1) for dy in (-1, 0, 1)], np.float64) / 64.0
    covered_total = 0
    for t in range(2500):
        kind = t % 4
        c = rng.normal(0, 1, 3) * [1.0, 1.0, 0] + [0, 0, -rng.uniform(0.2, 25.0)]
        spread = [0.3, 2.0, 8.0, 40.0][kind]
        pos = (c + rng.normal(0, spread, (3, 3)) * [1, 1, 0.5 if kind < 3 else 3.0]).astype(F32)
        m = depth.mesh_depth(_tri36(pos)[None, :], pvm, W, H).ravel()
        codes = np.rint(m.astype(np.float64) * 16777215.0)
        cov = codes < 16777215
        covered_total += int(cov.sum())
        clip = np.c_[pos.astype(np.float64), np.ones(3)] @ P.astype(F32).astype(np.float64).T
        inside_all = np.ones(W * H, bool)
        hit_any = np.zeros(W * H, bool)
        for dx, dy in off:
            b, wh, zh = _ray_hits(clip, Xc + dx * 2 / W, Yc + dy * 2 / H)
            ok = np.isfinite(b).all(axis=1) & (wh > 0)
            inb = ok & (b >= 0).all(axis=1) & (zh >= -wh) & (zh <= wh)
            strict = ok & (b > 1e-9).all(axis=1) & (zh > -wh * (1 - 1e-9)) & (zh < wh * (1 - 1e-9))
            hit_any |= inb
            inside_all &= strict
        assert hit_any[cov].all(), (t, np.flatnonzero(cov & ~hit_any))
        assert cov[inside_all].all(), (t, np.flatnonzero(inside_all & ~cov))
        if cov.any():
            b, wh, zh = _ray_hits(clip, Xc[cov], Yc[cov])
            zd = (zh / wh) * 0.5 + 0.5
            # the depth's change over 1/256 pixel in x and y: the snap moves each vertex by at most 1/512 pixel
            grad = 0.0
            for dx, dy in ((1, 0), (0, 1)):
                _, w2, z2 = _ray_hits(clip, Xc[cov] + dx * 2.0 / (256 * W), Yc[cov] + dy * 2.0 / (256 * H))
                grad = grad + np.abs((z2 / w2) * 0.5 + 0.5 - zd) * 16777215.0
            err = np.abs(codes[cov] - np.clip(zd, 0, 1) * 16777215.0)
            # the fp32 vertex stage: each clip coordinate carries a few roundings relative to the sum of its terms' sizes,
            # which z / w turns into a window-depth error of about 2^-22 (|z terms| + |z / w| |w terms|) / |w|
            Pf = P.astype(F32).astype(np.float64)
            ph = np.c_[pos.astype(np.float64), np.ones(3)]
            az, aw = np.abs(ph * Pf[2]).sum(axis=1), np.abs(ph * Pf[3]).sum(axis=1)
            front = clip[:, 3] > 0
            cond = ((az + np.abs(clip[:, 2] / clip[:, 3]) * aw) / np.abs(clip[:, 3]))[front].max() if front.any() else 0.0
            # a clipped vertex is an fp32 blend of two of them: its error is relative to their size, not to its own w
            poly = depth.poly(_tri36(pos), pvm).astype(np.float64)
            clipped = 2.0 ** -20 * np.abs(clip).max() / poly[:, 3].min() if len(poly) != 3 or not front.all() else 0.0
            tol = 2.0 + 2.0 * grad + 16777215.0 * (2.0 ** -22 * cond + clipped)
            assert (err <= tol).all(), (t, float(err.max()), float(tol.min()))
    assert covered_total > 50_000


def _depth_params(w=64, h=32):
    return _abi.make_mesh_depth_params(np.eye(4), np.eye(4), np.eye(4), w, h)


def test_mesh_depth_entry_points_reject_bad_arguments_without_a_gpu():
    L = _lib.lib()
    INV = _abi.M2S_E_INVALID
    ctx = C.cast(C.create_string_buffer(4096), C.c_void_p)
    scene = C.cast(C.create_string_buffer(4096), C.c_void_p)
    dmap = 0x40000
    p = _depth_params()
    assert L.m2s_mesh_depth(None, scene, C.byref(p), dmap, None) == INV
    assert L.m2s_mesh_depth(ctx, None, C.byref(p), dmap, None) == INV
    assert L.m2s_mesh_depth(ctx, scene, None, dmap, None) == INV
    assert L.m2s_mesh_depth(ctx, scene, C.byref(p), None, None) == INV and b"NULL" in L.m2s_last_error()
    assert L.m2s_mesh_depth(ctx, scene, C.byref(p), dmap + 2, None) == INV and b"aligned" in L.m2s_last_error()
    for w, h in ((0, 8), (8, 0), (4097, 8), (8, 4097)):
        assert L.m2s_mesh_depth(ctx, scene, C.byref(_depth_params(w, h)), dmap, None) == INV and b"4096" in L.m2s_last_error()
        assert L.m2s_mesh_depth_enqueue(ctx, scene, C.byref(_depth_params(w, h)), dmap, 10, None, None, None) == INV
    assert L.m2s_mesh_depth_enqueue(ctx, scene, C.byref(p), dmap, 1 << 30, None, None, None) == INV and b"max_pairs" in L.m2s_last_error()
    big = (C.c_uint64 * 512)()
    big[1] = 1 << 29   # m2s_dscene's triangle count, after the triangle pointer
    assert L.m2s_mesh_depth(ctx, C.cast(big, C.c_void_p), C.byref(p), dmap, None) == INV and b"triangles" in L.m2s_last_error()
    pp = _abi.make_prepass_params(np.eye(4), np.eye(4), np.eye(4), (64, 64), (0.1, 10.0), 0.01, 0, 0)
    rec, q, d, v = 0x10000, 0x20000, 0x30000, 0x50000
    pre = lambda *a: L.m2s_prepass_mesh_depth(ctx, rec, 4, C.byref(pp), *a)   # noqa: E731
    assert pre(None, 8, 8, q, d, None) == INV
    assert pre(dmap + 1, 8, 8, q, d, None) == INV
    for w, h in ((0, 8), (8, 0), (4097, 8), (8, 4097)):
        assert pre(dmap, w, h, q, d, None) == INV
    assert pre(dmap, 8, 8, q + 8, d, None) == INV
    assert L.m2s_prepass_mesh_depth_enqueue(ctx, rec, 4, None, C.byref(pp), dmap, 8, 8, q, d, None, None) == INV
    sing = _abi.make_prepass_params(np.eye(4), np.eye(4), np.zeros((4, 4)), (64, 64), (0.1, 10.0), 0.01, 0, 0)
    assert L.m2s_prepass_mesh_depth_enqueue(ctx, rec, 4, None, C.byref(sing), dmap, 8, 8, q, d, v, None) == INV


def test_no_gpu_gives_nogpu():
    from test_abi_host import _has_gpu
    if _has_gpu():
        pytest.skip("a CUDA device is present")
    L = _lib.lib()
    ctx = C.cast(C.create_string_buffer(4096), C.c_void_p)
    scene = C.cast(C.create_string_buffer(4096), C.c_void_p)
    p = _depth_params()
    assert L.m2s_mesh_depth(ctx, scene, C.byref(p), 0x40000, None) == _abi.M2S_E_NOGPU
    assert L.m2s_mesh_depth_enqueue(ctx, scene, C.byref(p), 0x40000, 10, None, None, None) == _abi.M2S_E_NOGPU
    pp = _abi.make_prepass_params(np.eye(4), np.eye(4), np.eye(4), (64, 64), (0.1, 10.0), 0.01, 0, 0)
    assert L.m2s_prepass_mesh_depth(ctx, 0x10000, 4, C.byref(pp), 0x40000, 8, 8, 0x20000, 0x30000, None) == _abi.M2S_E_NOGPU
    assert L.m2s_prepass_mesh_depth_enqueue(ctx, 0x10000, 4, None, C.byref(pp), 0x40000, 8, 8, 0x20000, 0x30000, 0x50000,
                                            None) == _abi.M2S_E_NOGPU


# ---- the oracle against the reference's own shaders (tests/golden/ref_depth_vectors.npz) --------------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_depth_vectors.npz")
CRAFTED, EYE_INF, EYE_NAN = 5, 6, 7   # case indices of make_golden_depth.py: the boundary scans, w = 0 with pos2d.z > 0 / = 0


def _case(z, k):
    p = z[f"params{k}"]
    return (z[f"g{k}"], z[f"view{k}"], z[f"proj{k}"], z[f"model{k}"], (float(p[0]), float(p[1])), (float(p[2]), float(p[3])),
            float(p[4]), z[f"map{k}"])


def test_vertex_invocations_match_the_reference_bit_for_bit():
    z = np.load(GOLDEN)
    n = 0
    for k in range(int(z["nvs"])):
        got = depth.vs(z[f"vs_pos{k}"], depth.pvm(z[f"vs_view{k}"], z[f"vs_proj{k}"], z[f"vs_model{k}"]))
        assert np.array_equal(got.view(np.uint32), z[f"vs_out{k}"].view(np.uint32)), k
        n += len(got)
    assert k == 6 and n == 7 * 360


def test_depth_test_mask_matches_the_reference_bit_for_bit():
    """Every gaussian the reference's prepass keeps with u_depthTestMesh = 0 is kept with it = 1 exactly when the
    oracle's mask keeps it, for u_format 0; with u_format 1 the test never drops anything."""
    z = np.load(GOLDEN)
    for k in range(int(z["ncases"])):
        g, V, P, M, res, nf, sd, dmap = _case(z, k)
        for fmt in (0, 1):
            on, off = z[f"keep{k}_f{fmt}"], z[f"cull{k}_f{fmt}"]
            assert not (on & ~off).any()
            mask = depth.test_mask(g, V, P, M, dmap, fmt)
            assert np.array_equal(mask[off], on[off]), (k, fmt, np.flatnonzero(mask[off] != on[off])[:10])
            if fmt == 1:
                assert mask.all() and np.array_equal(on, off)
        assert (z[f"cull{k}_f0"] & ~z[f"keep{k}_f0"]).any(), k   # the test drops something in every case


def test_the_golden_cases_sit_on_the_decision_boundaries():
    z = np.load(GOLDEN)
    on, off = z[f"keep{CRAFTED}_f0"], z[f"cull{CRAFTED}_f0"]
    scans = (on[: 24 * 49] ^ off[: 24 * 49]).reshape(24, 49)   # dropped by the test, per 49-ulp scan of view z
    # the scans cross myDepth = depth + eps (one lands on a texel of 1.0, past which nothing is ever dropped)
    assert sum(0 < s.sum() < 49 for s in scans) >= 22
    alpha = z[f"g{CRAFTED}"][24 * 49: 24 * 49 + 9, 7]
    dropped = (off & ~on)[24 * 49: 24 * 49 + 9]
    assert not dropped[alpha <= np.float32(0.95)].any() and dropped[alpha > np.float32(0.95)].all()
    for k, drops in ((EYE_INF, True), (EYE_NAN, False)):   # w = 0 at the eye: NaN uv, myDepth inf or NaN
        on, off, g = z[f"keep{k}_f0"], z[f"cull{k}_f0"], z[f"g{k}"]
        opaque = off[:3] & (g[:3, 7] > np.float32(0.95))
        assert opaque.any() and (on[:3][opaque] != drops).all(), k


def test_prepass_with_the_test_matches_the_reference():
    """orc_prepass of the records the mask keeps against the reference's whole prepass with the test on (input order)."""
    import oracle
    from util import assert_prepass_match
    z = np.load(GOLDEN)
    for k in range(int(z["ncases"])):
        g, V, P, M, res, nf, sd, dmap = _case(z, k)
        keep = depth.test_mask(g, V, P, M, dmap, 0)
        q, d = oracle.prepass(g[keep], V, P, M, res, nf, sd, 0, 0, 0)
        assert len(q) == len(z[f"quads{k}"]), k
        assert_prepass_match(q, d, z[f"quads{k}"], z[f"depths{k}"], res, ordered=True)
