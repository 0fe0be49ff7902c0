"""CPU tests of the viewer's shadow pass and deferred lighting (rows f-7, f-8): the contract pieces of the C
restatement (orc_light_*: pow / exp2 / log2 against fp64, cube face selection and texel coordinates against a direct
transcription of GL 4.6 table 8.19, D24 codes, the GLM uniforms), the shader quirks it keeps, and the argument checks of
the C entry points, which return before any CUDA call."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

from mesh2splat_b200 import _abi, _lib
from oracle import light

F32 = np.float32


def test_pow_against_fp64_within_the_stated_bound():
    """|pow(x, y) - x^y| <= x^y (2^-21 + |y log2 x| 2^-22) (DESIGN §2) for the shader's exponents and others, over
    (0, 1], subnormals and the whole positive range wherever x^y is a normal float."""
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.random(20000), rng.uniform(0, 1e-30, 2000), np.logspace(-44, 38, 3000)]).astype(F32)
    x = x[x > 0]
    for y in (2.2, 5.0, 1.0 / 2.2, 0.5, 3.0, -1.0, 17.0):
        y = F32(y)
        got = light.pow(x, y).astype(np.float64)
        with np.errstate(over="ignore"):
            want = np.power(x.astype(np.float64), np.float64(y))
        t = np.abs(np.float64(y) * np.log2(x.astype(np.float64)))
        ok = (want > 1.2e-38) & (want < 3e38)
        assert ok.sum() > 1000
        bound = want[ok] * (2.0 ** -21 + t[ok] * 2.0 ** -22)
        assert (np.abs(got[ok] - want[ok]) <= bound).all(), (float(y), float(np.max(np.abs(got[ok] - want[ok]) / bound)))


def test_pow_exp2_log2_edge_cases():
    assert light.pow([0.0], 2.2)[0] == 0.0 and light.pow([0.0], 5.0)[0] == 0.0
    assert light.pow([1.0], 2.2)[0] == 1.0 and light.pow([1.0], 1.0 / 2.2)[0] == 1.0
    assert np.isnan(light.pow([-0.5, np.nan], 2.2)).all()
    assert np.isnan(light.pow([0.5], np.nan)).all()
    assert np.isinf(light.pow([np.inf], 2.2)).all()
    assert light.log2([0.0])[0] == -np.inf and np.isnan(light.log2([-1.0, np.nan])).all() and light.log2([np.inf])[0] == np.inf
    assert light.log2([1.0, 2.0, 0.5, 1024.0, 2.0 ** -149]).tolist() == [0.0, 1.0, -1.0, 10.0, -149.0]
    assert light.exp2([0.0, 1.0, -1.0, 10.0, -149.0]).tolist() == [1.0, 2.0, 0.5, 1024.0, 2.0 ** -149]
    assert light.exp2([128.0, 1e4, np.inf]).tolist() == [np.inf] * 3
    assert light.exp2([-151.0, -1e4, -np.inf]).tolist() == [0.0] * 3
    assert np.isnan(light.exp2([np.nan])).all()


def gl_table_8_19(r, S):
    """GL 4.6 §8.13 table 8.19 written out, with the tie and sign rules DESIGN §2 fixes, and the texel of NEAREST +
    CLAMP_TO_EDGE."""
    rx, ry, rz = (F32(v) for v in r)
    ax, ay, az = abs(rx), abs(ry), abs(rz)
    if ax >= ay and ax >= az:
        face, sc, tc, ma = (0, -rz, -ry, rx) if rx > 0 else (1, rz, -ry, rx)
    elif ay >= ax and ay >= az:
        face, sc, tc, ma = (2, rx, rz, ry) if ry > 0 else (3, rx, -rz, ry)
    else:
        face, sc, tc, ma = (4, rx, -ry, rz) if rz > 0 else (5, -rx, -ry, rz)
    with np.errstate(all="ignore"):
        s = (F32(sc) / F32(abs(ma)) + F32(1)) * F32(0.5)
        t = (F32(tc) / F32(abs(ma)) + F32(1)) * F32(0.5)
        texel = lambda v: 0 if np.isnan(v) else int(min(max(np.floor(F32(v * F32(S))), 0), S - 1))  # noqa: E731
        return face, texel(s), texel(t)


def test_cube_texels_against_the_gl_table():
    rng = np.random.default_rng(2)
    dirs = rng.normal(0, 1, (100_000, 3)).astype(F32)
    ties = []
    for a in (1.0, 0.5, 3.0):
        for sx in (1, -1):
            for sy in (1, -1):
                for sz in (1, -1, 0):
                    ties += [(sx * a, sy * a, sz * a), (sx * a, sy * a, sz * a * 0.5), (sx * a, sy * a * 0.5, sz * a), (sx * a * 0.5, sy * a, sz * a)]
    ties += [(0, 0, 0), (-0.0, 0, 0), (np.nan, 1, 0), (1, np.nan, 0), (0, 0, np.nan), (np.inf, 1, 0), (np.inf, np.inf, 1), (-np.inf, 0, 0)]
    for S in (1, 17, 64, 1024):
        for d in list(dirs[:20000] if S != 64 else dirs) + [np.array(t, F32) for t in ties]:
            assert light.cube_texel(d, S) == gl_table_8_19(d, S), (d, S)


def test_face_selection_ties_and_nan():
    assert light.face(1, 1, 1) == 0 and light.face(-1, 1, 1) == 1 and light.face(0.5, 1, 1) == 2 and light.face(0.5, -1, 1) == 3
    assert light.face(0, 0, 1) == 4 and light.face(0, 0, -1) == 5 and light.face(0, 0, 0) == 1
    assert light.face(np.nan, 0, 0) == 5 and light.face(np.nan, np.nan, np.nan) == 5 and light.face(0, np.nan, 1) == 4


def test_d24_codes():
    assert light.d24(0.0) == 0 and light.d24(1.0) == 2 ** 24 - 1 and light.d24(-3.0) == 0 and light.d24(7.0) == 2 ** 24 - 1
    assert light.d24(np.nan) is None and light.d24(np.inf) == 2 ** 24 - 1 and light.d24(-np.inf) == 0
    rng = np.random.default_rng(3)
    for d in rng.random(20000).astype(F32):
        assert light.d24(float(d)) == int(np.rint(np.float64(d) * (2 ** 24 - 1)))   # exact product, ties to even
    # ties: d (2^24 - 1) = k + 1/2 exactly happens for no fp32 d in (0, 1); the rounding of the product is still exact
    for k in (1, 2, 3, 1000, 2 ** 23):
        d = F32(k / (2 ** 24 - 1))
        assert light.d24(float(d)) == k
    for c in (0, 1, 2, 12345, 2 ** 24 - 2, 2 ** 24 - 1):   # the stored sampler value round-trips to its code
        assert light.d24(float(F32(c) / F32(16777215.0))) == c


def test_uniforms_are_glms():
    """The face views are glm::lookAt(light, light + dir, up) (a rotation and the light's translation), the projection
    glm::perspective(90 deg, 1, near, far) with tan(pi/4) = 1 in fp32."""
    p = _abi.make_shadow_params(np.eye(4), (0.5, -0.25, 3.0), (0.1, 50.0), (1920, 1080), 0.01, 0, 64)
    V, P, R, s = light.uniforms(p)
    assert P[0] == 1.0 and P[5] == 1.0 and P[11] == -1.0 and P[10] == F32(-(F32(50.1) / F32(49.9)))
    dirs = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    for f in range(6):
        M = V[f].reshape(4, 4).T                    # row-major
        assert np.allclose(M[:3, :3] @ M[:3, :3].T, np.eye(3))
        assert np.allclose(M[:3, :3] @ np.array([0.5, -0.25, 3.0]) + M[:3, 3], 0, atol=1e-6)   # the light is the eye
        assert np.allclose(M[2, :3], -np.array(dirs[f]))                                       # looks along dir
    assert np.array_equal(R, np.eye(3, dtype=F32).ravel()) and np.array_equal(s, np.ones(3, F32))


def test_light_prepass_light_at_a_gaussian_and_face_buckets():
    """A light exactly at a gaussian gives the NaN direction, face 5; lights inside a cloud use all six faces."""
    rng = np.random.default_rng(4)
    g = np.zeros((600, 24), F32)
    g[:, 0:3] = rng.uniform(-1, 1, (600, 3))
    g[:, 8:11] = rng.uniform(1, 4, (600, 3))
    g[:, 16] = 1.0
    p = _abi.make_shadow_params(np.eye(4), (0.0, 0.0, 0.0), (0.01, 100.0), (1280, 720), 0.65 / 512, 0, 64)
    recs = light.prepass(g, len(g), p)
    faces = recs[:, 7].view(np.uint32)
    assert set(faces.tolist()) >= set(range(6))
    p2 = _abi.make_shadow_params(np.eye(4), tuple(g[7, :3]), (0.01, 100.0), (1280, 720), 0.65 / 512, 0, 64)
    r2 = light.prepass(g, len(g), p2)
    assert r2[7, 7].view(np.uint32) == 0xFFFFFFFF   # NaN direction -> face 5 -> behind the light: culled


def test_lighting_quirks():
    """Modes 0-4 copy the albedo, mode 5 the MR; a pixel with zero position, normal and albedo is still lit: its normal
    is normalize(-1, -1, -1) and it gets the specular term from F0 = 0.04 once its roughness is not 0 (an all-zero
    background pixel has roughness 0, so NDF = 0 and it stays black)."""
    g = {t: np.zeros((1, 1, 4), dt) for t, dt in _abi.GBUFFER_TARGETS}
    g["albedo"][:] = [10, 20, 30, 40]
    g["metallic_roughness"][:] = [50, 60, 70, 80]
    cube = np.ones((6, 4, 4), F32)
    for mode in range(5):
        assert light.deferred_light(g, None, _abi.make_light_params(1, 1, mode)).tolist() == [[[10, 20, 30, 255]]]
    assert light.deferred_light(g, None, _abi.make_light_params(1, 1, 5)).tolist() == [[[50, 60, 0, 255]]]
    z = {t: np.zeros((1, 1, 4), dt) for t, dt in _abi.GBUFFER_TARGETS}
    lp = _abi.make_light_params(1, 1, 6, (-1.0, -2.0, -3.0), (1, 1, 1), 30.0, (-2.0, -1.0, -1.0), 100.0, 4)
    assert light.deferred_light(z, cube, lp).tolist() == [[[0, 0, 0, 255]]]
    z["metallic_roughness"][:] = [0, 128, 0, 0]
    lit = light.deferred_light(z, cube, lp)
    assert lit[0, 0, 0] > 0 and lit[0, 0, 0] == lit[0, 0, 1] == lit[0, 0, 2] and lit[0, 0, 3] == 255


def _gbuf(**kw):
    g = _abi.m2s_gbuffer()
    for k, v in kw.items():
        setattr(g, k, v)
    return g


def test_light_entry_points_reject_bad_arguments_without_a_gpu():
    L = _lib.lib()
    INV = _abi.M2S_E_INVALID
    ctx = C.cast(C.create_string_buffer(4096), C.c_void_p)
    rec, cube, lq = 0x10000, 0x40000, 0x80000
    p = _abi.make_shadow_params(np.eye(4), (0, 0, 0), (0.1, 10), (64, 64), 0.01, 0, 64)
    sm = lambda *a: L.m2s_shadow_map(*a)   # noqa: E731
    enq = lambda *a: L.m2s_shadow_map_enqueue(*a)   # noqa: E731
    assert sm(None, rec, 4, C.byref(p), cube, None, None) == INV
    assert sm(ctx, rec, 4, None, cube, None, None) == INV
    assert sm(ctx, rec, 4, C.byref(p), None, None, None) == INV
    assert sm(ctx, None, 4, C.byref(p), cube, None, None) == INV
    assert b"NULL" in L.m2s_last_error()
    assert sm(ctx, rec + 8, 4, C.byref(p), cube, None, None) == INV and b"aligned" in L.m2s_last_error()
    assert sm(ctx, rec, 4, C.byref(p), cube, lq + 4, None) == INV
    assert sm(ctx, rec, 4, C.byref(p), cube + 2, None, None) == INV
    assert sm(ctx, rec, 1 << 30, C.byref(p), cube, None, None) == INV and b"2^30" in L.m2s_last_error()
    assert enq(ctx, rec, 4, None, C.byref(p), cube, None, 1 << 30, None, None, None) == INV
    for size in (0, 1025, 4096):
        pp = _abi.make_shadow_params(np.eye(4), (0, 0, 0), (0.1, 10), (64, 64), 0.01, 0, size)
        assert sm(ctx, rec, 4, C.byref(pp), cube, None, None) == INV
    assert b"1..1024" in L.m2s_last_error()
    pp = _abi.make_shadow_params(np.eye(4), (0, 0, 0), (0.1, 10), (64, 64), 0.01, 2, 64)
    assert sm(ctx, rec, 4, C.byref(pp), cube, None, None) == INV and b"layouts" in L.m2s_last_error()

    img = 0x90000
    full = _gbuf(position=0x20000, normal=0x28000, albedo=0x30000, metallic_roughness=0x38000)
    dl = lambda g, c, lp, im=img: L.m2s_deferred_light(ctx, C.byref(g), c, C.byref(lp), im)   # noqa: E731
    lp = _abi.make_light_params(64, 32, 6, shadow_size=64)
    assert L.m2s_deferred_light(None, C.byref(full), cube, C.byref(lp), img) == INV
    assert dl(full, cube, lp, None) == INV
    assert L.m2s_deferred_light_enqueue(ctx, None, cube, C.byref(lp), img, None) == INV
    for wh in ((0, 32), (64, 0), (4097, 32), (64, 4097)):
        assert dl(full, cube, _abi.make_light_params(wh[0], wh[1], 0)) == INV
    assert b"4096" in L.m2s_last_error()
    assert dl(full, cube, _abi.make_light_params(64, 32, 7)) == INV
    assert dl(full, None, lp) == INV and b"needs" in L.m2s_last_error()   # mode 6 without the cube
    for drop in ("position", "normal", "albedo", "metallic_roughness"):
        g = _gbuf(**{k: getattr(full, k) for k in ("position", "normal", "albedo", "metallic_roughness") if k != drop})
        assert dl(g, cube, lp) == INV
    assert dl(_gbuf(albedo=0x30000), None, _abi.make_light_params(64, 32, 5)) == INV   # mode 5 needs MR
    assert dl(_gbuf(metallic_roughness=0x38000), None, _abi.make_light_params(64, 32, 0)) == INV   # every mode needs albedo
    assert dl(full, cube, _abi.make_light_params(64, 32, 6, shadow_size=1025)) == INV
    assert dl(_gbuf(albedo=0x30002), None, _abi.make_light_params(64, 32, 0)) == INV and b"aligned" in L.m2s_last_error()
    assert dl(_gbuf(albedo=0x30000), None, _abi.make_light_params(64, 32, 0), img + 1) == INV


def test_no_gpu_gives_nogpu():
    from test_abi_host import _has_gpu
    if _has_gpu():
        pytest.skip("a CUDA device is present")
    L = _lib.lib()
    ctx = C.cast(C.create_string_buffer(4096), C.c_void_p)
    p = _abi.make_shadow_params(np.eye(4), (0, 0, 0), (0.1, 10), (64, 64), 0.01, 0, 64)
    assert L.m2s_shadow_map(ctx, 0x10000, 4, C.byref(p), 0x40000, None, None) == _abi.M2S_E_NOGPU
    assert L.m2s_shadow_map_enqueue(ctx, 0x10000, 4, None, C.byref(p), 0x40000, None, 10, None, None, None) == _abi.M2S_E_NOGPU
    g = _gbuf(albedo=0x30000)
    lp = _abi.make_light_params(64, 32, 0)
    assert L.m2s_deferred_light(ctx, C.byref(g), None, C.byref(lp), 0x90000) == _abi.M2S_E_NOGPU
    assert L.m2s_deferred_light_enqueue(ctx, C.byref(g), None, C.byref(lp), 0x90000, None) == _abi.M2S_E_NOGPU


# ---- the oracle against the reference's own shaders (tests/golden/ref_light_vectors.npz) --------------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_light_vectors.npz")
PREPASS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_prepass_vectors.npz")
SPLAT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_splat_vectors.npz")


def same_bits_nan(a, b) -> bool:
    """Bit for bit, with any NaN equal to any NaN (payloads are not part of the contract)."""
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.parametrize("case", range(5))
def test_light_prepass_matches_the_reference(case):
    """Light records (mean, axes, the cube pixel shader's depth, face) of the reference's compute shader, for four light
    placements per case: outside, inside (all six faces), on a diagonal (face ties) and at a gaussian."""
    z, zp = np.load(GOLDEN), np.load(PREPASS)
    g, prm, M = z[f"lg{case}"], zp[f"params{case}"], zp[f"model{case}"]
    faces = set()
    for k, lp in enumerate(z[f"lights{case}"]):
        p = _abi.make_shadow_params(M, tuple(float(v) for v in lp), (prm[2], prm[3]), (prm[0], prm[1]), prm[4], 0, 64)
        got, want = light.prepass(g, len(g), p), z[f"rec{case}_{k}"]
        assert same_bits_nan(got[:, :7], want[:, :7]) and np.array_equal(got[:, 7].view(np.uint32), want[:, 7].view(np.uint32)), (case, k)
        f = want[:, 7].view(np.uint32)
        faces |= set(f[f < 6].tolist())
    assert faces == set(range(6))


@pytest.mark.parametrize("case", range(5))
def test_cube_maps_match_the_reference(case):
    """The whole shadow pass (dispatch, six face draws, D24, LESS) with the light inside the cloud, S = 64."""
    z, zp = np.load(GOLDEN), np.load(PREPASS)
    g, prm, M = z[f"lg{case}"], zp[f"params{case}"], zp[f"model{case}"]
    p = _abi.make_shadow_params(M, tuple(float(v) for v in z["lights0"][1]), (prm[2], prm[3]), (prm[0], prm[1]), prm[4], 0, 64)
    want = z[f"cube{case}"]
    got = light.cube(light.prepass(g, len(g), p), 64)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int((got != want).sum())
    assert (want < 1.0).sum() > 100


def test_pixel_shader_invocations_match_the_reference():
    """2 400 invocations of gaussianSplattingDeferredPS.glsl on random texels (zeros, fp16 inf / NaN, negative normals,
    all modes): the oracle's FragColor bit for bit, NaN as NaN."""
    z = np.load(GOLDEN)
    cube = z["cube0"]
    n = 0
    for pos, nrm, alb, mr, q, want in zip(z["fs_pos"], z["fs_nrm"], z["fs_alb"], z["fs_mr"], z["fs_params"], z["fs_out"]):
        p = _abi.make_light_params(1, 1, int(q[11]), tuple(q[0:3]), tuple(q[3:6]), float(q[6]), tuple(q[7:10]), float(q[10]), 64)
        assert same_bits_nan(light.deferred_fs(pos, nrm, alb, mr, cube, p), want), n
        n += 1
    assert n >= 2000 and np.isnan(z["fs_out"]).any()
    assert np.isinf(z["fs_pos"].view(np.float16)).any() and np.isnan(z["fs_nrm"].view(np.float16)).any()


def test_pcf_at_the_bias_threshold_matches_the_reference():
    """Cube values exactly at currentDepth - 0.05 and one ulp either side: the comparison flips only below."""
    z = np.load(GOLDEN)
    outs = []
    for pos, lp, v, want in zip(z["th_pos"], z["th_light"], z["th_v"], z["th_out"]):
        p = _abi.make_light_params(1, 1, 6, tuple(float(c) for c in lp), (1.0, 1.0, 1.0), 5.0, (0.0, 0.0, 4.0), 1.0, 1)
        got = light.deferred_fs(pos, np.array([0.6, 0.7, 0.8, 1], np.float16), np.array([200, 150, 100, 255], np.uint8),
                                np.array([0, 128, 0, 255], np.uint8), np.full(6, v, F32), p)
        assert same_bits_nan(got, want)
        outs.append(got)
    t = np.array(outs).reshape(-1, 3, 4)
    assert (t[:, 1] == t[:, 0]).all() and (t[:, 2] != t[:, 0]).any(-1).all()


@pytest.mark.parametrize("case", range(5))
def test_images_match_the_reference(case):
    """The full lighting pass in modes 0-6 over the splat draw's golden G-buffers, RGBA8 bit for bit."""
    z, zs = np.load(GOLDEN), np.load(SPLAT)
    w, h = (int(v) for v in zs["img_size"])
    gb = {t: zs[f"img{case}_{t}"] for t in ("position", "normal", "albedo", "metallic_roughness")}
    for mode in range(7):
        p = _abi.make_light_params(w, h, mode, tuple(float(v) for v in z["lights0"][0]), (1.0, 0.9, 0.8), 25.0, (3.0, 2.0, 4.0), 100.0, 64)
        got, want = light.deferred_light(gb, z["cube0"], p), z[f"img{case}_{mode}"]
        assert np.array_equal(got, want), (mode, int((got != want).any(-1).sum()))
