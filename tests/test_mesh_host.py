"""The checker of the viewer's mesh G-buffer pass and of the split-screen composite (SURVEY 8 row 14) on the CPU: its
vertex and fragment stages against the reference's own meshRenderVS/PS.glsl (tests/golden/ref_mesh_vectors.npz), the
fixed fp64 sequences (log2 of the LOD, the sin of render mode 3), the host's normal matrix, the level rule, the nearest
surface against an fp64 ray cast, back-face culling, clipped against unclipped geometry, and the split column rule
against a literal restatement of the reference's scissor and stencil steps."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from oracle import mesh

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

EYE = np.eye(4, dtype=np.float32)
GOLDEN = os.path.join(HERE, "golden", "ref_mesh_vectors.npz")
HASH_ARGS = ((311.7, 0.0), (269.5, 1.3), (183.3, 2.7))


def _camera(eye, target, aspect, near=0.1, far=10.0, fov=60.0):
    V = column_major(look_at(np.array(eye, np.float64), np.array(target, np.float64), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(fov), aspect, near, far))
    return V, P


def _soup(pos, uv=None):
    """(T, 36) triangles from (T, 3, 3) positions; normal +z, tangent +x, uv = the given (T, 3, 2) or xy."""
    pos = np.asarray(pos, np.float32)
    t = np.zeros((len(pos), 36), np.float32)
    for k in range(3):
        t[:, 12 * k: 12 * k + 3] = pos[:, k]
        t[:, 12 * k + 5] = 1.0
        t[:, 12 * k + 6] = 1.0
        t[:, 12 * k + 9] = 1.0
        t[:, 12 * k + 10: 12 * k + 12] = pos[:, k, :2] if uv is None else np.asarray(uv, np.float32)[:, k]
    return t


def _scene(tris, factor=(0.8, 0.6, 0.4, 1.0), textures=(), maps=(-1, -1, -1)):
    return _abi.Scene(tris, [_abi.Primitive(0, len(tris), factor, *maps)], list(textures))


def test_log2_and_sin_sequences():
    rng = np.random.default_rng(1)
    for x in np.concatenate([2.0 ** rng.uniform(-140, 120, 500), [1.0, 2.0, 0.5, 3.0, 1e-45]]):
        assert abs(mesh.log2(x) - np.log2(x)) <= 4e-15 * max(1.0, abs(np.log2(x)))
    assert mesh.log2(0.0) == -np.inf and mesh.log2(np.inf) == np.inf and np.isnan(mesh.log2(np.nan))
    for x in np.concatenate([rng.uniform(-1e5, 1e5, 2000), [0.0, 1e-300, np.pi / 2, np.pi]]):
        assert abs(mesh.sin(x) - np.sin(x)) <= 2e-16 * max(1.0, abs(x) * 1e-5) + 1e-300
    assert np.isnan(mesh.sin(np.inf)) and np.isnan(mesh.sin(np.nan))


def test_vertex_stage_equals_the_reference_shader():
    """Every golden vertex invocation (two cameras x five model matrices, among them a mirrored, a non-uniformly scaled
    and a sheared one; zero, huge and tangent-parallel normals): gl_Position and the 13 varyings bit for bit, with the
    normal matrix from the host's GLM fp32 inverse."""
    z = np.load(GOLDEN)
    for c in range(len(z["vs_vtx"])):
        clip, vary = mesh.vs_vertices(z["vs_vtx"][c], z["vs_V"][c], z["vs_P"][c], z["vs_M"][c])
        assert np.array_equal(clip.view(np.uint32), z["vs_clip"][c].view(np.uint32)), c
        assert np.array_equal(vary.view(np.uint32), z["vs_vary"][c].view(np.uint32)), c


def _hash(s):
    v = np.float32(s) * np.float32(43758.5453)
    return np.float32(v - np.floor(v))


def test_fragment_stage_equals_the_reference_shader():
    """Every golden fragment invocation (every render mode, every combination of bound maps, zero and normal-parallel
    tangents, texels outside [0, 1]) bit for bit.  Render mode 3's colour is the one exception: there the shader called
    the C library's sinf, the pass its fixed sin (correctly rounded on these arguments); a channel may differ only where
    the two differ by one ulp, and then equals fract(sinf * 43758.5453).  Those channels are counted and bounded."""
    z = np.load(GOLDEN)
    n = len(z["fs_mode"])
    differing = mode3_channels = 0
    for i in range(n):
        got = mesh.fs(z["fs_vary"][i], z["fs_tex"][i], z["fs_has"][i], z["fs_factor"][i], z["fs_near_far"][i], z["fs_mode"][i],
                      z["fs_prim"][i])
        want = z["fs_out"][i]
        bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
        if z["fs_mode"][i] != 3:
            assert len(bad) == 0, (i, int(z["fs_mode"][i]), bad, got, want)
            continue
        mode3_channels += 3
        assert set(bad.tolist()) <= {8, 9, 10}, (i, bad)
        for ch in bad:
            m, c = HASH_ARGS[ch - 8]
            arg = np.float32(np.float32(z["fs_prim"][i]) * np.float32(m) + np.float32(c))
            fixed, libc = np.float32(mesh.sin(float(arg))), z["fs_sinf"][i][ch - 8]
            assert abs(int(fixed.view(np.int32)) - int(libc.view(np.int32))) == 1, (i, ch)
            assert _hash(libc) == want[ch], (i, ch)
            differing += 1
    assert mode3_channels > 0 and differing <= 0.05 * mode3_channels, (differing, mode3_channels)


def test_fixed_sin_is_correctly_rounded_on_mode3_arguments():
    """The fixed sin rounded to fp32 equals the correctly rounded sin of render mode 3's arguments, up to gl_PrimitiveID
    2^24 (the reduction's products are exact there)."""
    rng = np.random.default_rng(3)
    ids = np.concatenate([np.arange(2000), rng.integers(0, 1 << 24, 3000)])
    for i in ids:
        for m, c in HASH_ARGS:
            arg = np.float32(np.float32(i) * np.float32(m) + np.float32(c))
            assert np.float32(mesh.sin(float(arg))) == np.float32(np.sin(np.float64(arg))), (i, m)


def test_level_rule_and_non_finite_rho():
    """The LOD rule of DESIGN §2: magnification and lambda <= 0 on level 0, the blend between floor(lambda) and the next
    level, the clamp at the last level, and a non-finite rho: NaN (0 / 0 or inf - inf in the quad's steps) samples level
    0, +inf the last level."""
    assert mesh.level(64, 64, 5, 1 / 128, 0, 0, 1 / 128) == (0, 0.0)
    l0, f = mesh.level(64, 64, 5, 0.1, 0.0, 0.0, 0.05)
    assert l0 == 2 and 0.67 < f < 0.69   # log2(6.4) = 2.678
    assert mesh.level(64, 64, 5, 1e3, 0, 0, 0) == (4, 0.0)
    assert mesh.level(37, 23, 6, 1e3, 0, 0, 0)[0] == 5
    for bad in ((np.nan, 0, 0, 0), (0, 0, 0, np.nan), (np.inf, -np.inf, 0, 0), (np.nan, np.inf, 0, 0)):
        assert mesh.level(64, 64, 5, *bad)[0] in (0, 4)
    assert mesh.level(64, 64, 5, np.nan, 0, 0, 0) == (0, 0.0)
    assert mesh.level(64, 64, 5, 0, 0, np.nan, 1.0) == (0, 0.0)
    assert mesh.level(64, 64, 5, np.inf, 0, 0, 0) == (4, 0.0)
    assert mesh.level(64, 64, 5, 0, 3e38, 0, 0) == (4, 0.0)   # rho^2 overflows to +inf


def test_normal_matrix_is_the_inverse_transpose():
    rng = np.random.default_rng(2)
    for _ in range(50):
        A = rng.normal(size=(4, 4)).astype(np.float32)
        A[3] = (0, 0, 0, 1)
        N = mesh.normal_matrix(column_major(A))
        want = np.linalg.inv(A.astype(np.float64)).T[:3, :3]
        assert np.allclose(N.reshape(3, 3).T, want, rtol=1e-4, atol=1e-4 * np.abs(want).max())
    S = np.eye(4, dtype=np.float32)
    S[1, 1] = 0.0
    assert mesh.normal_matrix(column_major(S)) is None


def test_nearest_surface_equals_an_fp64_ray_cast():
    """Two overlapping quads at z = -2 and z = -3 (the nearer drawn second): every pixel away from the edges shows the
    nearer one, at the world position where the pixel centre's ray meets it (fp16 position target)."""
    W, H = 40, 30
    V, P = _camera((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), W / H)
    quad = lambda z, s: [[(-s, -s, z), (s, -s, z), (s, s, z)], [(-s, -s, z), (s, s, z), (-s, s, z)]]
    scene = _scene(_soup(quad(-3.0, 4.0) + quad(-2.0, 0.6)))
    g = mesh.mesh_render(scene, V, P, EYE, W, H, (0.1, 10.0))
    pos = g["position"].astype(np.float64)
    Pm = perspective(np.radians(60.0), W / H, 0.1, 10.0).astype(np.float64)
    checked = 0
    for j in range(H):
        for i in range(W):
            ndc = np.array([(i + 0.5) / W * 2 - 1, (j + 0.5) / H * 2 - 1])
            d = np.array([ndc[0] / Pm[0, 0], ndc[1] / Pm[1, 1], -1.0])   # view ray through the pixel centre
            hit = None
            for z, s in ((-2.0, 0.6), (-3.0, 4.0)):
                p = d * (-z)
                if abs(p[0]) < s - 0.02 and abs(p[1]) < s - 0.02:
                    hit = p
                    break
                if abs(abs(p[0]) - s) < 0.02 or abs(abs(p[1]) - s) < 0.02:
                    hit = "edge"
                    break
            if hit is None or isinstance(hit, str):
                continue
            assert pos[j, i, 3] == 1.0
            assert np.allclose(pos[j, i, :3], hit, rtol=2e-3, atol=2e-3), (i, j, pos[j, i], hit)
            checked += 1
    assert checked > W * H // 2


def test_culling_and_mirrored_model_matrix():
    W, H = 16, 16
    V, P = _camera((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), 1.0)
    ccw = [[(-1, -1, -2), (1, -1, -2), (0, 1, -2)]]
    cw = [[(-1, -1, -2), (0, 1, -2), (1, -1, -2)]]
    cov = lambda tris, M: mesh.mesh_render(_scene(_soup(tris)), V, P, M, W, H, (0.1, 10.0))["albedo"][..., 3] > 0
    assert cov(ccw, EYE).sum() > 20
    assert cov(cw, EYE).sum() == 0
    mirror = column_major(np.diag([-1.0, 1.0, 1.0, 1.0]).astype(np.float32))
    assert cov(ccw, mirror).sum() == 0
    assert cov(cw, mirror).sum() > 20


def test_clipped_and_unclipped_geometry_agree_inside_the_viewport():
    """One wall at z = -2 drawn as two huge triangles (clipped by the guard band) and as a grid of small ones (no
    clipping): the same pixels are covered, and the interpolated world positions, view depths and uvs agree.  The uv is
    read back through a uv-coded map (red = 4 x column, green = 4 x row, magnified: bilinear on level 0).  One tolerance:
    the targets' own rounding, 1/1024 on fp16 values in [0, 4] and one step on RGBA8."""
    W, H = 48, 36
    V, P = _camera((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), W / H)
    big = [[(-400, -400, -2), (400, -400, -2), (400, 400, -2)], [(-400, -400, -2), (400, 400, -2), (-400, 400, -2)]]
    small = []
    e = np.linspace(-3, 3, 13)
    for a in range(12):
        for b in range(12):
            x0, x1, y0, y1 = e[a], e[a + 1], e[b], e[b + 1]
            small += [[(x0, y0, -2), (x1, y0, -2), (x1, y1, -2)], [(x0, y0, -2), (x1, y1, -2), (x0, y1, -2)]]
    ramp = np.zeros((64, 64, 4), np.uint8)
    ramp[..., 0] = (np.arange(64) * 4)[None, :]
    ramp[..., 1] = (np.arange(64) * 4)[:, None]
    ramp[..., 3] = 255
    uvs = lambda tris: np.asarray(tris, np.float32)[..., :2] * np.float32(0.08) + np.float32(0.5)
    g = [mesh.mesh_render(_scene(_soup(t, uv=uvs(t)), factor=(1, 1, 1, 1), textures=[ramp], maps=(0, -1, -1)), V, P, EYE, W, H,
                          (0.1, 10.0)) for t in (big, small)]
    assert (g[0]["albedo"][..., 3] == 255).all() and (g[1]["albedo"][..., 3] == 255).all()
    for t, tol in (("position", 1 / 1024), ("depth", 1 / 1024), ("albedo", 1)):
        a, b = g[0][t].astype(np.float64), g[1][t].astype(np.float64)
        assert np.abs(a - b).max() <= tol, (t, np.abs(a - b).max())
    assert len(np.unique(g[0]["albedo"][..., 0])) > 10 and len(np.unique(g[0]["albedo"][..., 1])) > 10   # the uv varies


def test_near_plane_clipped_triangle_keeps_finite_attributes():
    """A triangle through the camera plane: clipped at the near plane, every covered pixel gets finite world positions."""
    W, H = 32, 32
    V, P = _camera((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), 1.0)
    tex = synth.random_texture(64, 64, 5)
    tri = [[(-2, -1, 1.0), (2, -1, 1.0), (0, 0.5, -3.0)]]
    scene = _scene(_soup(tri, uv=[[(0, 0), (8, 0), (4, 8)]]), textures=[tex], maps=(0, -1, -1))
    g = mesh.mesh_render(scene, V, P, EYE, W, H, (0.1, 10.0))
    cov = g["albedo"][..., 3] == 255
    assert cov.sum() > 10
    assert np.isfinite(g["position"][cov].astype(np.float32)).all()


def _split_literal(left, right, position):
    """GaussianRelightingPass.cpp:90-135 step by step: stencil cleared to 0, the scissor (0, 0, splitPixelX, h) cleared
    to 1, the splat side drawn where stencil == 0 and the mesh side where it is 1, then the scissored white clear."""
    h, w = left.shape[:2]
    split = int(np.float32(position) * np.float32(w))
    stencil = np.zeros((h, w), np.uint8)
    stencil[:, 0:max(0, min(split, w))] = 1
    out = np.where(stencil[..., None] == 0, right, left)
    x = max(0, split - 1)
    out[:, x:min(w, x + 2)] = 255
    return out


@pytest.mark.parametrize("w", [1, 2, 7, 640])
def test_split_column_rule(w):
    rng = np.random.default_rng(w)
    left = rng.integers(0, 255, size=(3, w, 4), dtype=np.uint8)
    right = rng.integers(0, 255, size=(3, w, 4), dtype=np.uint8)
    for pos in (0.0, 0.5, 1.0, 0.3, 1.0 / 3.0, 0.999, 5.0 / w, np.nextafter(np.float32(0.5), np.float32(0))):
        assert np.array_equal(mesh.split(left, right, pos), _split_literal(left, right, pos)), pos
