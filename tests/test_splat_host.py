"""CPU tests of the viewer's splat draw (row f-6, GaussianSplattingPass::execute): the C restatement (orc_splat_*)
against the reference's own shaders (tests/golden/ref_splat_vectors.npz), its exp against fp64, its coverage against a
brute-force pixel-centre test, and the argument checks of the C entry points, which return before any CUDA call."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import pytest

from mesh2splat_b200 import _abi, _lib
from oracle import splat

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_splat_vectors.npz")
PREPASS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_prepass_vectors.npz")


def prepass_quads_sorted(i: int) -> np.ndarray:
    """The quads of prepass golden case i, stably sorted by the bits of their depth (the depth sort's order)."""
    z = np.load(PREPASS)
    q, d = z[f"quads{i}"], z[f"depths{i}"]
    return np.ascontiguousarray(q[np.argsort(d.view(np.uint32), kind="stable")])


def same_bits(a: np.ndarray, b: np.ndarray) -> bool:
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def test_vertex_shader_invocations_match_the_reference():
    z = np.load(GOLDEN)
    for q, v, res, want in zip(z["vs_quads"], z["vs_vertex"], z["vs_resolution"], z["vs_out"]):
        assert same_bits(splat.vs(q, int(v), float(res[0]), float(res[1])), want)


def test_fragment_shader_invocations_match_the_reference():
    z = np.load(GOLDEN)
    n = 0
    for var, xy, mode, want in zip(z["fs_varyings"], z["fs_fragcoord"], z["fs_mode"], z["fs_out"]):
        got = splat.fs(var, float(xy[0]), float(xy[1]), int(mode))
        assert same_bits(np.where(np.isnan(got), np.float32(np.nan), got), np.where(np.isnan(want), np.float32(np.nan), want))
        n += 1
    assert n >= 2000 and np.isnan(z["fs_out"]).any() and np.isinf(z["fs_out"]).any()


@pytest.mark.parametrize("case", range(5))
def test_images_match_the_reference(case):
    z = np.load(GOLDEN)
    w, h = (int(v) for v in z["img_size"])
    mode = int(z["img_modes"][case])
    got = splat.draw(prepass_quads_sorted(case), w, h, mode)
    for t, _ in splat.TARGETS:
        want = z[f"img{case}_{t}"]
        assert same_bits(got[t], want), (t, int((got[t].view(np.uint8) != want.view(np.uint8)).sum()))
    assert (got["albedo"][..., 3] > 0).sum() > 100   # the case draws something


def test_exp_against_fp64():
    """The exp of DESIGN §2 stays within 2 ulp of exp over the range the fragment shader reaches ((-inf, 0] in practice,
    up to the overflow bound for odd conics), and gives 0 below the underflow bound, inf above the overflow bound."""
    rng = np.random.default_rng(1)
    x = np.concatenate([-rng.uniform(0, 104, 40000), rng.uniform(0, 88.72, 10000), -np.logspace(-8, 0, 2000),
                        [0.0, -0.0, -1e-30, 1e-30, -87.33, -103.9]]).astype(np.float32)
    got = splat.exp(x).astype(np.float64)
    want = np.exp(x.astype(np.float64))
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got - want) / ulp
    assert err.max() <= 2.0, (err.max(), x[np.argmax(err)])
    assert splat.exp(np.array([-104.0, -1e4, -np.inf], np.float32)).tolist() == [0.0, 0.0, 0.0]
    assert np.isinf(splat.exp(np.array([88.75, 1e4, np.inf], np.float32))).all()
    assert np.isnan(splat.exp(np.array([np.nan], np.float32))).all()


def random_parallelograms(rng, n: int, w: int, h: int) -> np.ndarray:
    q = np.zeros((n, 24), np.float32)
    q[:, 0:2] = rng.uniform(-1.2, 1.2, (n, 2))
    q[:, 4:8] = rng.normal(0, 1, (n, 4)) * rng.choice([0.002, 0.02, 0.2], (n, 1))
    q[:, 8:12] = rng.random((n, 4))
    q[:, 12:15] = rng.random((n, 3)) * 0.01
    return q


def brute_force_coverage(q: np.ndarray, tri: int, w: int, h: int) -> np.ndarray:
    """Pixel centres inside the snapped triangle, by the sign of each edge's cross product with the top-left rule,
    over the whole viewport in Python integers."""
    corners = np.array([[-1, -1], [-1, 1], [1, 1], [1, -1]], np.float32)
    X, Y = [], []
    for vx, vy in corners:
        nx = q[0] + (vx * q[4] + vy * q[6]); ny = q[1] + (vx * q[5] + vy * q[7])
        xw = np.float32(nx * np.float32(w * 0.5) + np.float32(w * 0.5)); yw = np.float32(ny * np.float32(h * 0.5) + np.float32(h * 0.5))
        X.append(int(np.rint(np.float32(xw * np.float32(256))))); Y.append(int(np.rint(np.float32(yw * np.float32(256)))))
    idx = [(0, 1, 2), (0, 2, 3)][tri]
    px, py = [X[i] for i in idx], [Y[i] for i in idx]
    area = (px[1] - px[0]) * (py[2] - py[0]) - (px[2] - px[0]) * (py[1] - py[0])
    mask = np.zeros((h, w), bool)
    if area == 0:
        return mask
    s = 1 if area > 0 else -1
    cy, cx = np.mgrid[0:h, 0:w].astype(np.int64) * 256 + 128
    inside = np.ones((h, w), bool)
    for k in range(3):
        ax, ay, bx, by = px[(k + 1) % 3], py[(k + 1) % 3], px[(k + 2) % 3], py[(k + 2) % 3]
        e = s * ((bx - ax) * (cy - ay) - (by - ay) * (cx - ax))
        a, b = s * (ay - by), s * (bx - ax)
        inside &= (e > 0) | ((e == 0) & ((a > 0) | ((a == 0) & (b > 0))))
    return inside


def test_coverage_against_brute_force_and_shared_edge_once():
    """10 000 random parallelograms: each triangle's coverage equals the brute-force pixel-centre test, and the two
    triangles of a quad whose snapped corners form a parallelogram (they share the diagonal exactly) cover every
    interior pixel exactly once."""
    rng = np.random.default_rng(7)
    w, h = 48, 40
    qs = random_parallelograms(rng, 10_000, w, h)
    overlaps = 0
    for q in qs:
        m0, m1 = splat.coverage(q, 0, w, h), splat.coverage(q, 1, w, h)
        assert np.array_equal(m0, brute_force_coverage(q, 0, w, h))
        assert np.array_equal(m1, brute_force_coverage(q, 1, w, h))
        overlaps += int((m0 & m1).sum())
    assert overlaps == 0   # the diagonal V0-V2 is shared exactly: the top-left rule gives its pixels to one triangle


def test_pair_counts_cover_every_drawn_tile():
    """Every tile a quad covers a pixel of is among the tiles its pairs name (the tile test is conservative)."""
    rng = np.random.default_rng(3)
    w, h = 70, 50
    qs = random_parallelograms(rng, 300, w, h)
    counts, total = splat.pairs(qs, w, h)
    assert total == int(counts.sum())
    for q, c in zip(qs, counts):
        m = splat.coverage(q, 0, w, h) | splat.coverage(q, 1, w, h)
        ys, xs = np.nonzero(m)
        assert len(set(zip(ys // 16, xs // 16))) <= c


def _gbuf(**kw):
    g = _abi.m2s_gbuffer()
    for k, v in kw.items():
        setattr(g, k, v)
    return g


def test_splat_entry_points_reject_bad_arguments_without_a_gpu():
    L = _lib.lib()
    INV = _abi.M2S_E_INVALID
    ctx = C.cast(C.create_string_buffer(4096), C.c_void_p)
    q = 0x10000
    g = _gbuf(position=0x20000, albedo=0x30000)
    p = _abi.m2s_splat_params(64, 32, 0)
    enq = lambda *a: L.m2s_splat_draw_enqueue(*a)   # noqa: E731
    assert L.m2s_splat_draw(None, q, 4, C.byref(p), C.byref(g), None) == INV
    assert enq(None, q, 4, None, C.byref(p), C.byref(g), 100, None, None, None) == INV
    assert b"NULL" in L.m2s_last_error()
    assert enq(ctx, None, 4, None, C.byref(p), C.byref(g), 100, None, None, None) == INV   # NULL quads, n > 0
    for qq in (q + 4, q + 8):
        assert enq(ctx, qq, 4, None, C.byref(p), C.byref(g), 100, None, None, None) == INV
    assert b"aligned" in L.m2s_last_error()
    for n in (1 << 30, 1 << 40):
        assert L.m2s_splat_draw(ctx, q, n, C.byref(p), C.byref(g), None) == INV
    assert b"2^30" in L.m2s_last_error()
    assert enq(ctx, q, 4, None, C.byref(p), C.byref(g), 1 << 30, None, None, None) == INV
    for wh in ((0, 32), (64, 0), (4097, 32), (64, 4097)):
        pp = _abi.m2s_splat_params(wh[0], wh[1], 0)
        assert L.m2s_splat_draw(ctx, q, 4, C.byref(pp), C.byref(g), None) == INV
    assert b"4096" in L.m2s_last_error()
    for mode in (7, 100):
        pp = _abi.m2s_splat_params(64, 32, mode)
        assert L.m2s_splat_draw(ctx, q, 4, C.byref(pp), C.byref(g), None) == INV
    assert L.m2s_splat_draw(ctx, q, 4, C.byref(p), C.byref(_gbuf()), None) == INV
    assert b"no targets" in L.m2s_last_error()
    assert L.m2s_splat_draw(ctx, q, 4, C.byref(p), None, None) == INV
    assert L.m2s_splat_draw(ctx, q, 4, C.byref(p), C.byref(_gbuf(normal=0x20004)), None) == INV   # fp16 target not 8-aligned


def test_no_gpu_gives_nogpu():
    from test_abi_host import _has_gpu
    if _has_gpu():
        pytest.skip("a CUDA device is present")
    L = _lib.lib()
    ctx = C.cast(C.create_string_buffer(4096), C.c_void_p)   # device 0, never reached past cudaSetDevice
    p = _abi.m2s_splat_params(64, 32, 0)
    g = _gbuf(albedo=0x30000)
    assert L.m2s_splat_draw(ctx, 0x10000, 4, C.byref(p), C.byref(g), None) == _abi.M2S_E_NOGPU
    assert L.m2s_splat_draw_enqueue(ctx, 0x10000, 4, None, C.byref(p), C.byref(g), 10, None, None, None) == _abi.M2S_E_NOGPU
