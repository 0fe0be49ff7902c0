"""A loaded .ply's view-dependent colour on the GPU (beyond the reference, which skips the SH rest coefficients):
m2s_ply_read_sh / m2s_ply_decode_sh_enqueue against a numpy gather of the file's f_rest bytes, and m2s_prepass_sh against
the C restatement (oracle/m2s_sh_oracle.c) and against m2s_prepass.

Accuracy rule: bit for bit.  The SH buffer holds the file's bytes; the records read with and without it are identical.
The prepass's quad colour (words 8-10 in render modes 0 and 6) equals orc_prepass_sh's; every other word equals
m2s_prepass's on the same input (the SH variant changes the colour and nothing else), and the survivors are the
restatement's.  m2s_prepass itself is held against orc_prepass within util.assert_prepass_match's bounds by
test_gpu_ply_load.py and test_gpu_parity.py: the conic and the axes are ill-conditioned for the near, large splats the
camera inside the capture sees here."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

from mesh2splat_b200 import _abi, api
from mesh2splat_b200._lib import check, lib
from oracle import sh as osh
from util import GuardedDevice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_ply_load import PBR, STANDARD, ply, vertex_rows  # noqa: E402
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "ref_ply_load_vectors.npz"))
NAMES = [str(n) for n in Z["names"]]
ACCEPTED = [n for n in NAMES if int(Z[f"ok_{n}"]) and not int(Z[f"dev_{n}"])]
STAGE_ROWS_256 = (32 << 20) // 256   # rows of one staging block of the degree-3 PBR layout (64 floats)


def _write(tmp_path, name, data: bytes) -> str:
    p = str(tmp_path / f"{name}.ply")
    with open(p, "wb") as f:
        f.write(data)
    return p


def _rest_file(tmp_path, rng, n, degree, prefix=(), pad=(), name="sh", fill=None):
    """n rows: `prefix`, then the standard and PBR properties and f_rest_0 .. f_rest_{3K-1} in shuffled order, then `pad`."""
    K = (degree + 1) ** 2 - 1
    core = [("float", k) for k in STANDARD + PBR] + [("float", f"f_rest_{k}") for k in range(3 * K)]
    props = list(prefix) + [core[i] for i in rng.permutation(len(core))] + list(pad)
    return _write(tmp_path, name, ply([("vertex", n, props, vertex_rows(rng, props, n, fill))]))


def _want_sh(path, info) -> np.ndarray:
    """The SH buffer m2s_ply_read_sh must write: the file's f_rest bytes gathered coefficient-major, zero padding;
    [n, M2S_SH_FLOATS] uint32 words."""
    n, d = info.vertex_count, info.sh_degree
    K = (d + 1) ** 2 - 1
    with open(path, "rb") as f:
        f.seek(info.body_offset)
        body = np.frombuffer(f.read(n * info.row_stride), np.uint8).reshape(n, info.row_stride)
    words = np.stack([body[:, o: o + 4].copy().view(np.uint32)[:, 0] for o in info.f_rest[: 3 * K]], 1)   # file order
    out = np.zeros((n, _abi.SH_FLOATS[d]), np.uint32)
    out[:, : 3 * K] = words.reshape(n, 3, K).transpose(0, 2, 1).reshape(n, 3 * K)
    return out


def _read_guarded(gpu_ctx, path, n, degree, what):
    """ply_read and ply_read_sh into guarded buffers: (records of ply_read, records of ply_read_sh, SH words [n, F])."""
    nf = _abi.SH_FLOATS[degree]
    g0, g1 = GuardedDevice(max(n, 1), 96, what=f"{what} records"), GuardedDevice(max(n, 1), 96, what=f"{what} records (sh)")
    import torch
    gs = GuardedDevice(max(n, 1), max(nf, 1) * 4, dtype=torch.float32, what=f"{what} sh")
    _, count0, _ = gpu_ctx.ply_read(path, out=g0.view)
    _, sh, count1, _, deg = gpu_ctx.ply_read_sh(path, out=g1.view, sh=gs.view)
    assert count0 == count1 == n and deg == degree, (what, count0, count1, deg)
    g0.check(n)
    g1.check(n)
    gs.check(n if nf else 0)
    rec0 = g0.view[: n * 96].cpu().numpy()
    rec1 = g1.view[: n * 96].cpu().numpy()
    words = sh.cpu().numpy().view(np.uint32) if sh is not None else None
    return rec0, rec1, words


# ---- the decode ---------------------------------------------------------------------------------------------------------
def test_read_sh_on_every_golden_fixture(gpu_ctx, tmp_path):
    """The records equal m2s_ply_read's bit for bit; a fixture with a full f_rest set (the reference writer's standard
    format: 45 zeros) gets its coefficients."""
    with_sh = 0
    for name in ACCEPTED:
        p = _write(tmp_path, name, Z[f"file_{name}"].tobytes())
        info = api.ply_parse_file(p)
        n = int(info.vertex_count)
        rec0, rec1, words = _read_guarded(gpu_ctx, p, n, int(info.sh_degree), name)
        assert np.array_equal(rec0, rec1), name
        if info.sh_degree:
            with_sh += 1
            assert np.array_equal(words, _want_sh(p, info)), name
    assert with_sh >= 1


@pytest.mark.parametrize("degree,n", [(d, n) for d in (1, 2, 3) for n in (1, 31, 32, 33, 1000)] + [(3, STAGE_ROWS_256 + 1)])
def test_sh_counts_around_warps_and_staging_blocks(gpu_ctx, tmp_path, degree, n):
    rng = np.random.default_rng(1000 * degree + n)
    p = _rest_file(tmp_path, rng, n, degree)
    info = api.ply_parse_file(p)
    assert info.sh_degree == degree
    rec0, rec1, words = _read_guarded(gpu_ctx, p, n, degree, f"degree {degree}, n = {n}")
    assert np.array_equal(rec0, rec1)
    assert np.array_equal(words, _want_sh(p, info))


@pytest.mark.parametrize("degree,prefix,pad", [
    (1, [("uchar", "red")], []),                                            # every float unaligned
    (2, [("uchar", "a"), ("ushort", "b")], [("uchar", "c")]),               # floats at 3 mod 4
    (3, [("char", "a")], [("double", f"p{k}") for k in range(479)]),        # stride 4089: two rows per warp pass
    (3, [], [("double", f"p{k}") for k in range(479)] + [("float", "q"), ("float", "r")]),   # stride 4096: the maximum
])
def test_sh_odd_strides_and_misaligned_rows(gpu_ctx, tmp_path, degree, prefix, pad):
    import torch
    rng = np.random.default_rng(len(pad) + degree)
    n = 700
    p = _rest_file(tmp_path, rng, n, degree, prefix, pad)
    info = api.ply_parse_file(p)
    assert info.sh_degree == degree
    want = _want_sh(p, info)
    rec0, rec1, words = _read_guarded(gpu_ctx, p, n, degree, f"stride {info.row_stride}")
    assert np.array_equal(rec0, rec1) and np.array_equal(words, want)
    with open(p, "rb") as f:
        f.seek(info.body_offset)
        body = np.frombuffer(f.read(n * info.row_stride), np.uint8)
    buf = torch.zeros(len(body) + 16, dtype=torch.uint8, device="cuda")
    nf = _abi.SH_FLOATS[degree]
    for mis in (1, 3, 8, 13):
        buf[mis: mis + len(body)] = torch.from_numpy(body.copy()).cuda()
        gr, gs = GuardedDevice(n, 96, what="records"), GuardedDevice(n, nf * 4, what="sh")
        torch.cuda.synchronize()
        check(lib().m2s_ply_decode_sh_enqueue(gpu_ctx.handle, C.byref(info), buf[mis:].data_ptr(), n, gr.view.data_ptr(), gs.view.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        gr.check(n)
        gs.check(n)
        assert np.array_equal(gr.view[: n * 96].cpu().numpy(), rec0), f"misaligned by {mis}"
        assert np.array_equal(gs.view[: n * nf * 4].cpu().numpy().view(np.uint32).reshape(n, nf), want), f"misaligned by {mis}"


def test_read_sh_capacity_and_degree_0(gpu_ctx, tmp_path):
    """A small SH buffer gives M2S_E_CAPACITY and writes nothing; a file of degree 0 writes no SH and returns None."""
    rng = np.random.default_rng(5)
    n = 100
    p = _rest_file(tmp_path, rng, n, 2)
    gr, gs = GuardedDevice(n, 96), GuardedDevice(n - 1, 96)
    info = _abi.m2s_ply_info()
    assert lib().m2s_ply_read_sh(gpu_ctx.handle, p.encode(), gr.view.data_ptr(), gs.view.data_ptr(), n - 1, C.byref(info)) == _abi.M2S_E_CAPACITY
    assert info.sh_degree == 2
    gr.check(0)
    gs.check(0)
    p0 = _rest_file(tmp_path, rng, n, 0, name="deg0")
    recs, sh, count, has_pbr, deg = gpu_ctx.ply_read_sh(p0)
    assert sh is None and deg == 0 and count == n and has_pbr
    assert np.array_equal(recs.cpu().numpy(), gpu_ctx.ply_read(p0)[0].cpu().numpy())


# ---- the prepass ----------------------------------------------------------------------------------------------------------
def _inputs(rng, n, buffer_degree, eye, rotated):
    g = np.zeros((n, 24), np.float32)
    g[:, 0:3] = (rng.random((n, 3)) - 0.5) * 2
    g[:, 3] = 1
    g[:, 4:7] = rng.normal(size=(n, 3)) * 0.28209479177387814 + 0.5
    g[:, 7] = rng.random(n)
    g[:, 8:11] = rng.random((n, 3)) * 0.05 + 0.001
    g[:, 12:15] = rng.normal(size=(n, 3))
    q = rng.normal(size=(n, 4))
    g[:, 16:20] = q / np.linalg.norm(q, axis=1, keepdims=True)
    g[:, 20:22] = rng.random((n, 2))
    nf = _abi.SH_FLOATS[buffer_degree]
    block = (rng.normal(size=(n, nf)) * 0.4).astype(np.float32)
    block[:, 3 * ((buffer_degree + 1) ** 2 - 1):] = 0
    V = column_major(look_at(np.asarray(eye, np.float64), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(60.0), 4 / 3, 0.01, 100.0))
    Mr = np.eye(4)
    if rotated:   # about an oblique axis, scaled non-uniformly, translated
        a, ax = np.radians(37.0), np.array([1.0, 2.0, -0.5]) / np.linalg.norm([1.0, 2.0, -0.5])
        Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
        Mr[:3, :3] = (np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx) @ np.diag([1.3, 0.7, 1.1])
        Mr[:3, 3] = (0.2, -0.1, 0.3)
    return g, block, V, P, column_major(Mr.astype(np.float32))


def _sorted_rows(q, cols):
    """The rows of q ordered by the bits of the given words: two outputs of one input set compared as multisets."""
    w = np.ascontiguousarray(q, np.float32).view(np.uint32)
    return w[np.lexsort(w[:, cols].T[::-1])]


def _run(gpu_ctx, g, block, layout, V, P, M, mode, sh_degree):
    import torch
    d = torch.from_numpy(g.view(np.uint8).reshape(-1).copy()).cuda()
    sh = torch.from_numpy(block).cuda()
    args = (d, len(g), layout, V, P, M, (800.0, 600.0), (0.01, 100.0), 1.0, mode)
    return gpu_ctx.prepass(*args, sh=sh, sh_degree=sh_degree), gpu_ctx.prepass(*args)


@pytest.mark.parametrize("buffer_degree,sh_degree", [(1, 1), (2, 2), (3, 3), (3, 1), (2, 1), (3, 2)])
@pytest.mark.parametrize("mode", [0, 1, 2, 6])
@pytest.mark.parametrize("rotated", [False, True])
def test_prepass_sh_matches_the_restatement(gpu_ctx, buffer_degree, sh_degree, mode, rotated):
    rng = np.random.default_rng(100 * buffer_degree + 10 * sh_degree + mode + 1000 * rotated)
    n = 20000
    eye = (0.4, 0.8, 3.0) if (mode + rotated) % 2 == 0 else (0.05, 0.1, 0.3)   # outside and inside the capture
    layout = _abi.VIEW_PLY_PBR if mode == 2 else _abi.VIEW_PLY
    g, block, V, P, M = _inputs(rng, n, buffer_degree, eye, rotated)
    (q, dep), (q0, dep0) = _run(gpu_ctx, g, block, layout, V, P, M, mode, sh_degree)
    wq, wd = osh.prepass_sh(g, V, P, M, (800.0, 600.0), (0.01, 100.0), 1.0, mode, layout == _abi.VIEW_PLY_PBR, block, buffer_degree, sh_degree)
    assert len(q) == len(q0) == len(wq) > 500
    # every word but the SH colour: m2s_prepass's, bit for bit (as multisets: atomic arrival order)
    colour = (8, 9, 10) if mode in (0, 6) else ()
    other = [c for c in range(24) if c not in colour]
    a, b = _sorted_rows(q, other), _sorted_rows(q0, other)
    assert np.array_equal(a[:, other], b[:, other])
    assert np.array_equal(np.sort(dep.view(np.uint32)), np.sort(dep0.view(np.uint32)))
    # the survivors are the restatement's: each quad paired with the restatement's at the same world position
    from scipy.spatial import cKDTree
    dist, idx = cKDTree(wq[:, 20:23].astype(np.float64)).query(q[:, 20:23].astype(np.float64))
    assert len(np.unique(idx)) == len(idx) and dist.max() < 1e-5
    if mode in (0, 6):   # the SH colour and the record's alpha: orc_prepass_sh's, bit for bit
        assert np.array_equal(q[:, 8:12].view(np.uint32), wq[idx, 8:12].view(np.uint32)), \
            f"{int((q[:, 8:12].view(np.uint32) != wq[idx, 8:12].view(np.uint32)).any(axis=1).sum())} colours differ"
        assert not np.array_equal(np.sort(q[:, 8]), np.sort(q0[:, 8]))


def test_prepass_sh_degree_0_is_the_prepass(gpu_ctx):
    rng = np.random.default_rng(3)
    g, block, V, P, M = _inputs(rng, 30000, 3, (0.4, 0.8, 3.0), True)
    for mode in (0, 6):
        (q, dep), (q0, dep0) = _run(gpu_ctx, g, block, _abi.VIEW_PLY, V, P, M, mode, 0)
        assert np.array_equal(_sorted_rows(q, list(range(24))), _sorted_rows(q0, list(range(24))))
        assert np.array_equal(np.sort(dep.view(np.uint32)), np.sort(dep0.view(np.uint32)))


def test_prepass_sh_staged_path_on_a_large_input(gpu_ctx):
    """2^21 + 4321 gaussians take the kernel that stages the records through shared memory; the colour of every
    survivor equals orc_sh_colours of its input (identity model: the world position is the record's, bit for bit)."""
    rng = np.random.default_rng(11)
    n = (2 << 20) + 4321
    g, block, V, P, M = _inputs(rng, n, 3, (0.2, 0.3, 1.5), False)
    (q, _), (q0, _) = _run(gpu_ctx, g, block, _abi.VIEW_PLY, V, P, M, 0, 3)
    assert len(q) == len(q0) > n // 4
    def key(xy):   # the bits of x and y: unique among the inputs (z is checked below)
        b = np.ascontiguousarray(xy, np.float32).view(np.uint32).astype(np.uint64)
        return (b[:, 0] << np.uint64(32)) | b[:, 1]
    keys = key(g[:, 0:2])
    order = np.argsort(keys)
    src = order[np.minimum(np.searchsorted(keys[order], key(q[:, 20:22])), n - 1)]
    assert np.array_equal(g[src, 0:3].view(np.uint32), q[:, 20:23].view(np.uint32))
    rgb = osh.colours(g[src], block[src], 3, 3, osh.camera(V, M))
    assert np.array_equal(q[:, 8:11].view(np.uint32), rgb.view(np.uint32))
    assert np.array_equal(q[:, 11].view(np.uint32), g[src, 7].view(np.uint32))


# ---- end to end -----------------------------------------------------------------------------------------------------------
def test_read_prepass_sort_draw_sees_the_capture_change_colour_with_the_side(gpu_ctx, tmp_path):
    """A degree-1 capture whose red channel follows the view direction's z (f_rest_1 = 1: coefficient 2 of red, basis
    C1 z), read with SceneManager.loadPly(withSh=True), then prepass_sh -> sort -> splat draw from +z and from -z: the
    albedo differs from the plain prepass's on both sides, darker red seen from +z and brighter from -z.  At degree 0
    every target is the plain prepass's, bit for bit."""
    import torch
    rng = np.random.default_rng(21)
    n, w, h = 20000, 320, 240

    def fill(name, v):
        if name.startswith("f_dc"):
            return np.zeros_like(v)
        if name.startswith("f_rest"):
            return np.ones_like(v) if name == "f_rest_1" else np.zeros_like(v)
        return np.abs(v) + 3 if name == "opacity" else v

    p = _rest_file(tmp_path, rng, n, 1, name="e2e", fill=fill)
    rc = api.RenderContext(0)
    sm = api.SceneManager(rc)
    assert sm.loadPly(p) and rc.shCoefficients is None and rc.shDegree == 0
    assert sm.loadPly(p, withSh=True) and rc.shDegree == 1 and tuple(rc.shCoefficients.shape) == (n, 12)
    ctx, recs = rc.ctx, rc.gaussianBuffer
    P = column_major(perspective(np.radians(60.0), w / h, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    quads = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
    depths = torch.empty(n, dtype=torch.float32, device="cuda")
    sq = torch.empty(n * 96, dtype=torch.uint8, device="cuda")

    def albedo(eye, **sh):
        V = column_major(look_at(np.asarray(eye, np.float64), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
        targets = tuple(t for t, _ in _abi.GBUFFER_TARGETS)
        qn, _ = ctx.prepass(recs, n, rc.viewLayout(), V, P, M, (w, h), (0.01, 100.0), 1.0, 0, quads=quads, depths=depths, **sh)
        m = len(qn)
        ctx.depth_sort(quads, depths, m, sorted_quads=sq)
        return ctx.splat_draw(sq, m, w, h, 0, targets=targets)[0]

    for eye, sign in (((0.0, 0.0, 6.0), -1), ((0.0, 0.0, -6.0), 1)):
        plain = albedo(eye)
        zero = albedo(eye, sh=rc.shCoefficients, sh_degree=0)
        assert all(np.array_equal(zero[t].view(np.uint8), plain[t].view(np.uint8)) for t in plain)
        lit = albedo(eye, sh=rc.shCoefficients)
        assert not np.array_equal(lit["albedo"], plain["albedo"])
        covered = plain["albedo"][..., 3] > 0
        assert covered.sum() > 1000
        red = lit["albedo"][..., 0][covered].astype(np.int64).sum() - plain["albedo"][..., 0][covered].astype(np.int64).sum()
        assert np.sign(red) == sign, (eye, red)
        assert np.array_equal(lit["albedo"][..., 1:], plain["albedo"][..., 1:])   # green and blue have no coefficients
    rc.ctx.close()
