"""The image comparison on the GPU (m2s_image_compare): the SSIM map bit for bit and the integer totals exactly against
the C restatement (oracle/m2s_compare_oracle.c), the fp64 sums against math.fsum of its per-window values, through
guarded buffers; determinism across calls and forms; the argument checks; and the comparison of a mesh-lit and a
splat-lit frame drawn by the real passes."""
from __future__ import annotations

import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._lib import M2SError, lib
from oracle import compare as oc
from util import GuardedDevice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

RESULT_BYTES = C.sizeof(_abi.m2s_compare_result)
INT_FIELDS = ("windows", "covered_windows", "pixels_both", "pixels_a_only", "pixels_b_only", "sq_err", "sq_err_covered")


def _images(w, h, seed):
    """Two related images (b a noisy, locally shifted copy of a smooth a) and two covers with holes."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    a = np.stack([(xx * 3 + yy) % 256, (yy * 5) % 256, ((xx // 7 + yy // 5) % 2) * 200 + 20, np.full_like(xx, 255)], -1).astype(np.uint8)
    b = np.clip(np.roll(a, 1, axis=1).astype(np.int64) + rng.integers(-20, 21, a.shape), 0, 255).astype(np.uint8)
    ca, cb = rng.integers(0, 256, a.shape, dtype=np.uint8), rng.integers(0, 256, a.shape, dtype=np.uint8)
    ca[(xx // 9) % 3 == 0, 3] = 0
    cb[(yy // 5) % 4 == 0, 3] = 255
    return a, b, ca, cb


def _dev(x):
    import torch
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x).reshape(-1)).cuda()


def _enqueue(gpu_ctx, A, B, CA, CB, w, h, cover_min, result_ptr, map_ptr, stream=None):
    p = _abi.m2s_compare_params(w, h, cover_min)
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    return lib().m2s_image_compare_enqueue(gpu_ctx.handle, ptr(A), ptr(B), ptr(CA), ptr(CB), C.byref(p), result_ptr, map_ptr, stream)


def _run(gpu_ctx, a, b, ca, cb, w, h, cover_min=128):
    """The enqueue form through guarded result and map buffers: (result dict, map (h - 10, w - 10) float32)."""
    import torch
    A, B, CA, CB = (_dev(x) for x in (a, b, ca, cb))
    nw = (w - 10) * (h - 10)
    gr = GuardedDevice(1, RESULT_BYTES, what="result")
    gm = GuardedDevice(nw, 4, dtype=torch.float32, what="map")
    torch.cuda.synchronize()
    st = _enqueue(gpu_ctx, A, B, CA, CB, w, h, cover_min, gr.view.data_ptr(), gm.view.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert st == _abi.M2S_OK, lib().m2s_last_error()
    torch.cuda.synchronize()
    gr.check(1)
    gm.check(nw)
    r = _abi.m2s_compare_result.from_buffer_copy(gr.view.cpu().numpy().tobytes())
    return _abi.compare_result_dict(r, w * h), gm.view[:nw].cpu().numpy().reshape(h - 10, w - 10)


def _check(got, m, want, wm, planes, covered):
    assert m.tobytes() == wm.tobytes(), f"{int((m != wm).sum())} of {m.size} map values differ"
    for f in INT_FIELDS:
        assert got[f] == want[f], (f, got[f], want[f])
    n = got["windows"]
    for c in range(3):
        for key, sel in (("ssim_sum", None), ("ssim_covered_sum", covered)):
            vals = planes[c].astype(np.float64)
            vals = vals.ravel() if sel is None else vals[sel]
            exact = math.fsum(vals)
            assert abs(got[key][c] - exact) <= n * 2.0 ** -52 * float(np.abs(vals).sum()), (key, c, got[key][c], exact)


@pytest.mark.parametrize("wh", [(11, 11), (11, 4096), (4096, 11), (43, 17), (1921, 1081), (3840, 2160), (4096, 4096)])
def test_map_and_totals_against_the_oracle(gpu_ctx, wh):
    w, h = wh
    a, b, ca, cb = _images(w, h, w + h)
    got, m = _run(gpu_ctx, a, b, ca, cb, w, h)
    want, wm, planes = oc.compare(a, b, w, h, ca, cb)
    covered = ((ca[..., 3] >= 128) | (cb[..., 3] >= 128))[5:-5, 5:-5]
    _check(got, m, want, wm, planes, covered)
    if w * h > 121:
        assert got["pixels_a_only"] > 0 and got["pixels_b_only"] > 0 and got["pixels_both"] > 0
    assert got["covered_windows"] == int(covered.sum())


@pytest.mark.parametrize("covers", ["none", "a", "b", "both"])
@pytest.mark.parametrize("cover_min", [1, 255])
def test_covers(gpu_ctx, covers, cover_min):
    w, h = 301, 157
    a, b, ca, cb = _images(w, h, 7)
    ca = ca if covers in ("a", "both") else None
    cb = cb if covers in ("b", "both") else None
    got, m = _run(gpu_ctx, a, b, ca, cb, w, h, cover_min)
    want, wm, planes = oc.compare(a, b, w, h, ca, cb, cover_min)
    cov = np.zeros((h, w), bool)
    for x in (ca, cb):
        if x is not None:
            cov |= x[..., 3] >= cover_min
    _check(got, m, want, wm, planes, cov[5:-5, 5:-5])
    if covers == "none":
        assert got["covered_windows"] == got["pixels_both"] == got["pixels_a_only"] == got["pixels_b_only"] == 0
        assert got["sq_err_covered"] == [0, 0, 0] and got["ssim_covered_sum"] == [0.0, 0.0, 0.0]


def test_identical_images_and_one_changed_pixel(gpu_ctx):
    w, h = 200, 90
    a, _, _, _ = _images(w, h, 3)
    got, m = _run(gpu_ctx, a, a.copy(), None, None, w, h)
    assert (m == np.float32(1.0)).all() and got["sq_err"] == [0, 0, 0] and got["psnr"] == math.inf and got["ssim"] == 1.0
    b = a.copy()
    b[40, 150, 2] ^= 0x55
    got, m = _run(gpu_ctx, a, b, None, None, w, h)
    d = int(b[40, 150, 2]) - int(a[40, 150, 2])
    assert got["sq_err"] == [0, 0, d * d]
    wy, wx = np.nonzero(m < 1)
    assert len(wy) == 121 and (abs(wy + 5 - 40) <= 5).all() and (abs(wx + 5 - 150) <= 5).all()


def test_two_calls_and_both_forms_are_bit_identical(gpu_ctx):
    import torch
    w, h = 1920, 1080
    a, b, ca, cb = _images(w, h, 11)
    A, B, CA, CB = (_dev(x) for x in (a, b, ca, cb))
    nw = (w - 10) * (h - 10)
    maps = [torch.empty(nw, dtype=torch.float32, device="cuda") for _ in range(3)]
    r1 = gpu_ctx.compare_images(A, B, w, h, CA, CB, ssim_map=maps[0])
    r2 = gpu_ctx.compare_images(A, B, w, h, CA, CB, ssim_map=maps[1])
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        r3 = gpu_ctx.compare_images(A, B, w, h, CA, CB, ssim_map=maps[2], enqueue=True)
    for r in (r2, r3):
        assert all(r[k] == r1[k] for k in r1 if not (isinstance(r1[k], float) and math.isnan(r1[k]))), (r, r1)
        assert [x.hex() for x in r["ssim_sum"] + r["ssim_covered_sum"]] == [x.hex() for x in r1["ssim_sum"] + r1["ssim_covered_sum"]]
    assert all(torch.equal(maps[0].view(torch.int32), m.view(torch.int32)) for m in maps[1:])
    assert 0.0 < r1["ssim"] < 1.0 and 0.0 < r1["psnr"] < 60.0


def test_invalid_arguments_write_nothing(gpu_ctx):
    import torch
    w, h = 64, 32
    a, b, ca, cb = _images(w, h, 5)
    big = torch.zeros(4097 * 12 * 4 + 16, dtype=torch.uint8, device="cuda")
    A, B = _dev(a), _dev(b)
    gr = GuardedDevice(1, RESULT_BYTES, what="result")
    gm = GuardedDevice((w - 10) * (h - 10), 4, dtype=torch.float32, what="map")
    cases = [(big, big, None, None, 10, 12, 128), (big, big, None, None, 12, 10, 128), (big, big, None, None, 4097, 12, 128),
             (big, big, None, None, 12, 4097, 128), (A, B, None, None, w, h, 0), (A, B, None, None, w, h, 256),
             (None, B, None, None, w, h, 128), (A, None, None, None, w, h, 128), (A[1:], B, None, None, w, h, 128),
             (A, B[2:], None, None, w, h, 128), (A, B, A[1:], None, w, h, 128), (A, B, None, B[3:], w, h, 128)]
    for i, (x, y, cx, cy, ww, hh, cm) in enumerate(cases):
        st = _enqueue(gpu_ctx, x, y, cx, cy, ww, hh, cm, gr.view.data_ptr(), gm.view.data_ptr())
        assert st == _abi.M2S_E_INVALID, (i, st)
    assert _enqueue(gpu_ctx, A, B, None, None, w, h, 128, gr.view.data_ptr() + 4, gm.view.data_ptr()) == _abi.M2S_E_INVALID
    assert _enqueue(gpu_ctx, A, B, None, None, w, h, 128, gr.view.data_ptr(), gm.view.data_ptr() + 2) == _abi.M2S_E_INVALID
    assert _enqueue(gpu_ctx, A, B, None, None, w, h, 128, None, gm.view.data_ptr()) == _abi.M2S_E_INVALID
    torch.cuda.synchronize()
    gr.check(0)
    gm.check(0)
    with pytest.raises(M2SError):
        gpu_ctx.compare_images(A, B, w, h, cover_min=0)
    # the largest size is accepted, and a map is optional
    got, _ = _run(gpu_ctx, a, b, None, None, w, h)
    assert got["windows"] == (w - 10) * (h - 10)
    assert gpu_ctx.compare_images(A, B, w, h)["sq_err"] == got["sq_err"]


def test_mesh_lit_against_splat_lit_frame(gpu_ctx):
    """A small synth scene at R = 64 drawn at 192 x 108 by the real passes: the mesh G-buffer lit, and convert -> prepass
    -> sort -> splat draw lit; the GPU comparison of the two images, with the albedo targets as covers, equals the
    oracle's comparison of the downloaded images."""
    import torch
    scene = synth.helmet_standin(64)
    ds = gpu_ctx.upload(scene)
    R, w, h = 64, 192, 108
    near_far = (0.01, 100.0)
    eye, tgt = (0.0, 0.5, 3.2), (0.0, 0.0, 0.0)
    V = column_major(look_at(np.array(eye), np.array(tgt), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(45.0), w / h, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    names = [t for t, _ in _abi.GBUFFER_TARGETS]
    alloc = lambda: {t: torch.empty(w * h * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda")  # noqa: E731
                     for t, dt in _abi.GBUFFER_TARGETS}
    mbuf, sbuf = alloc(), alloc()
    try:
        for mode in (0, 2):
            gpu_ctx.mesh_render(ds, V, P, M, w, h, near_far, mode, targets=tuple(names), gbuffer=mbuf)
            out = gpu_ctx.convert(ds, R, _abi.LAYOUT_REF96, 0.65, flags=_abi.FLAG_UNCAPPED)
            n = out.written
            quads = torch.empty(max(1, n) * _abi.QUAD_BYTES, dtype=torch.uint8, device="cuda")
            depths = torch.empty(max(1, n), dtype=torch.float32, device="cuda")
            q, _ = gpu_ctx.prepass(out.data, n, _abi.LAYOUT_REF96, V, P, M, (w, h), near_far, 0.65 / R, mode, quads=quads, depths=depths)
            sq = torch.empty(max(1, len(q)) * _abi.QUAD_BYTES, dtype=torch.uint8, device="cuda")
            gpu_ctx.depth_sort(quads, depths, len(q), sorted_quads=sq)
            gpu_ctx.splat_draw(sq, len(q), w, h, mode, targets=tuple(names), gbuffer=sbuf)
            mi = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
            si = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
            gpu_ctx.deferred_light(mbuf, None, w, h, mode, image=mi)
            gpu_ctx.deferred_light(sbuf, None, w, h, mode, image=si)
            smap = torch.empty((w - 10) * (h - 10), dtype=torch.float32, device="cuda")
            got = gpu_ctx.compare_images(mi, si, w, h, mbuf["albedo"], sbuf["albedo"], ssim_map=smap)
            host = lambda t: t.cpu().numpy().reshape(h, w, 4)  # noqa: E731
            want, wm, planes = oc.compare(host(mi), host(si), w, h, host(mbuf["albedo"]), host(sbuf["albedo"]))
            assert smap.cpu().numpy().tobytes() == wm.tobytes()
            for f in INT_FIELDS:
                assert got[f] == want[f], (mode, f)
            assert got["ssim"] == pytest.approx(want["ssim"], rel=1e-12) and got["psnr"] == want["psnr"]
            assert got["pixels_both"] > 0 and 0.0 < got["ssim_covered"] < 1.0 and math.isfinite(got["psnr_covered"])
    finally:
        ds.free()
