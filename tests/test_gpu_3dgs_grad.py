"""The 3DGS render's backward pass on the GPU (m2s_3dgs_render_grad, m2s_3dgs_backward_enqueue): the forward pass that
keeps its state bit for bit m2s_3dgs_render's; the backward pass bit for bit the C restatement
(oracle/m2s_3dgs_grad_oracle.c) through guarded buffers, across sizes, deep stacks, wide gaussians, pair budgets, empty
and culled inputs; determinism, independent states, the torch autograd route, a short refinement, and the argument
checks."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from mesh2splat_b200 import _abi
from mesh2splat_b200._lib import lib
from oracle import gs3d_grad
from util import GuardedDevice

from test_3dgs_grad_host import EYE, camera, packed56

pytestmark = pytest.mark.gpu


def _params(rec):
    import torch
    return torch.from_numpy(np.ascontiguousarray(rec, np.float32).reshape(-1, 14)).cuda()


def grad_forward(ctx, state, rec, V, P, w, h, max_pairs=None, **kw):
    """(image (h, w, 4) numpy, drawn, pairs) of the forward pass that keeps its state, into a guarded target."""
    import torch
    prm = _params(rec) if len(rec) else torch.zeros((0, 14), dtype=torch.float32, device="cuda")
    img = GuardedDevice(w * h, 16, dtype=torch.float32, what="rgba32f")
    p = _abi.make_3dgs_params(V, P, EYE, w, h, kw.get("near", 0.2), 1.0, 1.0, kw.get("background", (0, 0, 0)), _abi.LAYOUT_PACKED56)
    out = torch.zeros(4, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    if max_pairs is None:
        pairs = C.c_uint64(0)
        assert lib().m2s_3dgs_render_grad(ctx.handle, state.handle, prm.data_ptr() if len(rec) else None, len(rec), C.byref(p),
                                          img.view.data_ptr(), C.byref(pairs)) == 0, lib().m2s_last_error()
        drawn, npairs = len(rec), pairs.value
    else:
        assert lib().m2s_3dgs_render_grad_enqueue(ctx.handle, state.handle, prm.data_ptr() if len(rec) else None, len(rec), C.byref(p),
                                                  img.view.data_ptr(), max_pairs, out.data_ptr(), out[2:].data_ptr(), None) == 0
        torch.cuda.synchronize()
        o = out.cpu().numpy()
        drawn, npairs = int(o[2]), int(o[:2].view(np.uint64)[0])
    img.check(w * h)
    return img.view[: w * h * 4].cpu().numpy().reshape(h, w, 4).copy(), drawn, npairs, prm, p


def backward(ctx, state, prm, p, n, g):
    import torch
    gd = torch.from_numpy(np.ascontiguousarray(g, np.float32).reshape(-1)).cuda()
    out = GuardedDevice(max(n, 1), 56, dtype=torch.float32, what="grad")
    torch.cuda.synchronize()
    st = lib().m2s_3dgs_backward_enqueue(ctx.handle, state.handle, prm.data_ptr() if n else None, n, C.byref(p), gd.data_ptr(),
                                         out.view.data_ptr(), None)
    assert st == 0, lib().m2s_last_error()
    torch.cuda.synchronize()
    out.check(n)
    return out.view[: n * 14].cpu().numpy().reshape(n, 14).copy()


def _records_u8(rec):
    import torch
    return _params(rec).view(-1).view(torch.uint8) if len(rec) else torch.zeros(16, dtype=torch.uint8, device="cuda")


def forward_matches_render(ctx, state, rec, V, P, w, h, bg, max_pairs=None):
    """The forward pass keeping its state against render_3dgs on the same records: the RGBA32F image, the pair count and
    the drawn prefix bit for bit.  The synchronous forms report no drawn prefix, so the enqueue forms are also compared
    with the budget the synchronous form found.  Returns the state's forward (image, drawn, pairs, params tensor, params)
    with the budget asked for."""
    out = grad_forward(ctx, state, rec, V, P, w, h, max_pairs=max_pairs, background=bg)
    img, _, pairs, _, _ = out
    imgs, _, wpairs = ctx.render_3dgs(_records_u8(rec), len(rec), _abi.LAYOUT_PACKED56, V, P, EYE, w, h, background=bg,
                                      targets=("rgba32f",), max_pairs=max_pairs)
    assert img.tobytes() == imgs["rgba32f"][: w * h * 4].cpu().numpy().tobytes()
    assert pairs == wpairs
    budget = pairs if max_pairs is None else max_pairs
    img2, drawn2, pairs2, _, _ = grad_forward(ctx, state, rec, V, P, w, h, max_pairs=budget, background=bg)
    imgs2, wdrawn2, wpairs2 = ctx.render_3dgs(_records_u8(rec), len(rec), _abi.LAYOUT_PACKED56, V, P, EYE, w, h, background=bg,
                                              targets=("rgba32f",), max_pairs=budget)
    assert img2.tobytes() == imgs2["rgba32f"][: w * h * 4].cpu().numpy().tobytes()
    assert (drawn2, pairs2) == (wdrawn2, wpairs2)
    if max_pairs is None:
        assert img2.tobytes() == img.tobytes() and pairs2 == pairs
        return grad_forward(ctx, state, rec, V, P, w, h, background=bg)   # the state holds the synchronous form's pass again
    return out


def check(ctx, rec, w, h, seed=0, max_pairs=None, eye=(0.3, 0.4, 3.0), bg=(0.1, 0.2, 0.3)):
    V, P = camera(w, h, eye=eye)
    with ctx.gs3d_state() as state:
        img, drawn, pairs, prm, p = forward_matches_render(ctx, state, rec, V, P, w, h, bg, max_pairs)
        g = np.random.default_rng(seed).normal(size=(h, w, 4)).astype(np.float32)
        got = backward(ctx, state, prm, p, len(rec), g)
        want, wdrawn = gs3d_grad.backward(rec, V, P, EYE, w, h, g, background=bg, max_pairs=max_pairs)
        assert max_pairs is None or drawn == wdrawn   # the synchronous form draws every survivor
        bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
        assert got.tobytes() == want.tobytes(), (bad[:5], got[tuple(bad[0])] if len(bad) else None, want[tuple(bad[0])] if len(bad) else None)
        return got, drawn


@pytest.mark.parametrize("wh", [(1, 1), (17, 13), (64, 48), (256, 256)])
def test_backward_bit_for_bit(gpu_ctx, wh):
    w, h = wh
    check(gpu_ctx, packed56(3000 if w == 256 else 600, 1), w, h, seed=2)


def test_deep_stacks_that_stop(gpu_ctx):
    rec = packed56(4000, 5)
    rec[:, 0:3] *= 0.2
    rec[:, 13] = 4.0
    rec[7, 13] = np.nan     # drawn with alpha 0.99; its row is zero
    rec[9, 13] = np.inf
    got, _ = check(gpu_ctx, rec, 48, 40, seed=3)
    assert (got[7] == 0).all() and np.isfinite(got).all()


def test_wide_gaussians_over_many_tiles(gpu_ctx):
    rec = packed56(40, 6)
    rec[:, 7:10] = np.random.default_rng(1).uniform(-1.2, -0.5, (40, 3))
    rec[:, 13] = -1.0
    check(gpu_ctx, rec, 200, 150, seed=4)


def test_pair_budget_prefix(gpu_ctx):
    got, drawn = check(gpu_ctx, packed56(2000, 7), 96, 64, seed=5, max_pairs=700)
    assert 0 < drawn < 2000
    assert (got[np.abs(got).sum(1) == 0].shape[0]) >= 2000 - drawn   # the undrawn records' rows are zero


def test_count_zero_and_all_culled(gpu_ctx):
    check(gpu_ctx, np.zeros((0, 14), np.float32), 20, 20)
    rec = packed56(300, 8)
    rec[:, 2] = 10.0
    got, drawn = check(gpu_ctx, rec, 20, 20, max_pairs=100000)
    assert drawn == 0 and (got == 0).all()


def test_bench_scene_small_r(gpu_ctx):
    import torch
    from mesh2splat_b200 import synth
    scene = synth.helmet_standin(2048)
    ds = gpu_ctx.upload(scene)
    out = gpu_ctx.convert(ds, 64, _abi.LAYOUT_PACKED56)
    n = out.written
    rec = out.data[: n * 56].cpu().numpy().view(np.float32).reshape(n, 14).copy()
    ds.free()
    lo, hi = rec[:, 0:3].min(0), rec[:, 0:3].max(0)
    c = (lo + hi) / 2
    eye = tuple(c + np.array([0.0, 0.0, 2.5]) * float((hi - lo).max()))
    w, h = 160, 120
    V, P = camera(w, h, eye=eye, tgt=tuple(c))
    with gpu_ctx.gs3d_state() as state:
        img, drawn, pairs, prm, p = forward_matches_render(gpu_ctx, state, rec, V, P, w, h, (0.0, 0.0, 0.0))
        forward_matches_render(gpu_ctx, state, rec, V, P, w, h, (0.0, 0.0, 0.0), max_pairs=pairs // 2)
        img, drawn, pairs, prm, p = grad_forward(gpu_ctx, state, rec, V, P, w, h)
        g = np.random.default_rng(1).normal(size=(h, w, 4)).astype(np.float32)
        got = backward(gpu_ctx, state, prm, p, n, g)
    want, _ = gs3d_grad.backward(rec, V, P, EYE, w, h, g)
    assert got.tobytes() == want.tobytes()
    assert torch.cuda.is_available()


def test_deterministic_and_independent_states(gpu_ctx):
    w, h = 64, 48
    ra, rb = packed56(1500, 11), packed56(1200, 12)
    V, P = camera(w, h)
    ga = np.random.default_rng(1).normal(size=(h, w, 4)).astype(np.float32)
    gb = np.random.default_rng(2).normal(size=(h, w, 4)).astype(np.float32)
    with gpu_ctx.gs3d_state() as sa, gpu_ctx.gs3d_state() as sb:
        _, _, _, pa, p = grad_forward(gpu_ctx, sa, ra, V, P, w, h)
        _, _, _, pb, _ = grad_forward(gpu_ctx, sb, rb, V, P, w, h)
        a1 = backward(gpu_ctx, sa, pa, p, len(ra), ga)
        b1 = backward(gpu_ctx, sb, pb, p, len(rb), gb)
        a2 = backward(gpu_ctx, sa, pa, p, len(ra), ga)
    assert a1.tobytes() == a2.tobytes()
    assert a1.tobytes() == gs3d_grad.backward(ra, V, P, EYE, w, h, ga)[0].tobytes()
    assert b1.tobytes() == gs3d_grad.backward(rb, V, P, EYE, w, h, gb)[0].tobytes()


def test_autograd_equals_direct_call_and_adam_lowers_l1(gpu_ctx):
    import torch
    w, h = 64, 48
    V, P = camera(w, h)
    rec = packed56(800, 13)
    g = np.random.default_rng(3).normal(size=(h, w, 4)).astype(np.float32)
    with gpu_ctx.gs3d_state() as state:
        prm = _params(rec).requires_grad_(True)
        img = gpu_ctx.render_3dgs_grad(prm, state, V, P, EYE, w, h, background=(0.1, 0.2, 0.3))
        (img * torch.from_numpy(g).cuda()).sum().backward()
        torch.cuda.synchronize()
        want, _ = gs3d_grad.backward(rec, V, P, EYE, w, h, g, background=(0.1, 0.2, 0.3))
        assert prm.grad.cpu().numpy().tobytes() == want.tobytes()
        # a short seeded refinement towards the image of other gaussians lowers the L1 loss
        target = gpu_ctx.render_3dgs_grad(_params(packed56(800, 14)), state, V, P, EYE, w, h).detach().clone()
        x = _params(rec).requires_grad_(True)
        opt = torch.optim.Adam([x], lr=0.01)
        losses = []
        for _ in range(30):
            opt.zero_grad()
            loss = (gpu_ctx.render_3dgs_grad(x, state, V, P, EYE, w, h) - target).abs().mean()
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        assert losses[-1] < 0.8 * losses[0], losses


def test_argument_checks(gpu_ctx):
    import torch
    w, h = 16, 16
    V, P = camera(w, h)
    rec = packed56(50, 1)
    prm = _params(rec)
    img = torch.full((w * h * 4 + 4,), 5.0, dtype=torch.float32, device="cuda")
    p = _abi.make_3dgs_params(V, P, EYE, w, h, 0.2, 1.0, 1.0, (0, 0, 0), _abi.LAYOUT_PACKED56)
    bad_layout = _abi.make_3dgs_params(V, P, EYE, w, h, 0.2, 1.0, 1.0, (0, 0, 0), _abi.LAYOUT_REF96)
    grad = torch.full((50 * 14 + 4,), 7.0, dtype=torch.float32, device="cuda")
    gimg = torch.zeros(w * h * 4 + 4, dtype=torch.float32, device="cuda")
    L = lib()
    with gpu_ctx.gs3d_state() as state:
        # no forward pass yet
        assert L.m2s_3dgs_backward_enqueue(gpu_ctx.handle, state.handle, prm.data_ptr(), 50, C.byref(p), gimg.data_ptr(), grad.data_ptr(), None) == _abi.M2S_E_INVALID
        assert L.m2s_3dgs_render_grad(gpu_ctx.handle, state.handle, prm.data_ptr(), 50, C.byref(bad_layout), img.data_ptr(), None) == _abi.M2S_E_INVALID
        assert L.m2s_3dgs_render_grad(gpu_ctx.handle, None, prm.data_ptr(), 50, C.byref(p), img.data_ptr(), None) == _abi.M2S_E_INVALID
        assert L.m2s_3dgs_render_grad(gpu_ctx.handle, state.handle, prm.data_ptr(), 50, C.byref(p), None, None) == _abi.M2S_E_INVALID
        assert L.m2s_3dgs_render_grad(gpu_ctx.handle, state.handle, prm.data_ptr() + 4, 50, C.byref(p), img.data_ptr(), None) == _abi.M2S_E_INVALID
        assert L.m2s_3dgs_render_grad(gpu_ctx.handle, state.handle, prm.data_ptr(), 50, C.byref(p), img.data_ptr() + 4, None) == _abi.M2S_E_INVALID
        enq = L.m2s_3dgs_render_grad_enqueue
        assert enq(gpu_ctx.handle, state.handle, prm.data_ptr(), 50, C.byref(bad_layout), img.data_ptr(), 100, None, None, None) == _abi.M2S_E_INVALID
        assert enq(gpu_ctx.handle, state.handle, prm.data_ptr(), 50, C.byref(p), img.data_ptr(), 1 << 30, None, None, None) == _abi.M2S_E_INVALID
        torch.cuda.synchronize()
        assert (img == 5.0).all()   # nothing written by the rejected forward passes
        assert L.m2s_3dgs_render_grad(gpu_ctx.handle, state.handle, prm.data_ptr(), 50, C.byref(p), img.data_ptr(), None) == 0
        other = _abi.make_3dgs_params(V, P, EYE, w + 1, h, 0.2, 1.0, 1.0, (0, 0, 0), _abi.LAYOUT_PACKED56)
        for args in [(prm.data_ptr(), 49, C.byref(p), gimg.data_ptr(), grad.data_ptr()),           # count differs
                     (prm.data_ptr(), 50, C.byref(other), gimg.data_ptr(), grad.data_ptr()),       # size differs
                     (prm.data_ptr(), 50, C.byref(bad_layout), gimg.data_ptr(), grad.data_ptr()),  # layout differs
                     (prm.data_ptr(), 50, C.byref(p), None, grad.data_ptr()),
                     (prm.data_ptr(), 50, C.byref(p), gimg.data_ptr(), None),
                     (prm.data_ptr(), 50, C.byref(p), gimg.data_ptr() + 4, grad.data_ptr()),
                     (prm.data_ptr(), 50, C.byref(p), gimg.data_ptr(), grad.data_ptr() + 2)]:
            assert L.m2s_3dgs_backward_enqueue(gpu_ctx.handle, state.handle, *args, None) == _abi.M2S_E_INVALID, args
        torch.cuda.synchronize()
        assert (grad == 7.0).all()


def test_refined_ply_round_trip(gpu_ctx, tmp_path):
    """write_3dgs_ply's file loads through ply_read to the same fields, within the codec's rounding: position exact,
    colour SH0 C0 + 0.5, opacity sigmoid(logit), scale exp(log-scale), rotation q / |q|."""
    from mesh2splat_b200.api import write_3dgs_ply
    rec = packed56(500, 21)
    rec[3, 13] = np.inf
    path = str(tmp_path / "refined.ply")
    write_3dgs_ply(path, _params(rec))
    records, n, has_pbr = gpu_ctx.ply_read(path)
    assert n == 500 and not has_pbr
    got = records[: n * 96].cpu().numpy().view(np.float32).reshape(n, 24)
    r64 = rec.astype(np.float64)
    assert (got[:, 0:3] == rec[:, 0:3]).all()
    np.testing.assert_allclose(got[:, 4:7], r64[:, 10:13] * 0.28209479177387814 + 0.5, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(got[:, 7], 1.0 / (1.0 + np.exp(-r64[:, 13])), rtol=4e-6, atol=1e-7)
    np.testing.assert_allclose(got[:, 8:11], np.exp(r64[:, 7:10]), rtol=4e-6)
    q = r64[:, 3:7] / np.linalg.norm(r64[:, 3:7], axis=1, keepdims=True)
    np.testing.assert_allclose(got[:, 16:20], q, rtol=1e-5, atol=1e-6)


def test_autograd_backward_is_ordered_on_torch_stream(gpu_ctx):
    """The backward pass runs on torch's current stream: torch work right after .backward(), with no synchronisation,
    reads the finished gradient (on torch's default stream too), across states and counts that reuse freed memory."""
    import torch
    w, h = 128, 96
    V, P = camera(w, h)
    for n, seed in ((500, 31), (6000, 32), (3000, 33)):
        rec = packed56(n, seed)
        g = torch.from_numpy(np.random.default_rng(seed).normal(size=(h, w, 4)).astype(np.float32)).cuda()
        want, _ = gs3d_grad.backward(rec, V, P, EYE, w, h, g.cpu().numpy())
        for stream in (torch.cuda.default_stream(), torch.cuda.Stream()):
            with torch.cuda.stream(stream), gpu_ctx.gs3d_state() as state:
                prm = torch.full((n, 14), float("nan"), device="cuda").copy_(_params(rec)).requires_grad_(True)
                (gpu_ctx.render_3dgs_grad(prm, state, V, P, EYE, w, h) * g).sum().backward()
                snap = prm.grad.clone()   # on torch's stream, no synchronisation before it
            torch.cuda.synchronize()
            assert snap.cpu().numpy().tobytes() == want.tobytes()
