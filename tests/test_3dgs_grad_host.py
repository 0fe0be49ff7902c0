"""The 3DGS render's backward checker (oracle/m2s_3dgs_grad_oracle.c) against the fp64 torch-autograd statement of
graphdeco's forward pass (oracle/gs3d_grad.py), that statement against central finite differences of the fp64
gs3d.graphdeco_forward, and known answers.  CPU only.

Bound (DESIGN §2, backward).  Each partial is a short chain of fp32 operations on the forward values, whose own relative
error is within 2^-17 (test_3dgs_host.py); the per-pixel recovery T / (1 - alpha) loses at most one rounding per blended
term, and the sums over pixels and tiles add one rounding per term.  So each gradient component is held to
2^-10 (|g64| + s), s = the largest |component| of that field over the scene: a relative error a few hundred times the
fp32 step, with the field scale absorbing the cancellation in sums of terms of both signs."""
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from oracle import gs3d, gs3d_grad  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

EYE = column_major(np.eye(4, dtype=np.float32))
FIELDS = [(0, 3), (3, 7), (7, 10), (10, 13), (13, 14)]


def camera(w, h, eye=(0.3, 0.4, 3.0), tgt=(0.0, 0.0, 0.0), fov=50.0):
    V = column_major(look_at(np.array(eye, np.float64), np.array(tgt, np.float64), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(fov), w / h, 0.01, 100.0))
    return V, P


def packed56(n, seed):
    rng = np.random.default_rng(seed)
    r = np.zeros((n, 14), np.float32)
    r[:, 0:3] = rng.uniform(-1, 1, (n, 3))
    r[:, 3:7] = rng.normal(size=(n, 4))
    r[:, 7:10] = rng.uniform(-3.5, -1.5, (n, 3))
    r[:, 10:13] = rng.normal(size=(n, 3))
    r[:, 13] = rng.normal(size=n) * 2
    return r


def assert_close_fields(got, want, what, tol=2.0 ** -10):
    for a, b in FIELDS:
        s = np.abs(want[:, a:b]).max() if want.size else 0.0
        err = np.abs(got[:, a:b] - want[:, a:b])
        lim = tol * (np.abs(want[:, a:b]) + s) + 1e-30
        assert (err <= lim).all(), (what, a, b, np.argwhere(err > lim)[:4], float((err / lim).max()))


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("cam", [0, 1, 2])
@pytest.mark.parametrize("wh", [(64, 48), (33, 17)])
def test_checker_against_fp64_autograd(seed, cam, wh):
    w, h = wh
    eye = [(0.3, 0.4, 3.0), (-2.0, 1.0, 1.5), (0.1, -0.2, 1.2)][cam]
    V, P = camera(w, h, eye=eye)
    rec = packed56(60, seed)
    rng = np.random.default_rng(seed + 100)
    g = rng.normal(size=(h, w, 4)).astype(np.float32)
    bg = (0.1, 0.2, 0.3)
    got, drawn = gs3d_grad.backward(rec, V, P, EYE, w, h, g, background=bg)
    want = gs3d_grad.torch_backward(rec, V, P, EYE, w, h, g, background=bg)
    assert np.isfinite(got).all()
    assert_close_fields(got, want, (seed, cam, wh))


def test_fp64_autograd_against_finite_differences():
    """The torch statement's gradient is the derivative of graphdeco_forward's image, where no alpha is near 0.99, 1/255
    or the stop and no rectangle decides a gaussian."""
    w, h = 24, 20
    V, P = camera(w, h, eye=(0.2, 0.1, 2.5))
    bg = (0.2, 0.1, 0.3)

    def img(x):
        pos, scale, rot = x[:, 0:3], np.exp(x[:, 7:10]), x[:, 3:7]
        col, opac = x[:, 10:13] * gs3d.SH_C0 + 0.5, 1.0 / (1.0 + np.exp(-x[:, 13]))
        _, im, margin, rect_dep = gs3d.graphdeco_forward(pos, scale, rot, col, opac, V, P, w, h, 0.2, background=bg, model_to_world=EYE)
        return im, margin, rect_dep

    for seed in range(100):   # the first seeded scene whose every alpha is 1e-4 or more from each cut-off
        rng = np.random.default_rng(seed)
        rec = np.zeros((6, 14), np.float32)
        rec[:, 0:3] = rng.uniform(-0.25, 0.25, (6, 3))
        rec[:, 3:7] = rng.normal(size=(6, 4))
        rec[:, 7:10] = rng.uniform(-2.6, -1.9, (6, 3))
        rec[:, 10:13] = rng.uniform(-0.5, 1.0, (6, 3))
        rec[:, 13] = rng.uniform(-1.0, 0.5, 6)
        x64 = rec.astype(np.float64)
        _, margin, rect_dep = img(x64)
        if margin.min() > 1e-4 and not rect_dep.any():
            break
    else:
        pytest.fail("no scene with the margins")
    Wt = rng.normal(size=(h, w, 4))
    want = gs3d_grad.torch_backward(rec, V, P, EYE, w, h, Wt, background=bg)
    fd = np.zeros_like(x64)
    eps = 1e-7
    for i in range(x64.shape[0]):
        for k in range(14):
            xp, xm = x64.copy(), x64.copy()
            xp[i, k] += eps
            xm[i, k] -= eps
            fd[i, k] = ((img(xp)[0] * Wt).sum() - (img(xm)[0] * Wt).sum()) / (2 * eps)
    np.testing.assert_allclose(want, fd, rtol=1e-5, atol=1e-6 * np.abs(fd).max())


def V_single(w, h):
    return camera(w, h, eye=(0.0, 0.0, 3.0))


def test_one_gaussian_one_pixel_known_answer():
    """dL/dcolour = alpha T (T = 1) times C0 on SH0; the logit's derivative from the colour, background and alpha terms."""
    w = h = 1
    V, P = V_single(w, h)
    rec = np.zeros((1, 14), np.float32)
    rec[0, 3] = 1.0
    rec[0, 7:10] = -1.0
    rec[0, 10:13] = (0.5, -0.2, 0.1)
    rec[0, 13] = 0.3
    g = np.array([[[1.0, 0.0, 0.0, 0.0]]], np.float32)
    got, _ = gs3d_grad.backward(rec, V, P, EYE, w, h, g, background=(0.25, 0.5, 0.75))
    sp, _, _ = gs3d.preprocess(rec, 1, V, P, EYE, w, h)
    dx, dy = sp[0, 0] - 0.0, sp[0, 1] - 0.0
    power = -0.5 * (sp[0, 2] * dx * dx + sp[0, 4] * dy * dy) - sp[0, 3] * dx * dy
    o = 1.0 / (1.0 + np.exp(-0.3))
    alpha = o * np.exp(power)
    assert np.isclose(got[0, 10], alpha * gs3d.SH_C0, rtol=1e-5)
    assert got[0, 11] == 0.0 and got[0, 12] == 0.0
    # dL/dalpha = colour_r - background_r (T = 1, one term), times G o (1 - o) on the logit
    col_r = 0.5 * gs3d.SH_C0 + 0.5
    assert np.isclose(got[0, 13], (col_r - 0.25) * np.exp(power) * o * (1 - o), rtol=1e-4)


def test_culled_zero_rectangle_and_infinite_logit():
    w, h = 32, 32
    V, P = V_single(w, h)
    rec = np.zeros((3, 14), np.float32)
    rec[:, 3] = 1.0
    rec[:, 7:10] = -2.0
    rec[:, 10:13] = 0.3
    rec[0, 2] = 5.0        # behind the camera: culled
    rec[1, 0] = 100.0      # far off screen: an empty rectangle
    rec[2, 13] = np.inf    # alpha = 1, clamped to 0.99: the logit gets 0, the other fields theirs
    got, _ = gs3d_grad.backward(rec, V, P, EYE, w, h, np.ones((h, w, 4), np.float32))
    assert np.isfinite(got).all()
    assert (got[0] == 0).all() and (got[1] == 0).all()
    assert got[2, 13] == 0.0 and np.abs(got[2, :13]).max() > 0


def test_gaussian_past_the_stop_gets_nothing():
    """Ten opaque wide gaussians in front take T below 1e-4 around the centre; a small finite-logit gaussian behind them,
    inside that region, gets a row of exact zeros, and alone it gets a gradient."""
    w, h = 32, 32
    V, P = V_single(w, h)
    front = np.zeros((10, 14), np.float32)
    front[:, 2] = np.linspace(0.5, 0.05, 10)
    front[:, 3] = 1.0
    front[:, 7:10] = -0.5
    front[:, 10:13] = 0.4
    front[:, 13] = np.inf
    back = np.zeros((1, 14), np.float32)
    back[0, 2], back[0, 3], back[0, 7:10], back[0, 10:13], back[0, 13] = -0.5, 1.0, -4.0, (0.5, -0.3, 0.2), 2.0
    g = np.random.default_rng(4).normal(size=(h, w, 4)).astype(np.float32)
    got, _ = gs3d_grad.backward(np.concatenate([front, back]), V, P, EYE, w, h, g)
    assert np.isfinite(got).all() and np.abs(got[:10]).max() > 0
    assert (got[10] == 0).all(), got[10]
    alone, _ = gs3d_grad.backward(back, V, P, EYE, w, h, g)
    assert (np.abs(alone[0, [0, 1, 7, 10, 13]]) > 0).all(), alone


def test_nan_logit_row_is_zero():
    """A NaN logit is drawn with alpha 0.99 (min(0.99, NaN)); its row is zero and every other row finite."""
    w, h = 24, 24
    V, P = V_single(w, h)
    rec = packed56(40, 9)
    rec[:, 0:3] *= 0.3
    rec[5, 13] = np.nan
    got, _ = gs3d_grad.backward(rec, V, P, EYE, w, h, np.random.default_rng(1).normal(size=(h, w, 4)).astype(np.float32))
    assert (got[5] == 0).all() and np.isfinite(got).all()


def test_count_zero_and_all_culled():
    V, P = V_single(16, 16)
    g = np.ones((16, 16, 4), np.float32)
    got, drawn = gs3d_grad.backward(np.zeros((0, 14), np.float32), V, P, EYE, 16, 16, g)
    assert got.shape == (0, 14) and drawn == 0
    rec = packed56(10, 3)
    rec[:, 2] = 10.0
    got, drawn = gs3d_grad.backward(rec, V, P, EYE, 16, 16, g)
    assert drawn == 0 and (got == 0).all()
