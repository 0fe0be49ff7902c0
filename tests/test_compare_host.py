"""The image comparison's checker (oracle/m2s_compare_oracle.c) on the CPU: the window taps, the map against an fp64
statement of Wang et al.'s valid-window SSIM within the bound DESIGN §2 derives, known answers, and the coverage totals
against numpy."""
from __future__ import annotations

import math

import numpy as np
import pytest

from mesh2splat_b200 import _abi
from oracle import compare as oc

U = 2.0 ** -24
C1, C2 = oc.constants()
# DESIGN §2: each fp32 moment is within 24 u of its fp64 value relative to 255^2 (22 roundings in the two passes, one in
# the taps), so each variance and the covariance within 73 u 255^2; the numerator and denominator factors that carry them
# change by at most twice that, each over a factor >= C2 (the others move by far less): |s32 - s64| <= 4 (73 u 255^2) / C2
# + 1e-5 per channel, and so for the mean of the three.
BOUND = 4 * 73 * U * 255.0 ** 2 / float(C2) + 1e-5


def _images():
    rng = np.random.default_rng(1)
    h, w = 40, 57
    yield "random", rng.integers(0, 256, (h, w, 4), dtype=np.uint8), rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    g = np.stack([(xx * 4) % 256, (yy * 6) % 256, ((xx + yy) * 3) % 256, np.full_like(xx, 255)], -1).astype(np.uint8)
    yield "smooth gradient", g, np.clip(g.astype(int) + rng.integers(-3, 4, g.shape), 0, 255).astype(np.uint8)
    yield "flat", np.full((h, w, 4), 250, np.uint8), np.full((h, w, 4), 251, np.uint8)
    c = ((xx // 3 + yy // 3) % 2 * 255).astype(np.uint8)
    c = np.stack([c, c, 255 - c, c], -1)
    yield "high contrast", c, np.roll(c, 1, axis=1)
    yield "near 255", rng.integers(245, 256, (h, w, 4), dtype=np.uint8), rng.integers(245, 256, (h, w, 4), dtype=np.uint8)


def test_taps_are_the_fp64_gaussian_rounded_once():
    t = oc.taps()
    want = oc.gaussian_window().astype(np.float32)
    assert t.tobytes() == want.tobytes()
    assert np.array_equal(t, t[::-1])
    assert C1 == np.float32((0.01 * 255) ** 2) and C2 == np.float32((0.03 * 255) ** 2)


@pytest.mark.parametrize("case", range(5))
def test_map_within_the_derived_bound_of_fp64_ssim(case):
    name, a, b = list(_images())[case]
    r, m, planes = oc.compare(a, b, a.shape[1], a.shape[0])
    ref = oc.reference_ssim(a, b)
    err = float(np.abs(m.astype(np.float64) - ref).max())
    assert err <= BOUND, (name, err, BOUND)
    assert BOUND / max(err, 1e-300) > 5, f"{name}: margin {BOUND / err:.1f}x is thinner than DESIGN §2 states"
    for c in range(3):
        assert r["ssim_sum"][c] == pytest.approx(math.fsum(planes[c].astype(np.float64).ravel()), rel=1e-12)
    assert r["ssim"] == pytest.approx(ref.mean(), abs=BOUND)


@pytest.mark.parametrize("wh", [(11, 11), (12, 30), (64, 17)])
def test_identical_images_give_one_everywhere(wh):
    w, h = wh
    a = np.random.default_rng(w * h).integers(0, 256, (h, w, 4), dtype=np.uint8)
    r, m, planes = oc.compare(a, a.copy(), w, h)
    assert (m == np.float32(1.0)).all() and (planes == np.float32(1.0)).all()
    assert r["sq_err"] == [0, 0, 0] and r["psnr"] == math.inf and r["ssim"] == 1.0
    assert r["windows"] == (w - 10) * (h - 10)


def test_two_constant_images_closed_form():
    w, h = 20, 16
    a = np.empty((h, w, 4), np.uint8)
    b = np.empty((h, w, 4), np.uint8)
    a[...] = (10, 200, 255, 0)
    b[...] = (40, 190, 0, 255)
    r, m, planes = oc.compare(a, b, w, h)
    t = oc.taps()
    want = []
    for c in range(3):
        mom = []
        for q in (a[0, 0, c], b[0, 0, c], np.float32(a[0, 0, c]) * np.float32(a[0, 0, c]), np.float32(b[0, 0, c]) * np.float32(b[0, 0, c]),
                  np.float32(a[0, 0, c]) * np.float32(b[0, 0, c])):
            q = np.float32(q)
            row = t[0] * q
            for i in range(1, 11):
                row = np.float32(row + np.float32(t[i] * q))
            col = np.float32(t[0] * row)
            for j in range(1, 11):
                col = np.float32(col + np.float32(t[j] * row))
            mom.append(col)
        mx, my, exx, eyy, exy = mom
        mx2, my2, mxy = np.float32(mx * mx), np.float32(my * my), np.float32(mx * my)
        num = np.float32(np.float32(np.float32(2 * mxy) + C1) * np.float32(np.float32(2 * np.float32(exy - mxy)) + C2))
        den = np.float32(np.float32(np.float32(mx2 + my2) + C1) * np.float32(np.float32(np.float32(exx - mx2) + np.float32(eyy - my2)) + C2))
        want.append(np.float32(num / den))
        assert (planes[c] == want[-1]).all()
        assert oc.ssim_value(mx, my, exx, eyy, exy) == want[-1]
    assert (m == np.float32(np.float32(np.float32(want[0] + want[1]) + want[2]) / np.float32(3))).all()
    assert r["sq_err"] == [30 * 30 * w * h, 10 * 10 * w * h, 255 * 255 * w * h]


def test_one_changed_pixel():
    w, h = 40, 30
    a = np.random.default_rng(3).integers(0, 256, (h, w, 4), dtype=np.uint8)
    b = a.copy()
    x, y = 17, 12
    b[y, x, 1] = (int(a[y, x, 1]) + 77) % 256
    d = int(b[y, x, 1]) - int(a[y, x, 1])
    r, m, planes = oc.compare(a, b, w, h)
    assert r["sq_err"] == [0, d * d, 0]
    assert (planes[0] == 1).all() and (planes[2] == 1).all()
    wy, wx = np.nonzero(m < 1)
    inside = (abs(wx + 5 - x) <= 5) & (abs(wy + 5 - y) <= 5)
    assert inside.all() and len(wx) == 121
    assert r["psnr"] == pytest.approx(10 * math.log10(255 ** 2 * 3 * w * h / (d * d)))


def test_inverted_image():
    w, h = 33, 25
    a = np.random.default_rng(5).integers(0, 256, (h, w, 4), dtype=np.uint8)
    b = (255 - a).astype(np.uint8)
    r, m, _ = oc.compare(a, b, w, h)
    d = a[..., :3].astype(np.int64) - b[..., :3].astype(np.int64)
    assert r["sq_err"] == [int((d[..., c] ** 2).sum()) for c in range(3)]
    assert np.abs(m - oc.reference_ssim(a, b)).max() <= BOUND
    assert (m < 0.1).all()


@pytest.mark.parametrize("cover_min", [1, 128, 255])
def test_coverage_counts_and_covered_totals(cover_min):
    w, h = 47, 29
    rng = np.random.default_rng(cover_min)
    a, b = rng.integers(0, 256, (h, w, 4), dtype=np.uint8), rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    ca, cb = rng.integers(0, 256, (h, w, 4), dtype=np.uint8), rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    ca[::3, :, 3] = 0
    cb[:, ::4, 3] = 255
    d2 = (a[..., :3].astype(np.int64) - b[..., :3].astype(np.int64)) ** 2
    _, m, planes = oc.compare(a, b, w, h)
    for covers in ((ca, cb), (ca, None), (None, cb), (None, None)):
        r, _, _ = oc.compare(a, b, w, h, *covers, cover_min=cover_min)
        ia = covers[0][..., 3] >= cover_min if covers[0] is not None else np.zeros((h, w), bool)
        ib = covers[1][..., 3] >= cover_min if covers[1] is not None else np.zeros((h, w), bool)
        cov = ia | ib
        assert (r["pixels_both"], r["pixels_a_only"], r["pixels_b_only"]) == (int((ia & ib).sum()), int((ia & ~ib).sum()), int((ib & ~ia).sum()))
        assert r["sq_err_covered"] == [int(d2[..., c][cov].sum()) for c in range(3)]
        wc = cov[5:-5, 5:-5]
        assert r["covered_windows"] == int(wc.sum())
        for c in range(3):
            assert r["ssim_covered_sum"][c] == pytest.approx(math.fsum(planes[c][wc].astype(np.float64)), rel=1e-12, abs=0)
        if covers[0] is None and covers[1] is None:
            assert r["covered_windows"] == r["pixels_both"] == 0 and r["sq_err_covered"] == [0, 0, 0]
            assert math.isnan(r["ssim_covered"]) and math.isnan(r["psnr_covered"])


def test_sizes_and_cover_min_out_of_range_are_rejected():
    a = np.zeros((11, 11, 4), np.uint8)
    with pytest.raises(ValueError):
        oc.compare(np.zeros((11, 10, 4), np.uint8), np.zeros((11, 10, 4), np.uint8), 10, 11)
    for cm in (0, 256):
        with pytest.raises(ValueError):
            oc.compare(a, a, 11, 11, cover_min=cm)


def test_result_struct_layout():
    assert _abi.C.sizeof(_abi.m2s_compare_result) == 17 * 8
    assert _abi.C.sizeof(_abi.m2s_compare_params) == 12
