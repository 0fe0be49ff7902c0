"""CPU tests: the density bound that lets a PACKED56 conversion end in the raster kernel (m2s_dscene::r_small_max).

The bound is restated here over the oracle's orthographic uv, with the rule of small_box_density (m2s_plane.cuh): a
triangle whose uv spans eu x ev has a candidate box of at most floor(eu R + 1/64) + 1 columns (rows likewise), so its box
is small at every R <= max over w of min((w - 1/32) / eu, (min(32, 64 / w) - 1/32) / ev).  Every triangle's actual box,
as the oracle's set-up computes it, must then be small (<= 64 pixels, <= 32 rows) at densities up to the scene's bound:
seeded random meshes and the benchmark's scene, whose density (512) must be under its bound.
"""
from __future__ import annotations

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, synth

SMALL_CAND = 64   # kSmallCand


def ortho_uv(scene: _abi.Scene) -> np.ndarray:
    """(n, 3, 2) orthographic uv of every triangle over its primitive's box (the oracle's set-up)."""
    out = np.zeros((scene.triangle_count, 3, 2), np.float32)
    for p in scene.primitives:
        for t in range(p.first_triangle, p.first_triangle + p.triangle_count):
            out[t] = np.array(oracle.triangle_setup(scene.triangles[t], p.bbox_min, p.bbox_max, 64).ouv, np.float32)
    return out


def triangle_bounds(ouv: np.ndarray) -> np.ndarray:
    """Per triangle: the largest R at which its candidate box is certainly small (+inf where the uv is not finite)."""
    ext = (ouv.max(axis=1) - ouv.min(axis=1)).astype(np.float32)
    eu, ev = ext[:, 0], ext[:, 1]
    best = np.zeros(len(ext), np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        for w in range(1, SMALL_CAND + 1):
            h = min(32, SMALL_CAND // w)
            rw = np.where(eu > 0, np.float32(w - 0.03125) / eu, np.float32(np.inf))
            rh = np.where(ev > 0, np.float32(h - 0.03125) / ev, np.float32(np.inf))
            best = np.maximum(best, np.minimum(rw, rh))
    best[~np.isfinite(ext).all(axis=1)] = np.inf
    return best


def scene_r_small_max(scene: _abi.Scene) -> float:
    return float(triangle_bounds(ortho_uv(scene)).min())


def largest_box(scene: _abi.Scene, R: int) -> tuple:
    """(pixels, rows) of the largest candidate box the oracle's set-up gives any triangle at density R."""
    px, rows = 0, 0
    for p in scene.primitives:
        for t in range(p.first_triangle, p.first_triangle + p.triangle_count):
            s = oracle.triangle_setup(scene.triangles[t], p.bbox_min, p.bbox_max, R)
            w, h = s.x1 - s.x0 + 1, s.y1 - s.y0 + 1
            if s.valid and s.area2 != 0 and w > 0 and h > 0:
                px, rows = max(px, w * h), max(rows, h)
    return px, rows


def soup_scene(seed: int, n: int = 3000, tri_size: float = 0.02) -> _abi.Scene:
    s = _abi.Scene(synth.random_soup(n, seed, tri_size=tri_size), [_abi.Primitive(0, n, (1.0, 1.0, 1.0, 1.0), -1, -1, -1)], [])
    s.compute_bboxes()
    return s


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_meshes_small_under_the_bound(seed):
    scene = soup_scene(seed)
    r = scene_r_small_max(scene)
    assert 8 < r < 4096
    for R in sorted({int(r), int(r) - 1, int(0.75 * r), int(0.5 * r)}):
        px, rows = largest_box(scene, R)
        assert px <= SMALL_CAND and rows <= 32, (R, px, rows)
    # and the bound is not vacuous: well above it some box is not small
    px, rows = largest_box(scene, int(2 * r) + 2)
    assert px > SMALL_CAND or rows > 32


def test_bench_scene_is_eligible():
    """The benchmark's scene (helmet stand-in, R = 512) is under its bound, and every box is small at the bound."""
    scene = synth.helmet_standin(16)
    r = scene_r_small_max(scene)
    assert r >= 512
    for R in (512, int(r)):
        px, rows = largest_box(scene, R)
        assert px <= SMALL_CAND and rows <= 32, (R, px, rows)
