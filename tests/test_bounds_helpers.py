"""CPU tests of the helpers the GPU bounds tests stand on (tests/test_gpu_bounds.py): the layered tilings' totals, the
guarded buffers' checks and the triangle-soup .glb writer."""
from __future__ import annotations

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, synth
from util import GUARD_BYTE, GuardedHost, layered_tiling, write_soup_glb


@pytest.mark.parametrize("R", [16, 50])
@pytest.mark.parametrize("kind", ["delaunay", "strips"])
def test_layered_tiling_total_is_k_r2(oracle_lib, kind, R):
    """Each layer covers every pixel centre exactly once, so the oracle's total is k R^2 and every pixel of every layer
    appears once; with one primitive the reference's cap (6 R^2) stores 6 of 7 layers."""
    k = 7
    s = layered_tiling(k, R, kind, n=200 if kind == "delaunay" else 37, seed=1, wide=2 if kind == "strips" else 0)
    assert len(s.primitives) == 1
    rec, keys, total = oracle.convert(s, R, _abi.LAYOUT_PACKED56, flags=_abi.FLAG_UNCAPPED, capacity=k * R * R + 16)
    assert total == len(rec) == k * R * R
    per_layer = s.triangle_count // k
    layer = (keys >> np.uint64(24)).astype(np.int64) // per_layer
    pix = (keys & np.uint64(0xFFFFFF)).astype(np.int64)
    for i in range(k):
        assert len(np.unique(pix[layer == i])) == R * R
    _, _, capped = oracle.convert(s, R, _abi.LAYOUT_PACKED56, capacity=_abi.reference_capacity(R, 1))
    assert capped == k * R * R and _abi.reference_capacity(R, 1) == 6 * R * R


def test_strips_are_full_height_and_the_wide_ones_32_pixels():
    R = 256
    s = layered_tiling(1, R, "strips", n=40, wide=3)
    v = s.triangles.reshape(-1, 3, 12)
    assert np.all(v[:, :, 1].min(axis=1) == 0.0) and np.all(v[:, :, 1].max(axis=1) == 1.0)
    width = (v[:, :, 0].max(axis=1) - v[:, :, 0].min(axis=1)) * R
    np.testing.assert_allclose(width[:3], 32.0, rtol=1e-5)
    assert np.all(width[3:40] < 5.0)


def test_guarded_host_buffer_catches_overrun_and_hole():
    g = GuardedHost(10, 8, what="t")
    g.view[:5 * 8] = 0
    g.check(5)
    with pytest.raises(AssertionError, match="guard bytes"):
        g.check(4)                      # record 4 lies beyond `written`
    g.view[5 * 8] = 1
    with pytest.raises(AssertionError, match="guard bytes"):
        g.check(5)
    g.view[5 * 8] = GUARD_BYTE
    g.view[2 * 8: 3 * 8] = GUARD_BYTE   # an unwritten record below `written`
    with pytest.raises(AssertionError, match="never written"):
        g.check(5)
    g.raw[0] = 0
    with pytest.raises(AssertionError, match="guard bytes"):
        g.check(0)


def test_soup_glb_round_trips_through_the_loader(tmp_path):
    from mesh2splat_b200.gltf import load_glb
    s = layered_tiling(3, 32, "delaunay", n=40, seed=2)
    tex = synth.random_texture(16, 8, 5)
    p = tmp_path / "soup.glb"
    write_soup_glb(str(p), s.triangles, texture=tex, base_color=(0.5, 0.25, 1.0, 0.75))
    got = load_glb(str(p))
    assert got.triangle_count == s.triangle_count and len(got.primitives) == 1
    assert np.array_equal(got.triangles, s.triangles)
    pr = got.primitives[0]
    assert pr.albedo_texture == 0 and pr.normal_texture == -1 and pr.metallic_roughness_texture == -1
    np.testing.assert_allclose(pr.base_color_factor, (0.5, 0.25, 1.0, 0.75), rtol=1e-6)
    assert np.array_equal(got.textures[0], tex)
    assert pr.bbox_min == s.primitives[0].bbox_min and pr.bbox_max == s.primitives[0].bbox_max
    write_soup_glb(str(p), s.triangles)
    assert load_glb(str(p)).primitives[0].albedo_texture == -1
