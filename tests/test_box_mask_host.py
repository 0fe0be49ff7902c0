"""CPU test of the raster kernel's coverage walk of small triangles (box_mask, m2s_span.cuh): compiled for the host with
g++ and checked against the per-pixel coverage rule on random triangles (slivers, ties on pixel centres) and on every box
shape up to the small-triangle limits (w x h <= 64 pixels, h <= 32), each walked as the last lane and behind longer lanes."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_box_mask_matches_per_pixel_coverage(tmp_path):
    exe = str(tmp_path / "box_mask_harness")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "box_mask_harness.cpp")], check=True)
    r = subprocess.run([exe, "200000"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.startswith("ok ")
