#!/usr/bin/env python3
"""Generates tests/golden/ref_splat_vectors.npz from the REFERENCE's own splat shaders (row f-6).

Runs only where the reference checkout exists: oracle/build_splat.py compiles gaussianSplattingVS.glsl and
gaussianSplattingPS.glsl (token rewrites only) with the GL environment of oracle/ref_splat_harness.cpp into
oracle/_ref/libm2s_refsplat.so; this script feeds it seeded inputs and stores inputs + outputs:
  (a) vertex-shader invocations (quads of ref_prepass_vectors.npz, all four vertices, several viewports) and
      fragment-shader invocations (their varyings at pixel centres around the mean, plus extreme conics), modes 0 and 4;
  (b) full 192 x 108 images of every target for the five prepass cases, stably sorted by depth bits, one render mode
      per case (0, 1, 2, 4, 6).

    python tests/golden/make_golden_splat.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import splat  # noqa: E402
from oracle.build_splat import build_ref_splat  # noqa: E402

W, H = 192, 108
MODES = (0, 1, 2, 4, 6)


def sorted_case(z, i):
    q, d = z[f"quads{i}"], z[f"depths{i}"]
    return np.ascontiguousarray(q[np.argsort(d.view(np.uint32), kind="stable")])


def main():
    assert build_ref_splat() is not None, "needs the reference checkout"
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_prepass_vectors.npz"))
    rng = np.random.default_rng(20261015)
    out = {}
    # (a) invocations
    vq, vv, vres, vout = [], [], [], []
    for i in range(int(z["ncases"])):
        q = sorted_case(z, i)
        for k in rng.choice(len(q), 40, replace=False):
            for v in range(4):
                res = [(1280.0, 720.0), (1.0, 1.0), (4096.0, 4096.0), (17.0, 15.0)][int(rng.integers(0, 4))]
                vq.append(q[k]); vv.append(v); vres.append(res)
                vout.append(splat.vs(q[k], v, res[0], res[1], ref=True))
    out["vs_quads"] = np.array(vq, np.float32); out["vs_vertex"] = np.array(vv, np.int32)
    out["vs_resolution"] = np.array(vres, np.float32); out["vs_out"] = np.array(vout, np.float32)
    fv, fxy, fm, fo = [], [], [], []
    for j in range(len(vout)):
        var = vout[j][2:].copy()
        if j % 50 == 0:
            var[2:5] = [1e3, -1e3, 5e2] if j % 100 else [-3e4, 0.0, np.inf]   # positive exponents, inf and NaN
        for _ in range(3):
            xy = np.floor(var[0:2] + rng.normal(0, 3, 2)) + 0.5
            mode = 4 if rng.random() < 0.25 else int(rng.choice([0, 1, 2, 5, 6]))
            fv.append(var); fxy.append(xy); fm.append(mode)
            fo.append(splat.fs(var, float(xy[0]), float(xy[1]), mode, ref=True))
    out["fs_varyings"] = np.array(fv, np.float32); out["fs_fragcoord"] = np.array(fxy, np.float32)
    out["fs_mode"] = np.array(fm, np.int32); out["fs_out"] = np.array(fo, np.float32)
    # (b) images
    for i, mode in enumerate(MODES):
        img = splat.draw(sorted_case(z, i), W, H, mode, ref=True)
        for t, _ in splat.TARGETS:
            out[f"img{i}_{t}"] = img[t]
    out["img_modes"] = np.array(MODES, np.int32)
    out["img_size"] = np.array([W, H], np.int32)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_splat_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes;", len(vout), "vertex and", len(fo), "fragment invocations")


if __name__ == "__main__":
    main()
