#!/usr/bin/env python3
"""Writes tests/golden/ref_depth_vectors.npz: outputs of the REFERENCE's own depthPrepassVS.glsl and of its viewer prepass
with u_depthTestMesh = 1 (gaussianSplattingPrepassCS.glsl:78-91), compiled here by oracle/build_depth.py and run in the
GL environment of oracle/ref_depth_harness.cpp.  Needs the reference checkout; the tests only read the .npz.

  vs*        vertex invocations: random positions (some far out) under the five prepass golden cameras and two extra
             rotated, scaled, translated model matrices: gl_Position
  case*      prepass inputs (REF96 records, camera, a depth map) and, per gaussian, whether the reference keeps it with
             the test on and with the test off (run one gaussian at a time), for u_format 0 and 1, plus the full
             prepass output with the test on (u_format 0).  Cases: the five prepass golden cases over random maps (alpha
             forced to 1 on half the records so the test runs); a crafted case whose records scan, ulp by ulp, across
             myDepth = depth + eps, across alpha = 0.95, and across uv = 0 and uv = 1, with uv outside [0, 1]; two cases
             with w = 0 at the eye (pos2d.z > 0: myDepth = inf; pos2d.z = 0: NaN) that reach the test and read the map
             at a NaN uv.

    python tests/golden/make_golden_depth.py
"""
from __future__ import annotations

import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_prepass import column_major, perspective  # noqa: E402
from oracle import depth  # noqa: E402
from oracle.build_depth import build_ref_depth  # noqa: E402

F32 = np.float32


def _rot(ax, ang):
    c, s = np.cos(ang), np.sin(ang)
    R = np.eye(4)
    i, j = [(1, 2), (0, 2), (0, 1)][ax]
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def _scan(x: float, n: int):
    """2n + 1 consecutive floats centred on x."""
    v = [F32(x)]
    for _ in range(n):
        v.insert(0, np.nextafter(v[0], F32(-np.inf)))
        v.append(np.nextafter(v[-1], F32(np.inf)))
    return np.array(v, F32)


def _record(pos, alpha=1.0):
    g = np.zeros(24, F32)
    g[0:3] = pos
    g[3] = 1.0
    g[4:7] = 0.5
    g[7] = alpha
    g[8:11] = 0.01
    g[16] = 1.0
    g[23] = 1.0
    return g


def crafted(rng):
    """Identity model and view, a 60 degree perspective; records on the decision boundaries of a random map."""
    W, H = 53, 37
    P = perspective(np.radians(60.0), W / H, 0.1, 10.0).astype(F32)
    dmap = rng.uniform(0.9, 0.999, (H, W)).astype(F32)
    dmap[::7, ::5] = 1.0
    t = np.tan(np.radians(30.0))
    A, B = float(P[2, 2]), float(P[2, 3])
    rows = []
    for _ in range(24):   # myDepth across depth + eps: the view z scanned 24 ulps either side of the boundary's solution
        u, v = rng.uniform(0.02, 0.98, 2)
        i, j = int(np.floor(F32(u) * F32(W))), int(np.floor(F32(v) * F32(H)))
        target = float(F32(dmap[j, i]) + F32(0.00002))
        zz = -B / ((2 * target - 1) + A)
        for z in _scan(zz, 24):
            rows.append(_record(((2 * u - 1) * W / H * t * -z, (2 * v - 1) * t * -z, z)))
    for a in _scan(0.95, 4):   # alpha across 0.95, behind the map
        u, v = rng.uniform(0.1, 0.9, 2)
        rows.append(_record(((2 * u - 1) * W / H * t * 9.0, (2 * v - 1) * t * 9.0, -9.0), alpha=float(a)))
    for edge in (-1.0, 1.0):   # uv across 0 and 1 (and the texel index across 0 and W - 1) in x and in y
        for z in (-1.0, -4.0, -9.5):
            ex = edge * W / H * t * -z
            for x in _scan(ex, 16):
                rows.append(_record((x, rng.uniform(-0.5, 0.5) * t * -z, z)))
            for y in _scan(edge * t * -z, 16):
                rows.append(_record((rng.uniform(-0.5, 0.5) * W / H * t * -z, y, z)))
    for _ in range(300):   # random, uv well outside [0, 1] included (the 1.05 w cull lets 2.5 % through)
        u, v = rng.uniform(-0.1, 1.1, 2)
        z = -rng.uniform(0.2, 9.8)
        rows.append(_record(((2 * u - 1) * W / H * t * -z, (2 * v - 1) * t * -z, z), alpha=float(rng.choice([1.0, 0.96, 0.95, 0.5]))))
    return np.array(rows, F32), np.eye(4, dtype=F32), P, np.eye(4, dtype=F32), (float(W * 16), float(H * 16)), (0.1, 10.0), dmap


def at_the_eye(rng, p14):
    """w = 0: records at the eye under a projection whose z row gives pos2d.z = p14 there (the 1.05 w cull keeps
    pos2d.z >= 0), so the test reads the map at a NaN uv."""
    W, H = 16, 8
    P = perspective(np.radians(60.0), 2.0, 0.1, 10.0).astype(F32)
    P[2, 3] = p14
    dmap = rng.uniform(0.5, 1.0, (H, W)).astype(F32)
    g = np.array([_record((0.0, 0.0, 0.0), a) for a in (1.0, 0.96, 0.5)] +
                 [_record((rng.uniform(-1, 1), rng.uniform(-0.5, 0.5), -rng.uniform(0.5, 5))) for _ in range(20)], F32)
    return g, np.eye(4, dtype=F32), P, np.eye(4, dtype=F32), (256.0, 128.0), (0.1, 10.0), dmap


def save_npz(path: str, arrays: dict) -> None:
    """np.savez_compressed with a fixed member date, so a rerun writes the same bytes."""
    with zipfile.ZipFile(path, "w") as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    if build_ref_depth() is None:
        sys.exit("the reference checkout is needed to build oracle/_ref/libm2s_refdepth.so")
    rng = np.random.default_rng(20260415)
    pre = np.load(os.path.join(HERE, "ref_prepass_vectors.npz"))
    out = {}
    # ---- vertex invocations ----
    cams = [(pre[f"view{i}"], pre[f"proj{i}"], pre[f"model{i}"]) for i in range(int(pre["ncases"]))]
    M1 = column_major((_rot(1, 0.7) @ _rot(0, -0.3) @ np.diag([1.3, 0.8, 2.1, 1.0]) + np.array([[0, 0, 0, 0.4], [0, 0, 0, -1.2], [0, 0, 0, 0.3], [0, 0, 0, 0]])).astype(F32))
    M2 = column_major((_rot(2, 2.1) @ np.diag([0.01, 0.02, 0.015, 1.0])).astype(F32))
    cams += [(cams[1][0], cams[1][1], M1), (cams[2][0], cams[2][1], M2)]
    for k, (V, P, M) in enumerate(cams):
        pos = np.concatenate([rng.normal(0, 1, (300, 3)), rng.normal(0, 100, (50, 3)), rng.uniform(-1e4, 1e4, (10, 3))]).astype(F32)
        out[f"vs_pos{k}"], out[f"vs_view{k}"], out[f"vs_proj{k}"], out[f"vs_model{k}"] = pos, V, P, M
        out[f"vs_out{k}"] = depth.ref_vs(pos, V, P, M)
    out["nvs"] = np.array(len(cams))
    # ---- the prepass with the test ----
    cases = []
    for i in range(int(pre["ncases"])):
        g = pre[f"g{i}"].copy()
        g[::2, 7] = 1.0
        prm = pre[f"params{i}"]
        res = (float(prm[0]), float(prm[1]))
        w, h = max(1, int(res[0]) // 8), max(1, int(res[1]) // 8)
        dmap = rng.uniform(0.0, 1.0, (h, w)).astype(F32) ** 0.05   # mostly close to 1, some texels near the records' depths
        dmap[rng.random((h, w)) < 0.2] = 1.0
        cases.append((g, pre[f"view{i}"], pre[f"proj{i}"], pre[f"model{i}"], res, (float(prm[2]), float(prm[3])), float(prm[4]), dmap))
    g, V, P, M, res, nf, dmap = crafted(rng)
    cases.append((g, V, column_major(P), M, res, nf, 0.01, dmap))
    for p14 in (0.2, 0.0):
        g, V, P, M, res, nf, dmap = at_the_eye(rng, p14)
        cases.append((g, V, column_major(P), M, res, nf, 0.01, dmap))
    for k, (g, V, P, M, res, nf, sd, dmap) in enumerate(cases):
        out[f"g{k}"], out[f"view{k}"], out[f"proj{k}"], out[f"model{k}"], out[f"map{k}"] = g, V, P, M, dmap
        out[f"params{k}"] = np.array([res[0], res[1], nf[0], nf[1], sd], F32)
        for fmt in (0, 1):
            on, off = depth.ref_keep(g, V, P, M, res, nf, sd, fmt, dmap)
            out[f"keep{k}_f{fmt}"], out[f"cull{k}_f{fmt}"] = on, off
        out[f"quads{k}"], out[f"depths{k}"] = depth.ref_prepass(g, V, P, M, res, nf, sd, 0, 0, dmap)
    out["ncases"] = np.array(len(cases))
    path = os.path.join(HERE, "ref_depth_vectors.npz")
    save_npz(path, out)
    print("wrote", path, os.path.getsize(path), "bytes;",
          [(int(out[f"cull{k}_f0"].sum()), int(out[f"keep{k}_f0"].sum())) for k in range(len(cases))], "(survivors off, on)")


if __name__ == "__main__":
    main()
