#!/usr/bin/env python3
"""Writes tests/golden/ref_light_vectors.npz from the REFERENCE's own shadow-pass and lighting shaders, compiled here by
oracle/build_light.py (needs the reference checkout).  Contents:

  light prepass   the five prepass golden cases (ref_prepass_vectors.npz) with four lights each: outside the cloud,
                  inside its box (all six faces), on a diagonal (face ties; cases 0 and 3 also get gaussians on the
                  light's diagonals), and exactly at a gaussian's world position.  Records as the oracle writes them.
  cube maps       the whole shadow pass of each case with the light inside, S = 64.
  pixel shader    2 400 invocations of gaussianSplattingDeferredPS.glsl on random texels (zeros, fp16 inf / NaN,
                  negative normals, all modes), plus 402 whose PCF comparisons sit exactly at the 0.05 bias threshold or one ulp either side.
  images          the full lighting pass in modes 0-6 over the five G-buffers of ref_splat_vectors.npz.

    python tests/golden/make_golden_light.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from mesh2splat_b200 import _abi  # noqa: E402
from oracle import build_light, light  # noqa: E402

F32 = np.float32
HERE = os.path.dirname(os.path.abspath(__file__))
LIGHTS = [(3.0, 4.0, 2.5), (0.05, 0.02, -0.03), (2.0, 2.0, 2.0)]


def world(M, p):   # GLM mat4 * vec4(p, 1) in fp32: (m0 x + m1 y) + (m2 z + m3)
    M = np.asarray(M, F32).reshape(4, 4)   # rows are columns (column-major storage)
    return [F32(F32(F32(M[0, r] * F32(p[0])) + F32(M[1, r] * F32(p[1]))) + F32(F32(M[2, r] * F32(p[2])) + M[3, r])) for r in range(3)]


def light_params(rng, n, modes):
    out = []
    for k in range(n):
        out.append(_abi.make_light_params(1, 1, int(modes[k]), tuple(rng.normal(0, 2, 3)), tuple(rng.uniform(0, 2, 3)),
                                          float(rng.uniform(0.5, 40)), tuple(rng.normal(0, 3, 3)), float(rng.uniform(5, 100)), 64))
    return out


def main():
    assert build_light.build_ref_light() is not None, "needs the reference checkout"
    zp = np.load(os.path.join(HERE, "ref_prepass_vectors.npz"))
    zs = np.load(os.path.join(HERE, "ref_splat_vectors.npz"))
    out = {}
    for i in range(5):
        g = zp[f"g{i}"].copy()
        prm, M = zp[f"params{i}"], zp[f"model{i}"]
        if i in (0, 3):   # identity models: gaussians on the diagonal light's diagonals
            t = np.linspace(0.1, 1.0, 10, dtype=F32)[:, None]
            g[10:20, :3] = np.array(LIGHTS[2], F32) + t * np.array([1, -1, 1], F32)
            g[20:30, :3] = np.array(LIGHTS[2], F32) + t * np.array([0, -1, 1], F32)
        lights = LIGHTS + [tuple(float(v) for v in world(M, g[3, :3]))]
        out[f"lg{i}"] = g
        out[f"lights{i}"] = np.array(lights, F32)
        for k, lp in enumerate(lights):
            p = _abi.make_shadow_params(M, lp, (prm[2], prm[3]), (prm[0], prm[1]), prm[4], 0, 64)
            out[f"rec{i}_{k}"] = light.ref_prepass(g, p, int(prm[6]))
        p = _abi.make_shadow_params(M, LIGHTS[1], (prm[2], prm[3]), (prm[0], prm[1]), prm[4], 0, 64)
        out[f"cube{i}"] = light.ref_cube(g, p, int(prm[6]))
    cube = out["cube0"]

    rng = np.random.default_rng(20261015)
    n = 2400
    pos = rng.normal(0, 2, (n, 4)).astype(np.float16)
    nrm = rng.random((n, 4)).astype(np.float16)
    nrm[: n // 5, :3] = -nrm[: n // 5, :3]                              # negative normals
    alb = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    mr = rng.integers(0, 256, (n, 4), dtype=np.uint8)
    mr[n // 2:, 2] = 0                                                   # metallic as the splat draw writes it
    zero = rng.random(n) < 0.05
    pos[zero] = 0; nrm[zero] = 0; alb[zero] = 0; mr[zero] = 0           # empty pixels
    for a in (pos, nrm):
        flat = a.reshape(-1)
        idx = rng.choice(len(flat), 240, replace=False)
        flat[idx[:60]] = np.inf; flat[idx[60:120]] = -np.inf; flat[idx[120:180]] = np.nan; flat[idx[180:]] = 0
    modes = np.where(rng.random(n) < 0.75, 6, rng.integers(0, 6, n))
    params = light_params(rng, n, modes)
    fs_out = np.zeros((n, 4), F32)
    fs_par = np.zeros((n, 12), F32)
    for k in range(n):
        fs_out[k] = light.deferred_fs(pos[k], nrm[k], alb[k], mr[k], cube, params[k], ref=True)
        q = params[k]
        fs_par[k] = [*q.light_position, *q.light_color, q.light_intensity, *q.cam_pos, q.far_plane, q.render_mode]
    out.update(fs_pos=pos.view(np.uint16), fs_nrm=nrm.view(np.uint16), fs_alb=alb, fs_mr=mr, fs_params=fs_par, fs_out=fs_out)

    # PCF threshold: a uniform 1 x 1 cube whose value v makes closest = v * far (far = 1) equal currentDepth - 0.05, or a
    # neighbour of it
    m = 402   # 134 positions, each at the threshold and one ulp either side of it
    tpos = np.repeat(rng.normal(0, 1, (m // 3, 4)).astype(np.float16), 3, axis=0)
    nd = np.array([0.2, 0.4, 0.6]) / np.linalg.norm([0.2, 0.4, 0.6])   # the decoded normal below: lights in front of it
    tl = (tpos[:, :3].astype(np.float64) + np.repeat(nd * rng.uniform(0.5, 3, (m // 3, 1)) + rng.normal(0, 0.2, (m // 3, 3)), 3, axis=0)).astype(F32)
    tv = np.zeros(m, F32)
    tout = np.zeros((m, 4), F32)
    for k in range(m):
        ld = tpos[k, :3].astype(F32) - tl[k]
        cur = np.sqrt(F32(F32(F32(ld[0] * ld[0]) + F32(ld[1] * ld[1])) + F32(ld[2] * ld[2])))
        thr = F32(cur - F32(0.05))
        tv[k] = [thr, np.nextafter(thr, F32(np.inf)), np.nextafter(thr, F32(-np.inf))][k % 3]
        q = _abi.make_light_params(1, 1, 6, tuple(tl[k]), (1.0, 1.0, 1.0), 5.0, (0.0, 0.0, 4.0), 1.0, 1)
        tout[k] = light.deferred_fs(tpos[k], np.array([0.6, 0.7, 0.8, 1], np.float16), np.array([200, 150, 100, 255], np.uint8),
                                    np.array([0, 128, 0, 255], np.uint8), np.full(6, tv[k], F32), q, ref=True)
    out.update(th_pos=tpos.view(np.uint16), th_light=tl, th_v=tv, th_out=tout)

    w, h = (int(v) for v in zs["img_size"])
    for c in range(5):
        gb = {t: zs[f"img{c}_{t}"] for t in ("position", "normal", "albedo", "metallic_roughness")}
        for mode in range(7):
            q = _abi.make_light_params(w, h, mode, LIGHTS[0], (1.0, 0.9, 0.8), 25.0, (3.0, 2.0, 4.0), 100.0, 64)
            out[f"img{c}_{mode}"] = light.ref_deferred_light(gb, cube, q)
    path = os.path.join(HERE, "ref_light_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
