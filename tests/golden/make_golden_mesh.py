#!/usr/bin/env python3
"""Writes tests/golden/ref_mesh_vectors.npz: outputs of the REFERENCE's own meshRenderVS.glsl and meshRenderPS.glsl
(+ common.glsl), compiled here by oracle/build_mesh.py and run in the GL environment of oracle/ref_mesh_harness.cpp.
Needs the reference checkout; the tests only read the .npz.

  vs_*   vertex invocations: random vertices (some with zero or huge normals and tangents) under two cameras and five
         model matrices (identity, rotated and translated, mirrored, non-uniformly scaled, sheared): gl_Position and the
         13 varyings
  fs_*   fragment invocations: varyings (from the vertex stage and random, with zero tangents, tangents parallel to the
         normal and tangent.w in {-1, 0, 1}), texels (unorm values and arbitrary floats), every render mode, every
         combination of bound maps, base colour factors, near/far, gl_PrimitiveID (small and large): the five targets'
         fp32 values; fs_sinf holds the C library's sinf of render mode 3's three arguments, as the shader called it

    python tests/golden/make_golden_mesh.py
"""
from __future__ import annotations

import ctypes
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_prepass import column_major, look_at, perspective  # noqa: E402
from oracle import mesh  # noqa: E402
from oracle.build_mesh import build_ref_mesh  # noqa: E402

F32 = np.float32
OUT = os.path.join(HERE, "ref_mesh_vectors.npz")
HASH_ARGS = ((311.7, 0.0), (269.5, 1.3), (183.3, 2.7))


def _rot(ax, ang):
    c, s = np.cos(ang), np.sin(ang)
    m = np.eye(4)
    i, j = [(1, 2), (2, 0), (0, 1)][ax]
    m[i, i], m[i, j], m[j, i], m[j, j] = c, -s, s, c
    return m


def models():
    t = np.eye(4)
    t[:3, 3] = (0.3, -0.2, 0.5)
    shear = np.eye(4)
    shear[0, 1], shear[2, 0] = 0.4, -0.3
    return [np.eye(4), t @ _rot(1, 0.7) @ _rot(0, -0.3), np.diag([-1.0, 1.0, 1.0, 1.0]), np.diag([2.5, 0.3, 1.2, 1.0]) @ _rot(2, 0.4),
            shear @ _rot(1, 1.1)]


def cameras():
    out = []
    for eye, aspect, near, far in (((0.0, 0.5, 3.2), 16 / 9, 0.01, 100.0), ((2.0, -1.0, -1.5), 1.0, 0.1, 20.0)):
        V = look_at(np.array(eye), np.zeros(3), np.array([0.0, 1.0, 0.0]))
        out.append((column_major(V), column_major(perspective(np.radians(50.0), aspect, near, far)), (near, far)))
    return out


def vertices(rng, n):
    v = np.zeros((n, 12), F32)
    v[:, 0:3] = rng.normal(0, 1.5, (n, 3))
    v[:, 3:6] = rng.normal(0, 1, (n, 3))
    v[:, 6:9] = rng.normal(0, 1, (n, 3))
    v[:, 9] = rng.choice([-1.0, 1.0], n)
    v[:, 10:12] = rng.uniform(-3, 5, (n, 2))
    v[0, 3:6] = 0.0                 # zero normal
    v[1, 6:9] = 0.0                 # zero tangent
    v[2, 3:6] = (1e20, -3e19, 2e19)  # a normal whose dot overflows
    v[3, 6:9] = v[3, 3:6] * 2       # tangent parallel to the normal
    v[4, 0:3] = (1e5, -2e5, 3e4)    # far out
    return v


def main():
    if build_ref_mesh() is None:
        sys.exit("the reference checkout is needed to build oracle/_ref/libm2s_refmesh.so")
    rng = np.random.default_rng(20261017)
    a = {}
    vs_in, vs_V, vs_P, vs_M, vs_clip, vs_vary = [], [], [], [], [], []
    for V, P, _ in cameras():
        for M in models():
            Mc = column_major(M)
            v = vertices(rng, 64)
            clip, vary = mesh.ref_vs(v, V, P, Mc)
            vs_in.append(v); vs_V.append(V); vs_P.append(P); vs_M.append(Mc); vs_clip.append(clip); vs_vary.append(vary)
    a.update(vs_vtx=np.array(vs_in), vs_V=np.array(vs_V), vs_P=np.array(vs_P), vs_M=np.array(vs_M), vs_clip=np.array(vs_clip),
             vs_vary=np.array(vs_vary))

    n = 7 * 8 * 40
    pool = np.concatenate(vs_vary).reshape(-1, 13)
    vary = pool[rng.integers(0, len(pool), n)].copy()
    rnd = rng.random(n) < 0.4
    vary[rnd] = rng.normal(0, 2, (int(rnd.sum()), 13)).astype(F32)
    vary[:, 12] = np.where(rng.random(n) < 0.8, rng.uniform(-1, 30, n), vary[:, 12])
    k = rng.integers(0, 5, n)
    vary[k == 0, 6:9] = 0.0                                                   # zero tangent
    vary[k == 1, 6:9] = vary[k == 1, 3:6] * F32(-3.0)                         # tangent parallel to the normal
    vary[:, 9] = rng.choice([-1.0, 0.0, 1.0], n)
    tex = (rng.integers(0, 256, (n, 12)) / F32(255.0)).astype(F32)
    odd = rng.random(n) < 0.2
    tex[odd] = rng.uniform(-0.5, 1.5, (int(odd.sum()), 12)).astype(F32)
    tex[k == 2, 4:7] = 0.5                                                    # a normal-map texel of zero length
    mode = np.repeat(np.arange(7), n // 7).astype(np.int32)
    has = np.tile(np.repeat(np.arange(8), 40), 7).astype(np.int32)
    factor = rng.uniform(0, 1.2, (n, 4)).astype(F32)
    near_far = np.where(rng.random((n, 1)) < 0.5, np.array([[0.01, 100.0]]), np.array([[0.5, 8.0]])).astype(F32)
    prim = np.where(rng.random(n) < 0.5, rng.integers(0, 2000, n), rng.integers(0, 1 << 24, n)).astype(np.int32)
    out = np.array([mesh.ref_fs(vary[i], tex[i], has[i], factor[i], near_far[i], mode[i], prim[i]) for i in range(n)], F32)
    libm = ctypes.CDLL("libm.so.6")
    libm.sinf.restype, libm.sinf.argtypes = ctypes.c_float, [ctypes.c_float]
    sinf = np.array([[libm.sinf(float(F32(F32(p) * F32(m) + F32(c)))) for m, c in HASH_ARGS] for p in prim], F32)
    a.update(fs_vary=vary, fs_tex=tex, fs_has=has, fs_factor=factor, fs_near_far=near_far, fs_mode=mode, fs_prim=prim, fs_out=out,
             fs_sinf=sinf)
    with zipfile.ZipFile(OUT, "w") as z:   # a fixed member date: a rerun writes the same bytes
        for name in sorted(a):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(a[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
