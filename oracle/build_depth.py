#!/usr/bin/env python3
"""Build the checker of the viewer's mesh depth pre-pass and the prepass's mesh depth test (row f-9; TEST
INFRASTRUCTURE — never linked into the product).

  libm2s_depth_oracle.so      the plain-C restatement (m2s_depth_oracle.c), always built (gcc, no contraction)
  _ref/libm2s_refdepth.so     the REFERENCE's own depthPrepassVS.glsl, depthPrepassPS.glsl and
                              gaussianSplattingPrepassCS.glsl (+ common.glsl), read where they lie and turned into C++ by
                              the token rewrites of the splat draw and the prepass, compiled against the reference's
                              vendored GLM with ref_depth_harness.cpp (the GL environment: attributes, gl_Position,
                              gl_FragCoord, the SSBOs and counter, and the depth texture as a NEAREST / CLAMP_TO_EDGE
                              sampler with u_depthTestMesh = 1).  Only built when the reference checkout exists; the
                              generated files live in oracle/_ref/ (git-ignored).
"""
from __future__ import annotations

import os
import sys

from oracle.build import CFLAGS, HERE, REF, REF_OUT, _newer, _run, glsl_prepass_to_cpp
from oracle.build_splat import glsl_splat_to_cpp

SHADERS = ("depthPrepassVS.glsl", "depthPrepassPS.glsl", "gaussianSplattingPrepassCS.glsl", "common.glsl")


def build_depth_oracle(force: bool = False) -> str:
    src = os.path.join(HERE, "m2s_depth_oracle.c")
    out = os.path.join(HERE, "libm2s_depth_oracle.so")
    if force or not _newer(out, src, __file__):
        _run(["gcc", "-std=c11", *CFLAGS, "-o", out, src, "-lm"])
    return out


def build_ref_depth(force: bool = False) -> str | None:
    d = os.path.join(REF, "src", "shaders", "rendering")
    paths = [os.path.join(d, n) for n in SHADERS]
    glm = os.path.join(REF, "thirdParty", "glm")
    out = os.path.join(REF_OUT, "libm2s_refdepth.so")
    if not (all(os.path.exists(p) for p in paths) and os.path.isdir(glm)):
        return out if os.path.exists(out) else None
    harness = os.path.join(HERE, "ref_depth_harness.cpp")
    if not force and _newer(out, *paths, harness, __file__):
        return out
    os.makedirs(REF_OUT, exist_ok=True)
    text = {}
    for n, p in zip(SHADERS, paths):
        with open(p) as f:
            text[n] = f.read()
    incs = {"depthVS.inc": glsl_splat_to_cpp(text[SHADERS[0]]),
            "depthPS.inc": glsl_splat_to_cpp(text[SHADERS[1]]),
            "depthPrepassCS.inc": glsl_prepass_to_cpp(text[SHADERS[2]], text[SHADERS[3]])}
    for name, body in incs.items():
        with open(os.path.join(REF_OUT, name), "w") as f:
            f.write(body)
    _run(["g++", "-std=gnu++17", *CFLAGS, "-w", "-I", glm, "-I", REF_OUT, "-o", out, harness])
    return out


def build_all(force: bool = False) -> dict:
    return {"depth_oracle": build_depth_oracle(force), "ref_depth": build_ref_depth(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
