#!/usr/bin/env python3
"""Build the checker of the viewer's mesh G-buffer pass and of the split-screen composite (SURVEY 8 row 14; TEST
INFRASTRUCTURE — never linked into the product).

  libm2s_mesh_oracle.so      the plain-C restatement (m2s_mesh_oracle.c), linked with the splat draw's (fp16 conversion,
                             exp) and the depth pass's (D24 code) restatements; always built (gcc, no contraction)
  _ref/libm2s_refmesh.so     the REFERENCE's own meshRenderVS.glsl and meshRenderPS.glsl (+ common.glsl), read where they
                             lie and turned into C++ by the splat draw's token rewrites, compiled against the reference's
                             vendored GLM with ref_mesh_harness.cpp (the GL environment: attributes, uniforms,
                             gl_Position, gl_PrimitiveID, and texture() returning a texel supplied per invocation).  Only
                             built when the reference checkout exists; the generated files live in oracle/_ref/
                             (git-ignored).
"""
from __future__ import annotations

import os
import sys

import re

from oracle.build import CFLAGS, HERE, REF, REF_OUT, _newer, _run, glsl_prepass_to_cpp
from oracle.build_splat import glsl_splat_to_cpp

SHADERS = ("meshRenderVS.glsl", "meshRenderPS.glsl", "common.glsl")


def build_mesh_oracle(force: bool = False) -> str:
    srcs = [os.path.join(HERE, n) for n in ("m2s_mesh_oracle.c", "m2s_splat_oracle.c", "m2s_depth_oracle.c")]
    out = os.path.join(HERE, "libm2s_mesh_oracle.so")
    if force or not _newer(out, *srcs, __file__):
        _run(["gcc", "-std=c11", *CFLAGS, "-o", out, *srcs, "-lm"])
    return out


def mesh_ps_to_cpp(ps: str, common: str) -> str:
    """meshRenderPS.glsl with common.glsl spliced where it is included -> one C++ include (token rewrites only)."""
    common_cpp = re.sub(r"\bexp\(", "glsl_exp(", glsl_prepass_to_cpp("", common))   # the built-in the environment supplies
    s = glsl_splat_to_cpp(ps.replace('#include "common.glsl"', "@COMMON@"))
    s = re.sub(r"\.(bg)\b(?!\s*\()", r".\1()", s)                                    # the one other rvalue swizzle
    return s.replace("@COMMON@", common_cpp)


def build_ref_mesh(force: bool = False) -> str | None:
    d = os.path.join(REF, "src", "shaders", "rendering")
    paths = [os.path.join(d, n) for n in SHADERS]
    glm = os.path.join(REF, "thirdParty", "glm")
    out = os.path.join(REF_OUT, "libm2s_refmesh.so")
    if not (all(os.path.exists(p) for p in paths) and os.path.isdir(glm)):
        return out if os.path.exists(out) else None
    harness = os.path.join(HERE, "ref_mesh_harness.cpp")
    if not force and _newer(out, *paths, harness, __file__):
        return out
    os.makedirs(REF_OUT, exist_ok=True)
    text = {}
    for n, p in zip(SHADERS, paths):
        with open(p) as f:
            text[n] = f.read()
    incs = {"meshVS.inc": glsl_splat_to_cpp(text[SHADERS[0]]), "meshPS.inc": mesh_ps_to_cpp(text[SHADERS[1]], text[SHADERS[2]])}
    for name, body in incs.items():
        with open(os.path.join(REF_OUT, name), "w") as f:
            f.write(body)
    _run(["g++", "-std=gnu++17", *CFLAGS, "-w", "-I", glm, "-I", REF_OUT, "-o", out, harness])
    return out


def build_all(force: bool = False) -> dict:
    return {"mesh_oracle": build_mesh_oracle(force), "ref_mesh": build_ref_mesh(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
