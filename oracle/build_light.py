#!/usr/bin/env python3
"""Build the checkers of the viewer's shadow pass and deferred lighting (rows f-7, f-8; TEST INFRASTRUCTURE — never
linked into the product).

  libm2s_light_oracle.so      the plain-C restatement (m2s_light_oracle.c), always built (gcc, no contraction)
  _ref/libm2s_reflight.so     the REFERENCE's own gaussianPointShadowMappingCS.glsl (+ common.glsl),
                              gaussianPointLightCubeMapShadowVS/PS.glsl and gaussianSplattingDeferredVS/PS.glsl, read where
                              they lie and turned into C++ by the token rewrites below, compiled against the reference's
                              vendored GLM with ref_light_harness.cpp (the GL environment: dispatch with per-face counters,
                              the face draws, samplers, pow / exp2 / log2, RGBA8 store).  Only built when the reference
                              checkout exists; the generated files live in oracle/_ref/ (git-ignored).
"""
from __future__ import annotations

import os
import re
import sys

from oracle.build import CFLAGS, HERE, REF, REF_OUT, _newer, _run, glsl_prepass_to_cpp
from oracle.build_splat import glsl_splat_to_cpp

SHADERS = ("gaussianPointShadowMappingCS.glsl", "common.glsl", "gaussianPointLightCubeMapShadowVS.glsl",
           "gaussianPointLightCubeMapShadowPS.glsl", "gaussianSplattingDeferredVS.glsl", "gaussianSplattingDeferredPS.glsl")


def build_light_oracle(force: bool = False) -> str:
    src = os.path.join(HERE, "m2s_light_oracle.c")
    out = os.path.join(HERE, "libm2s_light_oracle.so")
    if force or not _newer(out, src, __file__):
        _run(["gcc", "-std=c11", *CFLAGS, "-o", out, src, "-lm"])
    return out


def glsl_shadow_cs_to_cpp(src: str, common: str) -> str:
    """gaussianPointShadowMappingCS.glsl + common.glsl -> one C++ include: the prepass shader's rewrites plus the
    uniform array declarator and the per-face indirect-command block."""
    src = re.sub(r"uniform\s+mat4\s*\[\s*6\s*\]\s+(\w+)\s*;", r"uniform mat4 \1[6];", src)
    src = re.sub(r"layout\s*\(std430,\s*binding\s*=\s*\d+\)\s*buffer\s+\w+\s*\{\s*(\w+)\s+(\w+\[\d+\]);\s*\}\s*;", r"static \1 \2;", src)
    return glsl_prepass_to_cpp(src, common).replace("void prepass_main()", "void main_cs()")


def glsl_deferred_to_cpp(src: str) -> str:
    """gaussianSplattingDeferredPS.glsl -> C++: the splat shaders' rewrites plus the array constructor, the .rg swizzle
    and the built-ins the environment supplies (texture, pow).  The PI macro is left to the C++ preprocessor."""
    s = re.sub(r"=\s*vec3\[\]\s*\((.*?)\)\s*;", r"= {\1};", src, flags=re.S)
    s = re.sub(r"\.rg\b(?!\s*\()", ".rg()", s)
    s = re.sub(r"\btexture\(", "glsl_texture(", s)
    s = re.sub(r"\bpow\(", "glsl_pow(", s)
    return glsl_splat_to_cpp(s)


def build_ref_light(force: bool = False) -> str | None:
    d = os.path.join(REF, "src", "shaders", "rendering")
    paths = [os.path.join(d, n) for n in SHADERS]
    glm = os.path.join(REF, "thirdParty", "glm")
    out = os.path.join(REF_OUT, "libm2s_reflight.so")
    if not (all(os.path.exists(p) for p in paths) and os.path.isdir(glm)):
        return out if os.path.exists(out) else None
    harness = os.path.join(HERE, "ref_light_harness.cpp")
    if not force and _newer(out, *paths, harness, __file__):
        return out
    os.makedirs(REF_OUT, exist_ok=True)
    text = {}
    for n, p in zip(SHADERS, paths):
        with open(p) as f:
            text[n] = f.read()
    incs = {"lightCS.inc": glsl_shadow_cs_to_cpp(text[SHADERS[0]], text[SHADERS[1]]),
            "lightCubeVS.inc": glsl_splat_to_cpp(text[SHADERS[2]]),
            "lightCubePS.inc": glsl_splat_to_cpp(text[SHADERS[3]]),
            "lightDeferredVS.inc": glsl_splat_to_cpp(text[SHADERS[4]]),
            "lightDeferredPS.inc": glsl_deferred_to_cpp(text[SHADERS[5]])}
    for name, body in incs.items():
        with open(os.path.join(REF_OUT, name), "w") as f:
            f.write(body)
    _run(["g++", "-std=gnu++17", *CFLAGS, "-w", "-I", glm, "-I", REF_OUT, "-o", out, harness])
    return out


def build_all(force: bool = False) -> dict:
    return {"light_oracle": build_light_oracle(force), "ref_light": build_ref_light(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
