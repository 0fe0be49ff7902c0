#!/usr/bin/env python3
"""Build the checkers of the viewer's splat draw (row f-6; TEST INFRASTRUCTURE — never linked into the product).

  libm2s_splat_oracle.so      the plain-C restatement (m2s_splat_oracle.c), always built (gcc)
  _ref/libm2s_refsplat.so     the REFERENCE's own gaussianSplattingVS.glsl and gaussianSplattingPS.glsl, read where they
                              lie and turned into C++ by the token rewrites below, compiled against the reference's
                              vendored GLM with ref_splat_harness.cpp (the GL environment: instanced draw loop,
                              rasteriser, blend, target formats, the exp built-in).  Only built when the reference
                              checkout exists; the generated files live in oracle/_ref/ (git-ignored).
"""
from __future__ import annotations

import os
import re
import sys

from oracle.build import _FLOAT_LIT, CFLAGS, REF, REF_OUT, HERE, _newer, _run


def build_splat_oracle(force: bool = False) -> str:
    src = os.path.join(HERE, "m2s_splat_oracle.c")
    out = os.path.join(HERE, "libm2s_splat_oracle.so")
    if force or not _newer(out, src, __file__):
        _run(["gcc", "-std=c11", *CFLAGS, "-o", out, src, "-lm"])
    return out


def glsl_splat_to_cpp(src: str) -> str:
    """gaussianSplattingVS.glsl / gaussianSplattingPS.glsl -> a C++ include (qualifier, literal and swizzle tokens only)."""
    s = re.sub(r"^\s*#version.*$", "", src, flags=re.M)
    s = _FLOAT_LIT.sub(lambda m: m.group(1) + "f", s)                          # GLSL literals are float
    s = re.sub(r"layout\s*\(\s*location\s*=\s*\d+\s*\)\s*(?:in|out)\s+", "static ", s)
    s = re.sub(r"^\s*(?:uniform|in|out)\s+(\w+\s+\w+\s*;)", r"static \1", s, flags=re.M)
    s = re.sub(r"\.(xyz|xzy|xy|zw|rgb)\b(?!\s*\()", r".\1()", s)               # rvalue swizzles -> GLM swizzle functions
    s = s.replace(".xy() + 1)", ".xy() + 1.0f)")                                # GLSL converts the int
    s = re.sub(r"\bexp\(", "glsl_exp(", s)                                      # the built-in the environment supplies
    return s.replace("void main()", "void shader_main()")


def build_ref_splat(force: bool = False) -> str | None:
    d = os.path.join(REF, "src", "shaders", "rendering")
    vs, ps = os.path.join(d, "gaussianSplattingVS.glsl"), os.path.join(d, "gaussianSplattingPS.glsl")
    glm = os.path.join(REF, "thirdParty", "glm")
    out = os.path.join(REF_OUT, "libm2s_refsplat.so")
    if not (os.path.exists(vs) and os.path.exists(ps) and os.path.isdir(glm)):
        return out if os.path.exists(out) else None
    harness = os.path.join(HERE, "ref_splat_harness.cpp")
    if not force and _newer(out, vs, ps, harness, __file__):
        return out
    os.makedirs(REF_OUT, exist_ok=True)
    for src, name in ((vs, "splatVS.inc"), (ps, "splatPS.inc")):
        with open(src) as f, open(os.path.join(REF_OUT, name), "w") as g:
            g.write(glsl_splat_to_cpp(f.read()))
    _run(["g++", "-std=gnu++17", *CFLAGS, "-w", "-I", glm, "-I", REF_OUT, "-o", out, harness])
    return out


def build_all(force: bool = False) -> dict:
    return {"splat_oracle": build_splat_oracle(force), "ref_splat": build_ref_splat(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
