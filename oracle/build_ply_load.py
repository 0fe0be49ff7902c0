#!/usr/bin/env python3
"""Build the checkers of the .ply loader (row f-10; TEST INFRASTRUCTURE — never linked into the product).

  libm2s_ply_oracle.so         the plain-C restatement of loadPlyFile's per-vertex arithmetic (m2s_ply_oracle.c), always
                               built (gcc, no contraction, glibc's expf)
  _ref/libm2s_refplyload.so    the REFERENCE's own parsers::loadPlyFile (src/parsers/parsers.cpp + src/utils/utils.cpp with
                               the vendored happly), compiled where it lies with ref_ply_load_harness.cpp.  Only built when
                               the reference checkout exists; the library lives in oracle/_ref/ (git-ignored).
"""
from __future__ import annotations

import os
import sys

from oracle.build import _STUBS, CFLAGS, HERE, REF, REF_OUT, _newer, _run


def build_ply_oracle(force: bool = False) -> str:
    src = os.path.join(HERE, "m2s_ply_oracle.c")
    out = os.path.join(HERE, "libm2s_ply_oracle.so")
    hdr = os.path.join(HERE, "..", "include", "m2s.h")
    if force or not _newer(out, src, hdr, __file__):
        _run(["gcc", "-std=c11", *CFLAGS, "-o", out, src, "-lm"])
    return out


def build_ref_ply_load(force: bool = False) -> str | None:
    srcs = [os.path.join(REF, "src", "parsers", "parsers.cpp"), os.path.join(REF, "src", "utils", "utils.cpp")]
    out = os.path.join(REF_OUT, "libm2s_refplyload.so")
    if not all(os.path.exists(x) for x in srcs):
        return out if os.path.exists(out) else None
    harness = os.path.join(HERE, "ref_ply_load_harness.cpp")
    if not force and _newer(out, *srcs, harness, __file__):
        return out
    stubs = os.path.join(REF_OUT, "stubs")
    os.makedirs(stubs, exist_ok=True)
    for name, text in _STUBS.items():
        with open(os.path.join(stubs, name), "w") as f:
            f.write(text)
    tp = os.path.join(REF, "thirdParty")
    inc = ["-I", stubs, "-I", os.path.join(REF, "src"), "-I", os.path.join(REF, "src", "utils"), "-I", tp, "-I", os.path.join(tp, "glm"),
           "-I", os.path.join(tp, "glew", "include"), "-I", os.path.join(tp, "GLFW", "include"), "-I", os.path.join(tp, "imgui"),
           "-I", os.path.join(tp, "imgui", "backends")]
    _run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-w", "-ffp-contract=off", "-DGLEW_NO_GLU", "-include", os.path.join(stubs, "compat.h"),
          *inc, "-o", out, *srcs, harness, "-lstdc++fs"])
    return out


def build_all(force: bool = False) -> dict:
    return {"ply_oracle": build_ply_oracle(force), "ref_ply_load": build_ref_ply_load(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
