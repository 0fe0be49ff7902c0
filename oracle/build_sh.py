#!/usr/bin/env python3
"""Build the checker of the prepass's view-dependent colour (m2s_prepass_sh; TEST INFRASTRUCTURE — never linked into the
product).

  libm2s_sh_oracle.so   the plain-C restatement of the SH colour (m2s_sh_oracle.c, gcc, no contraction), linked against
                        libm2s_oracle.so for orc_prepass.  It restates graphdeco's published formula, not the reference
                        (which skips the coefficients), so nothing here reads a reference checkout.
"""
from __future__ import annotations

import os
import sys

from oracle.build import CFLAGS, HERE, _newer, _run, build_oracle


def build_sh_oracle(force: bool = False) -> str:
    base = build_oracle(force)
    src = os.path.join(HERE, "m2s_sh_oracle.c")
    out = os.path.join(HERE, "libm2s_sh_oracle.so")
    if force or not _newer(out, src, base, __file__):
        _run(["gcc", "-std=c11", *CFLAGS, "-o", out, src, "-L", HERE, "-l:libm2s_oracle.so", "-Wl,-rpath,$ORIGIN", "-lm"])
    return out


def build_all(force: bool = False) -> dict:
    return {"sh_oracle": build_sh_oracle(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
