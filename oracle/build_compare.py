#!/usr/bin/env python3
"""Build the checker of the image comparison (m2s_image_compare; TEST INFRASTRUCTURE — never linked into the product).

  libm2s_compare_oracle.so   the plain-C restatement of the SSIM map and the totals (m2s_compare_oracle.c, gcc, OpenMP, no
                             contraction).  It restates the definition DESIGN §2 fixes (Wang et al. 2004), which the
                             reference does not have, so nothing here reads a reference checkout.
"""
from __future__ import annotations

import os
import sys

from oracle.build import CFLAGS, HERE, _newer, _run


def build_compare_oracle(force: bool = False) -> str:
    src = os.path.join(HERE, "m2s_compare_oracle.c")
    hdr = os.path.join(HERE, "..", "include", "m2s.h")
    out = os.path.join(HERE, "libm2s_compare_oracle.so")
    if force or not _newer(out, src, hdr, __file__):
        _run(["gcc", "-std=c11", "-fopenmp", *CFLAGS, "-o", out, src])
    return out


def build_all(force: bool = False) -> dict:
    return {"compare_oracle": build_compare_oracle(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
