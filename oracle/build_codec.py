#!/usr/bin/env python3
"""Build the checker of the codec's device functions (TEST INFRASTRUCTURE — never linked into the product).

  libm2s_codec_oracle.so   the writer's and the loader's per-value formulas with glibc's logf / expf
                           (m2s_codec_oracle.c), always built (gcc, OpenMP, no contraction).  It reads nothing of the
                           reference checkout, so it builds wherever the package does.
"""
from __future__ import annotations

import os
import sys

from oracle.build import CFLAGS, HERE, _newer, _run


def build_codec_oracle(force: bool = False) -> str:
    src = os.path.join(HERE, "m2s_codec_oracle.c")
    out = os.path.join(HERE, "libm2s_codec_oracle.so")
    if force or not _newer(out, src, __file__):
        _run(["gcc", "-std=c11", "-fopenmp", *CFLAGS, "-o", out, src, "-lm"])
    return out


def build_all(force: bool = False) -> dict:
    return {"codec_oracle": build_codec_oracle(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
