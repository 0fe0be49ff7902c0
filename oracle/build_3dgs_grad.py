#!/usr/bin/env python3
"""Build the checker of the standard 3DGS render's backward pass (m2s_3dgs_backward_enqueue; TEST INFRASTRUCTURE — never
linked into the product).

  libm2s_3dgs_grad_oracle.so   the plain-C restatement of DESIGN §2's backward pass (m2s_3dgs_grad_oracle.c, gcc, no
                               contraction), linked against the forward checker (orc_3dgs_preprocess) and the splat draw's
                               checker for its exp (orc_splat_exp = rn_exp).  It restates graphdeco's published backward
                               pass, so nothing here reads a reference checkout.
"""
from __future__ import annotations

import os
import sys

from oracle.build import CFLAGS, HERE, _newer, _run
from oracle.build_3dgs import build_3dgs_oracle
from oracle.build_splat import build_splat_oracle


def build_3dgs_grad_oracle(force: bool = False) -> str:
    deps = [build_3dgs_oracle(force), build_splat_oracle(force)]
    src = os.path.join(HERE, "m2s_3dgs_grad_oracle.c")
    out = os.path.join(HERE, "libm2s_3dgs_grad_oracle.so")
    if force or not _newer(out, src, *deps, __file__):
        _run(["gcc", "-std=c11", *CFLAGS, "-Wall", "-o", out, src, "-L", HERE, "-l:libm2s_3dgs_oracle.so", "-l:libm2s_splat_oracle.so",
              "-l:libm2s_sh_oracle.so", "-l:libm2s_oracle.so", "-Wl,-rpath,$ORIGIN", "-lm"])
    return out


def build_all(force: bool = False) -> dict:
    return {"3dgs_grad_oracle": build_3dgs_grad_oracle(force)}


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv))
