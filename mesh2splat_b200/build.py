#!/usr/bin/env python3
"""Builds mesh2splat_b200/libm2s.so — the C-ABI shared library (CUDA kernels for sm_90a + C++ host).

In-tree build with plain nvcc so the .so travels with the repository snapshot to the GPU box
(a JIT cache would not).  `python -m mesh2splat_b200.build [--force] [--verbose]`.
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libm2s.so")
# every translation unit and every header of csrc/, so that no edit can leave a stale library behind
SOURCES = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))
DEPS = sorted(glob.glob(os.path.join(CSRC, "*"))) + [os.path.join(HERE, "..", "include", "m2s.h"), os.path.abspath(__file__)]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force: bool = False, verbose: bool = False, out: str | None = None, defs: list | None = None) -> str:
    """out/defs: build a tuning or tracing variant (e.g. defs=['M2S_RASTER_WARPS=12'] or defs=['M2S_TRACE']) to another
    file; select it at run time with the M2S_LIB environment variable."""
    if out is None and not defs and not force and not _stale():
        return OUT
    out = out or OUT
    cmd = [_nvcc(), "-std=c++17", "-O3", "-lineinfo", *ARCH, "-shared", "-Xcompiler", "-fPIC,-fvisibility=hidden",
           "--cudart", "static", "-o", out, *[f"-D{d}" for d in (defs or [])], *SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("nvcc failed")
    if verbose:
        sys.stderr.write(r.stdout + r.stderr)
    return out


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    out = None
    defs = []
    for a in sys.argv[1:]:
        if a.startswith("--out="):
            out = a[6:]
        if a.startswith("--def="):
            defs.append(a[6:])
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, out=out, defs=defs))
