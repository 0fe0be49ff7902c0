#!/usr/bin/env python3
"""The 3DGS render's backward pass on the bench scene: the forward pass that keeps its state (m2s_3dgs_render_grad_enqueue)
against m2s_3dgs_render_enqueue, and the backward pass (m2s_3dgs_backward_enqueue), at R = 512 and 2048, 1920 x 1080,
from gs3d_bench.py's outside and inside views.  CUDA events around `--iters` enqueued calls after `--warmup`, the median of
`--reps` windows, each call with the pair budget the synchronous form found.  Prints one JSON document with the card's
name and power limit; `--out` also writes it to a file."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gs3d_bench import ROOT, VIEWS, camera, card, timed  # noqa: E402,F401

from mesh2splat_b200 import _abi, synth  # noqa: E402
from mesh2splat_b200.api import Context  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", default="512,2048")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from mesh2splat_b200._lib import check, lib
    L = lib()
    res = {"card": card(), "timing": []}
    scene = synth.helmet_standin(2048)
    M = np.eye(4, dtype=np.float32).T.copy()
    w, h = 1920, 1080
    with Context(0) as ctx, ctx.gs3d_state() as state:
        ds = ctx.upload(scene)
        side = torch.cuda.Stream()
        for R in [int(x) for x in args.res.split(",")]:
            out = ctx.convert(ds, R, _abi.LAYOUT_PACKED56)
            n = out.written
            prm = out.data[: n * 56].view(torch.float32)
            img = torch.empty(w * h * 4, dtype=torch.float32, device="cuda")
            gimg = torch.randn(w * h * 4, dtype=torch.float32, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
            grad = torch.empty(n * 14, dtype=torch.float32, device="cuda")
            words = torch.zeros(4, dtype=torch.int32, device="cuda")
            for view in VIEWS:
                V, P = camera(view, w, h)
                p = _abi.make_3dgs_params(V, P, M, w, h, 0.2, 1.0, 1.0, (0, 0, 0), _abi.LAYOUT_PACKED56)
                pairs = C.c_uint64(0)
                torch.cuda.synchronize()
                check(L.m2s_3dgs_render_grad(ctx.handle, state.handle, prm.data_ptr(), n, C.byref(p), img.data_ptr(), C.byref(pairs)))
                budget, s = pairs.value, side.cuda_stream
                render = lambda: check(L.m2s_3dgs_render_enqueue(ctx.handle, prm.data_ptr(), n, None, C.byref(p), None, 0, 0, img.data_ptr(),  # noqa: E731
                                                                 None, budget, words.data_ptr(), words[2:].data_ptr(), s))
                fwd = lambda: check(L.m2s_3dgs_render_grad_enqueue(ctx.handle, state.handle, prm.data_ptr(), n, C.byref(p), img.data_ptr(),  # noqa: E731
                                                                   budget, words.data_ptr(), words[2:].data_ptr(), s))
                bwd = lambda: check(L.m2s_3dgs_backward_enqueue(ctx.handle, state.handle, prm.data_ptr(), n, C.byref(p), gimg.data_ptr(),  # noqa: E731
                                                                grad.data_ptr(), s))
                row = {"R": R, "view": view, "width": w, "height": h, "gaussians": n, "pairs": budget,
                       "render_ms": timed(render, args.warmup, args.iters, args.reps, side),
                       "grad_forward_ms": timed(fwd, args.warmup, args.iters, args.reps, side)}
                fwd()
                row["backward_ms"] = timed(bwd, args.warmup, args.iters, args.reps, side)
                res["timing"].append(row)
                print(json.dumps(row), flush=True)
        ds.free()
    doc = json.dumps(res, indent=1)
    print(doc)
    if args.out:
        with open(args.out, "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
