#!/usr/bin/env python3
"""The standard 3DGS render (m2s_3dgs_render) on the bench scene, beside the reference-style chain (prepass -> sort ->
splat draw) on the same records, and the fidelity of its image against the mesh pass's albedo target.

Timing: R = 512 and 2048, 1920 x 1080 and 3840 x 2160, an outside and an inside view; CUDA events around `--iters`
enqueued calls after `--warmup`, the median of `--reps` windows.  Fidelity: R = 64 .. 2048 at 1920 x 1080 from the
outside view, m2s_image_compare of the 3DGS RGBA8 image against the mesh G-buffer's albedo, and of the splat draw's
albedo against the same, with both albedo targets as covers.  Prints one JSON document with the card's name and power
limit; `--out` also writes it to a file."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from make_golden_prepass import column_major, look_at, perspective  # noqa: E402
from mesh2splat_b200 import _abi, synth  # noqa: E402
from mesh2splat_b200.api import Context  # noqa: E402

VIEWS = {"outside": ((0.0, 0.5, 3.2), (0.0, 0.0, 0.0)), "inside": ((0.0, 0.0, 0.1), (0.0, 0.0, -1.0))}


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = (x.strip() for x in r.stdout.strip().splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def camera(view, w, h):
    eye, tgt = VIEWS[view]
    V = column_major(look_at(np.array(eye), np.array(tgt), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(60.0), w / h, 0.01, 100.0))
    return V, P


def timed(fn, warmup, iters, reps, stream):
    """median over reps of the mean ms per call of fn, every call enqueued on `stream` (a torch.cuda.Stream)"""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(iters):
            fn()
        b.record(stream)
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / iters)
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--timing-res", default="512,2048")
    ap.add_argument("--fidelity-res", default="64,128,256,512,1024,2048")
    ap.add_argument("--skip-fidelity", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    from mesh2splat_b200._lib import check, lib
    import ctypes as C
    res = {"card": card(), "timing": [], "fidelity": []}
    scene = synth.helmet_standin(2048)
    M = column_major(np.eye(4, dtype=np.float32))
    with Context(0) as ctx:
        ds = ctx.upload(scene)
        side = torch.cuda.Stream()   # a stream of its own: the events below time exactly the work enqueued on it
        stream = side.cuda_stream
        for R in [int(r) for r in args.timing_res.split(",")]:
            out = ctx.convert(ds, R, _abi.LAYOUT_REF96, 0.65, flags=_abi.FLAG_UNCAPPED)
            n = out.written
            quads = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
            depths = torch.empty(n, dtype=torch.float32, device="cuda")
            sq = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
            valid = torch.zeros(4, dtype=torch.int32, device="cuda")
            draw = torch.zeros(8, dtype=torch.int32, device="cuda")
            for (w, h) in ((1920, 1080), (3840, 2160)):
                for view in VIEWS:
                    V, P = camera(view, w, h)
                    _, _, pairs = ctx.render_3dgs(out.data, n, _abi.LAYOUT_REF96, V, P, M, w, h, near=0.01, std_dev=0.65 / R)
                    img8 = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
                    p3 = _abi.make_3dgs_params(V, P, M, w, h, 0.01, 0.65 / R, 1.0, (0, 0, 0), _abi.LAYOUT_REF96)
                    budget = min(pairs, (1 << 30) - 1)
                    t3 = timed(lambda: check(lib().m2s_3dgs_render_enqueue(ctx.handle, out.data.data_ptr(), n, None, C.byref(p3), None, 0, 0,
                                                                           None, img8.data_ptr(), budget, None, None, stream)),
                               args.warmup, args.iters, args.reps, side)
                    pp = _abi.make_prepass_params(V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 0, _abi.LAYOUT_REF96)
                    g = _abi.m2s_gbuffer()
                    alb = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
                    g.albedo = alb.data_ptr()
                    sp = _abi.m2s_splat_params(w, h, 0)
                    spairs = C.c_uint64(0)
                    q, _ = ctx.prepass(out.data, n, _abi.LAYOUT_REF96, V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 0, quads=quads, depths=depths)
                    ctx.depth_sort(quads, depths, len(q), sorted_quads=sq)
                    torch.cuda.synchronize()
                    lib().m2s_splat_draw(ctx.handle, sq.data_ptr(), len(q), C.byref(sp), C.byref(g), C.byref(spairs))
                    sbudget = min(int(spairs.value), (1 << 30) - 1)

                    def chain():
                        check(lib().m2s_prepass_enqueue(ctx.handle, out.data.data_ptr(), n, None, C.byref(pp), quads.data_ptr(),
                                                        depths.data_ptr(), valid.data_ptr(), stream))
                        check(lib().m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), n, valid.data_ptr(), sq.data_ptr(),
                                                           None, draw.data_ptr(), stream))
                        check(lib().m2s_splat_draw_enqueue(ctx.handle, sq.data_ptr(), n, draw.data_ptr(), C.byref(sp), C.byref(g), sbudget, None,
                                                           None, stream))
                    tc = timed(chain, args.warmup, args.iters, args.reps, side)
                    row = {"R": R, "gaussians": n, "width": w, "height": h, "view": view, "render_3dgs_ms": t3, "chain_ms": tc,
                           "pairs_3dgs": int(pairs), "pairs_splat_draw": int(spairs.value)}
                    print(json.dumps(row), flush=True)
                    res["timing"].append(row)
            del quads, depths, sq, out
            torch.cuda.empty_cache()
        w, h = 1920, 1080
        V, P = camera("outside", w, h)
        if args.skip_fidelity:
            args.fidelity_res = ""
        names = tuple(t for t, _ in _abi.GBUFFER_TARGETS)
        mbuf = {t: torch.empty(w * h * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda") for t, dt in _abi.GBUFFER_TARGETS}
        ctx.mesh_render(ds, V, P, M, w, h, (0.01, 100.0), 0, targets=names, gbuffer=mbuf)
        for R in [int(r) for r in args.fidelity_res.split(",") if r]:
            out = ctx.convert(ds, R, _abi.LAYOUT_REF96, 0.65, flags=_abi.FLAG_UNCAPPED)
            n = out.written
            imgs, _, _ = ctx.render_3dgs(out.data, n, _abi.LAYOUT_REF96, V, P, M, w, h, near=0.01, std_dev=0.65 / R, targets=("rgba8",))
            quads = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
            depths = torch.empty(n, dtype=torch.float32, device="cuda")
            sq = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
            q, _ = ctx.prepass(out.data, n, _abi.LAYOUT_REF96, V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 0, quads=quads, depths=depths)
            ctx.depth_sort(quads, depths, len(q), sorted_quads=sq)
            sbuf = {"albedo": torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")}
            ctx.splat_draw(sq, len(q), w, h, 0, targets=("albedo",), gbuffer=sbuf)
            a = ctx.compare_images(mbuf["albedo"], imgs["rgba8"], w, h, mbuf["albedo"], imgs["rgba8"])
            b = ctx.compare_images(mbuf["albedo"], sbuf["albedo"], w, h, mbuf["albedo"], sbuf["albedo"])
            row = {"R": R, "gaussians": n}
            for tag, r in (("3dgs", a), ("splat_draw", b)):
                for k in ("ssim", "psnr", "ssim_covered", "psnr_covered", "pixels_both", "pixels_a_only", "pixels_b_only"):
                    row[f"{tag}_{k}"] = r[k]
            print(json.dumps(row), flush=True)
            res["fidelity"].append(row)
            del quads, depths, sq, out
            torch.cuda.empty_cache()
        ds.free()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
