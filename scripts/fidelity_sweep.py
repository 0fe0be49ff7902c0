#!/usr/bin/env python3
"""How closely the splats reproduce their mesh at each conversion density (beyond the reference, whose split screen is
judged by eye), and what the comparison itself costs.

Scene and views: the bench scene (helmet stand-in, 70 074 triangles, three 2048^2 maps) at 1920 x 1080, seen from
mesh_bench.py's camera outside the model and from a second outside camera above and to the side.  Densities R in
{64, 128, 256, 512, 1024, 2048} (uncapped), render modes 0, 2 and 6.  Per case:
  - the mesh drawn into its G-buffer (m2s_mesh_render) and lit (m2s_deferred_light);
  - convert -> prepass -> sort -> splat draw (plus the shadow cube, S = 1024, in mode 6) and lit, the mesh lit with the
    same cube, as the split screen does;
  - the two lit images compared (m2s_image_compare, mesh = A, splats = B) with the albedo targets as covers
    (cover_min 128): gaussians, PSNR, SSIM, covered PSNR and SSIM, and the mesh-only / splat-only pixels.
Cost: m2s_image_compare_enqueue at 1920 x 1080 and 3840 x 2160 with both covers and the map, CUDA events around each
call, 5 warm-up calls, median of 50; bytes/s against the 16 B per pixel the call must read (two images, two covers),
and the share of the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run.

    python scripts/fidelity_sweep.py [--out results/fidelity.json] [--rs 64,128,...] [--modes 0,2,6]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from make_golden_prepass import column_major, look_at, perspective  # noqa: E402
from mesh2splat_b200 import _abi, synth  # noqa: E402
from mesh2splat_b200._lib import check, lib  # noqa: E402
from mesh2splat_b200.api import Context  # noqa: E402
from sort_bench import card  # noqa: E402

W, H, S = 1920, 1080, 1024
NEAR_FAR = (0.01, 100.0)
LIGHT = (1.5, 2.0, 2.5)
VIEWS = {"outside": ((0.0, 0.5, 3.2), (0.0, 0.0, 0.0)), "side": ((2.4, 1.4, 1.6), (0.0, 0.0, 0.0))}
HBM_PEAK = 3.35e12
BYTES_PER_PIXEL = 16


def time_compare(ctx, iters: int):
    rows = []
    stream = torch.cuda.Stream()
    for w, h in ((1920, 1080), (3840, 2160)):
        g = torch.Generator(device="cuda").manual_seed(w)
        imgs = [torch.randint(0, 256, (w * h * 4,), dtype=torch.uint8, device="cuda", generator=g) for _ in range(4)]
        res = torch.zeros(C.sizeof(_abi.m2s_compare_result), dtype=torch.uint8, device="cuda")
        smap = torch.empty((w - 10) * (h - 10), dtype=torch.float32, device="cuda")
        p = _abi.m2s_compare_params(w, h, 128)
        torch.cuda.synchronize()

        def call():
            check(lib().m2s_image_compare_enqueue(ctx.handle, *[t.data_ptr() for t in imgs], C.byref(p), res.data_ptr(), smap.data_ptr(),
                                                  stream.cuda_stream))
        for _ in range(5):
            call()
        times = []
        for _ in range(iters):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            call()
            b.record(stream)
            b.synchronize()
            times.append(a.elapsed_time(b) * 1e3)
        t = float(np.median(times))
        nb = BYTES_PER_PIXEL * w * h
        rows.append({"size": f"{w}x{h}", "us": t, "us_min": float(np.min(times)), "bytes": nb, "GBps": nb / (t * 1e-6) / 1e9,
                     "hbm_share": nb / (t * 1e-6) / HBM_PEAK})
        print(f"compare {w}x{h}: {t:8.1f} us (min {min(times):.1f})  {rows[-1]['GBps']:7.1f} GB/s of 16 B/px "
              f"({100 * rows[-1]['hbm_share']:.1f} % of 3.35 TB/s)", flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--rs", default="64,128,256,512,1024,2048")
    ap.add_argument("--modes", default="0,2,6")
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    ctx = Context(0)
    L, hc = lib(), ctx.handle
    results = {"card": card(), "size": f"{W}x{H}", "cases": []}
    print(f"# {results['card']}", flush=True)
    results["compare"] = time_compare(ctx, args.iters)

    scene = synth.helmet_standin(2048)
    ds = ctx.upload(scene)
    layout = _abi.LAYOUT_REF96
    M = column_major(np.eye(4, dtype=np.float32))
    alloc = lambda: {t: torch.empty(W * H * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda")  # noqa: E731
                     for t, dt in _abi.GBUFFER_TARGETS}
    mbuf, sbuf = alloc(), alloc()
    gm = _abi.m2s_gbuffer(*[mbuf[t].data_ptr() for t, _ in _abi.GBUFFER_TARGETS])
    gs = _abi.m2s_gbuffer(*[sbuf[t].data_ptr() for t, _ in _abi.GBUFFER_TARGETS])
    mimg = torch.empty(W * H * 4, dtype=torch.uint8, device="cuda")
    simg = torch.empty(W * H * 4, dtype=torch.uint8, device="cuda")
    cube = torch.empty(6 * S * S, dtype=torch.float32, device="cuda")
    draw = torch.zeros(5, dtype=torch.int32, device="cuda")
    print(f"{'view':8s} {'mode':>4s} {'R':>5s} {'gaussians':>10s} {'PSNR':>7s} {'SSIM':>7s} {'PSNRcov':>8s} {'SSIMcov':>8s} "
          f"{'mesh-only':>10s} {'splat-only':>10s}", flush=True)
    for vname, (eye, tgt) in VIEWS.items():
        V = column_major(look_at(np.array(eye), np.array(tgt), np.array([0.0, 1.0, 0.0])).astype(np.float32))
        P = column_major(perspective(np.radians(45.0), W / H, 0.01, 100.0))
        for mode in [int(m) for m in args.modes.split(",")]:
            mp = _abi.make_mesh_render_params(V, P, M, W, H, NEAR_FAR, mode)
            check(L.m2s_mesh_render(hc, ds.handle, C.byref(mp), C.byref(gm), None))
            lp = _abi.make_light_params(W, H, mode, LIGHT, (1.0, 1.0, 1.0), 10.0, eye, 100.0, S)
            for R in [int(r) for r in args.rs.split(",")]:
                out = ctx.convert(ds, R, layout, 0.65, flags=_abi.FLAG_UNCAPPED)
                assert not out.overflow
                n = out.written
                quads = torch.empty(max(1, n) * _abi.QUAD_BYTES, dtype=torch.uint8, device="cuda")
                depths = torch.empty(max(1, n), dtype=torch.float32, device="cuda")
                sq = torch.empty(max(1, n) * _abi.QUAD_BYTES, dtype=torch.uint8, device="cuda")
                pp = _abi.make_prepass_params(V, P, M, (W, H), NEAR_FAR, 0.65 / R, mode, layout)
                valid = C.c_uint32(0)
                check(L.m2s_prepass(hc, out.data.data_ptr(), n, C.byref(pp), quads.data_ptr(), depths.data_ptr(), C.byref(valid)))
                m = int(valid.value)
                check(L.m2s_depth_sort(hc, quads.data_ptr(), depths.data_ptr(), m, sq.data_ptr(), None, draw.data_ptr()))
                check(L.m2s_splat_draw(hc, sq.data_ptr(), m, C.byref(_abi.m2s_splat_params(W, H, mode)), C.byref(gs), None))
                d_cube = None
                if mode == 6:
                    shp = _abi.make_shadow_params(M, LIGHT, NEAR_FAR, (W, H), 0.65 / R, layout, S)
                    check(L.m2s_shadow_map(hc, out.data.data_ptr(), n, C.byref(shp), cube.data_ptr(), None, None))
                    d_cube = cube.data_ptr()
                check(L.m2s_deferred_light(hc, C.byref(gm), d_cube, C.byref(lp), mimg.data_ptr()))
                check(L.m2s_deferred_light(hc, C.byref(gs), d_cube, C.byref(lp), simg.data_ptr()))
                r = ctx.compare_images(mimg, simg, W, H, mbuf["albedo"], sbuf["albedo"], 128)
                row = {"view": vname, "mode": mode, "R": R, "gaussians": n, "in_view": m, "psnr": r["psnr"], "ssim": r["ssim"],
                       "psnr_covered": r["psnr_covered"], "ssim_covered": r["ssim_covered"], "pixels_both": r["pixels_both"],
                       "mesh_only": r["pixels_a_only"], "splat_only": r["pixels_b_only"]}
                results["cases"].append(row)
                print(f"{vname:8s} {mode:4d} {R:5d} {n:10d} {r['psnr']:7.2f} {r['ssim']:7.4f} {r['psnr_covered']:8.2f} "
                      f"{r['ssim_covered']:8.4f} {r['pixels_a_only']:10d} {r['pixels_b_only']:10d}", flush=True)
                del out, quads, depths, sq
                torch.cuda.empty_cache()
    ds.free()
    ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
