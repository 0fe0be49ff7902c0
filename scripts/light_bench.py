#!/usr/bin/env python3
"""Times the viewer's shadow pass and deferred lighting (rows f-7, f-8) on the GPU.

Inputs: the bench scene (helmet stand-in) converted at R = 512 and R = 2048 in both record layouts.  Per case:
  - the shadow pass at S = 1024 (m2s_shadow_map_enqueue) with a light outside the model and one inside it, as a whole
    (CUDA events, L2 flushed before each run, median) and split into the light prepass and the cube raster (the sum
    of each group's kernel times from torch.profiler, in a pass of its own);
  - the lighting pass in modes 0 and 6 at 1920 x 1080 and 3840 x 2160 over the splat draw's G-buffer (R = 512 only),
    with the bytes it must move (24 B of G-buffer read and 4 B written per pixel in mode 6, 4 + 4 in mode 0, cube taps
    not counted) against the H100 SXM data-sheet bandwidth (3350 GB/s, not a measured peak);
  - the whole one-stream frame convert -> prepass -> sort -> draw -> shadow -> light at 1920 x 1080.
The card's name and power limit are read in the same run.

    python scripts/light_bench.py [--iters 15] [--out results/light_bench.json]
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

HBM_GBS = 3350.0   # H100 SXM data sheet
S = 1024
LIGHTS = {"outside": (1.5, 2.0, 2.5), "inside": (0.0, 0.05, 0.0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    ctx = Context(0)
    L = lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    h = stream.cuda_stream
    results = {"card": card(), "peak_GBps": HBM_GBS, "peak_source": "H100 SXM data sheet (not measured)", "shadow": [], "light": [], "frame": []}
    print(f"# {results['card']}  (HBM {HBM_GBS:.0f} GB/s, data sheet)")

    def timed(fn):
        flush.zero_()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            a.record(stream)
            fn()
            b.record(stream)
        torch.cuda.synchronize()
        return a.elapsed_time(b) * 1e3   # us

    def median(fn):
        t = [timed(fn) for _ in range(args.iters + 3)][3:]
        return float(np.median(t))

    def kernel_split(fn):
        """(light prepass us, cube raster us) per call: device time of each group's kernels, summed, from the profiler."""
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                with torch.cuda.stream(stream):
                    fn()
            torch.cuda.synchronize()
        pre = ras = 0.0
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            if "light_prepass_kernel" in e.key:
                pre += t
            elif "shadow_" in e.key or "ShadowBins" in e.key or "sort_" in e.key:
                ras += t
        return pre / args.iters, ras / args.iters

    scene = synth.helmet_standin(2048)
    ds = ctx.upload(scene)
    V = column_major(look_at(np.array([0.0, 0.5, 3.2]), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(45.0), 16 / 9, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    cube = torch.empty(6 * S * S, dtype=torch.float32, device="cuda")
    lq_dev = None
    for R in (512, 2048):
        for layout, lname in ((_abi.LAYOUT_REF96, "ref96"), (_abi.LAYOUT_PACKED56, "packed56")):
            cap = 6 * R * R
            out = torch.empty(cap * _abi.STRIDES[layout], dtype=torch.uint8, device="cuda")
            total = torch.zeros(1, dtype=torch.int64, device="cuda")
            p = _abi.make_params(R, layout, 0.65, 0, _abi.FLAG_UNCAPPED)
            check(L.m2s_convert_enqueue(ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), h))
            stream.synchronize()
            n = int(total.item())
            lq_dev = torch.empty(n * 32, dtype=torch.uint8, device="cuda")
            res = torch.zeros(4, dtype=torch.int32, device="cuda")
            for lname2, lpos in LIGHTS.items():
                shp = _abi.make_shadow_params(M, lpos, (0.01, 100.0), (1920, 1080), 0.65 / R, layout, S)
                pairs_t = C.c_uint64(0)
                check(L.m2s_shadow_map(ctx.handle, out.data_ptr(), n, C.byref(shp), cube.data_ptr(), lq_dev.data_ptr(), C.byref(pairs_t)))
                pairs = int(pairs_t.value)
                budget = pairs + pairs // 8 + 1

                def shadow():
                    check(L.m2s_shadow_map_enqueue(ctx.handle, out.data_ptr(), n, None, C.byref(shp), cube.data_ptr(), lq_dev.data_ptr(),
                                                   budget, res.data_ptr(), res[2:].data_ptr(), h))
                t = median(shadow)
                t_pre, t_ras = kernel_split(shadow)
                o = res.cpu().numpy()
                assert int(o[2]) == n and int(o[:2].view(np.uint64)[0]) == pairs
                rb = n * _abi.STRIDES[layout] + n * 32   # the light prepass's bytes: records in, light records out
                row = {"case": f"R={R} {lname} light {lname2}", "gaussians": n, "pairs": pairs, "shadow_us": t, "light_prepass_us": t_pre,
                       "cube_raster_us": t_ras, "prepass_GBps": rb / (t_pre * 1e-6) / 1e9 if t_pre else None}
                results["shadow"].append(row)
                print(f"{row['case']:34s} n {n:9d} pairs {pairs:10d}  shadow {t:9.1f} us = light prepass {t_pre:8.1f} us "
                      f"({row['prepass_GBps'] or 0:6.0f} GB/s) + cube raster {t_ras:9.1f} us", flush=True)
            del out
            torch.cuda.empty_cache()

    # lighting over the splat draw's G-buffer, and the whole frame (R = 512)
    R, layout = 512, _abi.LAYOUT_REF96
    cap = 6 * R * R
    out = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    total = torch.zeros(1, dtype=torch.int64, device="cuda")
    quads = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    depths = torch.empty(cap, dtype=torch.float32, device="cuda")
    valid = torch.zeros(1, dtype=torch.int32, device="cuda")
    sq = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
    draw = torch.zeros(5, dtype=torch.int32, device="cuda")
    lq_dev = torch.empty(cap * 32, dtype=torch.uint8, device="cuda")
    res = torch.zeros(8, dtype=torch.int32, device="cuda")
    lpos = LIGHTS["outside"]
    for w, hgt in ((1920, 1080), (3840, 2160)):
        tg = {t: torch.empty(w * hgt * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda") for t, dt in _abi.GBUFFER_TARGETS}
        g = _abi.m2s_gbuffer(*[tg[t].data_ptr() for t, _ in _abi.GBUFFER_TARGETS])
        img = torch.empty(w * hgt * 4, dtype=torch.uint8, device="cuda")
        p = _abi.make_params(R, layout, 0.65, 0, _abi.FLAG_UNCAPPED)
        pp = _abi.make_prepass_params(V, P, M, (w, hgt), (0.01, 100.0), 0.65 / R, 6, layout)
        sp = _abi.m2s_splat_params(w, hgt, 6)
        shp = _abi.make_shadow_params(M, lpos, (0.01, 100.0), (w, hgt), 0.65 / R, layout, S)

        def frame(light_only=False, mode=6):
            lp = _abi.make_light_params(w, hgt, mode, lpos, (1.0, 1.0, 1.0), 10.0, (0.0, 0.5, 3.2), 100.0, S)
            if not light_only:
                check(L.m2s_convert_enqueue(ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), h))
                check(L.m2s_prepass_enqueue(ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                            depths.data_ptr(), valid.data_ptr(), h))
                check(L.m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(), sq.data_ptr(),
                                               None, draw.data_ptr(), h))
                check(L.m2s_splat_draw_enqueue(ctx.handle, sq.data_ptr(), cap, draw.data_ptr(), C.byref(sp), C.byref(g), 60_000_000,
                                               res.data_ptr(), res[2:].data_ptr(), h))
                check(L.m2s_shadow_map_enqueue(ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(shp), cube.data_ptr(),
                                               lq_dev.data_ptr(), 60_000_000, res[4:].data_ptr(), res[6:].data_ptr(), h))
            check(L.m2s_deferred_light_enqueue(ctx.handle, C.byref(g), cube.data_ptr(), C.byref(lp), img.data_ptr(), h))
        t_frame = median(frame)
        o = res.cpu().numpy()
        assert int(o[6]) == int(total.item()) and int(o[2]) == int(valid.item())
        if w == 1920:
            results["frame"].append({"case": f"R={R} ref96 {w}x{hgt}", "frame_us": t_frame})
            print(f"frame R={R} ref96 {w}x{hgt}: {t_frame:9.1f} us", flush=True)
        for mode in (0, 6):
            t = median(lambda: frame(True, mode))
            nbytes = w * hgt * ((24 if mode == 6 else 4) + 4)
            row = {"case": f"mode {mode} {w}x{hgt}", "light_us": t, "bytes": nbytes, "GBps": nbytes / (t * 1e-6) / 1e9,
                   "frac_of_datasheet": nbytes / (t * 1e-6) / 1e9 / HBM_GBS}
            results["light"].append(row)
            print(f"lighting {row['case']:18s} {t:8.1f} us  {row['GBps']:7.1f} GB/s = {row['frac_of_datasheet']:.2f} of data sheet", flush=True)
        del tg, img
        torch.cuda.empty_cache()
    ds.free()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
