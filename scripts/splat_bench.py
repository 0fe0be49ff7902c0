#!/usr/bin/env python3
"""Times the viewer's splat draw (row f-6, m2s_splat_draw_enqueue) on the GPU.

Inputs: the bench scene's survivors (helmet stand-in) at R = 512 and R = 2048 in both record layouts, through the camera
of scripts/sort_bench.py, sorted by the depth sort, drawn into all five targets at 1920 x 1080, and R = 512 also at
3840 x 2160.  Reports per case: the draw time (CUDA events, L2 flushed before each run), pairs and fragments per
second, the bytes the draw must move against the H100 SXM data-sheet bandwidth (3350 GB/s, not a measured peak), and
the one-stream convert -> prepass -> sort -> draw frame.  The card's name and power limit are read in the same run.

    python scripts/splat_bench.py [--iters 15] [--out results/splat_bench.json]
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
TARGET_BYTES_PER_PX = 3 * 8 + 2 * 4   # the G-buffer stores: 32 B per pixel
PAIR_BYTES = 4 + 8 + 8 + 8 + 8 + 4 + 96   # emission (key, value), two sort passes (read + write), ranges, quad read per pair


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
    results = {"card": card(), "peak_GBps": HBM_GBS, "peak_source": "H100 SXM data sheet (not measured)", "rows": []}
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

    scene = synth.helmet_standin(2048)
    ds = ctx.upload(scene)
    V = column_major(look_at(np.array([0.0, 0.5, 3.2]), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(45.0), 16 / 9, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    cases = [(512, 1920, 1080), (2048, 1920, 1080), (512, 3840, 2160)]
    for R, w, hgt in cases:
        for layout, lname in ((_abi.LAYOUT_REF96, "ref96"), (_abi.LAYOUT_PACKED56, "packed56")):
            cap = 6 * R * R
            out = torch.empty(cap * _abi.STRIDES[layout], dtype=torch.uint8, device="cuda")
            total = torch.zeros(1, dtype=torch.int64, device="cuda")
            quads = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
            depths = torch.empty(cap, dtype=torch.float32, device="cuda")
            valid = torch.zeros(1, dtype=torch.int32, device="cuda")
            sq = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
            draw = torch.zeros(5, dtype=torch.int32, device="cuda")
            tg = {t: torch.empty(w * hgt * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda")
                  for t, dt in _abi.GBUFFER_TARGETS}
            g = _abi.m2s_gbuffer(*[tg[t].data_ptr() for t, _ in _abi.GBUFFER_TARGETS])
            res = torch.zeros(4, dtype=torch.int32, device="cuda")
            p = _abi.make_params(R, layout, 0.65, 0, _abi.FLAG_UNCAPPED)
            pp = _abi.make_prepass_params(V, P, M, (w, hgt), (0.01, 100.0), 0.65 / R, 0, layout)
            sp = _abi.m2s_splat_params(w, hgt, 0)
            torch.cuda.synchronize()
            # the pair count of this frame, for the budget (a viewer keeps the last frame's count)
            check(L.m2s_convert_enqueue(ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), h))
            check(L.m2s_prepass_enqueue(ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                        depths.data_ptr(), valid.data_ptr(), h))
            check(L.m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(), sq.data_ptr(),
                                           None, draw.data_ptr(), h))
            pairs_t = C.c_uint64(0)
            stream.synchronize()
            n = int(valid.item())
            check(L.m2s_splat_draw(ctx.handle, sq.data_ptr(), n, C.byref(sp), C.byref(g), C.byref(pairs_t)))
            pairs = int(pairs_t.value)
            budget = pairs + pairs // 8 + 1

            def draw_only():
                check(L.m2s_splat_draw_enqueue(ctx.handle, sq.data_ptr(), n, None, C.byref(sp), C.byref(g), budget,
                                               res.data_ptr(), res[2:].data_ptr(), h))

            def frame():
                check(L.m2s_convert_enqueue(ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), h))
                check(L.m2s_prepass_enqueue(ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                            depths.data_ptr(), valid.data_ptr(), h))
                check(L.m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(),
                                               sq.data_ptr(), None, draw.data_ptr(), h))
                check(L.m2s_splat_draw_enqueue(ctx.handle, sq.data_ptr(), cap, draw.data_ptr(), C.byref(sp), C.byref(g), budget,
                                               res.data_ptr(), res[2:].data_ptr(), h))
            t_draw = median(draw_only)
            t_frame = median(frame)
            o = res.cpu().numpy()
            assert int(o[2]) == n and int(o[:2].view(np.uint64)[0]) == pairs
            # the tile pass tests every pixel of a tile against each of its pairs: pairs x 256 pixel-quad coverage tests
            # (the covered fragments are a subset; they are not counted on the device)
            nbytes = w * hgt * TARGET_BYTES_PER_PX + pairs * PAIR_BYTES + n * 96 * 2
            row = {"case": f"R={R} {lname} {w}x{hgt}", "quads": n, "pairs": pairs, "draw_us": t_draw, "frame_us": t_frame,
                   "pairs_per_s": pairs / (t_draw * 1e-6), "pixel_tests_per_s": pairs * 256 / (t_draw * 1e-6),
                   "bytes": nbytes, "GBps": nbytes / (t_draw * 1e-6) / 1e9, "frac_of_datasheet": nbytes / (t_draw * 1e-6) / 1e9 / HBM_GBS}
            results["rows"].append(row)
            print(f"{row['case']:28s} quads {n:9d} pairs {pairs:10d}  draw {t_draw:9.1f} us  {row['pairs_per_s'] / 1e9:6.2f} Gpairs/s "
                  f"{row['pixel_tests_per_s'] / 1e9:7.1f} G pixel-quad tests/s  {row['GBps']:7.1f} GB/s = {row['frac_of_datasheet']:.2f} "
                  f"of data sheet | frame {t_frame:9.1f} us", flush=True)
            del out, quads, depths, sq, tg
            torch.cuda.empty_cache()
    ds.free()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
