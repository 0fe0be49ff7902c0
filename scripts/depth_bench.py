#!/usr/bin/env python3
"""Times the viewer's mesh depth pre-pass and what the prepass's mesh depth test saves downstream (row f-9) on the GPU.

Inputs: the bench scene (helmet stand-in, 70 074 triangles, one opaque primitive) converted at R = 512 and R = 2048
(REF96), drawn at 1920 x 1080 and 3840 x 2160 with the chain test's camera outside the model and a camera inside it.
Per case:
  - the depth pass (m2s_mesh_depth_enqueue) as a whole (CUDA events, L2 flushed before each run, median) and split by
    torch.profiler (in a pass of its own) into set-up (count + scan), binning (emit + pair sort + ranges) and the tile
    kernel; triangles, pairs, and the bytes it must move by the count below;
  - the frame convert -> [mesh depth] -> prepass -> sort -> draw -> shadow (S = 1024) -> light with the test off and on,
    alternated in one run: survivors, the splat draw's pairs, and the median time of each stage and of the frame, from
    events recorded between the stages on one stream.
Bytes of the depth pass (a lower bound from shapes): every triangle's three positions read twice (count, emit: 2 x 48 B),
each pair's key and value written once (8 B) and read by the tile kernel (4 B), and the map written once (4 B per texel).
The card's name and power limit are read in the same run.

    python scripts/depth_bench.py [--iters 15] [--out results/depth_bench.json]
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

S = 1024
CAMS = {"outside": ((0.0, 0.5, 3.2), (0.0, 0.0, 0.0)), "inside": ((0.05, 0.02, -0.03), (1.0, 0.3, 0.2))}
STAGES = ["convert", "mesh_depth", "prepass", "sort", "draw", "shadow", "light"]


def depth_bytes(ntri: int, pairs: int, w: int, h: int) -> int:
    return 2 * 48 * ntri + 12 * pairs + 4 * w * h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    ctx = Context(0)
    L = lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    hs = stream.cuda_stream
    results = {"card": card(), "depth": [], "frame": []}
    print(f"# {results['card']}")

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
        return float(np.median([timed(fn) for _ in range(args.iters + 3)][3:]))

    def split(fn):
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                with torch.cuda.stream(stream):
                    fn()
            torch.cuda.synchronize()
        g = {"setup": 0.0, "binning": 0.0, "tile": 0.0}
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
            if "DepthBins" in e.key and ("bin_count" in e.key or "bin_scan" in e.key):
                g["setup"] += t
            elif ("DepthBins" in e.key and ("bin_emit" in e.key or "bin_ranges" in e.key)) or "sort_" in e.key:
                g["binning"] += t
            elif "depth_tile" in e.key:
                g["tile"] += t
        return {k: v / args.iters for k, v in g.items()}

    scene = synth.helmet_standin(2048)
    ds = ctx.upload(scene)
    ntri = scene.triangle_count
    M = column_major(np.eye(4, dtype=np.float32))
    layout = _abi.LAYOUT_REF96
    res = torch.zeros(16, dtype=torch.int32, device="cuda")
    cube = torch.empty(6 * S * S, dtype=torch.float32, device="cuda")
    for R in (512, 2048):
        cap = 6 * R * R
        out = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
        total = torch.zeros(1, dtype=torch.int64, device="cuda")
        quads = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
        depths = torch.empty(cap, dtype=torch.float32, device="cuda")
        valid = torch.zeros(1, dtype=torch.int32, device="cuda")
        sq = torch.empty(cap * 96, dtype=torch.uint8, device="cuda")
        draw = torch.zeros(5, dtype=torch.int32, device="cuda")
        lq = torch.empty(cap * 32, dtype=torch.uint8, device="cuda")
        for w, h in ((1920, 1080), (3840, 2160)):
            dmap = torch.empty(w * h, dtype=torch.float32, device="cuda")
            tg = {t: torch.empty(w * h * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda") for t, dt in _abi.GBUFFER_TARGETS}
            g = _abi.m2s_gbuffer(*[tg[t].data_ptr() for t, _ in _abi.GBUFFER_TARGETS])
            img = torch.empty(w * h * 4, dtype=torch.uint8, device="cuda")
            for cname, (eye, tgt) in CAMS.items():
                V = column_major(look_at(np.array(eye), np.array(tgt), np.array([0.0, 1.0, 0.0])).astype(np.float32))
                P = column_major(perspective(np.radians(45.0), w / h, 0.01, 100.0))
                dp = _abi.make_mesh_depth_params(V, P, M, w, h)
                pairs_t = C.c_uint64(0)
                check(L.m2s_mesh_depth(ctx.handle, ds.handle, C.byref(dp), dmap.data_ptr(), C.byref(pairs_t)))
                pairs = int(pairs_t.value)
                budget = pairs + pairs // 8 + 1

                def depth_pass():
                    check(L.m2s_mesh_depth_enqueue(ctx.handle, ds.handle, C.byref(dp), dmap.data_ptr(), budget, res[8:].data_ptr(),
                                                   res[10:].data_ptr(), hs))
                t = median(depth_pass)
                sp_ = split(depth_pass)
                o = res.cpu().numpy()
                assert int(o[10]) == ntri and int(o[8:10].view(np.uint64)[0]) == pairs
                nb = depth_bytes(ntri, pairs, w, h)
                row = {"case": f"R={R} {w}x{h} {cname}", "triangles": ntri, "pairs": pairs, "depth_us": t, "split_us": sp_,
                       "bytes": nb, "GBps": nb / (t * 1e-6) / 1e9}
                results["depth"].append(row)
                print(f"depth {row['case']:28s} tris {ntri} pairs {pairs:9d}  {t:8.1f} us (setup {sp_['setup']:7.1f}, binning "
                      f"{sp_['binning']:7.1f}, tile {sp_['tile']:7.1f})  {row['GBps']:6.1f} GB/s of the shape count", flush=True)

                p = _abi.make_params(R, layout, 0.65, 0, _abi.FLAG_UNCAPPED)
                pp = _abi.make_prepass_params(V, P, M, (w, h), (0.01, 100.0), 0.65 / R, 6, layout)
                spp = _abi.m2s_splat_params(w, h, 6)
                shp = _abi.make_shadow_params(M, (1.5, 2.0, 2.5), (0.01, 100.0), (w, h), 0.65 / R, layout, S)
                lp = _abi.make_light_params(w, h, 6, (1.5, 2.0, 2.5), (1.0, 1.0, 1.0), 10.0, eye, 100.0, S)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(STAGES) + 1)]

                def frame(test_on):
                    ev[0].record(stream)
                    check(L.m2s_convert_enqueue(ctx.handle, ds.handle, C.byref(p), out.data_ptr(), cap, None, total.data_ptr(), hs))
                    ev[1].record(stream)
                    if test_on:
                        check(L.m2s_mesh_depth_enqueue(ctx.handle, ds.handle, C.byref(dp), dmap.data_ptr(), budget, None, None, hs))
                    ev[2].record(stream)
                    if test_on:
                        check(L.m2s_prepass_mesh_depth_enqueue(ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp),
                                                               dmap.data_ptr(), w, h, quads.data_ptr(), depths.data_ptr(), valid.data_ptr(), hs))
                    else:
                        check(L.m2s_prepass_enqueue(ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(pp), quads.data_ptr(),
                                                    depths.data_ptr(), valid.data_ptr(), hs))
                    ev[3].record(stream)
                    check(L.m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), cap, valid.data_ptr(), sq.data_ptr(),
                                                   None, draw.data_ptr(), hs))
                    ev[4].record(stream)
                    check(L.m2s_splat_draw_enqueue(ctx.handle, sq.data_ptr(), cap, draw.data_ptr(), C.byref(spp), C.byref(g), 400_000_000,
                                                   res.data_ptr(), res[2:].data_ptr(), hs))
                    ev[5].record(stream)
                    check(L.m2s_shadow_map_enqueue(ctx.handle, out.data_ptr(), cap, total.data_ptr(), C.byref(shp), cube.data_ptr(),
                                                   lq.data_ptr(), 400_000_000, res[4:].data_ptr(), res[6:].data_ptr(), hs))
                    ev[6].record(stream)
                    check(L.m2s_deferred_light_enqueue(ctx.handle, C.byref(g), cube.data_ptr(), C.byref(lp), img.data_ptr(), hs))
                    ev[7].record(stream)

                samples = {False: [], True: []}
                counts = {}
                for it in range(2 * (args.iters + 3)):   # off, on, off, on, ...: both see the same host and device state
                    on = bool(it % 2)
                    flush.zero_()
                    torch.cuda.synchronize()
                    with torch.cuda.stream(stream):
                        frame(on)
                    torch.cuda.synchronize()
                    if it >= 6:
                        seg = [ev[k].elapsed_time(ev[k + 1]) * 1e3 for k in range(len(STAGES))]
                        samples[on].append(seg + [ev[0].elapsed_time(ev[-1]) * 1e3])
                    o = res.cpu().numpy()
                    counts[on] = {"gaussians": int(total.item()), "survivors": int(valid.item()), "draw_pairs": int(o[:2].view(np.uint64)[0]),
                                  "drawn": int(o[2])}
                    assert counts[on]["drawn"] == counts[on]["survivors"], "the draw budget holds every pair"
                for on in (False, True):
                    med = np.median(np.array(samples[on]), axis=0)
                    row = {"case": f"R={R} {w}x{h} {cname}", "test": "on" if on else "off", **counts[on],
                           **{f"{s}_us": float(med[k]) for k, s in enumerate(STAGES)}, "frame_us": float(med[-1])}
                    results["frame"].append(row)
                    print(f"frame {row['case']:28s} test {row['test']:3s} survivors {row['survivors']:9d} draw pairs {row['draw_pairs']:10d} | "
                          f"depth {row['mesh_depth_us']:7.1f} prepass {row['prepass_us']:7.1f} sort {row['sort_us']:7.1f} draw "
                          f"{row['draw_us']:8.1f} | frame {row['frame_us']:8.1f} us", flush=True)
            del tg, img, dmap
            torch.cuda.empty_cache()
        del out, quads, sq, lq
        torch.cuda.empty_cache()
    ds.free()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
