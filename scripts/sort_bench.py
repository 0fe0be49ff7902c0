"""Device time of the viewer's depth sort (m2s_depth_sort_enqueue) alone and chained behind the prepass on one stream
(the sort's count read from the prepass's valid counter), beside the obvious alternative in the same run: torch.sort
(stable) of the depth keys XOR 0x80000000 viewed as int32 (the uint32 order without a 64-bit sort), then index_select of
the quads.  Ours and torch's alternate launch by launch; every result is compared bit for bit between the two.

Inputs: the survivors of the bench scene (helmet stand-in) at R = 512 and 2048, both record layouts, and 7 000 000
synthetic quads whose depths are those of points uniform in the volume of a view frustum (near 0.5, far 50).
Reported: median device time over CUDA events (L2 flushed between launches), Gquads/s, and the bytes the sort moves
(256 per quad: keys and values through four passes, the order, two 96-byte quads; see DESIGN §4) over time against HBM
bandwidth.  `python scripts/sort_bench.py [--iters N] [--out results.json]`"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from make_golden_prepass import column_major, look_at, perspective  # noqa: E402
from mesh2splat_b200 import _abi, synth  # noqa: E402
from mesh2splat_b200._lib import check, lib  # noqa: E402
from mesh2splat_b200.api import Context  # noqa: E402

SORT_BYTES_PER_QUAD = 4 + (4 + 8) + 2 * (8 + 8) + (8 + 4) + (4 + 96 + 96)   # histogram, passes 0..3, gather = 256
FALLBACK_HBM_GBS = 3350.0   # H100 SXM data sheet


def peak():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    except Exception:  # noqa: BLE001
        return FALLBACK_HBM_GBS, "H100 SXM data sheet (not measured)"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return out or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--out", default="")
    ap.add_argument("--profile", action="store_true", help="per-kernel device times of the sort at 7 M (torch.profiler), in a run of their own")
    args = ap.parse_args()
    ctx = Context(0)
    L = lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    hbm, hbm_src = peak()
    results = {"card": card(), "peak_GBps": hbm, "peak_source": hbm_src, "bytes_per_quad": SORT_BYTES_PER_QUAD, "rows": []}
    print(f"# {results['card']}  (HBM {hbm:.0f} GB/s, {hbm_src})")

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

    def run_case(name, quads, depths, n, prepass=None):
        """quads: uint8 device tensor (>= n * 96 B), depths: n float32; prepass: (records, count, params) for the chain."""
        sorted_q = torch.empty(max(1, n) * 96, dtype=torch.uint8, device="cuda")
        order = torch.empty(max(1, n), dtype=torch.int32, device="cuda")
        draw = torch.empty(5, dtype=torch.int32, device="cuda")
        h = stream.cuda_stream

        def ours():
            check(L.m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), n, None, sorted_q.data_ptr(),
                                           order.data_ptr(), draw.data_ptr(), h))
        q24 = quads[: n * 96].view(torch.float32).view(n, 24)
        res = {}

        def baseline():
            keys = depths[:n].view(torch.int32) ^ torch.tensor(-0x80000000, dtype=torch.int32, device="cuda")
            _, idx = torch.sort(keys, stable=True)
            res["q"] = torch.index_select(q24, 0, idx)
            res["o"] = idx
        t_ours, t_torch = [], []
        for i in range(args.iters + 3):
            a = timed(ours)
            b = timed(baseline)
            if i >= 3:
                t_ours.append(a); t_torch.append(b)
        same = bool(torch.equal(res["o"].to(torch.int32), order[:n])) and bool(torch.equal(res["q"].view(torch.int32).reshape(-1),
                                                                                           sorted_q[: n * 96].view(torch.int32)))
        row = {"case": name, "n": n, "sort_us": float(np.median(t_ours)), "torch_us": float(np.median(t_torch)),
               "sort_us_min": float(np.min(t_ours)), "torch_us_min": float(np.min(t_torch)), "identical_to_torch": same}
        if prepass is not None:   # prepass + sort on one stream, the sort's n from the prepass's valid counter
            rec, count, p = prepass
            cq = torch.empty(max(1, count) * 96, dtype=torch.uint8, device="cuda")
            cd = torch.empty(max(1, count), dtype=torch.float32, device="cuda")
            valid = torch.zeros(1, dtype=torch.int32, device="cuda")
            cs = torch.empty(max(1, count) * 96, dtype=torch.uint8, device="cuda")

            def chain():
                check(L.m2s_prepass_enqueue(ctx.handle, rec.data_ptr(), count, None, C.byref(p), cq.data_ptr(), cd.data_ptr(),
                                            valid.data_ptr(), h))
                check(L.m2s_depth_sort_enqueue(ctx.handle, cq.data_ptr(), cd.data_ptr(), count, valid.data_ptr(), cs.data_ptr(),
                                               None, draw.data_ptr(), h))

            def prepass_only():
                check(L.m2s_prepass_enqueue(ctx.handle, rec.data_ptr(), count, None, C.byref(p), cq.data_ptr(), cd.data_ptr(),
                                            valid.data_ptr(), h))
            tc, tp = [], []
            for i in range(args.iters + 3):
                a = timed(chain)
                b = timed(prepass_only)
                if i >= 3:
                    tc.append(a); tp.append(b)
            assert int(draw[1].item()) == int(valid.item()) == n
            row.update(chain_us=float(np.median(tc)), prepass_us=float(np.median(tp)), gaussians=count)
        t = row["sort_us"] * 1e-6
        row["sort_Gquads_s"] = n / t / 1e9
        row["sort_GBps"] = n * SORT_BYTES_PER_QUAD / t / 1e9
        row["sort_frac_of_peak"] = row["sort_GBps"] / hbm
        row["torch_Gquads_s"] = n / (row["torch_us"] * 1e-6) / 1e9
        results["rows"].append(row)
        line = (f"{name:24s} n {n:9d}  sort {row['sort_us']:9.1f} us {row['sort_Gquads_s']:6.2f} Gquads/s "
                f"{row['sort_GBps']:7.1f} GB/s = {row['sort_frac_of_peak']:.2f} of peak | torch {row['torch_us']:9.1f} us "
                f"({row['torch_us'] / row['sort_us']:.2f}x)  identical {same}")
        if prepass is not None:
            line += f" | prepass {row['prepass_us']:8.1f} us, prepass+sort {row['chain_us']:8.1f} us"
        print(line, flush=True)

    # ---- the bench scene's survivors ----
    scene = synth.helmet_standin(2048)
    ds = ctx.upload(scene)
    V = column_major(look_at(np.array([0.0, 0.5, 3.2]), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(45.0), 16 / 9, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    for R in (() if args.profile else (512, 2048)):
        for layout, lname in ((_abi.LAYOUT_REF96, "ref96"), (_abi.LAYOUT_PACKED56, "packed56")):
            out = ctx.convert(ds, R, layout, flags=_abi.FLAG_UNCAPPED, capacity=6 * R * R)
            count = out.written
            p = _abi.make_prepass_params(V, P, M, (1920, 1080), (0.01, 100.0), 0.65 / R, 0, layout)
            quads = torch.empty(count * 96, dtype=torch.uint8, device="cuda")
            depths = torch.empty(count, dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            v = C.c_uint32(0)
            check(L.m2s_prepass(ctx.handle, out.data.data_ptr(), count, C.byref(p), quads.data_ptr(), depths.data_ptr(), C.byref(v)))
            n = int(v.value)
            run_case(f"R={R} {lname} survivors", quads, depths[:n].clone(), n, prepass=(out.data, count, p))
            del out
    ds.free()

    # ---- 7 000 000 synthetic quads, depths of points uniform in a frustum's volume ----
    n = 7_000_000
    g = torch.Generator(device="cuda").manual_seed(1)
    u = torch.rand(n, device="cuda", generator=g, dtype=torch.float64)
    z0, z1 = 0.5, 50.0
    depths = (-(z0 ** 3 + u * (z1 ** 3 - z0 ** 3)) ** (1.0 / 3.0)).to(torch.float32)
    quads = torch.randn(n * 24, device="cuda", generator=g).view(torch.uint8)
    if args.profile:   # per-kernel device times; no other timing in this run
        sorted_q = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
        order = torch.empty(n, dtype=torch.int32, device="cuda")
        for _ in range(3):
            check(L.m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), n, None, sorted_q.data_ptr(),
                                           order.data_ptr(), None, None))
        torch.cuda.synchronize()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                flush.zero_()
                check(L.m2s_depth_sort_enqueue(ctx.handle, quads.data_ptr(), depths.data_ptr(), n, None, sorted_q.data_ptr(),
                                               order.data_ptr(), None, None))
                torch.cuda.synchronize()
        print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=12, max_name_column_width=70))
        return
    run_case("synthetic 7M frustum", quads, depths, n)

    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
