#!/usr/bin/env python3
"""Cost of a loaded .ply's view-dependent colour (beyond the reference) on a seeded degree-3 standard file (62 floats =
248 B per row, 45 of them SH rest coefficients).

  m2s_ply_read against m2s_ply_read_sh end to end (file -> REF96 records, and the SH buffer), host clock around the
    synchronous call, median of --reps; the file was just written, so it is read from the page cache
  the decode kernel alone, without and with the SH buffer (m2s_ply_decode_enqueue / m2s_ply_decode_sh_enqueue on rows
    already on the device): CUDA events, median of 20 launches after 3 warm-up ones
  m2s_prepass against m2s_prepass_sh (degree 3, render mode 0) with the camera outside the capture (every gaussian in
    view) and inside it (the ones in front of the camera): CUDA events, median of 20 after 3 warm-up ones; the SH
    variant's added time per surviving gaussian
  achieved bytes/s = the bytes each call must move / time, against the H100 SXM data sheet's 3.35 TB/s: decode = rows
    read + records (+ SH blocks) written; prepass = records read + 100 B (quad + depth) per survivor (+ its 192-byte SH
    block)
  the card's name and power limit, read in the same run

    python scripts/sh_bench.py [--rows 4000000] [--out DIR]

The file is written under the output directory (default: a new temporary directory) and deleted at the end; one JSON
line goes to stdout and to <out>/sh_bench.json."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

from ply_load_bench import HBM_PEAK, card  # noqa: E402

SH_BLOCK = 48 * 4   # bytes of one degree-3 SH block


def timed(stream, fn, launches=23, warm=3) -> float:
    """Median seconds of fn() over launches - warm launches on `stream`, CUDA events."""
    import torch
    evs = []
    for _ in range(launches):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        fn()
        e1.record(stream)
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return float(np.median([e0.elapsed_time(e1) for e0, e1 in evs[warm:]])) * 1e-3


def write_file(path: str, n: int) -> None:
    """A standard-layout file (x y z nx ny nz f_dc_0..2 f_rest_0..44 opacity scale_0..2 rot_0..3) of n seeded rows, written
    in pieces so that the host holds one piece at a time."""
    from mesh2splat_b200 import api
    rng = np.random.default_rng(2026)
    with open(path, "wb") as f:
        f.write(api.ply_header(0, n))
        for a in range(0, n, 1 << 20):
            m = min(n - a, 1 << 20)
            r = np.zeros((m, 62), np.float32)
            r[:, 0:3] = rng.standard_normal((m, 3), np.float32)
            r[:, 3:6] = rng.standard_normal((m, 3), np.float32)
            r[:, 6:9] = rng.standard_normal((m, 3), np.float32)
            r[:, 9:54] = rng.standard_normal((m, 45), np.float32) * 0.2
            r[:, 54] = rng.standard_normal(m, np.float32) * 2
            r[:, 55:58] = rng.standard_normal((m, 3), np.float32) - 4
            r[:, 58:62] = rng.standard_normal((m, 4), np.float32)
            f.write(r.tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--out", default=None, help="output directory (default: a new temporary directory)")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from mesh2splat_b200 import _abi, api
    from mesh2splat_b200._lib import check, lib
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden_prepass import column_major, look_at, perspective

    if a.out is None:
        import tempfile
        a.out = tempfile.mkdtemp(prefix="sh_bench_")
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, "bench_sh3.ply")
    n = a.rows
    write_file(path, n)
    info = api.ply_parse_file(path)
    assert info.sh_degree == 3 and info.row_stride == 248
    size = os.path.getsize(path)
    res = {"rows": n, "file_bytes": size, "row_stride": info.row_stride, "sh_degree": 3, "card": card(), "page_cache": True}
    ctx = api.Context(0)
    L = lib()
    out = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
    sh = torch.empty(n * 48, dtype=torch.float32, device="cuda")
    try:
        # ---- m2s_ply_read against m2s_ply_read_sh, end to end ----
        ctx.ply_read(path, out=out)
        ctx.ply_read_sh(path, out=out, sh=sh)   # warm-up: pinned buffers, device slots, module load
        for key, call in (("ply_read_s", lambda: ctx.ply_read(path, out=out)), ("ply_read_sh_s", lambda: ctx.ply_read_sh(path, out=out, sh=sh))):
            ts = []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                call()
                ts.append(time.perf_counter() - t0)
            res[key] = float(np.median(ts))
            res[key[:-2] + "_file_gbs"] = size / res[key] / 1e9
        # ---- the decode kernel alone ----
        with open(path, "rb") as f:
            f.seek(info.body_offset)
            rows = torch.from_numpy(np.frombuffer(f.read(n * info.row_stride), np.uint8).copy()).cuda()
        rec2, sh2 = torch.empty_like(out), torch.empty_like(sh)
        stream = torch.cuda.Stream()
        hs = stream.cuda_stream
        for key, d_sh, extra in (("decode", None, 0), ("decode_sh", sh2.data_ptr(), n * SH_BLOCK)):
            t = timed(stream, lambda: check(L.m2s_ply_decode_sh_enqueue(ctx.handle, C.byref(info), rows.data_ptr(), n, rec2.data_ptr(), d_sh, hs)))
            moved = n * info.row_stride + n * 96 + extra
            res[f"{key}_kernel_s"] = t
            res[f"{key}_kernel_bytes_per_s"] = moved / t
            res[f"{key}_kernel_share_of_hbm_peak"] = moved / t / HBM_PEAK
        torch.cuda.synchronize()
        res["read_equals_decode"] = bool(torch.equal(out, rec2)) and bool(torch.equal(sh, sh2))
        del rows
        # ---- m2s_prepass against m2s_prepass_sh ----
        quads = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
        depths = torch.empty(n, dtype=torch.float32, device="cuda")
        valid = torch.zeros(1, dtype=torch.int32, device="cuda")
        w, h = 1920, 1080
        Pm = column_major(perspective(np.radians(60.0), w / h, 0.01, 100.0))
        M = column_major(np.eye(4, dtype=np.float32))
        for where, eye in (("outside", (0.0, 0.0, 12.0)), ("inside", (0.0, 0.0, 0.5))):
            V = column_major(look_at(np.array(eye), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
            p = _abi.make_prepass_params(V, Pm, M, (w, h), (0.01, 100.0), 1.0, 0, _abi.VIEW_PLY)
            plain = timed(stream, lambda: check(L.m2s_prepass_enqueue(ctx.handle, out.data_ptr(), n, None, C.byref(p), quads.data_ptr(),
                                                                      depths.data_ptr(), valid.data_ptr(), hs)))
            m = int(valid.item())
            with_sh = timed(stream, lambda: check(L.m2s_prepass_sh_enqueue(ctx.handle, out.data_ptr(), n, None, C.byref(p), sh.data_ptr(), 3, 3,
                                                                           quads.data_ptr(), depths.data_ptr(), valid.data_ptr(), hs)))
            assert int(valid.item()) == m
            moved = n * 96 + m * 100
            res[f"prepass_{where}"] = {"survivors": m, "prepass_s": plain, "prepass_sh_s": with_sh,
                                       "prepass_share_of_hbm_peak": moved / plain / HBM_PEAK,
                                       "prepass_sh_share_of_hbm_peak": (moved + m * SH_BLOCK) / with_sh / HBM_PEAK,
                                       "added_ns_per_survivor": (with_sh - plain) / max(m, 1) * 1e9}
    finally:
        os.remove(path)
        ctx.close()
    line = json.dumps(res)
    print(line)
    with open(os.path.join(a.out, "sh_bench.json"), "w") as f:
        f.write(line + "\n")
    print(f"ply_read {res['ply_read_s'] * 1e3:.1f} ms, ply_read_sh {res['ply_read_sh_s'] * 1e3:.1f} ms; decode {res['decode_kernel_s'] * 1e6:.0f} us "
          f"({res['decode_kernel_share_of_hbm_peak']:.2f} of 3.35 TB/s), with SH {res['decode_sh_kernel_s'] * 1e6:.0f} us "
          f"({res['decode_sh_kernel_share_of_hbm_peak']:.2f}); prepass outside {res['prepass_outside']['prepass_s'] * 1e6:.0f} -> "
          f"{res['prepass_outside']['prepass_sh_s'] * 1e6:.0f} us, inside {res['prepass_inside']['prepass_s'] * 1e6:.0f} -> "
          f"{res['prepass_inside']['prepass_sh_s'] * 1e6:.0f} us", file=sys.stderr)


if __name__ == "__main__":
    main()
