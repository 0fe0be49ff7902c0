#!/usr/bin/env python3
"""Throughput of the .ply loader (SURVEY 8 f-10) on a seeded standard-format file (62 floats = 248 B per row).

  m2s_ply_read end to end (file -> REF96 records on the device), host clock around the synchronous call, in file GB/s.
    The file was just written, so it is read from the page cache: this is the loader's own speed, not the disk's.
  the decode kernel alone (m2s_ply_decode_enqueue on rows already on the device): CUDA events, median of 20 launches
    after 3 warm-up ones; achieved bytes/s = (rows read + records written) / time, against the H100 SXM data sheet's
    3.35 TB/s
  the H2D bytes of one read (m2s_ply_h2d_bytes)
  baselines: the reference's own parsers::loadPlyFile (oracle/_ref/libm2s_refplyload.so, when built) and a numpy decode
  of the same rows
  the card's name and power limit, read in the same run

    python scripts/ply_load_bench.py [--rows 4000000] [--out DIR]

The file is written under the output directory (default: a new temporary directory) and deleted at the end; one JSON
line goes to stdout and to <out>/ply_load_bench.json."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def card() -> dict:
    import torch
    r = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        r["nvidia_smi"] = q[0] if q else ""
    except (OSError, subprocess.SubprocessError) as e:
        r["nvidia_smi"] = f"unavailable: {e}"
    return r


def numpy_decode(rows: np.ndarray) -> np.ndarray:
    """loadPlyFile's per-vertex formulas, vectorised (standard layout: x y z nx ny nz f_dc 0..2 f_rest 0..44 opacity
    scale 0..2 rot 0..3)."""
    f = rows.view(np.float32).reshape(len(rows), 62)
    g = np.zeros((len(f), 24), np.float32)
    g[:, 0:3] = f[:, 0:3]; g[:, 3] = 1
    g[:, 4:7] = f[:, 6:9] * np.float32(0.28209479177387814) + np.float32(0.5)
    g[:, 7] = 1.0 / (1.0 + np.exp(-f[:, 54]).astype(np.float64))
    g[:, 8:11] = np.exp(f[:, 55:58]); g[:, 11] = 1
    q = f[:, 58:62]
    ln = np.sqrt((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + (q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3]))
    ok = ln > 0
    with np.errstate(divide="ignore", invalid="ignore"):
        g[:, 16:20] = np.where(ok[:, None], q * (np.float32(1) / ln)[:, None], np.array([1, 0, 0, 0], np.float32))
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--out", default=None, help="output directory (default: a new temporary directory)")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from mesh2splat_b200 import api
    from mesh2splat_b200._lib import check, lib
    from oracle import ply_load

    if a.out is None:
        import tempfile
        a.out = tempfile.mkdtemp(prefix="ply_load_bench_")
    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, "bench_standard.ply")
    rng = np.random.default_rng(2026)
    n = a.rows
    g = np.zeros((n, 24), np.float32)
    g[:, 0:3] = rng.standard_normal((n, 3), np.float32); g[:, 3] = 1
    g[:, 4:7] = rng.random((n, 3), np.float32); g[:, 7] = rng.random(n, np.float32) * 0.98 + 0.01
    g[:, 8:11] = rng.random((n, 3), np.float32) * 8 + 0.5
    g[:, 12:15] = rng.standard_normal((n, 3), np.float32)
    g[:, 16:20] = rng.standard_normal((n, 4), np.float32)   # unnormalised, as trained captures store them
    api.ply_write(path, g, 0, 0.65 / 512)
    del g
    info = api.ply_parse_file(path)
    size = os.path.getsize(path)
    res = {"rows": n, "file_bytes": size, "row_stride": info.row_stride, "card": card(), "page_cache": True}
    ctx = api.Context(0)
    out = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
    try:
        # ---- m2s_ply_read end to end ----
        ctx.ply_read(path, out=out)   # warm-up: pinned buffers, device slots, module load
        ts = []
        for _ in range(a.reps):
            h0 = ctx.ply_h2d_bytes()
            t0 = time.perf_counter()
            ctx.ply_read(path, out=out)
            ts.append(time.perf_counter() - t0)
            res["h2d_bytes"] = ctx.ply_h2d_bytes() - h0
        t = float(np.median(ts))
        res["ply_read_s"] = t
        res["ply_read_file_gbs"] = size / t / 1e9
        # ---- the decode kernel alone ----
        with open(path, "rb") as f:
            f.seek(info.body_offset)
            body = np.frombuffer(f.read(n * info.row_stride), np.uint8)
        rows = torch.from_numpy(body.copy()).cuda()
        rec2 = torch.empty_like(out)
        stream = torch.cuda.Stream()
        evs = []
        for i in range(23):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            check(lib().m2s_ply_decode_enqueue(ctx.handle, C.byref(info), rows.data_ptr(), n, rec2.data_ptr(), stream.cuda_stream))
            e1.record(stream)
            evs.append((e0, e1))
        torch.cuda.synchronize()
        kt = float(np.median([e0.elapsed_time(e1) for e0, e1 in evs[3:]])) * 1e-3
        moved = n * info.row_stride + n * 96
        res["decode_kernel_s"] = kt
        res["decode_kernel_bytes_per_s"] = moved / kt
        res["decode_kernel_share_of_hbm_peak"] = moved / kt / HBM_PEAK
        same = torch.equal(out[: n * 96], rec2[: n * 96])
        res["read_equals_decode"] = bool(same)
        # ---- baselines ----
        t0 = time.perf_counter()
        want = numpy_decode(body.reshape(n, info.row_stride))
        res["numpy_decode_s"] = time.perf_counter() - t0
        res["numpy_decode_file_gbs"] = size / res["numpy_decode_s"] / 1e9
        got = out[: n * 96].cpu().numpy().view(np.float32).reshape(n, 24)
        res["numpy_max_abs_diff"] = float(np.nanmax(np.abs(got.astype(np.float64) - want)))
        if ply_load.ref_lib() is not None:
            pbr = C.c_int(0)
            t0 = time.perf_counter()
            r = ply_load.ref_lib().ref_load_ply(path.encode(), None, 0, C.byref(pbr))   # the whole load; nothing copied out
            res["reference_loadPlyFile_s"] = time.perf_counter() - t0
            res["reference_loadPlyFile_file_gbs"] = size / res["reference_loadPlyFile_s"] / 1e9
            res["reference_rows"] = int(r)
        else:
            res["reference_loadPlyFile_s"] = None
    finally:
        os.remove(path)
        ctx.close()
    line = json.dumps(res)
    print(line)
    with open(os.path.join(a.out, "ply_load_bench.json"), "w") as f:
        f.write(line + "\n")
    print(f"m2s_ply_read {res['ply_read_s'] * 1e3:.1f} ms = {res['ply_read_file_gbs']:.2f} GB/s of file; decode kernel "
          f"{kt * 1e6:.0f} us = {moved / kt / 1e12:.2f} TB/s ({moved / kt / HBM_PEAK:.2f} of 3.35 TB/s); numpy "
          f"{res['numpy_decode_s']:.2f} s; reference {res['reference_loadPlyFile_s']}", file=sys.stderr)


if __name__ == "__main__":
    main()
