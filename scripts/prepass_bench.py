"""Device time of the viewer prepass (m2s_prepass_enqueue) on the bench scene's conversion output, both record layouts:
CUDA events on the launching stream, L2 flushed between launches; achieved GB/s = (records read + quads and depths
written) / time against the measured HBM peak."""
import os, sys, json, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mesh2splat_b200 import synth, _abi
from mesh2splat_b200.api import Context
from mesh2splat_b200._lib import lib, check

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden"))
from make_golden_prepass import look_at, perspective, column_major

ctx = Context(0)
scene = synth.helmet_standin(2048)
ds = ctx.upload(scene)
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
peak = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists("MEASURED_PEAKS.json") else 3350.0   # H100 SXM data sheet
V = column_major(look_at(np.array([0.0, 0.5, 3.2]), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
P = column_major(perspective(np.radians(45.0), 16 / 9, 0.01, 100.0))
M = column_major(np.eye(4, dtype=np.float32))
stream = torch.cuda.Stream()
for R in (512, 2048):
    for layout, name in ((_abi.LAYOUT_REF96, "ref96"), (_abi.LAYOUT_PACKED56, "packed56")):
        out = ctx.convert(ds, R, layout, flags=_abi.FLAG_UNCAPPED, capacity=6 * R * R)
        n = out.written
        quads = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
        depths = torch.empty(n, dtype=torch.float32, device="cuda")
        valid = torch.zeros(1, dtype=torch.int32, device="cuda")
        p = _abi.make_prepass_params(V, P, M, (1920, 1080), (0.01, 100.0), 0.65 / R, 0, layout)
        ts = []
        with torch.cuda.stream(stream):
            for i in range(12):
                flush.zero_(); torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                check(lib().m2s_prepass_enqueue(ctx.handle, out.data.data_ptr(), n, None, C.byref(p), quads.data_ptr(), depths.data_ptr(), valid.data_ptr(), stream.cuda_stream))
                b.record(stream); torch.cuda.synchronize()
                ts.append(a.elapsed_time(b))
        m = int(valid.item())
        t = float(np.median(ts[3:])) * 1e-3
        byts = n * _abi.STRIDES[layout] + m * 100
        print(f"prepass R={R:5d} {name:9s} gaussians {n:9d} survivors {m:9d}  {t * 1e6:8.2f} us  {n / t / 1e9:6.2f} Ggaussians/s  {byts / t / 1e9:7.1f} GB/s = {byts / t / 1e9 / peak:.2f} of the measured HBM peak")
        del out
