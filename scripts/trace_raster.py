"""Per-phase account of the raster kernel's warps (needs a -DM2S_TRACE build selected with M2S_LIB).

Every raster warp sums the SM cycles (clock64) it spends in each phase over ALL its units; the kernel also records each
warp's cycles and globaltimer nanoseconds from entry to exit, which give the SM clock the cycles convert at.
usage: trace_raster.py [packed56|ref96] [density] [helmet|dh|quad]"""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mesh2splat_b200 import synth, _abi, _lib
from mesh2splat_b200.api import Context
layout = {"ref96": 0, "packed56": 1}[sys.argv[1] if len(sys.argv) > 1 else "packed56"]
R = int(sys.argv[2]) if len(sys.argv) > 2 else 512
which = sys.argv[3] if len(sys.argv) > 3 else "helmet"
ctx = Context(0)
scene = {"helmet": lambda: synth.helmet_standin(2048), "quad": synth.unit_quad, "dh": lambda: synth.damaged_helmet_standin(2048)}[which]()
ds = ctx.upload(scene)
nw = torch.cuda.get_device_properties(0).multi_processor_count * 16
tr = torch.zeros(nw * 16, dtype=torch.int64, device="cuda")
_lib.lib().m2s_debug_set_trace(C.c_void_p(tr.data_ptr()))
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
out = None
for i in range(5):
    flush.zero_(); tr.zero_(); torch.cuda.synchronize()   # cold L2, as in bench.py
    out = ctx.convert(ds, R, layout, flags=_abi.FLAG_UNCAPPED, capacity=6 * R * R, out=out.data if out else None)
t = tr.cpu().numpy().reshape(nw, 16).astype(np.float64)
_lib.lib().m2s_debug_set_trace(None)
# slots: enum TraceSlot in m2s_raster.cu
PHASES = ["triangle-load wait", "set-up", "walk + scan", "larger tris + flush", "reservation wait", "listing",
          "direct shading", "unit end (stores)", "tail (help, last CTA)"]
UNITS, DUNITS, GROUPS, CYC, NS, ENTRY = 9, 10, 11, 12, 13, 14
live = t[:, CYC] > 0
t = t[live]
mhz = t[:, CYC].sum() / t[:, NS].sum() * 1e3
print(f"{which} R={R} layout={layout}: device_ms={out.device_ms:.4f} total={out.total} warps={len(t)} SM clock {mhz:.0f} MHz (clock64 / globaltimer)")
print(f"units/warp p50 {np.median(t[:, UNITS]):.0f} max {t[:, UNITS].max():.0f}; direct units/warp p50 {np.median(t[:, DUNITS]):.0f}; "
      f"32-fragment groups/warp p50 {np.median(t[:, GROUPS]):.1f} max {t[:, GROUPS].max():.0f} total {t[:, GROUPS].sum():.0f}")
us = lambda c: c / mhz
print(f"{'phase (per-warp sum)':24s} {'p50 us':>8s} {'p90 us':>8s} {'mean us':>8s}")
for k, n in enumerate(PHASES + ["entry (tables)"]):
    v = us(t[:, ENTRY if n == "entry (tables)" else k])
    print(f"{n:24s} {np.median(v):8.2f} {np.percentile(v, 90):8.2f} {v.mean():8.2f}")
v = us(t[:, CYC])
print(f"{'warp entry -> exit':24s} {np.median(v):8.2f} {np.percentile(v, 90):8.2f} {v.mean():8.2f}")
g = t[:, GROUPS] > 0
if g.any():
    pg = us(t[g, 6]) / t[g, GROUPS]
    print(f"direct shading per 32-fragment group: p50 {np.median(pg):.3f} us  p90 {np.percentile(pg, 90):.3f} us")
