"""Per-phase account of the raster kernel's warps (needs a -DM2S_TRACE build selected with M2S_LIB).

Every raster warp sums the SM cycles (clock64) it spends in each phase over ALL its units; the kernel also records each
warp's cycles and globaltimer nanoseconds from entry to exit, which give the SM clock the cycles convert at.  Globaltimer
stamps at each warp's entry, unit-loop exit and exit, and the fragment kernel's (its first CTA's start and release from
griddepcontrol.wait, its last CTA's end; on a single launch the raster kernel's last CTA stamps the end), place the raster
warps' work inside the step, whose length comes from the events
of the same call.  The trace build shows shape, not timing: its
atomics and stamps lengthen the step.
usage: trace_raster.py [packed56|ref96] [density] [helmet|dh|quad] [single|two]   (two: the fragment kernel is launched
even where the conversion could end in the raster kernel)"""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from mesh2splat_b200 import synth, _abi, _lib
from mesh2splat_b200.api import Context
layout = {"ref96": 0, "packed56": 1}[sys.argv[1] if len(sys.argv) > 1 else "packed56"]
R = int(sys.argv[2]) if len(sys.argv) > 2 else 512
which = sys.argv[3] if len(sys.argv) > 3 else "helmet"
_lib.lib().m2s_debug_set_single_off(int(len(sys.argv) > 4 and sys.argv[4] == "two"))
ctx = Context(0)
scene = {"helmet": lambda: synth.helmet_standin(2048), "quad": synth.unit_quad, "dh": lambda: synth.damaged_helmet_standin(2048)}[which]()
ds = ctx.upload(scene)
nw = torch.cuda.get_device_properties(0).multi_processor_count * 16
HEADER, SLOTS = 32, 32   # kTraceHeader, kTraceWarpSlots (m2s_device.cuh)
tr = torch.zeros(HEADER + nw * SLOTS, dtype=torch.int64, device="cuda")
_lib.lib().m2s_debug_set_trace(C.c_void_p(tr.data_ptr()))
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
out = None
for i in range(5):
    flush.zero_(); tr.zero_(); tr[1:3] = -1; torch.cuda.synchronize()   # cold L2, as in bench.py; ~0 under the atomicMin stamps
    out = ctx.convert(ds, R, layout, flags=_abi.FLAG_UNCAPPED, capacity=6 * R * R, out=out.data if out else None)
trn = tr.cpu().numpy()
frag_end, frag_start, frag_wait = (int(v) for v in trn[:3])   # kTrFragEndNs, kTrFragStartNs, kTrFragWaitNs
ts = trn[HEADER:].reshape(nw, SLOTS)   # the globaltimer stamps, exact in int64
t = ts.astype(np.float64)
_lib.lib().m2s_debug_set_trace(None)
# slots: enum TraceSlot in m2s_raster.cu
PHASES = ["triangle-load wait", "set-up", "walk + scan", "larger tris + flush", "reservation wait", "listing",
          "direct shading", "unit end (stores)", "tail (help, exit)"]
UNITS, DUNITS, GROUPS, CYC, NS, ENTRY, ENTRY_NS, LOOP_NS, EXIT_NS = 9, 10, 11, 12, 13, 14, 15, 16, 17
live = t[:, CYC] > 0
t = t[live]
ts = ts[live]
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

# where the raster warps' work sits in the step: the step starts its event time before the fragment kernel's end
plan = ctx.convert_plan(ds, R, layout, capacity=6 * R * R)
cta = np.arange(nw)[live] // (plan.raster_warps // plan.grid)   # raster warp -> CTA (slots are laid out CTA by CTA)
step_ns = out.device_ms * 1e6
start = frag_end - step_ns
first_entry = np.array([ts[cta == c, ENTRY_NS].min() for c in np.unique(cta)])
cta_exit = np.array([ts[cta == c, EXIT_NS].max() for c in np.unique(cta)])
print(f"spans of the step (globaltimer, us): CTAs {len(cta_exit)}, first entries spread {(first_entry.max() - first_entry.min()) / 1e3:.2f}, "
      f"exits spread {(cta_exit.max() - cta_exit.min()) / 1e3:.2f}")
print(f"  launch -> first warp entry            {(first_entry.min() - start) / 1e3:8.2f}")
print(f"  last unit-loop exit -> last CTA exit  {(cta_exit.max() - ts[:, LOOP_NS].max()) / 1e3:8.2f}")
last = cta_exit.max()   # the last raster CTA's exit; < 0 below: before it
if plan.single_launch:   # no fragment grid: the step ends when the raster kernel's last CTA has published the count
    print(f"  single launch (no fragment kernel)")
else:
    print(f"  last raster CTA exit -> first fragment CTA resident  {(frag_start - last) / 1e3:8.2f}")
    print(f"  last raster CTA exit -> first fragment wait released {(frag_wait - last) / 1e3:8.2f}")
print(f"  last raster CTA exit -> step end                     {(frag_end - last) / 1e3:8.2f}")
print(f"  step (events)                         {step_ns / 1e3:8.2f}")
