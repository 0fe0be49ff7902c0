"""m2s_convert_host on the bench scene (pinned buffers), a few repetitions; prints the mean time."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from mesh2splat_b200 import _abi, synth
from mesh2splat_b200.api import Context
scene = synth.helmet_standin(2048)
ctx = Context(0)
layout = _abi.LAYOUT_PACKED56
stride = 56
cap = 6 * 512 * 512
ps, keep = bench.pinned_scene(scene, torch)
cs = ps.c_struct()
h = torch.empty(cap * stride, dtype=torch.uint8).pin_memory().numpy()
for _ in range(3):
    ctx.convert_host(ps, 512, layout, flags=_abi.FLAG_UNCAPPED, capacity=cap, out=h, c_scene=cs)
torch.cuda.synchronize()
t0 = time.perf_counter()
n = 10
for _ in range(n):
    rec, _, res = ctx.convert_host(ps, 512, layout, flags=_abi.FLAG_UNCAPPED, capacity=cap, out=h, c_scene=cs)
torch.cuda.synchronize()
print(f"e2e ms {1e3 * (time.perf_counter() - t0) / n:.3f} written {res.written}")
