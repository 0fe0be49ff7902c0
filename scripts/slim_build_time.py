"""Time of the kernel that builds a scene's 64-byte position/uv stream at upload (slim_tris_kernel, m2s_scene.cu), and
the memory it adds.  Uploads the scene several times under torch.profiler and reports the kernel's median duration.
usage: slim_build_time.py [helmet|sphere_1m|sponza] [uploads]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
from mesh2splat_b200 import synth
from mesh2splat_b200.api import Context

which = sys.argv[1] if len(sys.argv) > 1 else "helmet"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 8
scene = {"helmet": lambda: synth.helmet_standin(2048), "sphere_1m": lambda: synth.sphere_1m(2048),
         "sponza": lambda: synth.sponza_standin(1024)}[which]()
ctx = Context(0)
ctx.upload(scene).free()   # module load, pool warm-up
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(n):
        ctx.upload(scene).free()
    torch.cuda.synchronize()
us = [e.device_time for e in prof.events() if "slim_tris_kernel" in e.name]
T = scene.triangle_count
print(f"{which}: {T} triangles; stream {T * 64 / 1e6:.2f} MB (+64 B per triangle, the 144-byte triangles: {T * 144 / 1e6:.2f} MB); "
      f"slim_tris_kernel median {np.median(us):.2f} us over {len(us)} uploads "
      f"({(T * (144 + 64)) / (np.median(us) * 1e-6) / 1e9:.0f} GB/s of {T * 144 / 1e6:.1f} MB read (every 32-byte sector of a triangle "
      f"holds a value it needs) + {T * 64 / 1e6:.1f} MB written)")
ctx.close()
