"""PCIe probe: H2D and D2H alone and concurrently (pinned memory, two streams), and with the argument `host` the
per-call times of m2s_convert_host.  Explains the e2e number of bench.py."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

dev = torch.device("cuda", 0)
up_mb, down_mb = 27, 36
h_up = torch.empty(up_mb << 20, dtype=torch.uint8).pin_memory()
h_dn = torch.empty(down_mb << 20, dtype=torch.uint8).pin_memory()
d_up = torch.empty(up_mb << 20, dtype=torch.uint8, device=dev)
d_dn = torch.empty(down_mb << 20, dtype=torch.uint8, device=dev)
s1, s2 = torch.cuda.Stream(dev), torch.cuda.Stream(dev)


def timed(fn, reps=10):
    fn(); torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
        torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def up():
    with torch.cuda.stream(s1):
        d_up.copy_(h_up, non_blocking=True)


def down():
    with torch.cuda.stream(s2):
        h_dn.copy_(d_dn, non_blocking=True)


def both():
    up(); down()


tu, td, tb = timed(up), timed(down), timed(both)
print(f"H2D {up_mb} MiB: {tu:.3f} ms ({up_mb * 1.048576 / tu:.1f} GB/s)   D2H {down_mb} MiB: {td:.3f} ms ({down_mb * 1.048576 / td:.1f} GB/s)"
      f"   concurrent: {tb:.3f} ms (sum {tu + td:.3f}, max {max(tu, td):.3f})")

# one direction split over several streams (several copy engines): does the link carry more than one engine delivers?
for n in (2, 4):
    ss = [torch.cuda.Stream(dev) for _ in range(n)]
    def up_split():
        step = (up_mb << 20) // n
        for i, st in enumerate(ss):
            with torch.cuda.stream(st):
                d_up[i * step:(i + 1) * step].copy_(h_up[i * step:(i + 1) * step], non_blocking=True)
    t = timed(up_split)
    print(f"H2D {up_mb} MiB over {n} streams: {t:.3f} ms ({up_mb * 1.048576 / t:.1f} GB/s)")
# page-locked by cudaHostRegister instead of cudaHostAlloc, and write-combined
try:
    rt = torch.cuda.cudart()
    import ctypes
    lib = ctypes.CDLL("libcudart.so.12")
    pwc = ctypes.c_void_p()
    if lib.cudaHostAlloc(ctypes.byref(pwc), ctypes.c_size_t(up_mb << 20), ctypes.c_uint(4)) == 0:  # cudaHostAllocWriteCombined
        ctypes.memset(pwc, 1, up_mb << 20)
        def up_wc():
            lib.cudaMemcpyAsync(ctypes.c_void_p(d_up.data_ptr()), pwc, ctypes.c_size_t(up_mb << 20), ctypes.c_int(1), ctypes.c_void_p(s1.cuda_stream))
        t = timed(up_wc)
        print(f"H2D {up_mb} MiB from write-combined memory: {t:.3f} ms ({up_mb * 1.048576 / t:.1f} GB/s)")
except Exception as e:  # noqa: BLE001
    print("write-combined probe unavailable:", e)

if len(sys.argv) > 1 and sys.argv[1] == "host":
    import numpy as np
    from mesh2splat_b200 import synth, _abi
    from mesh2splat_b200.api import Context
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    scene = synth.helmet_standin(2048)
    ctx = Context(0)
    pscene, keep = bench.pinned_scene(scene, torch)
    cs = pscene.c_struct()
    cap = 6 * 512 * 512
    h_out = torch.empty(cap * 56, dtype=torch.uint8).pin_memory()
    for i in range(4):
        t0 = time.perf_counter()
        rec, _, res = ctx.convert_host(pscene, 512, _abi.LAYOUT_PACKED56, flags=_abi.FLAG_UNCAPPED, capacity=cap, out=h_out.numpy(), c_scene=cs)
        print(f"call {i}: {(time.perf_counter() - t0) * 1e3:.3f} ms, {res.written} records", file=sys.stderr)
