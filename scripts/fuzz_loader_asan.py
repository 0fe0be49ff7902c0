"""Mutation fuzz of the .glb loader under AddressSanitizer + UBSan.

  g++ -std=c++17 -g -O1 -fsanitize=address,undefined -o build/glb_asan scripts/glb_asan_main.cpp \
      mesh2splat_b200/csrc/m2s_glb.cpp mesh2splat_b200/csrc/m2s_image.cpp mesh2splat_b200/csrc/m2s_host.cpp
  python scripts/fuzz_loader_asan.py <count> [first seed]
"""
import subprocess, sys, os, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
g = np.load(os.path.join(ROOT, "tests", "golden", "ref_loader_vectors.npz")); names = [str(n) for n in g["names"]]
n = int(sys.argv[1]); seed0 = int(sys.argv[2]) if len(sys.argv) > 2 else 0
FZ = os.path.join(ROOT, "build", "fz")
os.makedirs(FZ, exist_ok=True)
bad = 0
for s0 in range(seed0, seed0 + n, 200):
    files = []
    for seed in range(s0, min(s0 + 200, seed0 + n)):
        rng = np.random.default_rng(seed)
        blob = bytearray(g[names[seed % len(names)] + "/glb"].tobytes())
        kind = seed % 4
        if kind == 0:
            for _ in range(int(rng.integers(1, 8))): blob[int(rng.integers(0, len(blob)))] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1: blob = blob[: int(rng.integers(0, len(blob)))]
        elif kind == 2:
            i = int(rng.integers(0, max(1, len(blob) - 4))); blob[i:i + 4] = int(rng.integers(0, 2**32)).to_bytes(4, "little")
        else:
            i = int(rng.integers(0, len(blob))); j = int(rng.integers(0, len(blob))); blob[i], blob[j] = blob[j], blob[i]
            blob[int(rng.integers(0, len(blob)))] = int(rng.integers(0, 256))
        f = os.path.join(FZ, f"{seed}.glb"); open(f, "wb").write(bytes(blob)); files.append(f)
    r = subprocess.run([os.path.join(ROOT, "build", "glb_asan"), *files], capture_output=True, text=True, timeout=900,
                       env={**os.environ, "ASAN_OPTIONS": "detect_leaks=0:allocator_may_return_null=1", "UBSAN_OPTIONS": "print_stacktrace=0"})
    errs = [l for l in (r.stderr + r.stdout).splitlines() if "runtime error" in l or "ERROR: AddressSanitizer" in l or "SUMMARY" in l]
    if r.returncode != 0 or errs:
        bad += 1
        last = [l for l in r.stdout.splitlines() if "status" in l][-1:] 
        print("batch", s0, "rc", r.returncode, "after", last, *sorted(set(errs))[:6], sep="\n   ")
    for f in files: os.remove(f)
print("bad batches:", bad)
