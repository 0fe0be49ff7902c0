"""Static SASS instruction counts of raster_kernel<1> (PACKED56) by phase: the per-triangle set-up, the small triangles'
coverage walk, and the direct path's group loop (direct_run), split into the shading and staging of a group, the record
emission (capacity cut, copy, keys) and the rest of the loop.

Compiles m2s_raster.cu of a source tree for sm_90a with -lineinfo into a cubin, disassembles it with nvdisasm -gi (the
disassembler cuobjdump -sass uses, plus the line table) and gives every instruction of raster_kernel<1> to the phase of
the outermost m2s_raster.cu line it was inlined from.  Static counts: a loop body counts once, however often it runs.
usage: raster_sass_phases.py [tree ...]   (default: this repository; e.g. a git worktree of another commit to compare)"""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_ZN3m2s13raster_kernelILi1EEEvNS_11ConvertArgsE"
ANNOT = re.compile(r'//## File "([^"]+)", line (\d+)')
INSTR = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+(\S.*?)\s*;")


def source_lines(src):
    with open(src) as f:
        lines = f.read().split("\n")
    find = lambda pat, start=0: next(i + 1 for i in range(start, len(lines)) if re.search(pat, lines[i]))
    setup = find(r"cnt = setup_triangle<RK>\(")
    walk0, walk1 = find(r"const uint32_t mine = "), find(r"const uint32_t nh = ")
    d0 = find(r"__noinline__ \w+ direct_run\(")
    d1 = find(r"^}", d0)
    return lines, setup, (walk0, walk1), (d0, d1)


def phases(tree):
    csrc = os.path.join(tree, "mesh2splat_b200", "csrc")
    src = os.path.join(csrc, "m2s_raster.cu")
    lines, setup, walk, drun = source_lines(src)
    with tempfile.TemporaryDirectory() as tmp:
        cubin = os.path.join(tmp, "raster.cubin")
        subprocess.run(["nvcc", "-std=c++17", "-O3", "-lineinfo", "-gencode", "arch=compute_90a,code=sm_90a", "-cubin",
                        "-o", cubin, src], check=True, cwd=csrc)
        sass = subprocess.run(["nvdisasm", "-gi", cubin], check=True, capture_output=True, text=True).stdout
    counts = {k: 0 for k in ("set-up", "coverage walk", "direct_run: shade + stage", "direct_run: record emission",
                             "direct_run: rest of the loop", "rest of the kernel")}
    inside, chain, fresh = False, [], True
    for ln in sass.split("\n"):
        if ln.startswith(".text."):
            inside = ln.startswith(f".text.{KERNEL}:")
            continue
        if not inside:
            continue
        m = ANNOT.search(ln)
        if m:
            if fresh:
                chain, fresh = [], False
            chain.append((m.group(1), int(m.group(2))))
            continue
        if not INSTR.match(ln):
            continue
        fresh = True
        outer = [l for f, l in chain if f.endswith("m2s_raster.cu")]
        line = outer[-1] if outer else 0
        if line == setup:
            counts["set-up"] += 1
        elif walk[0] <= line < walk[1]:
            counts["coverage walk"] += 1
        elif drun[0] <= line <= drun[1]:
            text = lines[line - 1]
            if re.search(r"\bshade", text):
                counts["direct_run: shade + stage"] += 1
            elif re.search(r"emit_records|bulk_span|fragment_key|keys|room", text):
                counts["direct_run: record emission"] += 1
            else:
                counts["direct_run: rest of the loop"] += 1
        else:
            counts["rest of the kernel"] += 1
    return counts


def main():
    trees = sys.argv[1:] or [ROOT]
    res = [phases(os.path.abspath(t)) for t in trees]
    print(f"{'raster_kernel<1> static SASS':32s}" + "".join(f"{os.path.basename(os.path.abspath(t)) or t:>14s}" for t in trees))
    for k in res[0]:
        print(f"{k:32s}" + "".join(f"{r[k]:14d}" for r in res))
    print(f"{'total':32s}" + "".join(f"{sum(r.values()):14d}" for r in res))


if __name__ == "__main__":
    main()
