#!/usr/bin/env python3
"""Generates tests/golden/ref_shader_vectors.npz from the REFERENCE's own shaders.

Runs only in the build container (needs /root/reference): oracle/build.py compiles
src/shaders/conversion/converter{GS,FS}.glsl (unmodified arithmetic, token-level GLSL->C++
rewrites) against the reference's vendored GLM into oracle/_ref/libm2s_refshader.so; this script
feeds it seeded inputs and stores inputs + outputs.  The committed .npz is what travels: the tests
that consume it (CPU: oracle vs golden; GPU: CUDA vs golden) never touch /root/reference.

    python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import oracle  # noqa: E402
from oracle import build as obuild  # noqa: E402


def gs_inputs(rng, n):
    tris = np.zeros((n, 36), np.float32)
    bmin = np.zeros((n, 3), np.float32)
    bmax = np.zeros((n, 3), np.float32)
    for i in range(n):
        kind = i % 8
        ext = rng.random(3).astype(np.float32) * 4 + 0.5
        lo = (rng.random(3).astype(np.float32) - 0.5) * 10
        if kind == 0:    # generic
            p = lo + rng.random((3, 3)).astype(np.float32) * ext
        elif kind == 1:  # axis aligned right triangle in a random plane, exact ties likely
            ax = rng.integers(0, 3)
            p = np.tile(lo + ext * 0.5, (3, 1)).astype(np.float32)
            a, b = [k for k in range(3) if k != ax]
            p[1, a] += 1.0; p[2, a] += 1.0; p[2, b] += 1.0
        elif kind == 2:  # equilateral-ish: equal edge lengths
            c = lo + ext * 0.5
            p = np.stack([c + [1, 0, 0], c + [0, 1, 0], c + [0, 0, 1]]).astype(np.float32)
        elif kind == 3:  # tiny
            p = lo + ext * 0.5 + rng.random((3, 3)).astype(np.float32) * 1e-3
        elif kind == 4:  # 45 degree tilt: |nx| == |ny|
            c = lo + ext * 0.25
            p = np.stack([c, c + [1, -1, 0], c + [0, 0, 1]]).astype(np.float32)
        elif kind == 5:  # degenerate in projection (collinear) -> inverse2x2 returns 0
            c = lo + ext * 0.25
            d = rng.random(3).astype(np.float32)
            p = np.stack([c, c + d, c + 2 * d]).astype(np.float32)
        elif kind == 6:  # long thin
            c = lo + ext * 0.1
            d = rng.random(3).astype(np.float32) * ext * 0.8
            p = np.stack([c, c + d, c + d * 0.5 + rng.random(3).astype(np.float32) * 1e-2]).astype(np.float32)
        else:            # unit-quad triangles (SURVEY 8c KAT i)
            q = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float32)
            p = q[[0, 1, 2]] if (i // 8) % 2 == 0 else q[[0, 2, 3]]
            lo = np.zeros(3, np.float32); ext = np.array([1, 1, 0], np.float32)
        v = tris[i].reshape(3, 12)
        v[:, 0:3] = p
        v[:, 3:6] = rng.normal(size=(3, 3))
        v[:, 6:10] = rng.normal(size=(3, 4))
        v[:, 10:12] = rng.random((3, 2))
        mn = np.minimum(p.min(axis=0), lo); mx = np.maximum(p.max(axis=0), lo + ext)
        bmin[i] = mn; bmax[i] = mx
    return tris, bmin, bmax


def main():
    obuild.build_all()
    if oracle.ref_lib() is None:
        raise SystemExit("oracle/_ref is not built (no /root/reference here)")
    rng = np.random.default_rng(20260922)
    n = 256
    tris, bmin, bmax = gs_inputs(rng, n)
    glpos = np.zeros((n, 3, 4), np.float32); scale = np.zeros((n, 3), np.float32); quat = np.zeros((n, 4), np.float32)
    for i in range(n):
        glpos[i], scale[i], quat[i] = oracle.ref_gs(tris[i], bmin[i], bmax[i])
    m = 256
    vary = rng.normal(size=(m, 19)).astype(np.float32)
    vary[:, 9] = np.where(rng.random(m) < 0.5, -1.0, 1.0)  # tangent.w
    tex = rng.integers(0, 256, size=(m, 3, 4)).astype(np.float32) / np.float32(255.0)
    flags = rng.integers(0, 8, size=m).astype(np.uint32)
    factor = rng.random((m, 4)).astype(np.float32)
    start = rng.integers(0, 1000, size=m).astype(np.uint32)
    maxg = np.where(rng.random(m) < 0.8, 1 << 20, 500).astype(np.int32)
    rec = np.zeros((m, 24), np.float32); written = np.zeros(m, np.uint8); after = np.zeros(m, np.uint32)
    for i in range(m):
        w, r, c = oracle.ref_fs(vary[i], tex[i, 0], tex[i, 1], tex[i, 2], int(flags[i]), factor[i], int(start[i]), int(maxg[i]))
        written[i] = w; rec[i] = r; after[i] = c
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_shader_vectors.npz")
    np.savez_compressed(out, gs_tris=tris, gs_bmin=bmin, gs_bmax=bmax, gs_glpos=glpos, gs_scale=scale, gs_quat=quat,
                        fs_varyings=vary, fs_texels=tex, fs_flags=flags, fs_factor=factor, fs_counter_start=start,
                        fs_max_gaussians=maxg, fs_rec=rec, fs_written=written, fs_counter_after=after)
    print("wrote", out, os.path.getsize(out), "bytes")
    ply_vectors(rng)
    loader_vectors()


def ply_vectors(rng):
    """ref_ply_vectors.npz: REF96 records -> the bytes the REFERENCE's own parsers::savePlyVector writes
    (src/parsers/parsers.cpp + src/utils/utils.cpp compiled where they lie, oracle/_ref/libm2s_refply.so)."""
    import tempfile
    if oracle.ref_ply_lib() is None:
        raise SystemExit("oracle/_ref/libm2s_refply.so is not built (no /root/reference here)")
    n = 200
    rec = np.zeros((n, 24), np.float32)
    rec[:, 0:3] = rng.normal(size=(n, 3)) * 3                      # position
    rec[:, 3] = 1.0
    rec[:, 4:8] = rng.random((n, 4))                               # colour
    rec[:, 8:10] = np.exp(rng.normal(size=(n, 2)) * 2 - 3); rec[:, 10] = 1e-7   # raw scale
    nrm = rng.normal(size=(n, 3)); rec[:, 12:15] = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    q = rng.normal(size=(n, 4)); rec[:, 16:20] = q / np.linalg.norm(q, axis=1, keepdims=True)
    rec[:, 20:22] = rng.random((n, 2)); rec[:, 23] = 1.0          # pbr
    # edge cases: alpha 1 (opacity +inf) and 0, colours outside [0,1], zero scale, axis normals, unnormalised normal
    rec[0, 7] = 1.0; rec[1, 7] = 0.0; rec[2, 4:7] = (1.5, -0.25, 0.5); rec[3, 8:10] = 0.0
    rec[4, 12:15] = (0, 0, 1); rec[5, 12:15] = (0, 0, -1); rec[6, 12:15] = (-1, 0, 0); rec[7, 12:15] = (3.0, 0.5, -2.0)
    rec[8, 9] = rec[8, 8]; rec[9, 20:22] = (1.7, -0.3)
    rec = rec.astype(np.float32)
    mult = np.float32(0.65) / np.float32(512)
    files = {}
    with tempfile.TemporaryDirectory() as d:
        for fmt in (0, 1, 2, 9):
            path = os.path.join(d, f"ref{fmt}.ply")
            oracle.ref_save_ply(path, rec, fmt, float(mult))
            files[f"ply_format_{fmt}"] = np.frombuffer(open(path, "rb").read(), np.uint8)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_ply_vectors.npz")
    np.savez_compressed(out, records=rec, scale_multiplier=np.float32(mult), **files)
    print("wrote", out, os.path.getsize(out), "bytes")


def loader_vectors():
    """ref_loader_vectors.npz: small .glb files (geometry variants, node transforms, PNG / JPEG images) and what the
    REFERENCE's own parser — SceneManager::parseGltfFile with tinygltf + stb_image, compiled where they lie
    (oracle/_ref/libm2s_refloader.so) — makes of them: faces (pos, normal, tangent, uv), base colour, decoded images."""
    import io
    import tempfile
    from PIL import Image
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from util import png_encode, write_image_glb, write_quad_glb
    if oracle.ref_loader_lib() is None:
        raise SystemExit("oracle/_ref/libm2s_refloader.so is not built (no /root/reference here)")
    rng = np.random.default_rng(424242)
    store = {}
    names = []

    def add(name, path):
        ok, meshes = oracle.ref_load_glb(path)
        assert ok and meshes, name
        names.append(name)
        store[f"{name}/glb"] = np.frombuffer(open(path, "rb").read(), np.uint8)
        store[f"{name}/faces"] = np.vstack([m["faces"] for m in meshes])
        store[f"{name}/mesh_faces"] = np.array([len(m["faces"]) for m in meshes], np.int64)
        store[f"{name}/mesh_names"] = np.array([m["name"] for m in meshes])
        store[f"{name}/base_color"] = np.stack([m["base_color"] for m in meshes])
        for which, t in meshes[0]["textures"].items():
            if t.ndim == 3 and t.shape[2] == 4:       # 8-bit RGBA (16-bit PNGs come back as 8 bytes per pixel: not compared)
                store[f"{name}/tex{which}"] = t
        # per-primitive texture presence (3 flags) for the multi-mesh cases
        store[f"{name}/tex_present"] = np.array([[int(w in m["textures"]) for w in range(3)] for m in meshes], np.int64)
        for mi, m in enumerate(meshes[1:], start=1):
            for which, t in m["textures"].items():
                if t.ndim == 3 and t.shape[2] == 4:
                    store[f"{name}/m{mi}tex{which}"] = t

    def rnd_mat():
        M = np.eye(4, dtype=np.float32); M[:3, :3] = rng.normal(size=(3, 3)); M[:3, 3] = rng.normal(size=3) * 5
        return M

    with tempfile.TemporaryDirectory() as d:
        k = 0
        for indexed in (True, False):
            for with_normals in (True, False):
                for with_tangents in (True, False):
                    for xf in ("none", "matrix", "trs"):
                        kw = dict(indexed=indexed, with_normals=with_normals, with_tangents=with_tangents, two_prims=(k % 4 == 0),
                                  with_uv=(k % 5 != 4), with_texture=(k % 3 == 0))
                        if xf == "matrix":
                            kw["matrix"] = rnd_mat()
                        elif xf == "trs":
                            q = rng.normal(size=4); q /= np.linalg.norm(q)
                            kw["trs"] = ([float(v) for v in rng.normal(size=3) * 3], [float(v) for v in q], [float(v) for v in rng.random(3) * 3 + 0.1])
                        path = os.path.join(d, f"g{k}.glb")
                        write_quad_glb(path, **kw)
                        add(f"geom{k:02d}", path)
                        k += 1
        # images: every 8-bit-or-less PNG type (plain + Adam7), JPEG baseline/progressive x subsampling, gray
        for ctype, depth in [(0, 1), (0, 2), (0, 4), (0, 8), (2, 8), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (6, 8)]:
            ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
            smp = rng.integers(0, 1 << depth, size=(11, 13, ch))
            plte = trns = None
            if ctype == 3:
                n = 1 << depth
                plte = rng.integers(0, 256, size=(n, 3), dtype=np.uint8).tobytes()
                trns = rng.integers(0, 256, size=(max(1, n // 2),), dtype=np.uint8).tobytes()
            if ctype == 0:
                trns = int(smp[2, 3, 0]).to_bytes(2, "big")
            if ctype == 2:
                trns = b"".join(int(v).to_bytes(2, "big") for v in smp[4, 5])
            for il in (False, True):
                path = os.path.join(d, "p.glb")
                write_image_glb(path, png_encode(smp, ctype, depth, il, plte, trns), "image/png")
                add(f"png_c{ctype}_d{depth}_i{int(il)}", path)
        for (w, h) in [(64, 48), (37, 70), (17, 9), (1, 1)]:
            yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
            img = np.stack([128 + 100 * np.sin(xx / 9), 128 + 100 * np.cos(yy / 7), 128 + 60 * np.sin((xx + yy) / 11)], axis=-1)
            img = np.clip(img + rng.normal(0, 12, img.shape), 0, 255).astype(np.uint8)
            for prog in (False, True):
                for ss in (0, 1, 2):
                    b = io.BytesIO()
                    Image.fromarray(img).save(b, "JPEG", quality=80, subsampling=ss, progressive=prog)
                    path = os.path.join(d, "j.glb")
                    write_image_glb(path, b.getvalue(), "image/jpeg")
                    add(f"jpeg_{w}x{h}_p{int(prog)}_s{ss}", path)
            b = io.BytesIO()
            Image.fromarray(img[..., 0]).save(b, "JPEG", quality=80)
            path = os.path.join(d, "j.glb")
            write_image_glb(path, b.getvalue(), "image/jpeg")
            add(f"jpeg_{w}x{h}_gray", path)
        # random multi-mesh scene graphs (nested matrix / TRS nodes, instancing, several materials sharing images,
        # u8 / u16 / u32 / no indices, skipped LINES and POSITION-less primitives, two scenes)
        from util import make_complex_glb
        for seed in range(40):
            path = os.path.join(d, "c.glb")
            make_complex_glb(path, 1000 + seed)
            ok, meshes = oracle.ref_load_glb(path)
            if ok and meshes:
                add(f"graph{seed:02d}", path)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_loader_vectors.npz")
    np.savez_compressed(out, names=np.array(names), **store)
    print("wrote", out, os.path.getsize(out), "bytes,", len(names), "cases")


if __name__ == "__main__":
    main()
