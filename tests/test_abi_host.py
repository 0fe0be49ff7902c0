"""CPU tests of the C-ABI library's host side: exports, error behaviour without a GPU, .ply writer
bytes, bbox rule, .glb loader.  No compute kernels are launched here."""
from __future__ import annotations

import ctypes as C
import json
import os
import re
import struct

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, _lib, synth
from mesh2splat_b200._abi import Primitive, Scene
from util import write_glb, write_image_glb, write_quad_glb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu() -> bool:
    h = C.c_void_p(0)
    st = _lib.lib().m2s_ctx_create(0, C.byref(h))
    if st == _abi.M2S_OK:
        _lib.lib().m2s_ctx_destroy(h)
        return True
    return False


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "m2s.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(m2s_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    L = C.CDLL(_lib.LIB_PATH)
    missing = [n for n in sorted(declared) if not hasattr(L, n)]
    assert not missing, f"libm2s.so does not export {missing}"
    assert declared == set(_lib.SYMBOLS), f"binding list out of sync: {declared ^ set(_lib.SYMBOLS)}"
    assert _lib.lib().m2s_version() == 100


def test_struct_layouts_match_the_header():
    # sizes the C compiler gives the structs in include/m2s.h (checked against ctypes mirrors)
    assert C.sizeof(_abi.m2s_texture) == 16
    assert C.sizeof(_abi.m2s_primitive) == 72
    assert C.sizeof(_abi.m2s_scene) == 48
    assert C.sizeof(_abi.m2s_params) == 48
    assert C.sizeof(_abi.m2s_result) == 32
    L = _lib.lib()
    for layout, stride in _abi.STRIDES.items():
        assert L.m2s_record_stride(layout) == stride == oracle.lib().orc_record_stride(layout)
        assert _abi.record_dtype(layout).itemsize == stride
    assert L.m2s_record_stride(99) == 0
    assert L.m2s_reference_capacity(64, 1) == 24576
    assert L.m2s_reference_capacity(64, 0) == 24576
    assert L.m2s_reference_capacity(1024, 100) == 7_000_000
    p = _abi.m2s_params()
    L.m2s_params_default(C.byref(p))
    assert p.resolution == 520 and abs(p.gaussian_std - 0.65) < 1e-7 and p.layout == 0


def test_no_gpu_means_loud_failure_not_cpu_fallback():
    if _has_gpu():
        pytest.skip("a CUDA device is present")
    L = _lib.lib()
    h = C.c_void_p(0)
    st = L.m2s_ctx_create(0, C.byref(h))
    assert st == _abi.M2S_E_NOGPU and not h.value
    assert b"CUDA" in L.m2s_last_error()
    from mesh2splat_b200.api import Context
    with pytest.raises(_lib.M2SError) as e:
        Context(0)
    assert e.value.status == _abi.M2S_E_NOGPU
    # compute entry points reject a NULL context instead of computing anything
    assert L.m2s_convert(None, None, None, None, 0, None, None) == _abi.M2S_E_INVALID


def test_compute_bboxes_matches_reference_rule():
    a = synth.displaced_sphere(8, 4, seed=1); b = synth.displaced_sphere(8, 4, seed=2, center=(4, 1, -2))
    s = Scene(np.concatenate([a, b]), [Primitive(0, len(a)), Primitive(len(a), len(b))])
    for cumulative in (1, 0):
        s.compute_bboxes(cumulative=bool(cumulative))
        cs, keep = s.c_struct()
        prims = (_abi.m2s_primitive * 2)()
        for i in range(2):
            prims[i].first_triangle = cs.primitives[i].first_triangle
            prims[i].triangle_count = cs.primitives[i].triangle_count
        assert _lib.lib().m2s_compute_bboxes(s.triangles.ctypes.data, prims, 2, cumulative) == 0
        o = (_abi.m2s_primitive * 2)()
        for i in range(2):
            o[i].first_triangle = prims[i].first_triangle; o[i].triangle_count = prims[i].triangle_count
        oracle.lib().orc_compute_bboxes(s.triangles.ctypes.data, o, 2, cumulative)
        for i in range(2):
            assert tuple(prims[i].bbox_min) == s.primitives[i].bbox_min == tuple(o[i].bbox_min)
            assert tuple(prims[i].bbox_max) == s.primitives[i].bbox_max == tuple(o[i].bbox_max)


@pytest.mark.parametrize("fmt", [0, 1, 2, 7])
def test_ply_writer_is_byte_identical_to_the_restated_savePlyVector(tmp_path, fmt):
    from mesh2splat_b200.api import ply_header, ply_write
    tri = synth.displaced_sphere(16, 8, seed=3)
    s = Scene(tri, [Primitive(0, len(tri), (0.9, 0.7, 0.8, 0.9), 0, 1, 2)], synth.make_material_textures(32, 2))
    s.compute_bboxes()
    rec, _, _ = oracle.convert(s, 48, want_keys=False)
    assert len(rec) > 500
    mult = float(np.float32(0.65) / np.float32(48))
    path = tmp_path / f"out{fmt}.ply"
    ply_write(str(path), rec, fmt, mult)
    eff = fmt if fmt <= 2 else 0     # default branch of savePlyVector (parsers.cpp:646-648)
    want = oracle.ply_bytes(rec, eff, mult)
    got = path.read_bytes()
    assert ply_header(eff, len(rec)) == oracle.ply_header(eff, len(rec))
    assert got[:200] == want[:200]
    assert got == want
    hdr = want[: want.index(b"end_header\n") + 11].decode()
    assert hdr.startswith("ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % len(rec))
    assert (len(want) - len(hdr)) == len(rec) * {0: 248, 1: 76, 2: 48}[eff]
    assert hdr.count("property") == {0: 62, 1: 19, 2: 18}[eff]


@pytest.mark.parametrize("fmt", [0, 1, 2, 9])
def test_ply_writer_matches_reference_savePlyVector_golden(tmp_path, fmt):
    """m2s_ply_write vs the files the reference's own parsers::savePlyVector wrote (tests/golden/ref_ply_vectors.npz)."""
    from mesh2splat_b200.api import ply_write
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ply_vectors.npz"))
    rec = g["records"].view(_abi.record_dtype(_abi.LAYOUT_REF96)).reshape(-1)
    path = tmp_path / f"g{fmt}.ply"
    ply_write(str(path), rec, fmt, float(g["scale_multiplier"]))
    assert path.read_bytes() == g[f"ply_format_{fmt}"].tobytes()


# ---- .glb loader ------------------------------------------------------------------------------------
def test_glb_loader_basic(tmp_path):
    from mesh2splat_b200.gltf import load_glb
    p = tmp_path / "a.glb"
    src = write_quad_glb(str(p))
    s = load_glb(str(p))
    assert s.triangle_count == 2 and len(s.primitives) == 1 and s.primitives[0].name == "quad_0"
    v = s.triangles.reshape(2, 3, 12)
    tri_idx = src["idx"].reshape(2, 3)
    assert np.array_equal(v[:, :, 0:3], src["pos"][tri_idx])
    assert np.array_equal(v[:, :, 3:6], src["nrm"][tri_idx])
    assert np.array_equal(v[:, :, 6:10], src["tan"][tri_idx])
    assert np.array_equal(v[:, :, 10:12], src["uv"][tri_idx])
    pr = s.primitives[0]
    np.testing.assert_allclose(pr.base_color_factor, (0.5, 0.6, 0.7, 0.8), rtol=1e-6)
    assert pr.albedo_texture == 0 and pr.normal_texture == 0 and pr.metallic_roughness_texture == 1  # images shared
    assert np.array_equal(s.textures[0], src["img"])
    assert np.array_equal(s.textures[1][..., :3], src["img_rgb"]) and np.all(s.textures[1][..., 3] == 255)
    assert pr.bbox_min == (0.0, 0.0, 0.0) and pr.bbox_max == (1.0, 1.0, 0.5)


def test_glb_loader_fallbacks_and_transforms(tmp_path):
    from mesh2splat_b200.gltf import load_glb
    p = tmp_path / "b.glb"
    M = np.eye(4, dtype=np.float32); M[:3, :3] = np.diag([2.0, 1.0, 0.5]); M[:3, 3] = (1, 2, 3)
    src = write_quad_glb(str(p), indexed=False, with_normals=False, with_tangents=False, with_texture=False, matrix=M,
                    trs=([0.5, 0.0, 0.0], [0.0, 0.0, 0.70710678, 0.70710678], [1.0, 1.0, 2.0]), two_prims=True)
    s = load_glb(str(p))
    assert [q.name for q in s.primitives] == ["quad_0", "quad_1"]     # the LINES primitive is skipped, no counter bump
    assert s.triangle_count == 4
    # world = M * (T R S)
    c = 0.70710678
    R = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]], np.float32)       # 90 deg about z
    L = np.eye(4, dtype=np.float32); L[:3, :3] = R @ np.diag([1, 1, 2]).astype(np.float32); L[:3, 3] = (0.5, 0, 0)
    W = M @ L
    pos = src["pos"][src["idx"]]
    want = (np.c_[pos, np.ones(len(pos))] @ W.T)[:, :3].reshape(2, 3, 3)
    v = s.triangles.reshape(4, 3, 12)
    np.testing.assert_allclose(v[:2, :, 0:3], want, rtol=1e-5, atol=1e-6)
    for t in range(2):                                                 # flat face normal (SceneManager.cpp:406-413)
        fn = np.cross(want[t, 1] - want[t, 0], want[t, 2] - want[t, 0]); fn /= np.linalg.norm(fn)
        np.testing.assert_allclose(v[t, :, 3:6], np.tile(fn, (3, 1)), atol=1e-5)
        assert abs(np.linalg.norm(v[t, 0, 6:9]) - 1) < 1e-5 and abs(v[t, 0, 9]) == 1.0   # per-face tangent + handedness
    assert np.all(v[2:, :, 10:12] == 0)                                # no TEXCOORD_0 -> zeros
    # cumulative bbox: primitive 1 includes primitive 0's extent
    assert s.primitives[1].bbox_min[0] <= s.primitives[0].bbox_min[0]
    assert s.primitives[1].albedo_texture == -1


def test_glb_loader_errors(tmp_path):
    from mesh2splat_b200.gltf import load_glb
    with pytest.raises(OSError):
        load_glb(str(tmp_path / "missing.glb"))
    bad = tmp_path / "bad.glb"
    bad.write_bytes(b"not a glb at all, definitely")
    with pytest.raises(ValueError):
        load_glb(str(bad))
    from mesh2splat_b200.api import SceneManager

    class _RC:  # loadModel prints and returns False on failure, like the reference (SceneManager.cpp:24-27)
        deviceScene = None
    assert SceneManager(_RC()).loadModel(str(bad)) is False


def _rewrite_glb_json(src: str, dst: str, edit) -> None:
    """Re-serialise a .glb after `edit(gltf_dict)` changed its JSON chunk (BIN chunk untouched)."""
    raw = open(src, "rb").read()
    jlen = struct.unpack_from("<I", raw, 12)[0]
    g = json.loads(raw[20:20 + jlen])
    edit(g)
    blen = struct.unpack_from("<I", raw, 20 + jlen)[0]
    write_glb(dst, g, raw[28 + jlen:28 + jlen + blen])


_HOSTILE = [-1, -3, -1000000, 2**31, 2**40, 2**63, 1e300, 0.5, -0.5]


def test_glb_loader_rejects_hostile_sizes(tmp_path):
    """ADVICE r1: negative / huge / fractional byteOffset, byteLength and count must come back as a format error —
    not wrap through size_t into an out-of-bounds read, not throw std::length_error across the C boundary.
    Loaded in a child process so that a crash is a test failure, not the end of the test run."""
    import subprocess
    import sys as _sys
    base = tmp_path / "base.glb"
    write_quad_glb(str(base))
    cases = []
    for i, bad in enumerate(_HOSTILE):
        def e_img_off(g, bad=bad): g["bufferViews"][g["images"][0]["bufferView"]]["byteOffset"] = bad
        def e_img_len(g, bad=bad): g["bufferViews"][g["images"][0]["bufferView"]]["byteLength"] = bad
        def e_img_wrap(g, bad=bad):
            v = g["bufferViews"][g["images"][0]["bufferView"]]
            v["byteOffset"] = -1000000; v["byteLength"] = 1000016
        def e_idx_count(g, bad=bad): g["accessors"][g["meshes"][0]["primitives"][0]["indices"]]["count"] = bad
        def e_pos_count(g, bad=bad): g["accessors"][g["meshes"][0]["primitives"][0]["attributes"]["POSITION"]]["count"] = bad
        def e_acc_off(g, bad=bad): g["accessors"][g["meshes"][0]["primitives"][0]["attributes"]["POSITION"]]["byteOffset"] = bad
        def e_view_off(g, bad=bad): g["bufferViews"][0]["byteOffset"] = bad
        for j, ed in enumerate((e_img_off, e_img_len, e_img_wrap, e_idx_count, e_pos_count, e_acc_off, e_view_off)):
            p = tmp_path / f"h_{i}_{j}.glb"
            _rewrite_glb_json(str(base), str(p), ed)
            cases.append(str(p))
    child = (
        "import sys; sys.path.insert(0, %r)\n"
        "from mesh2splat_b200.gltf import load_glb\n"
        "n = 0\n"
        "for p in sys.argv[1:]:\n"
        "    try:\n"
        "        load_glb(p)\n"
        "    except ValueError:\n"
        "        n += 1\n"
        "print('rejected', n, 'of', len(sys.argv) - 1)\n"
    ) % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([_sys.executable, "-c", child, *cases], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, f"loader crashed (rc {r.returncode}): {r.stderr[-400:]}"
    assert r.stdout.strip() == f"rejected {len(cases)} of {len(cases)}", r.stdout


def _loader_golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_loader_vectors.npz"))


def test_glb_loader_matches_the_reference_parser_golden(tmp_path):
    """tests/golden/ref_loader_vectors.npz: 110+ small .glb files (geometry variants, every image type, 40 random
    multi-mesh scene graphs) and what the REFERENCE's own parser made of them
    (SceneManager::parseGltfFile + tinygltf + stb_image compiled from /root/reference; make_golden.py).
    m2s_glb_load must reproduce it BIT FOR BIT: world-space positions, normals (normal matrix or flat fallback),
    tangents (transformed or per-face fallback), uvs, primitive names and skipping rules, base colour, and every
    decoded texel (all <= 8-bit PNG types incl. Adam7, baseline and progressive JPEG in 4:4:4 / 4:2:2 / 4:2:0)."""
    from mesh2splat_b200.gltf import load_glb
    g = _loader_golden()
    checked_tex = 0
    for name in g["names"]:
        name = str(name)
        p = tmp_path / "case.glb"
        p.write_bytes(g[f"{name}/glb"].tobytes())
        s = load_glb(str(p))
        want = g[f"{name}/faces"]
        assert s.triangles.shape == want.shape, name
        assert np.array_equal(s.triangles.view(np.uint32), want.view(np.uint32)), f"{name}: triangle data differs"
        assert [pr.name for pr in s.primitives] == [str(x) for x in g[f"{name}/mesh_names"]], name
        assert [pr.triangle_count for pr in s.primitives] == list(g[f"{name}/mesh_faces"]), name
        for pr, bc in zip(s.primitives, g[f"{name}/base_color"]):
            assert np.array_equal(np.asarray(pr.base_color_factor, np.float32), bc), name
        present = g[f"{name}/tex_present"] if f"{name}/tex_present" in g.files else None
        for mi, pr in enumerate(s.primitives):
            for which, idx in ((0, pr.albedo_texture), (1, pr.normal_texture), (2, pr.metallic_roughness_texture)):
                if present is not None:
                    assert (idx >= 0) == bool(present[mi][which]), f"{name}: primitive {mi} texture slot {which}"
                key = f"{name}/tex{which}" if mi == 0 else f"{name}/m{mi}tex{which}"
                if key in g.files:
                    assert idx >= 0, name
                    assert np.array_equal(s.textures[idx], g[key]), f"{name}: primitive {mi} texture {which} differs from stb_image's decode"
                    checked_tex += 1
    assert checked_tex >= 150


@pytest.mark.parametrize("mode,subsampling,size", [("RGB", 0, (64, 48)), ("RGB", 2, (70, 37)), ("RGB", 1, (33, 65)), ("L", 0, (40, 24))])
def test_glb_loader_decodes_baseline_jpeg(tmp_path, mode, subsampling, size):
    """Sanity bound of the own JPEG decoder against Pillow (libjpeg) on smooth images.  The decoder follows
    stb_image's arithmetic (the reference's decoder; bit-exactness against it is what tests/test_oracle.py checks
    with golden files); libjpeg rounds its IDCT and 4:2:2 upsampling slightly differently."""
    import io
    from PIL import Image
    from mesh2splat_b200.gltf import load_glb
    w, h = size
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([128 + 100 * np.sin(xx / 9.0), 128 + 100 * np.cos(yy / 7.0), 128 + 60 * np.sin((xx + yy) / 11.0)], axis=-1)
    img = np.clip(img, 0, 255).astype(np.uint8)
    pil = Image.fromarray(img if mode == "RGB" else img[..., 0], mode)
    buf = io.BytesIO()
    kw = {"quality": 92} if mode == "L" else {"quality": 92, "subsampling": subsampling}
    pil.save(buf, "JPEG", **kw)
    want = np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert("RGB")).astype(np.int32)
    p = tmp_path / "j.glb"
    write_image_glb(str(p), buf.getvalue(), "image/jpeg")
    s = load_glb(str(p))
    got = s.textures[0]
    assert got.shape == (h, w, 4) and np.all(got[..., 3] == 255)
    d = np.abs(got[..., :3].astype(np.int32) - want)
    if subsampling == 0:
        assert d.max() <= 3, d.max()
    else:
        assert d.mean() < 1.0 and d.max() <= 12, (d.mean(), d.max())


_PNG_CASES = [(0, 1), (0, 2), (0, 4), (0, 8), (0, 16), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16), (6, 8), (6, 16)]


@pytest.mark.parametrize("interlace", [False, True])
@pytest.mark.parametrize("ctype,depth", _PNG_CASES)
def test_glb_loader_decodes_every_png_type(tmp_path, ctype, depth, interlace):
    """Every PNG colour type / bit depth, plain and Adam7, all five filters, tRNS (palette alpha and colour key):
    the expected RGBA8 is computed from the source samples (16-bit -> high byte; sub-byte gray scaled to 0..255,
    as stb_image — tinygltf's decoder in the reference — does)."""
    from mesh2splat_b200.gltf import load_glb
    from util import png_encode
    rng = np.random.default_rng(ctype * 100 + depth)
    w, h = 13, 11                        # not multiples of 8: exercises partial bytes and short Adam7 passes
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[ctype]
    smp = rng.integers(0, 1 << depth, size=(h, w, ch), dtype=np.int64)
    plte = trns = None
    to8 = (lambda v: v >> 8) if depth == 16 else (lambda v: v)
    want = np.zeros((h, w, 4), np.int64)
    if ctype == 3:
        n = 1 << depth
        pal = rng.integers(0, 256, size=(n, 3), dtype=np.int64)
        alpha = rng.integers(0, 256, size=(max(1, n // 2),), dtype=np.int64)   # tRNS shorter than the palette: rest opaque
        plte, trns = pal.astype(np.uint8).tobytes(), alpha.astype(np.uint8).tobytes()
        idx = smp[..., 0]
        want[..., :3] = pal[idx]
        want[..., 3] = np.where(idx < len(alpha), alpha[np.minimum(idx, len(alpha) - 1)], 255)
    elif ctype == 0:
        key = int(smp[2, 3, 0])
        trns = int(key).to_bytes(2, "big")
        scale = 255 // ((1 << depth) - 1) if depth < 8 else 1
        want[..., :3] = (to8(smp[..., :1]) * scale)
        want[..., 3] = np.where(smp[..., 0] == key, 0, 255)
    elif ctype == 2:
        key = smp[4, 5]
        trns = b"".join(int(v).to_bytes(2, "big") for v in key)
        want[..., :3] = to8(smp)
        want[..., 3] = np.where(np.all(smp == key, axis=-1), 0, 255)
    elif ctype == 4:
        want[..., :3] = to8(smp[..., :1]); want[..., 3] = to8(smp[..., 1])
    else:
        want[...] = to8(smp)
    blob = png_encode(smp, ctype, depth, interlace, plte, trns)
    p = tmp_path / "p.glb"
    write_image_glb(str(p), blob, "image/png")
    got = load_glb(str(p)).textures[0]
    assert got.shape == (h, w, 4)
    assert np.array_equal(got.astype(np.int64), want)
    if ctype in (0, 2, 6) and depth == 8 or ctype == 3:     # cross-check the test's own encoder against Pillow
        import io
        from PIL import Image
        pil = np.asarray(Image.open(io.BytesIO(blob)).convert("RGBA")).astype(np.int64)
        assert np.array_equal(pil, want)


@pytest.mark.parametrize("mode,subsampling,size,restart", [("RGB", 0, (64, 48), 0), ("RGB", 2, (70, 37), 0), ("RGB", 1, (33, 65), 0),
                                                          ("L", 0, (40, 24), 0), ("RGB", 2, (129, 95), 3), ("RGB", 0, (17, 9), 0)])
@pytest.mark.parametrize("quality", [35, 92])
def test_glb_loader_decodes_progressive_jpeg(tmp_path, mode, subsampling, size, restart, quality):
    """Progressive JPEG (spectral selection + successive approximation, per-component AC scans, EOB runs,
    refinement passes; stb_image — the reference's decoder — reads these too): same bounds vs Pillow/libjpeg
    as the baseline decoder, and bit-identical to OUR decoding of the same picture saved as baseline when the
    coefficients are the same (libjpeg quantises before choosing the scan script)."""
    import io
    from PIL import Image
    from mesh2splat_b200.gltf import load_glb
    w, h = size
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    rng = np.random.default_rng(w * h)
    img = np.stack([128 + 100 * np.sin(xx / 9.0), 128 + 100 * np.cos(yy / 7.0), 128 + 60 * np.sin((xx + yy) / 11.0)], axis=-1)
    img = np.clip(img + rng.normal(0, 6, img.shape), 0, 255).astype(np.uint8)   # noise: many non-zero AC coefficients
    pil = Image.fromarray(img if mode == "RGB" else img[..., 0], mode)
    kw = {"quality": quality} if mode == "L" else {"quality": quality, "subsampling": subsampling}
    if restart:
        kw["restart_marker_rows"] = restart
    outs = {}
    for prog in (True, False):
        buf = io.BytesIO()
        pil.save(buf, "JPEG", progressive=prog, **kw)
        if prog:
            assert b"\xff\xc2" in buf.getvalue()
            want = np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert("RGB")).astype(np.int32)
        p = tmp_path / f"j{int(prog)}.glb"
        write_image_glb(str(p), buf.getvalue(), "image/jpeg")
        outs[prog] = load_glb(str(p)).textures[0]
    got = outs[True]
    assert got.shape == (h, w, 4) and np.all(got[..., 3] == 255)
    assert np.array_equal(got, outs[False])          # same coefficients, whatever the scan script
    d = np.abs(got[..., :3].astype(np.int32) - want)
    if subsampling == 0 or mode == "L":   # IDCT / colour-conversion rounding only (libjpeg islow vs stb's fixed point)
        assert d.max() <= 4 and d.mean() < 0.6, (d.max(), d.mean())
    else:                                  # + chroma upsampling differences on noisy content
        assert d.mean() < 1.5 and d.max() <= 16, (d.mean(), d.max())


def test_glb_loader_rejects_arithmetic_jpeg(tmp_path):
    """Arithmetic-coded frames (SOF9..SOF11) are rejected loudly, not mis-decoded."""
    import io
    from PIL import Image
    from mesh2splat_b200.gltf import load_glb
    buf = io.BytesIO()
    Image.fromarray(np.full((16, 16, 3), 90, np.uint8)).save(buf, "JPEG")
    blob = buf.getvalue().replace(b"\xff\xc0", b"\xff\xc9", 1)
    p = tmp_path / "p.glb"
    write_image_glb(str(p), blob, "image/jpeg")
    with pytest.raises(ValueError, match="arithmetic"):
        load_glb(str(p))


def test_glb_loader_survives_corrupt_files():
    """600 deterministic mutants (bit flips, truncations, clobbered length fields, byte swaps) of the golden .glb
    files, loaded in a child process: every one must end in a status code — never a crash.  (scripts/fuzz_loader.py
    runs the same mutation engine at scale; the decoder was also run under ASan/UBSan on 40 k mutants.)"""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import fuzz_loader
    ok, msg = fuzz_loader.run(0, 600)
    assert ok, msg


def test_every_entry_point_rejects_null_arguments_with_a_status():
    """Error behaviour of the boundary: integer status + thread-local message, never a crash (the reference prints
    to std::cerr and carries on, or exit(1)s — SURVEY 8b)."""
    from mesh2splat_b200 import _lib
    L = _lib.lib()
    INV = _abi.M2S_E_INVALID
    assert L.m2s_ply_write(None, None, 0, 0, C.c_float(1.0)) == INV
    assert L.m2s_ply_write(b"/tmp/never_written.ply", None, 5, 0, C.c_float(1.0)) == INV
    small = C.create_string_buffer(16)
    need = L.m2s_ply_header(0, 10, small, 16)
    assert need > 16 and L.m2s_ply_header(0, 10, None, 0) == need   # returns the size needed, writes at most cap bytes
    h = C.c_void_p(0)
    assert L.m2s_glb_load(None, 1, C.byref(h)) == INV and L.m2s_glb_load(b"/nonexistent.glb", 1, None) == INV
    assert not L.m2s_hscene_view(None) and L.m2s_hscene_primitive_name(None, 0) == b""
    L.m2s_hscene_free(None); L.m2s_ctx_destroy(None); L.m2s_scene_free(None, None)
    assert L.m2s_record_stride(99) == 0 and L.m2s_status_string(99) == b"unknown"
    assert L.m2s_compute_bboxes(None, None, 3, 1) == INV
    assert L.m2s_ctx_create(0, None) == INV
    assert L.m2s_convert(None, None, None, None, 0, None, None) == INV
    assert L.m2s_convert_host(None, None, None, None, 0, None, None) == INV
    assert L.m2s_convert_file(None, None, 64, C.c_float(0.65), 0, None, None) == INV
    assert L.m2s_scene_upload(None, None, None) == INV
    assert b"NULL" in L.m2s_last_error()


def test_prepass_entry_points_reject_bad_arguments_without_a_gpu():
    """m2s_prepass / m2s_prepass_enqueue: NULL context or parameters -> M2S_E_INVALID before any CUDA call."""
    import ctypes as C
    L = _lib.lib()
    p = _abi.make_prepass_params(np.eye(4).ravel(), np.eye(4).ravel(), np.eye(4).ravel(), (640, 480), (0.1, 10.0), 0.001, 0, _abi.LAYOUT_REF96)
    v = C.c_uint32(0)
    assert L.m2s_prepass(None, None, 0, C.byref(p), None, None, C.byref(v)) == _abi.M2S_E_INVALID
    assert L.m2s_prepass_enqueue(None, None, 0, None, C.byref(p), None, None, None, None) == _abi.M2S_E_INVALID
    assert C.sizeof(_abi.m2s_prepass_params) == 3 * 64 + 8 + 8 + 16
