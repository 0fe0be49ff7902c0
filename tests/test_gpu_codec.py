"""The codec's device functions (mesh2splat_b200/csrc/m2s_codec.cuh) against glibc, and the outputs that use them against
the project's .ply writer and loader.

Function level: each function through m2s_debug_codec_eval on every input bit pattern of its domain, in chunks of 2^26
made on the device, against the checker (oracle/m2s_codec_oracle.c), which computes the reference's formulas with glibc's
logf / expf.  NaN compares equal to NaN.  The device ports glibc's FMA variant of logf and expf (the one glibc selects on
an x86-64 CPU with FMA and AVX2, and the only one on aarch64): against that glibc every value is bit-identical.  Against
a glibc that runs its other variant the rule is 1 ulp; util.GLIBC_MAX_ULP decides it once, from the CPU.

Integration (guarded outputs, rows matched by fragment key): every .ply layout a conversion writes equals the writer's
bytes of the REF96 record of the same fragment; m2s_ply_encode equals m2s_ply_write; convert -> .ply -> m2s_ply_read
equals the writer's file of the REF96 conversion decoded by the loader's restatement."""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, api, synth
from mesh2splat_b200._abi import (FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_REF96, PLY_FORMAT_LAYOUT, Primitive, Scene)
from oracle import codec, ply_load
from util import GLIBC_MAX_ULP, GuardedDevice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CHUNK = 1 << 26
BENCH_MULT = float(np.float32(0.65) / np.float32(512))


MAX_ULP = GLIBC_MAX_ULP
EXACT = MAX_ULP == 0


def _ulp_diff(got, want):
    """|got - want| in ulp (fp32 ordered as integers) on the device, 0 for NaN vs NaN."""
    import torch
    gi, wi = got.view(torch.int32).to(torch.int64), want.view(torch.int32).to(torch.int64)
    gi = torch.where(gi < 0, -(1 << 31) - gi, gi)
    wi = torch.where(wi < 0, -(1 << 31) - wi, wi)
    d = (gi - wi).abs()
    return torch.where(torch.isnan(got) & torch.isnan(want), torch.zeros_like(d), d)


def _check(ctx, fn, ref, x_host, x_dev, arg, what):
    import torch
    got = ctx.codec_eval(fn, x_dev, arg)
    want = torch.from_numpy(ref(x_host)).cuda()
    d = _ulp_diff(got, want)
    bad = d > MAX_ULP
    nbad = int(bad.sum())
    if nbad:
        i = int(torch.nonzero(bad)[0])
        return nbad, (f"{what}: input {x_host[i]!r} (0x{int(x_host.view(np.uint32)[i]):08x}) -> {float(got[i])!r} "
                      f"(0x{int(got.view(torch.int32)[i]) & 0xffffffff:08x}), glibc {float(want[i])!r}")
    return 0, None


def _sweep(ctx, fn, ref, lo, hi, what, arg=1.0, extra=()):
    """fn on the float bit patterns [lo, hi) and on `extra` values; asserts no value is more than MAX_ULP away."""
    import torch
    t0 = time.perf_counter()
    nbad, first = 0, None
    for a in range(lo, hi, CHUNK):
        b = min(hi, a + CHUNK)
        x = torch.arange(a, b, dtype=torch.int64, device="cuda")
        x = torch.where(x >= (1 << 31), x - (1 << 32), x).to(torch.int32).view(torch.float32)
        n, msg = _check(ctx, fn, ref, np.arange(a, b, dtype=np.uint64).astype(np.uint32).view(np.float32), x, arg, what)
        nbad, first = nbad + n, first or msg
    if len(extra):
        xh = np.asarray(extra, np.float32)
        n, msg = _check(ctx, fn, ref, xh, torch.from_numpy(xh.copy()).cuda(), arg, what)
        nbad, first = nbad + n, first or msg
    torch.cuda.synchronize()
    print(f"{what}: {hi - lo + len(extra)} inputs, {nbad} differ ({'bit for bit' if EXACT else '1 ulp'} rule), "
          f"{time.perf_counter() - t0:.1f} s")
    assert nbad == 0, f"{nbad} values differ; first {first}"


def _f(bits):
    return np.array(bits, np.uint32).view(np.float32)


NEG_AND_NAN = _f([0x80000000, 0x80000001, 0x807fffff, 0x80800000, 0xbf800000, 0xff7fffff, 0xff800000,
                  0x7fc00000, 0x7f800001, 0x7fbfffff, 0xffc00000, 0xffffffff])


# ---- function level, exhaustive --------------------------------------------------------------------------------------------
def test_decoder_expf_every_input(gpu_ctx):
    _sweep(gpu_ctx, _abi.CODEC_EXPF, codec.expf, 0, 1 << 32, "expf")


def test_decoder_sigmoid_every_input(gpu_ctx):
    _sweep(gpu_ctx, _abi.CODEC_SIGMOID, codec.sigmoid, 0, 1 << 32, "sigmoid")


@pytest.mark.parametrize("mult", [1.0, BENCH_MULT])
def test_log_scale_every_positive_input(gpu_ctx, mult):
    """+0, every subnormal and normal, +inf (bit patterns 0 .. 0x7f800000), then -0, negatives, -inf and NaNs."""
    _sweep(gpu_ctx, _abi.CODEC_LOG_SCALE, lambda x: codec.log_scale(x, mult), 0, 0x7f800001, f"log(s * {mult:.9g})",
           arg=mult, extra=NEG_AND_NAN)


def test_opacity_logit_every_alpha(gpu_ctx):
    """Every alpha in [+0, 1] (bit patterns 0 .. 0x3f800000), then the clamp's inputs: -0, negatives, above 1, +-inf,
    NaN; and by name the values where the formula turns: 1 - 1 ulp, 0.5 +- a few ulp, the alphas around 1e-8 and 6e-8
    where a + 1e-8f starts to round."""
    one_m = np.nextafter(np.float32(1), np.float32(0))
    half = np.float32(0.5)
    named = [one_m, np.nextafter(one_m, np.float32(0))] + [half + k * np.spacing(half) for k in (-3, -2, -1, 1, 2, 3)] + \
            [np.float32(v) for v in (1e-8, 5e-9, 6e-8, 1.2e-7, 5.96e-8, 1.5e-45)]
    above = _f([0x3f800001, 0x3fc00000, 0x40000000, 0x7f7fffff, 0x7f800000])
    _sweep(gpu_ctx, _abi.CODEC_LOGIT, codec.logit, 0, 0x3f800001, "opacity logit",
           extra=np.concatenate([NEG_AND_NAN, above, np.array(named, np.float32)]))


def test_sh0_every_input(gpu_ctx):
    _sweep(gpu_ctx, _abi.CODEC_SH0, codec.sh0, 0, 1 << 32, "sh0")


# ---- the conversion's layouts against the writer -----------------------------------------------------------------------
def _scene(name):
    if name == "three_map_sphere":
        tri = synth.displaced_sphere(48, 24, seed=3, amplitude=0.1)
        s = Scene(tri, [Primitive(0, len(tri), (0.9, 0.8, 0.7, 1.0), 0, 1, 2)], synth.make_material_textures(256, 11))
        s.compute_bboxes()
        return s, 128, 0
    if name == "helmet_standin":
        return synth.helmet_standin(2048), 512, 0
    tri = synth.random_soup(600, seed=5, tri_size=0.3)
    tex = [synth.random_texture(100, 37, 1), synth.random_texture(17, 129, 2), synth.random_texture(1, 1, 3),
           synth.random_texture(5, 3, 4)]
    prims = [Primitive(0, 200, (1, 1, 1, 1), 0, 1, 2), Primitive(200, 200, (0.3, 0.6, 0.9, 0.5), 3, -1, 0),
             Primitive(400, 200, (1, 1, 1, 1), -1, 2, -1)]
    s = Scene(tri, prims, tex)
    s.compute_bboxes(cumulative=True)
    return s, 200, FLAG_UNCAPPED


def _guarded_convert(ctx, ds, R, layout, flags, n):
    import torch
    stride = _abi.STRIDES[layout]
    out, keys = GuardedDevice(n, stride, what=f"layout {layout}"), GuardedDevice(n, 8, torch.int64, what="keys")
    o = ctx.convert(ds, R, layout, flags=flags, capacity=n, out=out.view, keys=keys.view, want_keys=True)
    assert o.total == n and o.written == n
    out.check(n)
    keys.check(n)
    rows = out.view[: n * stride].cpu().numpy().reshape(n, stride)
    k = keys.view[:n].cpu().numpy().view(np.uint64)
    order = np.argsort(k, kind="stable")
    return rows[order], k[order]


def _same_bits(g, w, what, byte_lanes=()):
    """Rows equal byte for byte, except that a float lane where both hold a NaN is equal (the device's NaN pattern is
    not the host's).  byte_lanes: 4-byte lanes that hold bytes, not a float."""
    g, w = np.ascontiguousarray(g), np.ascontiguousarray(w)
    gb, wb = g.view(np.uint8).reshape(len(g), -1), w.view(np.uint8).reshape(len(w), -1)
    same = gb == wb
    if gb.shape[1] % 4 == 0:
        gf, wf = gb.view(np.float32), wb.view(np.float32)
        nan = np.isnan(gf) & np.isnan(wf)
        nan[:, list(byte_lanes)] = False
        same |= np.repeat(nan, 4, axis=1)
    bad = np.flatnonzero(~same.all(axis=1))
    assert len(bad) == 0, f"{what}: {len(bad)} of {len(g)} rows differ, first row {bad[0]}: {g[bad[0]]!r} vs {w[bad[0]]!r}"


@pytest.mark.parametrize("scene", ["three_map_sphere", "helmet_standin", "npot_repeat_soup"])
def test_ply_layouts_equal_the_writer_of_the_ref96_records(gpu_ctx, scene):
    s, R, flags = _scene(scene)
    mult = float(np.float32(0.65) / np.float32(R))
    ds = gpu_ctx.upload(s)
    n = gpu_ctx.convert(ds, R, LAYOUT_REF96, flags=flags).total
    ref, rk = _guarded_convert(gpu_ctx, ds, R, LAYOUT_REF96, flags, n)
    r = ref.view(np.float32).reshape(n, 24)
    for fmt in (0, 1, 2):
        layout = PLY_FORMAT_LAYOUT[fmt]
        rows, k = _guarded_convert(gpu_ctx, ds, R, layout, flags, n)
        assert np.array_equal(k, rk), f"format {fmt}: coverage differs from REF96"
        want = np.frombuffer(oracle.ply_bytes(r, fmt, mult)[len(oracle.ply_header(fmt, n)):], np.uint8).reshape(n, -1)
        # the carried fields first: position, normal, quaternion
        carried = {0: [(0, 12, "position"), (12, 24, "normal"), (232, 248, "rotation")],
                   1: [(0, 12, "position"), (12, 24, "normal"), (60, 76, "rotation")],
                   2: [(0, 12, "position"), (16, 32, "rotation"), (44, 46, "octahedral normal")]}[fmt]
        for a, b, what in carried:
            _same_bits(rows[:, a:b], want[:, a:b], f"{scene} format {fmt} {what}")
        _same_bits(rows, want, f"{scene} format {fmt} row", byte_lanes=(3, 11) if fmt == 2 else ())
    # PACKED56: position and uv come from planes and the colour may differ in the last bits; log-scale and rotation are
    # the REF96 record's exactly
    pk, k = _guarded_convert(gpu_ctx, ds, R, LAYOUT_PACKED56, flags, n)
    assert np.array_equal(k, rk)
    p = pk.view(_abi.record_dtype(LAYOUT_PACKED56)).reshape(n)
    _same_bits(p["rot"], r[:, 16:20], f"{scene} PACKED56 rotation")
    want_ls = np.stack([codec.log_scale(r[:, 8], mult), codec.log_scale(r[:, 9], mult),
                        codec.log_scale(r[:, 10], mult)], 1)
    _same_bits(p["log_scale"], want_ls, f"{scene} PACKED56 log_scale")
    ds.free()


# ---- m2s_ply_encode against m2s_ply_write --------------------------------------------------------------------------------
def _adversarial_ref96(fmt):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_prepass import gaussians
    rng = np.random.default_rng(77 + fmt)
    g = np.ascontiguousarray(gaussians(rng, 4096, 0.02), np.float32)
    one_m = np.nextafter(np.float32(1), np.float32(0))
    half = np.float32(0.5)
    alphas = np.array([0, -0.0, 1, one_m, half, np.nextafter(half, 0), np.nextafter(half, 1), half + 3 * np.spacing(half),
                       np.nan, -0.5, 1.5, -np.inf, np.inf, 1e-8, 6e-8, 1.5e-45], np.float32)
    scales = np.array([0, -0.0, 1.5e-45, 1e-40, np.inf, np.nan, -1, -1e-30, 3.4e38, 1e-7], np.float32)
    colours = np.array([0, -0.0, 1, one_m, half, -1e30, 1e30, np.inf, -np.inf, 1.5e-45, 2], np.float32)
    m = max(len(alphas), len(scales), len(colours))
    a = np.resize(alphas, 4 * m)
    if fmt == 2:   # a NaN alpha has no byte (the C++ float -> uint8 conversion of NaN is undefined)
        a = np.where(np.isnan(a), np.float32(0.25), a)
    g[: 4 * m, 7] = a
    for c in range(3):
        g[: 4 * m, 8 + c] = np.roll(np.resize(scales, 4 * m), c)
        g[: 4 * m, 4 + c] = np.roll(np.resize(colours, 4 * m), 2 * c)
    return g


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_ply_encode_equals_the_writer_byte_for_byte(gpu_ctx, tmp_path, fmt):
    import torch
    g = _adversarial_ref96(fmt)
    n = len(g)
    for mult in (1.0, BENCH_MULT):
        d = torch.from_numpy(g.view(np.uint8).reshape(-1).copy()).cuda()
        rows = gpu_ctx.ply_encode(d, n, fmt, mult).cpu().numpy()
        p = tmp_path / f"w{fmt}.ply"
        api.ply_write(str(p), g, fmt, mult)
        data = p.read_bytes()
        want = np.frombuffer(data[len(api.ply_header(fmt, n)):], np.uint8).reshape(n, -1)
        _same_bits(rows.reshape(n, -1), want, f"format {fmt}, mult {mult:.9g}", byte_lanes=(3, 11) if fmt == 2 else ())


def test_ply_encode_rejects_misaligned_buffers(gpu_ctx):
    """The encoder's wide loads and stores need 16-byte aligned buffers: a misaligned one is an argument error, not a
    fault.  count = 0: nothing is ever launched, whatever the check does."""
    import torch
    from mesh2splat_b200._lib import lib
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    assert lib().m2s_ply_encode(gpu_ctx.handle, p, 0, 0, 1.0, p + 16, None) == _abi.M2S_OK
    for ref96, rows in ((p + 4, p), (p, p + 4)):
        assert lib().m2s_ply_encode(gpu_ctx.handle, ref96, 0, 0, 1.0, rows, None) == _abi.M2S_E_INVALID


# ---- export -> import ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1])
def test_convert_file_then_ply_read_equals_the_writer_then_the_loader(gpu_ctx, tmp_path, fmt):
    """m2s_convert_file then m2s_ply_read equals orc_ply_load of m2s_ply_write's bytes of the REF96 conversion of the same
    .glb, bit for bit (as multisets of records: both files are in atomic arrival order)."""
    from mesh2splat_b200.gltf import load_glb
    from util import write_quad_glb
    glb, ply, ref_ply = tmp_path / "m.glb", tmp_path / f"m{fmt}.ply", tmp_path / f"r{fmt}.ply"
    write_quad_glb(str(glb), two_prims=True)
    R, std = 96, 0.65
    res = gpu_ctx.convert_file(str(glb), R, str(ply), std, fmt)
    ds = gpu_ctx.upload(load_glb(str(glb)))
    out = gpu_ctx.convert(ds, R, LAYOUT_REF96, gaussian_std=std)
    ds.free()
    assert res.total == out.total and res.written == out.written > 1000
    api.ply_write(str(ref_ply), out.numpy(), fmt, float(np.float32(std) / np.float32(R)))
    want = ply_load.load_file(str(ref_ply), api.ply_parse_file(str(ref_ply)))
    recs, count, _ = gpu_ctx.ply_read(str(ply))
    got = recs[: count * 96].cpu().numpy().view(np.float32).reshape(count, 24)
    assert count == len(want)

    def canon(x):
        u = np.where(np.isnan(x), np.float32(np.nan), x).view(np.uint32)
        return u[np.lexsort(u.T[::-1])]
    _same_bits(canon(got), canon(want), f"format {fmt} record")
