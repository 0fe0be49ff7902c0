"""The .ply loader on the GPU (SURVEY 8 f-10): m2s_ply_read / m2s_ply_decode_enqueue against the reference's own
loadPlyFile (golden fixtures) and the C restatement (oracle/m2s_ply_oracle.c) at sizes and strides no fixture holds, and
the viewer passes on loaded records (M2S_VIEW_PLY / M2S_VIEW_PLY_PBR) against the reference's prepass shader and the C
restatements.

Accuracy rule: every field bit for bit.  The kernel evaluates expf with glibc's own table-driven fp64 algorithm
(m2s_codec.cuh; CUDA's expf is up to 2 ulp away, and through the sigmoid that becomes 2 ulp in color.a), so the records
equal the reference loader's golden records exactly, and the restatement's wherever this host's glibc runs the same
variant (util.GLIBC_MAX_ULP; against glibc's other variant scale.xyz and color.a are within 1 ulp).  test_gpu_codec.py
checks the expf and the sigmoid on all 2^32 inputs.  NaN compares equal to NaN (the device's NaN pattern is not the
host's)."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, api
from mesh2splat_b200._lib import M2SError, check, lib
from oracle import light, ply_load
from util import GLIBC_MAX_ULP, GuardedDevice, assert_prepass_match

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
Z = np.load(os.path.join(HERE, "golden", "ref_ply_load_vectors.npz"))
PP = np.load(os.path.join(HERE, "golden", "ref_prepass_ply_vectors.npz"))
NAMES = [str(n) for n in Z["names"]]
EXP_COLS = [7, 8, 9, 10]   # color.a, scale.xyz
STAGE_ROWS_248 = (32 << 20) // 248   # rows of one staging block of the standard layout


def _ulp_diff(a, b):
    """|a - b| in units in the last place (fp32 ordered as integers), 0 for NaN vs NaN."""
    ia = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    ib = np.ascontiguousarray(b, np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, np.int64(-(1 << 31)) - ia, ia)
    ib = np.where(ib < 0, np.int64(-(1 << 31)) - ib, ib)
    d = np.abs(ia - ib)
    return np.where(np.isnan(a) & np.isnan(b), 0, d)


def assert_records(got, want, what="", max_ulp=GLIBC_MAX_ULP):
    """The accuracy rule above (max_ulp: of the exp fields; 0 against the golden records); returns the number of values
    that differ."""
    g, w = np.asarray(got, np.float32).reshape(-1, 24), np.asarray(want, np.float32).reshape(-1, 24)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    d = _ulp_diff(g, w)
    exact = [c for c in range(24) if c not in EXP_COLS]
    bad = np.argwhere(d[:, exact] != 0)
    assert len(bad) == 0, f"{what}: {len(bad)} values differ outside the exp fields, first record {bad[0][0]} field {exact[bad[0][1]]}"
    assert d[:, EXP_COLS].max(initial=0) <= max_ulp, f"{what}: exp fields differ by {d[:, EXP_COLS].max()} ulp"
    return int((d != 0).sum())


def _records(t, n):
    return t[: n * 96].cpu().numpy().view(np.float32).reshape(n, 24)


def _write(tmp_path, name, data: bytes) -> str:
    p = str(tmp_path / f"{name}.ply")
    with open(p, "wb") as f:
        f.write(data)
    return p


def _random_ref96(rng, n):
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_prepass import gaussians
    g = gaussians(rng, n, 0.02)
    g[:, 7] = np.clip(g[:, 7], 1e-3, 1 - 1e-3)
    return np.ascontiguousarray(g, np.float32)


# ---- golden fixtures ------------------------------------------------------------------------------------------------------
def test_ply_read_matches_the_reference_loader_on_every_fixture(gpu_ctx, tmp_path):
    differ = total = 0
    for name in NAMES:
        p = _write(tmp_path, name, Z[f"file_{name}"].tobytes())
        if not int(Z[f"ok_{name}"]) or int(Z[f"dev_{name}"]):
            with pytest.raises(M2SError) as e:
                gpu_ctx.ply_read(p)
            assert e.value.status == _abi.M2S_E_FORMAT, (name, e.value)
            continue
        want = Z[f"rec_{name}"]
        n = len(want)
        guard = GuardedDevice(max(n, 1), 96, what=name)
        recs, count, has_pbr = gpu_ctx.ply_read(p, out=guard.view)
        guard.check(n)
        assert count == n and has_pbr == bool(int(Z[f"pbr_{name}"])), name
        differ += assert_records(_records(recs, n), want, name, max_ulp=0)
        total += n * 24
    assert differ == 0 and total > 0


def test_capacity_below_the_count_writes_nothing(gpu_ctx, tmp_path):
    p = _write(tmp_path, "w1", Z["file_writer_fmt1"].tobytes())
    n = len(Z["rec_writer_fmt1"])
    guard = GuardedDevice(n - 1, 96)
    info = _abi.m2s_ply_info()
    assert lib().m2s_ply_read(gpu_ctx.handle, p.encode(), guard.view.data_ptr(), n - 1, C.byref(info)) == _abi.M2S_E_CAPACITY
    assert info.vertex_count == n and info.has_pbr == 1
    guard.check(0)
    probe = _abi.m2s_ply_info()
    check(lib().m2s_ply_read(gpu_ctx.handle, p.encode(), None, 0, C.byref(probe)))
    assert bytes(probe) == bytes(info)


# ---- round trips through the project's own writer -------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [0, 1])
def test_device_round_trip_encode_then_decode(gpu_ctx, fmt):
    """REF96 -> m2s_ply_encode (format 0 / 1) -> m2s_ply_decode_enqueue equals the restatement on the same rows."""
    import torch
    rng = np.random.default_rng(10 + fmt)
    n = 5000
    g = _random_ref96(rng, n)
    d = torch.from_numpy(g.view(np.uint8).reshape(-1).copy()).cuda()
    rows = gpu_ctx.ply_encode(d, n, fmt, 0.65 / 512)
    info = api.ply_parse_header(api.ply_header(fmt, n) + rows.cpu().numpy().tobytes())
    out = gpu_ctx.ply_decode(rows, info)
    assert_records(_records(out, n), ply_load.load(rows.cpu().numpy(), info, n), f"format {fmt}")


@pytest.mark.parametrize("fmt", [0, 1])
def test_file_round_trip_write_then_read(gpu_ctx, tmp_path, fmt):
    rng = np.random.default_rng(20 + fmt)
    n = 3000
    p = str(tmp_path / f"rt{fmt}.ply")
    api.ply_write(p, _random_ref96(rng, n), fmt, 0.65 / 512)
    info = api.ply_parse_file(p)
    recs, count, has_pbr = gpu_ctx.ply_read(p)
    assert count == n and has_pbr == (fmt == 1)
    assert_records(_records(recs, n), ply_load.load_file(p, info), f"format {fmt}")


# ---- counts and strides ---------------------------------------------------------------------------------------------------
def _rows_file(tmp_path, rng, n, prefix=(), pad=(), name="f"):
    """A file of n rows: `prefix` (type, name) properties, the standard properties with PBR values, then `pad`."""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_ply_load import PBR, STANDARD, ply, vertex_rows
    props = list(prefix) + [("float", k) for k in STANDARD[:3] + PBR + STANDARD[3:]] + list(pad)
    return _write(tmp_path, name, ply([("vertex", n, props, vertex_rows(rng, props, n))]))


@pytest.mark.parametrize("n", [0, 1, 31, 33, STAGE_ROWS_248 - 1, STAGE_ROWS_248, STAGE_ROWS_248 + 1, 2 * STAGE_ROWS_248 + 12345])
def test_counts_around_warps_and_staging_blocks(gpu_ctx, tmp_path, n):
    """The standard 248-byte layout (62 floats): counts around a warp's 32 rows, around one 32 MB staging block, and
    more than two blocks with a partial last one."""
    import torch
    rng = np.random.default_rng(n)
    p = str(tmp_path / "c.ply")
    api.ply_write(p, _random_ref96(rng, n), 0, 0.65 / 512)
    info = api.ply_parse_file(p)
    assert info.row_stride == 248
    guard = GuardedDevice(max(n, 1), 96)
    h0 = gpu_ctx.ply_h2d_bytes()
    recs, count, _ = gpu_ctx.ply_read(p, out=guard.view)
    assert count == n and gpu_ctx.ply_h2d_bytes() - h0 == n * 248
    guard.check(n)
    assert_records(_records(recs, n), ply_load.load_file(p, info), f"n = {n}")
    torch.cuda.synchronize()


@pytest.mark.parametrize("prefix,pad", [
    ([("uchar", "red")], []),                                               # stride 77: every float unaligned
    ([("uchar", "a"), ("ushort", "b")], [("uchar", "c")]),                  # stride 80, floats at 3 mod 4
    ([("char", "a")], [("double", f"p{k}") for k in range(502)]),           # stride 4093
    ([], [("double", f"p{k}") for k in range(502)] + [("float", "q")]),     # stride 4096: the maximum
])
def test_odd_and_maximum_strides(gpu_ctx, tmp_path, prefix, pad):
    import torch
    rng = np.random.default_rng(len(pad) + len(prefix))
    n = 1000
    p = _rows_file(tmp_path, rng, n, prefix, pad)
    info = api.ply_parse_file(p)
    want = ply_load.load_file(p, info)
    recs, count, has_pbr = gpu_ctx.ply_read(p)
    assert count == n and has_pbr
    assert_records(_records(recs, n), want, f"stride {info.row_stride}")
    # the decode on device rows at every byte misalignment of the first row
    with open(p, "rb") as f:
        f.seek(info.body_offset)
        body = np.frombuffer(f.read(n * info.row_stride), np.uint8)
    buf = torch.zeros(len(body) + 16, dtype=torch.uint8, device="cuda")
    for mis in (1, 3, 8, 13):
        buf[mis: mis + len(body)] = torch.from_numpy(body.copy()).cuda()
        guard = GuardedDevice(n, 96)
        gpu_ctx.ply_decode(buf[mis: mis + len(body)], info, out=guard.view, count=n)
        guard.check(n)
        assert_records(_records(guard.view, n), want, f"stride {info.row_stride}, misaligned by {mis}")


# ---- the passes on loaded records -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(4))
def test_prepass_on_loaded_records_matches_the_reference_shader(gpu_ctx, case):
    import torch
    g = PP[f"g{case}"]
    prm = PP[f"params{case}"]
    res, nf, sd, mode, has_pbr = (prm[0], prm[1]), (prm[2], prm[3]), float(prm[4]), int(prm[5]), int(prm[6])
    layout = _abi.VIEW_PLY_PBR if has_pbr else _abi.VIEW_PLY
    V, P, M = PP[f"view{case}"], PP[f"proj{case}"], PP[f"model{case}"]
    d = torch.from_numpy(g.view(np.uint8).reshape(-1).copy()).cuda()
    q, dep = gpu_ctx.prepass(d, len(g), layout, V, P, M, res, nf, sd, mode)
    assert_prepass_match(q, dep, PP[f"quads{case}"], PP[f"depths{case}"], res, ordered=False)
    wq, wd = oracle.prepass(g, V, P, M, res, nf, sd, mode, fmt=1, ply_has_pbr=has_pbr)
    assert_prepass_match(q, dep, wq, wd, res, ordered=False)
    # u_format 1 never reads the mesh depth map: a map in front of everything changes nothing
    near = torch.zeros((64, 48), dtype=torch.float32, device="cuda")
    q2, d2 = gpu_ctx.prepass(d, len(g), layout, V, P, M, res, nf, sd, mode, mesh_depth=near)
    assert_prepass_match(q2, d2, q, dep, res, ordered=False)


@pytest.mark.parametrize("layout", [_abi.VIEW_PLY, _abi.VIEW_PLY_PBR])
def test_shadow_map_on_loaded_records_matches_the_light_oracle(gpu_ctx, layout):
    import torch
    g = PP["g0"] if layout == _abi.VIEW_PLY else PP["g2"]
    n, S = len(g), 128
    M = PP["model1"]
    d = torch.from_numpy(g.view(np.uint8).reshape(-1).copy()).cuda()
    cube, lq, drawn, _ = gpu_ctx.shadow_map(d, n, layout, M, (0.3, 0.2, -0.1), (0.01, 100.0), (1280.0, 720.0), 0.65 / 512, S)
    p = ply_load.light_params(_abi.make_shadow_params(M, (0.3, 0.2, -0.1), (0.01, 100.0), (1280.0, 720.0), 0.65 / 512, layout, S))
    want = light.prepass(g, n, p)
    assert drawn == n
    same = (lq.view(np.uint32) == want.view(np.uint32)) | (np.isnan(lq) & np.isnan(want))
    assert same.all(), f"{int((~same).any(axis=1).sum())} light records differ"
    assert np.array_equal(cube.view(np.uint32), light.cube(lq, S).view(np.uint32))
    # the reference's light prepass with u_format 1 agrees on the culled set
    ref = light.ref_prepass(g, p, 1) if light.ref_lib() is not None else None
    if ref is not None:
        assert np.array_equal(ref[:, 7].view(np.uint32), want[:, 7].view(np.uint32))


def test_read_prepass_sort_draw_shadow_light_chain_on_one_stream(gpu_ctx, tmp_path):
    """A PBR .ply read from disk, then prepass -> sort -> draw -> shadow -> light enqueued on one non-default stream with no
    host synchronisation, at 1280 x 720.  The records equal the restatement of the file's rows, the light records and the
    cube the light oracle's, the image the oracle's lighting of the drawn G-buffer and that cube."""
    import torch
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_prepass import column_major, look_at, perspective
    rng = np.random.default_rng(99)
    n, S, w, h = 200_000, 256, 1280, 720
    g = _random_ref96(rng, n)
    g[:, 8:11] = rng.random((n, 3)).astype(np.float32) * 2 + 0.1
    p = str(tmp_path / "frame.ply")
    api.ply_write(p, g, 1, 0.65 / 512)
    info = api.ply_parse_file(p)
    recs_t, count, has_pbr = gpu_ctx.ply_read(p)
    assert count == n and has_pbr
    recs = _records(recs_t, n)
    assert_records(recs, ply_load.load_file(p, info), "frame records")
    V = column_major(look_at(np.array([0.0, 0.5, 4.0]), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(45.0), w / h, 0.01, 100.0))
    M = column_major(np.eye(4, dtype=np.float32))
    lpos = (1.5, 2.0, 2.5)
    stream = torch.cuda.Stream()
    quads = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
    depths = torch.empty(n, dtype=torch.float32, device="cuda")
    valid = torch.zeros(1, dtype=torch.int32, device="cuda")
    sq = torch.empty(n * 96, dtype=torch.uint8, device="cuda")
    draw = torch.zeros(5, dtype=torch.int32, device="cuda")
    names = [t for t, _ in _abi.GBUFFER_TARGETS]
    gbuf = {t: torch.empty(w * h * 4, dtype=torch.int16 if dt == np.float16 else torch.uint8, device="cuda") for t, dt in _abi.GBUFFER_TARGETS}
    gb_c = _abi.m2s_gbuffer(*[gbuf[t].data_ptr() for t in names])
    gc, gl, gi = GuardedDevice(6 * S * S, 4, what="cube"), GuardedDevice(n, 32, what="light records"), GuardedDevice(w * h, 4, what="image")
    res = torch.zeros(8, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    pp = _abi.make_prepass_params(V, P, M, (w, h), (0.01, 100.0), 0.65 / 512, 6, _abi.VIEW_PLY_PBR)
    sp = _abi.m2s_splat_params(w, h, 6)
    shp = _abi.make_shadow_params(M, lpos, (0.01, 100.0), (w, h), 0.65 / 512, _abi.VIEW_PLY_PBR, S)
    lp = _abi.make_light_params(w, h, 6, lpos, (1.0, 1.0, 1.0), 10.0, (0.0, 0.5, 4.0), 100.0, S)
    L, hs = lib(), stream.cuda_stream
    check(L.m2s_prepass_enqueue(gpu_ctx.handle, recs_t.data_ptr(), n, None, C.byref(pp), quads.data_ptr(), depths.data_ptr(), valid.data_ptr(), hs))
    check(L.m2s_depth_sort_enqueue(gpu_ctx.handle, quads.data_ptr(), depths.data_ptr(), n, valid.data_ptr(), sq.data_ptr(), None, draw.data_ptr(), hs))
    check(L.m2s_splat_draw_enqueue(gpu_ctx.handle, sq.data_ptr(), n, draw.data_ptr(), C.byref(sp), C.byref(gb_c), 60_000_000,
                                   res.data_ptr(), res[2:].data_ptr(), hs))
    check(L.m2s_shadow_map_enqueue(gpu_ctx.handle, recs_t.data_ptr(), n, None, C.byref(shp), gc.view.data_ptr(), gl.view.data_ptr(),
                                   60_000_000, res[4:].data_ptr(), res[6:].data_ptr(), hs))
    check(L.m2s_deferred_light_enqueue(gpu_ctx.handle, C.byref(gb_c), gc.view.data_ptr(), C.byref(lp), gi.view.data_ptr(), hs))
    stream.synchronize()
    o = res.cpu().numpy()
    assert int(o[6]) == n, "the budget holds every pair"
    gc.check(6 * S * S)
    gl.check(n)
    gi.check(w * h)
    m = int(valid.item())
    assert 0 < m <= n and int(draw[1].item()) == m
    lq = gl.view[: n * 32].cpu().numpy().view(np.float32).reshape(n, 8)
    want = light.prepass(recs, n, ply_load.light_params(shp))
    assert ((lq.view(np.uint32) == want.view(np.uint32)) | (np.isnan(lq) & np.isnan(want))).all()
    cube = gc.view[: 6 * S * S * 4].cpu().numpy().view(np.float32).reshape(6, S, S)
    assert np.array_equal(cube.view(np.uint32), light.cube(lq, S).view(np.uint32))
    gb = {t: gbuf[t].view(torch.uint8)[: w * h * 4 * np.dtype(dt).itemsize].cpu().numpy().view(dt).reshape(h, w, 4)
          for t, dt in _abi.GBUFFER_TARGETS}
    img = gi.view[: w * h * 4].cpu().numpy().reshape(h, w, 4)
    wimg = light.deferred_light(gb, cube, lp)
    assert np.array_equal(img, wimg), int((img != wimg).any(axis=-1).sum())
    assert (img[..., :3] > 0).any()


def test_scene_manager_load_ply_sets_the_render_context(tmp_path):
    p = _write(tmp_path, "w1", Z["file_writer_fmt1"].tobytes())
    rc = api.RenderContext(0)
    sm = api.SceneManager(rc)
    assert sm.loadPly(p) is True
    assert rc.format == 1 and rc.plyHasPbr is True and rc.numberOfGaussians == len(Z["rec_writer_fmt1"])
    assert rc.viewLayout() == _abi.VIEW_PLY_PBR
    assert_records(_records(rc.gaussianBuffer, rc.numberOfGaussians), Z["rec_writer_fmt1"])
    bad = _write(tmp_path, "bad", Z["file_writer_fmt2"].tobytes())
    assert sm.loadPly(bad) is False and rc.numberOfGaussians == len(Z["rec_writer_fmt1"])
    rc.ctx.close()
