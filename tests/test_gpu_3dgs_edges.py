"""The standard 3DGS render on the GPU (m2s_3dgs_render) at its edges: both targets and the pair count bit for bit
against the checker (oracle/m2s_3dgs_oracle.c) through guarded buffers, on the input classes of
tests/test_3dgs_host_edges.py (held there against fp64), non-finite and degenerate records, exact tile-boundary ties,
the batch and early-stop edges of the tile loop, survivor counts past the binner's 1 024 scan blocks, d_count and the
pair budget at exact boundaries, SH read from a .ply file, and the .ply export round trip within a per-pixel bound
derived from the codec's roundings.

Round-trip bound.  ply_write stores log(s), logit(o) and (c - 0.5) / C0; ply_read decodes with expf, the sigmoid and
C0 f + 0.5, each within 1 ulp of glibc (tests/test_gpu_codec.py pins them bit for bit).  So per record the scale
moves by e_s = 2^-23 (2 + |log s|) relative (log's ulp is that of |log s|, then exp's), the opacity by e_o = 2^-20
relative (the logit's 1e-8 guard, the quotient, the log and the sigmoid, each a few ulp of o) and the colour by e_c =
2^-22 absolute (a few ulp of 0.5 + |C0 f|), and the writer's normalised rotation by e_q = 2^-21 per component; these
are asserted record by record.  A rotation change e_q turns Sigma by an angle of about 2 e_q, which moves the power
by at most 2 e_q kappa |power| (kappa as in test_3dgs_host_edges).  A relative scale change e_s moves
Sigma within (1 +- e_s)^2 in the Loewner order, hence cov and the conic, hence the power by at most 2 e_s |power|, and
the alpha by alpha (2 e_s |power| + e_o).  Through the blend (see tests/test_3dgs_host_edges.py: d out <= sum_i T_i
d alpha_i max(colour, background) + T_i alpha_i d c_i) the two exact images differ by at most
    cmax (sum_i T_i alpha_i 2 e_s |power_i| + e_o (1 - T)) + e_c (1 - T),
and each fp32 image differs from its exact one by the fp32 bound of test_3dgs_host_edges (taken twice).  Pixels where
an alpha lies within 2^-16 of 1/255 or 0.99, a T of the stop, or a rectangle decides a gaussian are excluded and
counted (under 10 %: 1 500 gaussians on 128 x 96 put many pixels near an edge of some tile rectangle)."""
from __future__ import annotations

import numpy as np
import pytest

from mesh2splat_b200 import _abi
from oracle import gs3d
from test_3dgs_host_edges import (CAMERAS, CLAMP_V, U, camera, clamp_scene, huge_scene, image_scene, near_scene,
                                  octant_cameras, perspective, random_quats, shaped_scene, sh_scene)
from test_3dgs_host import ref96
from test_gpu_3dgs import _dev, check_against_oracle, render_guarded

pytestmark = pytest.mark.gpu
EYE = np.eye(4, dtype=np.float32)


# ---- the host edge classes on the GPU --------------------------------------------------------------------------------
def _host_case(name):
    """(records, V, P, w, h, near, kwargs) of each input class of test_3dgs_host_edges."""
    if name in ("iso", "needle", "flat"):
        V, P = camera(96, 64)
        return shaped_scene(name, 1500, 1), V, P, 96, 64, 0.2, {}
    if name == "clamp":
        P = perspective(50.0, 96 / 64, 0.1, 100.0)
        return clamp_scene(96, 64, P, 4), CLAMP_V, P, 96, 64, 0.2, {}
    if name.startswith("near"):
        near = float(np.float32(float(name[4:])))
        return near_scene(near, int(float(name[4:]) * 1e4)), CLAMP_V, perspective(60.0, 1.5, 0.001, 100.0), 96, 64, near, {}
    if name.startswith("view"):
        w, h = (int(x) for x in name[4:].split("x"))
        V, P = camera(w, h)
        return image_scene(3000, 5), V, P, w, h, 0.2, {}
    if name == "huge":
        return huge_scene(6), CLAMP_V, perspective(60.0, 1920 / 1080, 0.01, 100.0), 1920, 1080, 0.01, {}
    if name.startswith("image"):
        cam, w, h = name[6:].split("_")
        V, P = camera(int(w), int(h), cam)
        return image_scene(150, 2), V, P, int(w), int(h), 0.2, {"background": (0.1, 0.2, 0.3)}
    raise ValueError(name)


HOST_CASES = (["iso", "needle", "flat", "clamp", "near0.001", "near0.01", "near0.2", "huge", "view1920x1080", "view4096x4096",
               "view4096x1", "view1x4096"] + [f"image_{c}_640_360" for c in CAMERAS])


@pytest.mark.parametrize("case", HOST_CASES)
def test_host_edge_classes_bit_for_bit(gpu_ctx, case):
    rec, V, P, w, h, near, kw = _host_case(case)
    check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=near, **kw)


def test_sh_octants_bit_for_bit(gpu_ctx):
    rec, sh = sh_scene(4000, 23, 3)
    P = perspective(120.0, 1.0, 0.05, 100.0)
    for V in octant_cameras()[::3]:
        for degree in (1, 3):
            check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, 64, 64, sh=sh, buffer_degree=3, sh_degree=degree, near=0.05)


# ---- non-finite and degenerate records --------------------------------------------------------------------------------
W_ODD, H_ODD = 63, 47   # the mean of a gaussian on the axis lands exactly on pixel ((W - 1) / 2, (H - 1) / 2)


def _axis_camera():
    return CLAMP_V, perspective(50.0, W_ODD / H_ODD, 0.1, 100.0)


def degenerate_records():
    """One record per degenerate case, each at its own place in front of the camera at (0, 0, 4)."""
    rng = np.random.default_rng(30)
    cases = []

    def add(pos=None, s=(0.05, 0.05, 0.05), q=(1.0, 0.0, 0.0, 0.0), op=0.7):
        p = rng.uniform(-0.6, 0.6, 3) if pos is None else np.asarray(pos, np.float64)
        cases.append(ref96(np.array([p]), np.array([s]), np.array([q]), rng.uniform(0, 1, (1, 3)), np.array([op])))

    for bad in (np.nan, np.inf, -np.inf):
        for k in range(3):
            p = rng.uniform(-0.6, 0.6, 3)
            p[k] = bad
            add(pos=p)
            s = np.full(3, 0.05)
            s[k] = bad
            add(s=s)
        add(op=bad)
    add(q=(0.0, 0.0, 0.0, 0.0))                       # the 1e-12 floor of |q|
    add(q=(1e-30, 0.0, 0.0, 0.0))
    for zeros in ((0,), (0, 1), (0, 1, 2)):           # only the +0.3 dilation keeps det > 0
        s = np.full(3, 0.05)
        s[list(zeros)] = 0.0
        add(s=s)
    cut = float(np.float32(1.0 / 255.0))
    for op in (cut, float(np.nextafter(np.float32(cut), np.float32(0))), float(np.nextafter(np.float32(cut), np.float32(1))),
               0.99, float(np.nextafter(np.float32(0.99), np.float32(1))), 1.0):
        add(op=op, s=(0.3, 0.3, 0.3))
    return np.concatenate(cases)


def test_non_finite_and_degenerate_records(gpu_ctx):
    V, P = _axis_camera()
    rec = degenerate_records()
    splats, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, W_ODD, H_ODD, near=0.2)
    gs, gk, galive = gpu_ctx.gs3d_preprocess(_dev(rec), len(rec), _abi.VIEW_PLY, V, P, EYE, W_ODD, H_ODD, near=0.2)
    assert galive == alive and gk.tobytes() == keys.tobytes() and gs.tobytes() == splats.tobytes()
    assert 0 < alive < len(rec)
    # every record alone (its own image) and all together
    for i in range(len(rec)):
        check_against_oracle(gpu_ctx, rec[i:i + 1], _abi.VIEW_PLY, V, P, EYE, W_ODD, H_ODD, near=0.2, background=(0.2, 0.4, 0.6))
    check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, W_ODD, H_ODD, near=0.2)


@pytest.mark.parametrize("which", ["at", "below"])
def test_alpha_exactly_at_the_cut(gpu_ctx, which):
    """A gaussian on the axis: its mean is exactly pixel ((W - 1) / 2, (H - 1) / 2), where power = -0 and alpha = the
    opacity.  An opacity of exactly 1/255 is composited there (the cut is alpha < 1/255); one ulp less is not."""
    V, P = _axis_camera()
    cut = np.float32(1.0 / 255.0)
    op = cut if which == "at" else np.nextafter(cut, np.float32(0))
    rec = ref96(np.array([[0.0, 0.0, 0.0]]), np.full((1, 3), 0.05), np.array([[1.0, 0, 0, 0]]), np.array([[1.0, 1.0, 1.0]]), np.array([op]))
    splats, *_ = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, W_ODD, H_ODD, near=0.2)
    assert splats[0, 0] == (W_ODD - 1) / 2 and splats[0, 1] == (H_ODD - 1) / 2
    f32, _, _ = check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, W_ODD, H_ODD, near=0.2)
    centre = f32[(H_ODD - 1) // 2, (W_ODD - 1) // 2]
    assert (centre[3] > 0) == (which == "at"), centre
    assert np.count_nonzero(f32[..., 3]) == (1 if which == "at" else 0)


# ---- tile-boundary ties ------------------------------------------------------------------------------------------------
def tie_records(w, h, V, P):
    """Gaussians whose u - r, u + r + 15, v - r or v + r + 15 is exactly a multiple of 16: the x (then y) of each is
    walked over neighbouring fp32 values until the checker's mean lands on the wanted integer."""
    out = []
    P00, P11 = float(P.ravel()[0]), float(P.ravel()[5])
    d = 4.0
    rng = np.random.default_rng(40)
    for s in (0.02, 0.05, 0.1):
        probe = ref96(np.array([[0.0, 0.0, 0.0]]), np.full((1, 3), s), np.array([[1.0, 0, 0, 0]]), np.ones((1, 3)), np.array([0.8]))
        r = int(gs3d.preprocess(probe, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)[0][0, 11])
        for k in range(1, 5):
            for mode in ("lo", "hi"):
                tu = 16 * k + r if mode == "lo" else 16 * k + 1 - r   # u - r = 16 k, or u + r + 15 = 16 (k + 1)
                tv = 16 * (k % 3 + 1) + r if mode == "hi" else 16 * (k % 3 + 1) + 1 - r
                if not (0 <= tu < w and 0 <= tv < h):
                    continue
                x0 = ((2 * tu + 1) / w - 1) * d / P00
                y0 = ((2 * tv + 1) / h - 1) * d / P11
                best = None
                for axis, target in ((0, tu), (1, tv)):
                    base = np.array([x0, y0, 0.0], np.float32) if best is None else best
                    c0 = np.float32(base[axis])
                    cand = c0 + np.arange(-300, 301, dtype=np.float32) * np.spacing(c0)
                    pos = np.repeat(base[None], len(cand), 0)
                    pos[:, axis] = cand
                    rr = ref96(pos, np.full((len(cand), 3), s), np.tile([1.0, 0, 0, 0], (len(cand), 1)), rng.uniform(0, 1, (len(cand), 3)),
                               np.full(len(cand), 0.8))
                    sp, *_ = gs3d.preprocess(rr, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)
                    hit = np.nonzero((sp[:, axis] == target) & (sp[:, 11] == r))[0]
                    if len(hit) == 0:
                        break
                    best = pos[hit[0]].copy()
                else:
                    out.append(ref96(best[None].astype(np.float64), np.full((1, 3), s), np.array([[1.0, 0, 0, 0]]), rng.uniform(0, 1, (1, 3)),
                                     np.array([0.8])))
    return np.concatenate(out)


def test_tile_boundary_ties(gpu_ctx):
    w, h = 127, 95
    V, P = CLAMP_V, perspective(50.0, w / h, 0.1, 100.0)
    rec = tie_records(w, h, V, P)
    splats, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)
    u, v, r = splats[:, 0], splats[:, 1], splats[:, 11]
    on16 = lambda x: np.mod(x, 16) == 0   # noqa: E731
    tied_x = on16(u - r) | on16(u + r + 15)
    tied_y = on16(v - r) | on16(v + r + 15)
    assert (tied_x & tied_y).sum() >= 8, (tied_x.sum(), tied_y.sum(), len(rec))
    assert on16(u - r).any() and on16(u + r + 15).any() and on16(v - r).any() and on16(v + r + 15).any()
    check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)


# ---- batches and the early stop of the tile loop --------------------------------------------------------------------
def layers(n, opaque_at=(), w=16, h=16, seed=50):
    """n broad gaussians over a w x h viewport, front to back by index (depth 1 + i / n); those at `opaque_at`
    opaque (0.95), the others faint (0.01: 769 of them leave T = 0.99^769 > 1e-4)."""
    rng = np.random.default_rng(seed)
    i = np.arange(n)
    pos = np.c_[rng.uniform(-0.05, 0.05, (n, 2)), 3.0 - (1.0 + i / n)]
    op = np.full(n, 0.01)
    op[list(opaque_at)] = 0.95
    return ref96(pos, np.full((n, 3), 3.0), random_quats(rng, n), rng.uniform(0, 1, (n, 3)), op)


@pytest.mark.parametrize("n", [255, 256, 257, 3 * 256 + 1])
def test_runs_around_the_batch_size(gpu_ctx, n):
    V, P = CLAMP_V, perspective(60.0, 1.0, 0.1, 100.0)
    f32, _, pairs = check_against_oracle(gpu_ctx, layers(n), _abi.VIEW_PLY, V, P, EYE, 16, 16, near=0.2)
    assert pairs == n   # one tile: every gaussian is one pair of it
    assert np.all(f32[..., 3] < 1 - 1e-4)   # nothing stopped: every batch ran


@pytest.mark.parametrize("at", [10, 255, 300, 700])
def test_early_stop_in_first_middle_and_last_batch(gpu_ctx, at):
    V, P = CLAMP_V, perspective(60.0, 1.0, 0.1, 100.0)
    rec = layers(769, opaque_at=range(at, at + 6))
    f32, _, _ = check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, 16, 16, near=0.2)
    assert np.all(f32[..., 3] > 0.99)   # every pixel stopped within the opaque run


def test_one_tile_stops_its_neighbour_does_not(gpu_ctx):
    """32 x 16: three layers of opaque pinpoint gaussians on every pixel of the left tile, in front of 600 faint
    broad ones over both tiles.  Every pixel of the left tile stops at its second layer (T = 0.01 * 0.01 < 1e-4), so the
    tile stops within its fourth batch; the right one runs all its pairs."""
    w, h = 32, 16
    V, P = CLAMP_V, perspective(60.0, w / h, 0.1, 100.0)
    P00, P11 = float(P.ravel()[0]), float(P.ravel()[5])
    ys, xs = np.mgrid[0:16, 0:16].reshape(2, -1).astype(np.float64)
    front = []
    for layer in range(3):
        d = 2.0 + 0.01 * layer
        pos = np.c_[((2 * xs + 1) / w - 1) * d / P00, ((2 * ys + 1) / h - 1) * d / P11, np.full(256, 4.0 - d)]
        front.append(ref96(pos, np.full((256, 3), 1e-4), np.tile([1.0, 0, 0, 0], (256, 1)), np.full((256, 3), 0.5), np.full(256, 1.0)))
    back = layers(600, w=w, h=h)
    back[:, 0] *= 4
    back[:, 2] -= 1.0   # behind every front layer
    rec = np.concatenate(front + [back])
    f32, _, pairs = check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)
    alone, *_ = gs3d.render(np.concatenate(front), _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)
    assert pairs > 2 * 768
    assert f32[:, :16].tobytes() == alone[:, :16].tobytes()   # the left tile stopped before any back gaussian
    assert np.all(f32[:, 17:, 3] > alone[:, 17:, 3])           # the right one composited them


# ---- counts ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257])
def test_survivor_counts(gpu_ctx, n):
    w, h = 80, 48
    V, P = camera(w, h)
    check_against_oracle(gpu_ctx, image_scene(max(n, 1), 60)[:n], _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)


def test_survivors_past_1024_scan_blocks(gpu_ctx):
    """2^20 + 1 survivors: 2 049 blocks of 512 items, so the scan of the block sums carries across three passes of
    its 1 024 threads.  One run."""
    w, h = 256, 256
    V, P = camera(w, h)
    n = (1 << 20) + 1
    rec = image_scene(n, 61)
    rec[:, 0:3] *= 0.4
    rec[:, 8:11] = 0.004
    _, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)
    assert alive == n
    check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)


def test_mostly_culled(gpu_ctx):
    """Nine in ten records behind the camera: their keys (0xFFFFFFFF) sort past every survivor."""
    w, h = 96, 64
    V, P = camera(w, h)
    rec = image_scene(5000, 62)
    rec[np.arange(5000) % 10 != 3, 2] += 10.0
    _, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)
    assert 400 <= alive <= 600
    check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)


@pytest.mark.parametrize("d", [0, 1, 128, 1000, 3000, 5000])
def test_d_count(gpu_ctx, d):
    """d_count limits n to min(count, *d_count): 0, inside the first 256-thread block, mid-block, the count, past it."""
    import torch
    w, h = 96, 64
    V, P = camera(w, h)
    rec = image_scene(3000, 63)
    dc = torch.tensor([d], dtype=torch.int64, device="cuda")
    f32, u8, drawn, pairs = render_guarded(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, max_pairs=(1 << 30) - 1, d_count=dc)
    wf, wu, wdrawn, wpairs = gs3d.render(rec[:min(d, len(rec))], _abi.VIEW_PLY, V, P, EYE, w, h)
    assert f32.tobytes() == wf.tobytes() and u8.tobytes() == wu.tobytes() and (drawn, pairs) == (wdrawn, wpairs)


# ---- the pair budget at exact boundaries ------------------------------------------------------------------------------
def test_pair_budget_boundaries(gpu_ctx):
    w, h = 128, 96
    V, P = camera(w, h)
    rec = image_scene(2000, 64)
    rec[np.arange(2000) % 7 == 0, 2] += 10.0   # culled records: they sort last and never count
    splats, keys, alive = gs3d.preprocess(rec, _abi.VIEW_PLY, V, P, EYE, w, h, near=0.2)
    order = np.lexsort((np.arange(len(rec)), keys))[:alive]
    rx, ry = splats[order, 9].view(np.uint32), splats[order, 10].view(np.uint32)
    counts = ((rx >> 16) - (rx & 0xFFFF)).astype(np.int64) * ((ry >> 16) - (ry & 0xFFFF))
    incl = np.cumsum(counts)
    total = int(incl[-1])
    # a prefix ending on an item with no pair: counts are >= 1 for survivors, so the zero-pair items are the culled
    # ones past the survivors; a prefix ending at the survivors' end is the total
    k = int(np.searchsorted(incl, total // 2))
    for budget in sorted({0, 1, int(incl[k]), int(incl[k]) - 1, total - 1, total}):
        f32, u8, drawn, pairs = render_guarded(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, max_pairs=budget)
        wf, wu, wdrawn, wpairs = gs3d.render(rec, _abi.VIEW_PLY, V, P, EYE, w, h, max_pairs=budget)
        assert pairs == wpairs == total
        assert drawn == wdrawn == int(np.searchsorted(incl, budget, side="right")), (budget, drawn, wdrawn)
        assert f32.tobytes() == wf.tobytes() and u8.tobytes() == wu.tobytes()


# ---- SH from a file -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("degree", [1, 2, 3])
def test_sh_from_a_ply_file(gpu_ctx, tmp_path, degree):
    """A .ply with f_rest of `degree`, read by m2s_ply_read_sh; rendered at every sh_degree <= degree against the
    checker on the decoded records and coefficients."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden_ply_load import STANDARD, ply, vertex_rows
    rng = np.random.default_rng(70 + degree)
    n = 3000
    K = (degree + 1) ** 2 - 1
    props = [("float", k) for k in STANDARD] + [("float", f"f_rest_{k}") for k in range(3 * K)]
    props = [props[i] for i in rng.permutation(len(props))]

    def fill(name, v):
        if name in ("x", "y", "z"):
            return v * 0.5
        return v * 0.4 if name.startswith("f_rest") else v

    path = str(tmp_path / "sh.ply")
    with open(path, "wb") as f:
        f.write(ply([("vertex", n, props, vertex_rows(rng, props, n, fill))]))
    records, sh, count, _, deg = gpu_ctx.ply_read_sh(path)
    assert count == n and deg == degree
    rec = records.cpu().numpy().view(np.float32).reshape(n, 24)
    shh = sh.cpu().numpy()
    w, h = 120, 80
    V, P = camera(w, h, "oblique")
    for sd in range(degree + 1):
        f32, _, pairs = check_against_oracle(gpu_ctx, rec, _abi.VIEW_PLY, V, P, EYE, w, h, sh=shh, buffer_degree=degree, sh_degree=sd,
                                             near=0.2)
        assert pairs > 0


# ---- export round trip, within the codec's roundings -------------------------------------------------------------------
def test_export_round_trip_within_codec_bound(gpu_ctx, tmp_path):
    from mesh2splat_b200 import api
    w, h = 128, 96
    V, P = camera(w, h)
    rec = image_scene(1500, 12)
    rec[:, 4:7] = np.clip(rec[:, 4:7], 0.02, 0.98)
    a = gpu_ctx.render_3dgs(_dev(rec), len(rec), _abi.LAYOUT_REF96, V, P, EYE, w, h, std_dev=1.0)[0]
    path = str(tmp_path / "rt.ply")
    api.ply_write(path, rec, 0, 1.0)
    loaded, n, _ = gpu_ctx.ply_read(path)
    back = loaded.cpu().numpy().view(np.float32).reshape(n, 24)
    # the codec's roundings, record by record
    s = rec[:, 8:11].astype(np.float64)
    e_s = 2.0 ** -23 * (2 + np.abs(np.log(s)))
    e_o, e_c, e_q = 2.0 ** -20, 2.0 ** -22, 2.0 ** -21
    assert np.all(np.abs(back[:, 8:11] / s - 1) <= e_s)
    assert np.all(np.abs(back[:, 7] / rec[:, 7].astype(np.float64) - 1) <= e_o)
    assert np.all(np.abs(back[:, 4:7] - rec[:, 4:7].astype(np.float64)) <= e_c)
    assert np.array_equal(back[:, 0:3], rec[:, 0:3])
    assert np.all(np.abs(back[:, 16:20] - rec[:, 16:20]) <= e_q)
    b, _, _ = check_against_oracle(gpu_ctx, back, _abi.VIEW_PLY, V, P, EYE, w, h)
    fa = a["rgba32f"].cpu().numpy().reshape(h, w, 4).astype(np.float64)
    # per pixel: the codec's term and twice the fp32 term of test_3dgs_host_edges
    dec = gs3d.decode(rec, _abi.VIEW_PLY)
    pre, *_ = gs3d.graphdeco_forward(*dec, V, P, w, h, 0.2, render=False)
    ca, cb, cc = pre["cov"].T
    lam = 0.5 * (ca + cc) + np.sqrt(0.25 * (ca - cc) ** 2 + cb * cb)
    kappa = pre["mag"] / ((ca * cc - cb * cb) / lam)
    mean_err = 16 * U * (np.abs(pre["u"]) + np.abs(pre["v"]) + w + h)
    info, img, margin, rect_dep = gs3d.graphdeco_forward(*dec, V, P, w, h, 0.2, power_err=(2 * 64 * U + 2 * e_q) * kappa + 2 * e_s.max(1),
                                                         mean_err=2 * mean_err)
    cover = img[..., 3]
    cmax = max(1.0, float(rec[:, 4:7].max()))
    bound = cmax * (info["dalpha"] + (8 * U + e_o) * cover) + e_c * cover + 8 * U * info["blended"] + 4 * U
    clean = (margin > 2.0 ** -16) & ~rect_dep
    assert 1.0 - clean.mean() < 0.1, 1.0 - clean.mean()
    ratio = (np.abs(fa - b) / bound[..., None])[clean]
    assert ratio.max() <= 1.0, ratio.max()
    assert ratio.max() >= 1e-2, ratio.max()   # the bound is within 100 x of what the round trip moves
