"""The direct path's cutting of a set-up pass into groups and shared pieces (raster kernel, PACKED56, paired launches).

A paired pass lists the direct fragments of its two 16-triangle units as one list, cut into groups of 32 from fragment 0
across the boundary of the units.  The owner shades the first 192 fragments; the rest is posted to the CTA's help queue
in pieces of 64.  Each case converts a scene on the paired direct route and again with the direct path off
(m2s_debug_set_direct_off: every small triangle goes to the fragment kernel), and the two results must be the same
multiset of records, bit for bit, with the same count.  The scenes are rows of tiny triangles whose fragment counts are
chosen per triangle, so that each case has the pass shapes it names; the fragment-kernel route's keys confirm them.
All marked gpu.
"""
from __future__ import annotations

from contextlib import contextmanager

import numpy as np
import pytest

from mesh2splat_b200 import _abi, _lib, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56, STRIDES
from util import GuardedDevice

pytestmark = pytest.mark.gpu

L = LAYOUT_PACKED56
R = 512
UNIT = 16   # triangles per unit on a paired launch


@contextmanager
def direct_off():
    _lib.lib().m2s_debug_set_direct_off(1)
    try:
        yield
    finally:
        _lib.lib().m2s_debug_set_direct_off(0)


def _warps(ctx):
    ds = ctx.upload(synth.unit_quad())
    w = int(ctx.convert_plan(ds, 64, L).raster_warps)
    ds.free()
    return w


def row_scene(frags: np.ndarray, big: np.ndarray | None = None) -> _abi.Scene:
    """Triangle t covers the centres of frags[t] consecutive pixels of one row (0 <= frags[t] <= 32: a box of at most
    2 frags[t] x 1 pixels, a small triangle); where big[t], a right triangle of 20 x 20 pixels instead (a larger triangle,
    counted in row blocks for the fragment kernel).  z = 0, uv = xy, one textured primitive over the unit square."""
    n = len(frags)
    t = np.arange(n)
    i0 = (t % 7) * 70 + 3 + (t // 7) % 5          # the box stays inside [0, R)
    j = (t // 7) % (R - 40) + 8
    k = frags.astype(np.float64)
    # apex above the left end, base from (i0 + 0.1) to (i0 + 2k - 0.1): the top edge crosses the centre line at i0 + k
    x = np.stack([i0 + 0.1, i0 + 2 * k - 0.1, i0 + 0.1], axis=1)
    y = np.stack([j + 0.25, j + 0.25, j + 0.75], axis=1)
    empty = frags == 0                             # a box without a pixel centre
    x[empty] = np.stack([i0 + 0.1, i0 + 0.4, i0 + 0.1], axis=1)[empty]
    y[empty] = np.stack([j + 0.1, j + 0.1, j + 0.4], axis=1)[empty]
    if big is not None:
        x[big] = np.stack([i0 + 0.0, i0 + 20.0, i0 + 0.0], axis=1)[big]
        y[big] = np.stack([j + 0.0, j + 0.0, j + 20.0], axis=1)[big]
    v = np.zeros((n, 3, 12), np.float32)
    v[:, :, 0] = x / R
    v[:, :, 1] = y / R
    v[:, :, 5] = 1.0                               # normal (0, 0, 1)
    v[:, :, 6] = 1.0; v[:, :, 9] = 1.0             # tangent (1, 0, 0, 1)
    v[:, :, 10] = v[:, :, 0]; v[:, :, 11] = v[:, :, 1]
    prim = _abi.Primitive(0, n, (0.9, 1.0, 0.8, 1.0), 0, -1, -1, bbox_min=(0.0, 0.0, 0.0), bbox_max=(1.0, 1.0, 0.0))
    return _abi.Scene(v.reshape(n, 36), [prim], synth.make_material_textures(256, 6)[:1])


def pass_scene(ctx, unit0: np.ndarray, unit1: np.ndarray, late: int = 64, big0: bool = False) -> _abi.Scene:
    """Every paired pass of the launch: unit 0 with the per-triangle fragment counts `unit0`, unit 1 with `unit1`
    (16 each); then `late` units of unit-0 shape, claimed one at a time.  big0: unit 0's triangle 0 is a larger one."""
    w = _warps(ctx)
    pair = np.concatenate([unit0, unit1])
    frags = np.concatenate([np.tile(pair, w), np.tile(unit0, late)])
    big = None
    if big0:
        big = np.zeros(len(frags), bool)
        big[np.arange(len(frags)) % (2 * UNIT) == 0] = True
        big[2 * UNIT * w:] = False
    return row_scene(frags, big)


def rows_sorted(rec: np.ndarray) -> np.ndarray:
    """The records as a multiset: rows of 7 u64 words in lexicographic order."""
    words = np.ascontiguousarray(rec).view(np.uint8).reshape(len(rec), STRIDES[L]).view(np.uint64)
    return words[np.lexsort(words.T[::-1])]


def convert_both(ctx, ds, capacity, want_keys):
    plan = ctx.convert_plan(ds, R, L, capacity=capacity, flags=FLAG_UNCAPPED)
    assert plan.multi_round and plan.direct_ok and plan.claim_late and plan.pair_first
    got = ctx.convert(ds, R, L, flags=FLAG_UNCAPPED, capacity=capacity, want_keys=want_keys)
    with direct_off():
        assert not ctx.convert_plan(ds, R, L, capacity=capacity, flags=FLAG_UNCAPPED).direct_ok
        ref = ctx.convert(ds, R, L, flags=FLAG_UNCAPPED, capacity=capacity, want_keys=True)
    assert got.total == ref.total and got.written == ref.written
    return got, ref


def assert_same(got, ref, want_keys):
    a, b = got.numpy(), ref.numpy()
    if want_keys:
        ak, bk = got.keys_numpy(), ref.keys_numpy()
        oa, ob = np.argsort(ak, kind="stable"), np.argsort(bk, kind="stable")
        assert np.array_equal(ak[oa], bk[ob]), "the direct path's fragment identities differ"
        assert a[oa].tobytes() == b[ob].tobytes(), "direct path and fragment-kernel path disagree"
    else:
        assert np.array_equal(rows_sorted(a), rows_sorted(b)), "direct path and fragment-kernel path disagree"


def unit_weights(ref, n_units):
    tri = (ref.keys_numpy() >> np.uint64(24)).astype(np.int64)
    return np.bincount(tri // UNIT, minlength=n_units)


def check_scene(ctx, s, shape=None, want_keys=True):
    """shape: (fragments of unit 0, of unit 1, passes) that every paired pass must have (the fragment kernel's keys)."""
    ds = ctx.upload(s)
    got, ref = convert_both(ctx, ds, 8 * R * R, want_keys)
    assert got.total > 0
    if shape is not None:
        wt = unit_weights(ref, (s.triangle_count + UNIT - 1) // UNIT)
        n = 2 * shape[2]
        assert np.all(wt[0:n:2] == shape[0]) and np.all(wt[1:n:2] == shape[1]), wt[:8]
    assert_same(got, ref, want_keys)
    ds.free()


@pytest.mark.parametrize("want_keys", [True, False], ids=["keys", "no_keys"])
def test_bench_scene_direct_groups(gpu_ctx, want_keys):
    """The benchmark's scene (helmet stand-in, R = 512): every fragment goes through the direct path."""
    check_scene(gpu_ctx, synth.helmet_standin(2048), want_keys=want_keys)


U0_MID = np.array([5] * 8 + [0] * 8)       # 40 fragments
U1_MID = np.array([17] * 4 + [16] * 12)    # 260


def test_unit0_list_ends_mid_group(gpu_ctx):
    """Unit 0 lists 40 fragments, unit 1 260: the group of fragments [32, 64) holds 8 of unit 0's and 24 of unit 1's,
    and the pieces [192, 256) and [256, 300) are posted."""
    w = _warps(gpu_ctx)
    check_scene(gpu_ctx, pass_scene(gpu_ctx, U0_MID, U1_MID), (40, 260, w))


def test_only_unit1_direct(gpu_ctx):
    """Unit 0 has no small-triangle fragment (one larger triangle, counted for the fragment kernel, and empty ones):
    the pass's list is unit 1's alone."""
    u0 = np.zeros(UNIT, int)
    u1 = np.array([19] * 10 + [18] * 6)   # 298: two posted pieces
    w = _warps(gpu_ctx)
    s = pass_scene(gpu_ctx, u0, u1, big0=True)
    ds = gpu_ctx.upload(s)
    got, ref = convert_both(gpu_ctx, ds, 8 * R * R, True)
    wt = unit_weights(ref, (s.triangle_count + UNIT - 1) // UNIT)
    assert np.all(wt[1:2 * w:2] == 298) and np.all(wt[0:2 * w:2] > 0)   # unit 0: the larger triangle's fragments only
    assert_same(got, ref, True)
    ds.free()


def test_only_unit0_direct(gpu_ctx):
    """Unit 1 emits nothing: the pass's list is unit 0's alone (two posted pieces, the last partial)."""
    u0 = np.array([19] * 12 + [18] * 4)
    u1 = np.zeros(UNIT, int)
    w = _warps(gpu_ctx)
    check_scene(gpu_ctx, pass_scene(gpu_ctx, u0, u1), (300, 0, w))


def test_queue_capacity_overflow_owner_keeps_the_rest(gpu_ctx):
    """Passes of 2 x 304 fragments: 7 posted pieces per warp, 112 per CTA of 16 warps, more than the CTA's queue holds;
    the pieces past its capacity stay with their owners."""
    u0 = np.array([19] * UNIT)
    w = _warps(gpu_ctx)
    check_scene(gpu_ctx, pass_scene(gpu_ctx, u0, u0), (304, 304, w))


def test_capacity_cut_inside_straddling_group_and_shared_piece(gpu_ctx):
    """Every pass lists 300 fragments (unit 0: 40, unit 1: 260); each reservation is one pass's 300 (the late units
    reserve after the pairs), so a cap of
    k * 300 + 50 falls inside the group [32, 64) that straddles the units, and k * 300 + 220 inside the posted piece
    [192, 256).  The records stored are a subset of the uncapped result, bit for bit, and nothing is written past the cap."""
    import torch
    s = pass_scene(gpu_ctx, U0_MID, U1_MID)
    ds = gpu_ctx.upload(s)
    _, ref = convert_both(gpu_ctx, ds, 8 * R * R, True)
    rk = ref.keys_numpy()
    order = np.argsort(rk)
    rk, rrec = rk[order], ref.numpy()[order]
    total = int(ref.total)
    k = total // 300 // 3
    for cap in (k * 300 + 50, k * 300 + 220):
        out = GuardedDevice(cap, STRIDES[L], what="records")
        keys = GuardedDevice(cap, 8, torch.int64, what="keys")
        o = gpu_ctx.convert(ds, R, L, flags=FLAG_UNCAPPED, capacity=cap, out=out.view, keys=keys.view, want_keys=True)
        out.check(o.written)
        keys.check(o.written)
        assert o.total == total and o.written == cap and o.overflow
        kk = o.keys_numpy()
        assert len(np.unique(kk)) == len(kk), f"cap {cap}: duplicate fragment identities"
        pos = np.minimum(np.searchsorted(rk, kk), len(rk) - 1)
        assert np.array_equal(rk[pos], kk), "a stored key is not a fragment of the uncapped result"
        assert o.numpy().tobytes() == rrec[pos].tobytes(), f"cap {cap}: records differ from the fragment kernel's"
    ds.free()
