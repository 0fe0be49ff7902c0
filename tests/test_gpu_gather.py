"""The fused multi-GPU gather (m2s_convert_gather_enqueue) on ONE GPU, with W ranks emulated in one process.  All marked
gpu.

Each emulated rank has its own context (so its own epoch counter; every case makes fresh ones, so the epochs of its
three rounds are 1, 2, 3), its own upload of its shard (m2s_scene_upload_range, as a real rank does; the whole scene for
row bands), a guarded final buffer (util.GuardedDevice) and a zeroed exchange block of M2S_MAX_PEERS * 4 int64.
m2s_peers carries these plain device pointers, so every "peer store" is a local store and each record is written W
times, once into every final buffer.

No device wait depends on work that has not been enqueued.  The ranks run one after another, with a device synchronise
between calls.  Before rank r's call the harness writes, into rank r's exchange block, the slot {count, count epoch,
done epoch} = {c_q, e, e} of every rank q > r (not yet run), with c_q from a plain m2s_convert of q's range with the
same parameters.  The slots of the ranks q < r were written by their own kernels; the harness asserts that they hold
c_q and e before relying on them.  Rank r's own slots are written by its raster and fragment kernels, on the same stream
before the waits that read them.  So every wait is satisfied at its first load, or by an earlier kernel of the same
stream, and after each call m2s_ctx_status must be M2S_OK: no wait timed out.  Once the call has finished, the slots
pre-published in r's block go back to the previous epoch, so the slot check at the end of a round sees only what the
kernels wrote.

What one GPU cannot show is the ordering of the peer stores and flags between GPUs over NVLink: that stays with
test_gpu_multi, on boxes with at least 2 GPUs.

Checks of every round, with c_r the records rank r stores (min(generated, its cap)), n = min(sum c, capacity) and
o_r = sum_{q<r} c_q:
  - every final buffer holds the same bytes on [0, n), its guard bytes outside [0, n) are intact and no record below
    n is unwritten;
  - rank r's slice [o_r, min(o_r + c_r, capacity)) is, as a multiset of records, the plain conversion of r's range bit
    for bit, or where r's own cap or the capacity cuts it, a part of it (test_gpu_bounds pins the plain conversions
    of these scene shapes to the oracle; test_direct_path_and_queue_path_write_the_same_records shows that the direct
    path and the queue path write the same records);
  - rank r's count and done slots hold c_r and the epoch in every exchange block;
  - d_total_global == n on every rank.
The scenes are util.layered_tiling stacks as in test_gpu_bounds, and each route case asserts its premise on the launch
plan (m2s_debug_convert_plan: its fields other than direct_ok do not depend on the world size).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from functools import lru_cache

import numpy as np
import pytest

from mesh2splat_b200 import _abi, synth
from mesh2splat_b200._abi import (FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_PLY_STANDARD, LAYOUT_REF96, M2S_E_INVALID, M2S_OK,
                                  MAX_PEERS, STRIDES)
from mesh2splat_b200._lib import check, lib
from mesh2splat_b200.api import Context
from mesh2splat_b200.shard import estimate_cost, plan_shards, plan_work
from util import GUARD_BYTE, GUARD_HEAD, GuardedDevice, layered_tiling

pytestmark = pytest.mark.gpu

ROUNDS = 3
STALE = -1   # the count of a pre-published slot once the call that read it has finished


@dataclass
class Shard:
    first: int
    count: int
    row_begin: int = 0
    row_end: int = 0
    max_gaussians: int = 0   # 0: the rank's cap is the final buffers' capacity (FLAG_UNCAPPED)


@lru_cache(maxsize=None)
def _tiling(k, R, kind, n, seed=0, wide=0):
    return layered_tiling(k, R, kind, n=n, seed=seed, wide=wide)


def _small():
    """42 k sub-pixel triangles at R = 64 (7 layers): cheap, and most units are micro items."""
    return _tiling(7, 64, "delaunay", 3000, seed=5)


def _warps(ctx, layout):
    ds = ctx.upload(synth.unit_quad())
    w = int(ctx.convert_plan(ds, 64, layout).raster_warps)
    ds.free()
    return w


def _totals(scene, R, layout, shards):
    """Records each shard generates (a plain conversion of its range)."""
    with Context(0) as ctx:
        ds = ctx.upload(scene)
        t = [_convert(ctx, ds, R, layout, sh, 0, max_gaussians=0).total for sh in shards]
        ds.free()
    return t


def _convert(ctx, ds, R, layout, sh, capacity, max_gaussians=None, keys=False):
    return ctx.convert(ds, R, layout, max_gaussians=sh.max_gaussians if max_gaussians is None else max_gaussians,
                       flags=FLAG_UNCAPPED, first_triangle=sh.first, triangle_count=sh.count, capacity=capacity,
                       want_keys=keys, row_begin=sh.row_begin, row_end=sh.row_end)


def _rows(t, stride):
    """A uint8 device tensor of whole records -> (records, stride / 8) int64; the gather's strides, 96 and 56, are
    multiples of 8."""
    import torch
    return t.view(torch.int64).view(-1, stride // 8)


def assert_rows(got, want, part, what):
    """got == want as multisets of records, bit for bit; part: got is a sub-multiset of want."""
    import torch
    if not part:
        assert got.shape == want.shape, f"{what}: {got.shape[0]} records, the plain conversion has {want.shape[0]}"
    if got.shape[0] == 0:
        return
    ug, cg = torch.unique(got, dim=0, return_counts=True)
    uw, cw = torch.unique(want, dim=0, return_counts=True)
    if not part:
        assert torch.equal(ug, uw) and torch.equal(cg, cw), f"{what}: not the records of the plain conversion"
        return
    _, inv = torch.unique(torch.cat([ug, uw]), dim=0, return_inverse=True)
    have = torch.zeros(ug.shape[0] + uw.shape[0], dtype=torch.int64, device=got.device).index_add_(0, inv[ug.shape[0]:], cw)
    need = torch.zeros_like(have).index_add_(0, inv[: ug.shape[0]], cg)
    bad = int((need > have).sum())
    assert bad == 0, f"{what}: {bad} distinct records are not records of the plain conversion, or occur more often"


def _out_ptr(buf):
    """The address of a GuardedDevice's records, also when it holds none (an empty view's data_ptr() is 0)."""
    return buf.raw.data_ptr() + GUARD_HEAD


def _peers(world, rank, outs, xch):
    p = _abi.m2s_peers()
    p.world, p.rank = world, rank
    for q in range(min(world, MAX_PEERS)):
        p.out[q] = _out_ptr(outs[q])
        p.xch[q] = xch[q].data_ptr()
    return p


def run_gather(scene, R, layout, shards, gcap, whole=False, premise=None):
    """ROUNDS fused gathers of `shards` (one emulated rank each) into final buffers of `gcap` records, every round
    checked as the module docstring says.  whole: the ranks partition the scene, so the gathered records are the
    whole scene's conversion.  premise(plan, unit_weights): asserted for every rank's launch plan.  Returns the stored
    counts c of the last round."""
    import torch
    W, stride = len(shards), STRIDES[layout]
    ctxs = [Context(0) for _ in shards]
    dss = []
    try:
        for ctx, sh in zip(ctxs, shards):
            dss.append(ctx.upload_range(scene, layout, sh.first, sh.count))
        full = []   # every rank's whole range, uncapped: what its slice holds, or a part of it where a cap cuts it
        for ctx, ds, sh in zip(ctxs, dss, shards):
            t = _convert(ctx, ds, R, layout, sh, 0, max_gaussians=0).total
            o = _convert(ctx, ds, R, layout, sh, t, max_gaussians=0, keys=premise is not None)
            assert o.total == o.written == t
            full.append(o)
        if premise is not None:
            for ctx, ds, sh, o in zip(ctxs, dss, shards, full):
                plan = ctx.convert_plan(ds, R, layout, capacity=gcap, max_gaussians=sh.max_gaussians, flags=FLAG_UNCAPPED,
                                        first_triangle=sh.first, triangle_count=sh.count)
                unit = ((o.keys_numpy() >> np.uint64(24)).astype(np.int64) - sh.first) // int(plan.unit_tris)
                premise(plan, np.bincount(unit, minlength=int(plan.n_units)))
        want_whole = None
        if whole:
            ds = ctxs[0].upload(scene)
            t = ctxs[0].convert(ds, R, layout, flags=FLAG_UNCAPPED, capacity=0).total
            want_whole = _rows(ctxs[0].convert(ds, R, layout, flags=FLAG_UNCAPPED, capacity=t).data[: t * stride], stride)
            ds.free()
        outs = [GuardedDevice(gcap, stride, what=f"final buffer of rank {r}") for r in range(W)]
        xch = [torch.zeros(MAX_PEERS * 4, dtype=torch.int64, device="cuda") for _ in range(W)]
        tot = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(W)]
        peers = [_peers(W, r, outs, xch) for r in range(W)]
        params = [_abi.make_params(R, layout, 0.65, sh.max_gaussians, FLAG_UNCAPPED, sh.first, sh.count, sh.row_begin,
                                   sh.row_end) for sh in shards]
        for e in range(1, ROUNDS + 1):
            # a plain conversion of every range at the final buffers' capacity gives the count the rank stores; it also
            # runs on the gather's own contexts between two rounds
            c = [_convert(ctx, ds, R, layout, sh, gcap).written for ctx, ds, sh in zip(ctxs, dss, shards)]
            for o in outs:
                o.raw.fill_(GUARD_BYTE)
            for t in tot:
                t.fill_(-1)
            torch.cuda.synchronize()
            for r in range(W):
                slots = xch[r].view(MAX_PEERS, 4)
                assert slots[:r, :3].cpu().tolist() == [[c[q], e, e] for q in range(r)], \
                    f"round {e}: the earlier ranks' slots in rank {r}'s block"
                if r + 1 < W:
                    slots[r + 1: W, :3] = torch.tensor([[c[q], e, e] for q in range(r + 1, W)], dtype=torch.int64, device="cuda")
                torch.cuda.synchronize()
                check(lib().m2s_convert_gather_enqueue(ctxs[r].handle, dss[r].handle, C.byref(params[r]), C.byref(peers[r]),
                                                       gcap, tot[r].data_ptr(), None))
                torch.cuda.synchronize()
                assert lib().m2s_ctx_status(ctxs[r].handle) == M2S_OK, f"round {e}, rank {r}: a gather wait timed out"
                if r + 1 < W:
                    slots[r + 1: W, :3] = torch.tensor([STALE, e - 1, e - 1], dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            n = min(sum(c), gcap)
            for b in range(W):
                got = xch[b].view(MAX_PEERS, 4)[:, :3].cpu().tolist()
                assert got[:W] == [[c[q], e, e] for q in range(W)], f"round {e}: rank {b}'s exchange block {got[:W]}, counts {c}"
                assert got[W:] == [[0, 0, 0]] * (MAX_PEERS - W), f"round {e}: a slot past the world in rank {b}'s block"
            for r in range(W):
                assert int(tot[r].item()) == n, (f"round {e}, rank {r}: d_total_global {int(tot[r].item())}, but the final "
                                                 f"buffer holds {n} records (stored counts {c}, capacity {gcap})")
                outs[r].check(n)
                if r:
                    assert torch.equal(outs[r].view[: n * stride], outs[0].view[: n * stride]), \
                        f"round {e}: the final buffers of ranks 0 and {r} differ"
            o_r = 0
            for r in range(W):
                lo, hi = min(o_r, gcap), min(o_r + c[r], gcap)
                assert_rows(_rows(outs[0].view[lo * stride: hi * stride], stride),
                            _rows(full[r].data[: full[r].total * stride], stride), hi - lo < full[r].total,
                            f"round {e}, rank {r}'s records [{lo}, {hi}) of the final buffer")
                o_r += c[r]
            if want_whole is not None:
                assert n == want_whole.shape[0], (f"round {e}: {n} records gathered, the whole scene converts to "
                                                  f"{want_whole.shape[0]}: the ranks' ranges do not partition the scene "
                                                  f"(stored counts {c})")
                assert_rows(_rows(outs[0].view[: n * stride], stride), want_whole, False, f"round {e}: the gathered records")
            for r, sh in enumerate(shards):
                if sh.count == 0:
                    assert c[r] == 0, f"rank {r}: the empty range ({sh.first}, 0) stores {c[r]} records"
        return c
    finally:
        for ds in dss:
            ds.free()
        for ctx in ctxs:
            ctx.close()


def _shards(T, world):
    return [Shard(f, n) for f, n in plan_shards(T, world)]


# ---- the routes of the fragment kernel's output ------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3])
def test_route_micro_items(gpu_ctx, world):
    """REF96, sub-pixel Delaunay tilings at R = 64: most units emit <= 32 fragments and become micro items, which take
    their own global-offset path (micro_item)."""
    s = _small()

    def premise(plan, wt):
        assert not plan.direct_ok
        assert np.count_nonzero((wt >= 1) & (wt <= 32)) >= 0.5 * plan.n_units

    run_gather(s, 64, LAYOUT_REF96, _shards(s.triangle_count, world), 7 * 64 * 64 + 64, whole=True, premise=premise)


@pytest.mark.parametrize("world", [2, 3])
def test_route_unit_items(gpu_ctx, world):
    """PACKED56 in one round (32 triangles per raster warp): every unit's small triangles are one unit item."""
    w = _warps(gpu_ctx, LAYOUT_PACKED56)
    K, R = 4, 512
    s = _tiling(K, R, "delaunay", 3 * 32 * w // (2 * K) + 64, seed=3)
    assert s.triangle_count >= world * 32 * w

    def premise(plan, wt):
        assert not plan.multi_round and not plan.direct_ok and plan.unit_tris == 32
        assert np.count_nonzero(wt > 32) >= 0.9 * len(wt)   # unit items, not micro items

    run_gather(s, R, LAYOUT_PACKED56, [Shard(r * 32 * w, 32 * w) for r in range(world)], K * R * R + 64, premise=premise)


@pytest.mark.parametrize("world", [2, 3])
def test_route_block_split_and_help_queue_items(gpu_ctx, world):
    """REF96, full-height strips at R = 512: every triangle is counted in row blocks of 32 rows; the 32-pixel-wide
    strips make blocks of more fragments than an item (split items); units of >= 2 triangles of 16 blocks each post
    to their CTA's help queue."""
    w = _warps(gpu_ctx, LAYOUT_REF96)
    K, R = 2, 512
    s = _tiling(K, R, "strips", max(300, -(-world * w // K)), wide=8)   # about 2 w triangles per rank

    def premise(plan, wt):
        assert plan.unit_tris >= 2 and not plan.direct_ok
        assert plan.item_max < 32 * 31

    run_gather(s, R, LAYOUT_REF96, _shards(s.triangle_count, world), K * R * R + 64, whole=True, premise=premise)


@pytest.mark.parametrize("world", [2, 3])
def test_route_multi_round_packed56(gpu_ctx, world):
    """PACKED56 with 65 triangles per raster warp (three rounds): on one GPU the raster kernel shades these light units
    itself (the plan's direct_ok), but the gather turns the direct path off, so only here are a multi-round launch's
    units queued for the fragment kernel."""
    w = _warps(gpu_ctx, LAYOUT_PACKED56)
    K, R, per = 2, 512, 65 * w
    s = _tiling(K, R, "delaunay", 3 * per // (2 * K) + 64, seed=3)
    assert s.triangle_count >= world * per

    def premise(plan, wt):
        assert plan.multi_round and plan.direct_ok   # the one-GPU plan
        assert np.count_nonzero((wt >= 1) & (wt <= plan.direct_max)) >= 0.9 * plan.n_units

    run_gather(s, R, LAYOUT_PACKED56, [Shard(r * per, per) for r in range(world)], K * R * R + 64, premise=premise)


@pytest.mark.parametrize("layout", [LAYOUT_REF96, LAYOUT_PACKED56], ids=["ref96", "packed56"])
def test_world_8(gpu_ctx, layout):
    """M2S_MAX_PEERS ranks: the raster kernel publishes its count with all 8 lanes, and every span is written to 8
    destinations in rotated order."""
    s = _small()
    run_gather(s, 64, layout, _shards(s.triangle_count, 8), 7 * 64 * 64 + 64, whole=True)


# ---- caps ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", [LAYOUT_PACKED56, LAYOUT_REF96], ids=["packed56", "ref96"])
def test_a_ranks_own_cap_cuts_its_slice(gpu_ctx, layout):
    """max_gaussians < t_0 on rank 0: it stores c_0 = 17 mod 32 records (odd: the later ranks' PACKED56 spans start 8
    bytes into a 16-byte line), and the later ranks' records start at c_0, not at the t_0 rank 0 generated."""
    s = _small()
    shards = _shards(s.triangle_count, 3)
    t0 = _totals(s, 64, layout, shards[:1])[0]
    shards[0].max_gaussians = t0 // 2 - (t0 // 2) % 32 + 17
    c = run_gather(s, 64, layout, shards, 7 * 64 * 64 + 64)
    assert c[0] == shards[0].max_gaussians < t0 and c[0] % 2 == 1


CUTS = ["zero", "inside_rank0", "at_o1", "inside_last", "sum_minus_1", "sum", "sum_plus_1"]


@pytest.mark.parametrize("where", CUTS)
@pytest.mark.parametrize("layout", [LAYOUT_PACKED56, LAYOUT_REF96], ids=["packed56", "ref96"])
def test_cut_at_the_final_buffers_capacity(gpu_ctx, layout, where):
    """The final buffers' capacity (which is also every rank's cap here) at 0, inside rank 0's records (17 mod 32),
    exactly where rank 1's start, inside the last rank's records, and at sum c - 1, sum c, sum c + 1.  Every span is
    clipped there, and d_total_global is what the buffers hold, not the sum of the ranks' counts."""
    s = _small()
    shards = _shards(s.triangle_count, 3)
    t = _totals(s, 64, layout, shards)
    S, last = sum(t), t[-1] // 2 - (t[-1] // 2) % 32 + 17
    gcap = {"zero": 0, "inside_rank0": t[0] // 2 - (t[0] // 2) % 32 + 17, "at_o1": t[0], "inside_last": S - t[-1] + last,
            "sum_minus_1": S - 1, "sum": S, "sum_plus_1": S + 1}[where]
    assert max(t) <= gcap or where in ("zero", "inside_rank0", "at_o1")
    c = run_gather(s, 64, layout, shards, gcap)
    assert c == [min(x, gcap) for x in t]
    n = min(sum(c), gcap)
    assert n == {"zero": 0, "inside_rank0": gcap, "at_o1": t[0], "inside_last": gcap, "sum_minus_1": S - 1,
                 "sum": S, "sum_plus_1": S}[where]
    if where == "inside_last":
        assert S - t[-1] < gcap < S


# ---- plans ----------------------------------------------------------------------------------------------------------
def test_row_bands(gpu_ctx):
    """plan_work's row-band mode: the unit quad on 3 ranks at R = 300, every rank converts both triangles and a band
    of 100 rows.  (Not compared with the whole grid's conversion bit for bit: PACKED56 interpolates from planes based
    at the triangle's box origin, which the band moves, so the last bits of a record may differ.  test_multi_rank
    shows with the oracle that the bands partition the grid's fragments.)"""
    s, R = synth.unit_quad(), 300
    plan = plan_work(s.triangle_count, 3, R, estimate_cost(s.triangles, s.primitives[0].bbox_min, s.primitives[0].bbox_max, R))
    assert [p[:2] for p in plan] == [(0, 2)] * 3 and [p[2:] for p in plan] == [(0, 100), (100, 200), (200, 300)]
    c = run_gather(s, R, LAYOUT_PACKED56, [Shard(*p) for p in plan], R * R + 64)
    assert c == [100 * R] * 3


def test_empty_shards_plan_work(gpu_ctx):
    """plan_work with its cost: the 2-triangle unit quad on 4 ranks at R = 2 (fewer rows than ranks, so no row bands)
    leaves two ranks without triangles.  Their range must be (2, 0), after the ranks with triangles: (1, 0) would mean
    "triangle 1 to the end" and convert triangle 1 twice.  An empty rank stores no records but still publishes its
    count and flags."""
    s, R = synth.unit_quad(), 2
    plan = plan_work(s.triangle_count, 4, R, estimate_cost(s.triangles, s.primitives[0].bbox_min, s.primitives[0].bbox_max, R))
    assert sorted(p[1] for p in plan) == [0, 0, 1, 1]
    c = run_gather(s, R, LAYOUT_PACKED56, [Shard(*p) for p in plan], 2 * R * R + 64, whole=True)
    assert sum(c) == R * R
    assert plan == [(0, 1, 0, 0), (1, 1, 0, 0), (2, 0, 0, 0), (2, 0, 0, 0)]
    ds = gpu_ctx.upload_range(s, LAYOUT_PACKED56, s.triangle_count, 0)
    assert ds.h2d_bytes() == 0
    ds.free()


def test_empty_shards_plan_shards(gpu_ctx):
    """plan_shards without a cost: the unit quad on 3 ranks leaves one rank without triangles, as (2, 0); (0, 0)
    would convert both triangles."""
    s, R = synth.unit_quad(), 64
    shards = plan_shards(s.triangle_count, 3)
    assert sorted(n for _, n in shards) == [0, 1, 1]
    c = run_gather(s, R, LAYOUT_REF96, [Shard(*p) for p in shards], 2 * R * R + 64, whole=True)
    assert sum(c) == R * R
    assert shards == [(0, 1), (1, 1), (2, 0)]


def test_empty_rank_0(gpu_ctx):
    """An empty range on rank 0 (the C ABI takes the ranks' ranges in any order): rank 0 publishes a count of 0 and
    rank 1's records start at offset 0."""
    s, R = synth.unit_quad(), 64
    c = run_gather(s, R, LAYOUT_PACKED56, [Shard(2, 0), Shard(0, 1), Shard(1, 1)], R * R + 64, whole=True)
    assert c[0] == 0 and sum(c) == R * R


# ---- world = 1 and the argument checks -----------------------------------------------------------------------------
@pytest.mark.parametrize("cut", [False, True], ids=["uncut", "cut"])
def test_world_1_is_a_plain_conversion(gpu_ctx, cut):
    """world = 1: a plain conversion into out[0]; d_total_global is the generated total, even above the capacity."""
    import torch
    s, R, layout = _small(), 64, LAYOUT_PACKED56
    stride = STRIDES[layout]
    with Context(0) as ctx:
        ds = ctx.upload(s)
        t = ctx.convert(ds, R, layout, flags=FLAG_UNCAPPED, capacity=0).total
        want = _rows(ctx.convert(ds, R, layout, flags=FLAG_UNCAPPED, capacity=t).data[: t * stride], stride)
        gcap = t // 2 - (t // 2) % 32 + 17 if cut else t + 1
        out = GuardedDevice(gcap, stride, what="final buffer")
        xch = torch.zeros(MAX_PEERS * 4, dtype=torch.int64, device="cuda")
        p = _abi.make_params(R, layout, 0.65, 0, FLAG_UNCAPPED)
        for _ in range(ROUNDS):
            out.raw.fill_(GUARD_BYTE)
            total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            check(lib().m2s_convert_gather_enqueue(ctx.handle, ds.handle, C.byref(p), C.byref(_peers(1, 0, [out], [xch])),
                                                   gcap, total.data_ptr(), None))
            torch.cuda.synchronize()
            assert lib().m2s_ctx_status(ctx.handle) == M2S_OK
            assert int(total.item()) == t
            n = min(t, gcap)
            out.check(n)
            assert_rows(_rows(out.view[: n * stride], stride), want, cut, "the records of out[0]")
            assert int(torch.count_nonzero(xch)) == 0
        ds.free()


BAD = ["rank_not_below_world", "world_9", "ply_layout", "null_out", "null_xch", "misaligned_out"]


@pytest.mark.parametrize("bad", BAD)
def test_argument_checks(gpu_ctx, bad):
    """M2S_E_INVALID, and nothing launched: the final buffers, the exchange blocks and d_total_global stay as they were.
    (Rank 1's slot in rank 0's block is published beforehand, so that a call accepted by mistake would not wait.)"""
    import torch
    s, R = synth.unit_quad(), 16
    with Context(0) as ctx:
        ds = ctx.upload(s)
        outs = [GuardedDevice(64, STRIDES[LAYOUT_REF96], what=f"final buffer of rank {r}") for r in range(2)]
        xch = [torch.zeros(MAX_PEERS * 4, dtype=torch.int64, device="cuda") for _ in range(2)]
        xch[0][4:7] = torch.tensor([0, 1, 1], dtype=torch.int64, device="cuda")
        before = [x.clone() for x in xch]
        total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        peers = _peers(2, 0, outs, xch)
        layout = LAYOUT_PLY_STANDARD if bad == "ply_layout" else LAYOUT_REF96
        if bad == "rank_not_below_world":
            peers.rank = 2
        elif bad == "world_9":
            peers.world = MAX_PEERS + 1
        elif bad == "null_out":
            peers.out[1] = None
        elif bad == "null_xch":
            peers.xch[1] = None
        elif bad == "misaligned_out":
            peers.out[1] = _out_ptr(outs[1]) + 8
        p = _abi.make_params(R, layout, 0.65, 0, FLAG_UNCAPPED)
        torch.cuda.synchronize()
        st = lib().m2s_convert_gather_enqueue(ctx.handle, ds.handle, C.byref(p), C.byref(peers), 64, total.data_ptr(), None)
        torch.cuda.synchronize()
        assert st == M2S_E_INVALID, (bad, st)
        assert lib().m2s_ctx_status(ctx.handle) == M2S_OK
        for o in outs:
            o.check(0)
        assert all(torch.equal(x, b) for x, b in zip(xch, before)) and int(total.item()) == -1
        ds.free()
