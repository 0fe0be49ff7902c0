"""The conversion's scheduler state alternates between two sets by launch: launch k claims units and counts fragments and
work items in set k & 1, and its fragment kernel zeroes the other set for launch k + 1.  Here launches of every route
run back to back on one context, twice over, so that each route runs on both sets and after every other route.  Each
launch's count and its records (sorted by their fragment keys, or as a multiset where a route has no keys) must equal
those of the same launch on a fresh context, bit for bit.  All marked gpu.
"""
from __future__ import annotations

from contextlib import contextmanager

import numpy as np
import pytest

from mesh2splat_b200 import _abi, _lib, synth
from mesh2splat_b200._abi import FLAG_UNCAPPED, LAYOUT_PACKED56, LAYOUT_PLY_STANDARD, LAYOUT_REF96, STRIDES
from mesh2splat_b200.api import Context

pytestmark = pytest.mark.gpu

R = 512


@pytest.fixture(scope="module")
def scene():
    return synth.helmet_standin(256)   # 70 074 triangles: more units than raster warps, the direct path's premise


@contextmanager
def direct_off():
    _lib.lib().m2s_debug_set_direct_off(1)
    try:
        yield
    finally:
        _lib.lib().m2s_debug_set_direct_off(0)


def keyed(out):
    """(total, keys in ascending order, the records in that order)"""
    k = out.keys_numpy()
    o = np.argsort(k, kind="stable")
    return out.total, k[o].tobytes(), out.numpy()[o].tobytes()


def multiset(raw: np.ndarray, n: int, stride: int) -> bytes:
    rows = np.ascontiguousarray(raw[: n * stride]).reshape(n, stride)
    return rows[np.lexsort(rows.T[::-1])].tobytes()


def _convert(ctx, ds, layout, **kw):
    return keyed(ctx.convert(ds, R, layout, flags=FLAG_UNCAPPED, want_keys=True, **kw))


def run_direct(ctx, ds, s):
    plan = ctx.convert_plan(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED)
    assert plan.direct_ok and plan.multi_round
    return _convert(ctx, ds, LAYOUT_PACKED56)


def run_direct_off(ctx, ds, s):
    with direct_off():
        assert not ctx.convert_plan(ds, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED).direct_ok
        return _convert(ctx, ds, LAYOUT_PACKED56)


def run_ref96(ctx, ds, s):
    return _convert(ctx, ds, LAYOUT_REF96)


def run_ply(ctx, ds, s):
    return _convert(ctx, ds, LAYOUT_PLY_STANDARD)


def run_timed(ctx, ds, s):
    """m2s_convert_timed returns no count: every record it wrote (and nothing past them) stands for it"""
    import torch
    stride = STRIDES[LAYOUT_PACKED56]
    cap = 6 * R * R
    out = torch.full((cap * stride,), 0xA5, dtype=torch.uint8, device="cuda")
    p = _abi.make_params(R, LAYOUT_PACKED56, 0.65, 0, FLAG_UNCAPPED)
    ctx.convert_timed(ds, p, out, cap)
    raw = out.cpu().numpy()
    n = cap - int(np.argmax(np.any(raw.reshape(cap, stride)[::-1] != 0xA5, axis=1)))   # the last record written, + 1
    return n, multiset(raw, n, stride)


def run_capacity_then_good(ctx, ds, s):
    """a launch whose records overflow its capacity (M2S_E_CAPACITY, the count still complete), then a good one"""
    cut = ctx.convert(ds, R, LAYOUT_PACKED56, max_gaussians=1000, capacity=1000)
    assert cut.overflow and cut.written == 1000 and cut.total > 1000
    return cut.total, _convert(ctx, ds, LAYOUT_PACKED56)


def run_host(ctx, ds, s):
    rec, keys, res = ctx.convert_host(s, R, LAYOUT_PACKED56, flags=FLAG_UNCAPPED, want_keys=True)
    o = np.argsort(keys, kind="stable")
    return int(res.total), keys[o].tobytes(), np.ascontiguousarray(rec)[o].tobytes()


ROUTES = [run_direct, run_direct_off, run_ref96, run_ply, run_timed, run_capacity_then_good, run_host]


def test_mixed_routes_alternate_the_scheduler_sets(scene):
    want = {}
    for f in ROUTES:   # each launch on a fresh context
        with Context(0) as fresh:
            ds = fresh.upload(scene)
            want[f.__name__] = f(fresh, ds, scene)
            ds.free()
    with Context(0) as ctx:
        ds = ctx.upload(scene)
        # one round is 11 launches (two for the capacity case, four chunks in m2s_convert_host), an odd number: over
        # two rounds every route runs on both sets
        for rnd in range(2):
            for f in ROUTES:
                assert f(ctx, ds, scene) == want[f.__name__], f"{f.__name__}, round {rnd}"
        ds.free()
