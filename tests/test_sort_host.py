"""CPU tests of the viewer's depth sort (SURVEY 8 f-5, RadixSortPass::execute): a literal numpy restatement of the
reference's three steps (reference_depth_sort: 8 x 4-bit radix sort, gather, draw command) against numpy's stable
argsort, and the argument checks of the C entry points, which return before any CUDA call.  The key sets are shared with
tests/test_gpu_sort.py."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from mesh2splat_b200 import _abi, _lib

# bit patterns of the special depths: +0, -0, denormals, positive z, +-inf, NaNs (quiet, signalling, negative, all ones)
SPECIAL_BITS = np.array([0x00000000, 0x80000000, 0x00000001, 0x007FFFFF, 0x80000001, 0x807FFFFF, 0x3F800000, 0x42C80000,
                         0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFC00000, 0xFFFFFFFF, 0x7FFFFFFF], np.uint32)

KEY_SETS = ["uniform", "sixteen_values", "all_equal", "sorted", "reverse_sorted",
            "byte0", "byte1", "byte2", "byte3", "specials"]


def make_depths(kind: str, n: int, seed: int = 0) -> np.ndarray:
    """n float32 view depths of one key set (the prepass's gaussian_vs.z: visible gaussians have z < 0)."""
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return -rng.uniform(0.01, 100.0, n).astype(np.float32)
    if kind == "sixteen_values":   # many equal keys: stability
        vals = -rng.uniform(0.5, 50.0, 16).astype(np.float32)
        return vals[rng.integers(0, 16, n)]
    if kind == "all_equal":
        return np.full(n, -3.25, np.float32)
    if kind in ("sorted", "reverse_sorted"):
        d = -rng.uniform(0.01, 100.0, n).astype(np.float32)
        d = d[np.argsort(d.view(np.uint32), kind="stable")]
        return d if kind == "sorted" else d[::-1].copy()
    if kind.startswith("byte"):    # only byte b varies: pass b alone carries the order
        b = int(kind[4:])
        base = np.uint32(0xC1234567) & ~np.uint32(0xFF << (8 * b))
        return (base | (rng.integers(0, 256, n).astype(np.uint32) << np.uint32(8 * b))).view(np.float32)
    if kind == "specials":
        bits = -rng.uniform(0.01, 100.0, n).astype(np.float32).view(np.uint32)
        pick = rng.random(n) < 0.5
        bits[pick] = SPECIAL_BITS[rng.integers(0, len(SPECIAL_BITS), int(pick.sum()))]
        return bits.view(np.float32)
    raise ValueError(kind)


def make_quads(n: int) -> np.ndarray:
    """n distinct 96-byte quads: word j of quad i holds the bits of i * 24 + j + 1 (no two rows alike)."""
    return (np.arange(n * 24, dtype=np.uint32) + np.uint32(1)).view(np.float32).reshape(n, 24)


def expected_sort(quads: np.ndarray, depths: np.ndarray):
    order = np.argsort(np.ascontiguousarray(depths, np.float32).view(np.uint32), kind="stable").astype(np.uint32)
    return quads[order], order, np.array([6, len(depths), 0, 0, 0], np.uint32)


def reference_depth_sort(quads, depths):
    """RadixSortPass::execute restated in numpy, step for step (no np.argsort):
    radixSortPrepass.glsl   key = floatBitsToUint(depth), value = index;
    glu::RadixSort          8 LSD passes of 4 bits (RadixSort.hpp:1393-1562); each pass counts the digits per 1024-key
                            block, scans every digit's block counts in block order, adds the global digit offsets and the
                            block-local exclusive prefix (the reorder shader), and scatters keys and values;
    radixSortGather.glsl    sorted[i] = quads[value[i]]; DrawElementsIndirectCommand {6, n, 0, 0} (+ the 0 the fifth
                            word keeps from its initialisation, renderer.cpp:82-92).
    Returns (sorted [n, 24] float32, order [n] uint32, draw [5] uint32)."""
    q = np.ascontiguousarray(quads, np.float32).reshape(-1, 24)
    keys = np.ascontiguousarray(depths, np.float32).view(np.uint32).copy()
    n = len(keys)
    vals = np.arange(n, dtype=np.uint32)
    if n > 1:   # the reference skips the sort for count <= 1
        block = 1024
        nblocks = (n + block - 1) // block
        blk = np.arange(n) // block
        first = blk * block                                                                # each key's block start
        for step in range(8):
            digit = ((keys >> np.uint32(4 * step)) & np.uint32(15)).astype(np.int64)
            # counting shader: per block and digit
            counts = np.zeros((16, nblocks), np.int64)
            np.add.at(counts, (digit, blk), 1)
            glob = np.concatenate(([0], np.cumsum(counts.sum(axis=1))[:-1]))              # exclusive over the digits
            block_off = np.cumsum(counts, axis=1) - counts                                 # exclusive over the blocks, per digit
            # reorder shader: per digit, the block-local exclusive prefix of "my digit == radix"
            dst = np.empty(n, np.int64)
            for radix in range(16):
                place = digit == radix
                excl = np.cumsum(place, dtype=np.int64) - place                            # exclusive over the whole array
                local = excl - excl[first]                                                 # ... restarted at every block
                dst[place] = glob[radix] + block_off[radix, blk[place]] + local[place]
            nk = np.empty_like(keys)
            nv = np.empty_like(vals)
            nk[dst] = keys
            nv[dst] = vals
            keys, vals = nk, nv
    draw = np.array([6, n, 0, 0, 0], np.uint32)
    return q[vals].copy(), vals, draw


@pytest.mark.parametrize("kind", KEY_SETS)
@pytest.mark.parametrize("n", [0, 1, 2, 33, 1023, 1025, 100_000])
def test_reference_radix_sort_is_the_stable_sort(kind, n):
    d = make_depths(kind, n, seed=n)
    q = make_quads(n)
    got_q, got_o, got_d = reference_depth_sort(q, d)
    want_q, want_o, want_d = expected_sort(q, d)
    assert got_o.dtype == np.uint32 and np.array_equal(got_o, want_o)
    assert np.array_equal(got_q.view(np.uint32), want_q.view(np.uint32))
    assert np.array_equal(got_d, want_d)


@pytest.mark.parametrize("kind", ["uniform", "sixteen_values", "specials"])
def test_reference_radix_sort_millions(kind):
    n = 2_000_003
    d = make_depths(kind, n, seed=7)
    q = make_quads(n)
    got_q, got_o, _ = reference_depth_sort(q, d)
    want_q, want_o, _ = expected_sort(q, d)
    assert np.array_equal(got_o, want_o)
    assert np.array_equal(got_q.view(np.uint32), want_q.view(np.uint32))


def test_key_sets_have_the_intended_shape():
    n = 50_000
    assert len(np.unique(make_depths("sixteen_values", n))) == 16
    assert len(np.unique(make_depths("all_equal", n))) == 1
    s = make_depths("sorted", n).view(np.uint32)
    assert np.all(s[1:] >= s[:-1])
    for b in range(4):
        k = make_depths(f"byte{b}", n).view(np.uint32)
        other = k & ~np.uint32(0xFF << (8 * b))
        assert len(np.unique(other)) == 1 and len(np.unique((k >> np.uint32(8 * b)) & np.uint32(255))) == 256
    sp = make_depths("specials", n).view(np.uint32)
    assert set(SPECIAL_BITS.tolist()) <= set(np.unique(sp).tolist())


def test_depth_sort_entry_points_reject_bad_arguments_without_a_gpu():
    """m2s_depth_sort / m2s_depth_sort_enqueue return M2S_E_INVALID before any CUDA call: NULL context, NULL buffers with
    count > 0, quad buffers not 16-byte aligned, count >= 2^30.  The context stands in as an opaque non-NULL pointer: the
    checks never dereference it."""
    L = _lib.lib()
    INV = _abi.M2S_E_INVALID
    fake_ctx = C.create_string_buffer(256)
    ctx = C.cast(fake_ctx, C.c_void_p)
    q, d, s = 0x10000, 0x20000, 0x30000          # aligned stand-ins for device pointers, never touched
    o, w = 0x40000, 0x50000
    # NULL context
    assert L.m2s_depth_sort(None, q, d, 10, s, o, w) == INV
    assert L.m2s_depth_sort_enqueue(None, q, d, 10, None, s, o, w, None) == INV
    assert L.m2s_depth_sort(None, None, None, 0, None, None, None) == INV
    assert b"NULL" in L.m2s_last_error()
    # NULL buffers with count > 0
    for args in ((None, d, s), (q, None, s), (q, d, None)):
        assert L.m2s_depth_sort(ctx, args[0], args[1], 5, args[2], o, w) == INV
        assert L.m2s_depth_sort_enqueue(ctx, args[0], args[1], 5, None, args[2], o, w, None) == INV
    # misaligned quad buffers
    for qq, ss in ((q + 8, s), (q, s + 4), (q + 1, s + 1)):
        assert L.m2s_depth_sort(ctx, qq, d, 5, ss, o, w) == INV
        assert L.m2s_depth_sort_enqueue(ctx, qq, d, 5, None, ss, o, w, None) == INV
    assert b"aligned" in L.m2s_last_error()
    # count = 2^30 and beyond
    for n in (1 << 30, (1 << 30) + 1, 1 << 40):
        assert L.m2s_depth_sort(ctx, q, d, n, s, o, w) == INV
        assert L.m2s_depth_sort_enqueue(ctx, q, d, n, None, s, o, w, None) == INV
    assert b"2^30" in L.m2s_last_error()


def test_sort_tile_is_exposed():
    from mesh2splat_b200.api import depth_sort_tile
    t = depth_sort_tile()
    assert t >= 1024 and t % 32 == 0
