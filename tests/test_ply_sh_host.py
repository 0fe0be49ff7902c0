"""A loaded .ply's view-dependent colour, host half (beyond the reference, which skips the SH rest coefficients):
m2s_ply_parse_header's sh_degree and f_rest offsets, the C restatement of the SH colour (oracle/m2s_sh_oracle.c) against
an fp64 statement of graphdeco's computeColorFromSH, and the argument checks of m2s_prepass_sh and
m2s_ply_decode_sh_enqueue, all without a GPU."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np
import pytest

import oracle
from mesh2splat_b200 import _abi, api
from mesh2splat_b200._lib import lib
from oracle import sh as osh

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_ply_load import PBR, STANDARD, ply, vertex_rows  # noqa: E402
from make_golden_prepass import column_major, look_at, perspective  # noqa: E402

Z = np.load(os.path.join(HERE, "golden", "ref_ply_load_vectors.npz"))
NAMES = [str(n) for n in Z["names"]]
TYPE_BYTES = {"float": 4, "double": 8, "uchar": 1, "ushort": 2, "int": 4}


class _InfoPrefix(C.Structure):
    """m2s_ply_info up to (not including) sh_degree: the fields every load had before the SH fields were appended."""
    _fields_ = _abi.m2s_ply_info._fields_[:5]


PREFIX = _abi.m2s_ply_info.sh_degree.offset


def _header(props, n=3, seed=0) -> bytes:
    if len({name for _, name in props}) < len(props):   # a repeated name: the body's values do not matter
        return ply([("vertex", n, props, bytes(n * sum(TYPE_BYTES[t] for t, _ in props)))])
    return ply([("vertex", n, props, vertex_rows(np.random.default_rng(seed), props, n))])


def _offsets(props) -> dict:
    offs, o = {}, 0
    for t, name in props:
        offs.setdefault(name, o)
        o += TYPE_BYTES[t]
    return offs


def _standard_with_rest(rng, nrest, rest_type="float", names=None):
    names = names if names is not None else [f"f_rest_{k}" for k in range(nrest)]
    props = [("float", k) for k in STANDARD] + [(rest_type, n) for n in names]
    return [props[i] for i in rng.permutation(len(props))]


@pytest.mark.parametrize("nrest,degree", [(0, 0), (9, 1), (24, 2), (45, 3)])
def test_sh_degree_and_offsets_in_shuffled_property_order(nrest, degree):
    rng = np.random.default_rng(nrest)
    for trial in range(4):
        props = _standard_with_rest(rng, nrest)
        info = api.ply_parse_header(_header(props, seed=trial))
        offs = _offsets(props)
        assert info.sh_degree == degree
        want = [offs[f"f_rest_{k}"] if k < nrest else -1 for k in range(_abi.SH_REST_MAX)]
        assert list(info.f_rest) == want
        assert info.offsets() == {n: offs[n] for n in _abi.PLY_PROPS if n in offs}


@pytest.mark.parametrize("case", ["partial_8", "partial_44", "odd_10", "gap", "duplicate", "leading_zero", "non_float", "suffix"])
def test_other_rest_sets_give_degree_0_without_error(case):
    rng = np.random.default_rng(7)
    names = [f"f_rest_{k}" for k in range(9)]
    rest_type = "float"
    if case == "partial_8":
        names = names[:8]
    elif case == "partial_44":
        names = [f"f_rest_{k}" for k in range(44)]
    elif case == "odd_10":
        names = [f"f_rest_{k}" for k in range(10)]
    elif case == "gap":            # nine properties, f_rest_8 missing and f_rest_9 instead
        names = names[:8] + ["f_rest_9"]
    elif case == "duplicate":      # nine properties, f_rest_3 twice
        names = names[:8] + ["f_rest_3"]
    elif case == "leading_zero":   # f_rest_08 is not f_rest_8
        names = names[:8] + ["f_rest_08"]
    elif case == "non_float":
        rest_type = "double"
    elif case == "suffix":
        names = names[:8] + ["f_rest_8x"]
    props = _standard_with_rest(rng, 0, rest_type, names)
    info = api.ply_parse_header(_header(props))
    assert info.sh_degree == 0 and list(info.f_rest) == [-1] * _abi.SH_REST_MAX
    offs = _offsets(props)
    assert info.row_stride == sum(TYPE_BYTES[t] for t, _ in props)
    assert info.offsets() == {n: offs[n] for n in _abi.PLY_PROPS if n in offs}


def test_every_golden_fixture_gives_the_same_info_prefix_as_before():
    """The fields before sh_degree keep their offsets and values: the prefix of m2s_ply_info equals a struct of the old
    layout filled from an independent reading of the header; the files refused before are still refused."""
    assert PREFIX == C.sizeof(_InfoPrefix) - 4 and _abi.m2s_ply_info.offset.offset == _InfoPrefix.offset.offset
    for name in NAMES:
        data = Z[f"file_{name}"].tobytes()
        if not int(Z[f"ok_{name}"]) or int(Z[f"dev_{name}"]):
            with pytest.raises(api.M2SError):
                api.ply_parse_header(data)
            continue
        info = api.ply_parse_header(data)
        old = _InfoPrefix()
        old.vertex_count, old.body_offset, old.row_stride = info.vertex_count, info.body_offset, info.row_stride
        old.has_pbr = int(Z[f"pbr_{name}"])
        assert old.vertex_count == len(Z[f"rec_{name}"])
        names = data[: data.index(b"end_header")].decode("latin-1").replace("\r", "").split("\n")
        vertex = names.index(next(line for line in names if line.startswith("element vertex")))
        props, o, offs = [], 0, {}
        for line in names[vertex + 1:]:
            t = line.split()
            if not t or t[0] == "element":
                break
            if t[0] == "property":
                offs.setdefault(t[-1], o)
                props.append(t[-1])
                o += {"float": 4, "float32": 4, "double": 8, "float64": 8, "uchar": 1, "char": 1, "ushort": 2, "short": 2,
                      "int": 4, "uint": 4}[t[1]]
        for k, n in enumerate(_abi.PLY_PROPS):
            old.offset[k] = offs.get(n, -1)
        assert bytes(info)[:PREFIX] == bytes(old)[:PREFIX], name
        rest = [p for p in props if p.startswith("f_rest_")]
        assert info.sh_degree == {9: 1, 24: 2, 45: 3}.get(len(rest), 0), name


# ---- the SH colour: the C restatement against fp64 --------------------------------------------------------------------------
def _records(rng, n):
    g = np.zeros((n, 24), np.float32)
    g[:, 0:3] = (rng.random((n, 3)) - 0.5) * 2
    g[:, 3] = 1
    g[:, 4:7] = rng.normal(size=(n, 3)) * 0.28209479177387814 + 0.5
    g[:, 7] = rng.random(n)
    g[:, 8:11] = rng.random((n, 3)) * 0.05 + 0.001
    q = rng.normal(size=(n, 4))
    g[:, 16:20] = q / np.linalg.norm(q, axis=1, keepdims=True)
    return g


def _camera_matrices(eye, target=(0.0, 0.0, 0.0)):
    V = column_major(look_at(np.asarray(eye, np.float64), np.asarray(target, np.float64), np.array([0.0, 1.0, 0.0])).astype(np.float32))
    P = column_major(perspective(np.radians(60.0), 4 / 3, 0.01, 100.0))
    return V, P


@pytest.mark.parametrize("buffer_degree,sh_degree", [(1, 1), (2, 2), (3, 3), (3, 1), (3, 2), (2, 1)])
def test_restatement_matches_fp64_compute_color_from_sh(buffer_degree, sh_degree):
    """Random directions (the camera outside and inside the gaussians) and coefficients.  Bound: the fp32 evaluation
    rounds about 20 times along each term's path, the camera's position once (its error reaches the direction as
    |c| eps / |d|); 32 eps of (|colour| + sum |B_k coeff_k|), plus that direction term, holds with margin."""
    rng = np.random.default_rng(100 * buffer_degree + sh_degree)
    n = 20000
    g = _records(rng, n)
    K = (sh_degree + 1) ** 2 - 1
    block = (rng.normal(size=(n, _abi.SH_FLOATS[buffer_degree])) * 0.5).astype(np.float32)
    block[:, 3 * ((buffer_degree + 1) ** 2 - 1):] = 0
    for eye in ((0.3, 1.5, 4.0), (0.05, -0.1, 0.2)):
        V, _ = _camera_matrices(eye)
        M = column_major(np.eye(4, dtype=np.float32))
        cam = osh.camera(V, M)
        assert np.allclose(cam, eye, rtol=1e-6, atol=1e-6)
        got = osh.colours(g, block, buffer_degree, sh_degree, cam).astype(np.float64)
        d = g[:, 0:3].astype(np.float64) - cam.astype(np.float64)
        coeffs = block[:, : 3 * K].reshape(n, K, 3)
        want = osh.reference_rgb(d, coeffs, g[:, 4:7])
        # |B_k| <= 1.1 on the sphere (graphdeco's normalised basis)
        mag = np.abs(g[:, 4:7]).astype(np.float64) + 1.1 * np.abs(coeffs).astype(np.float64).sum(axis=1)
        dist = np.linalg.norm(d, axis=1, keepdims=True)
        eps = 2.0 ** -24
        bound = 32 * eps * mag + 8 * eps * (np.abs(cam).max() + np.abs(g[:, 0:3]).max(axis=1, keepdims=True)) / dist * mag
        err = np.abs(got - want)
        assert (err <= bound).all(), f"max error {err.max()} at bound {bound[np.unravel_index(err.argmax(), err.shape)]}"
        assert (err > 0).any() or sh_degree == 0   # the comparison is not vacuous: fp32 and fp64 do differ


def test_zero_length_direction_gives_the_record_colour():
    g = _records(np.random.default_rng(1), 4)
    g[:, 4] = (-0.25, 0.0, 0.5, 2.0)
    cam = g[0, 0:3].copy()
    block = np.ones((4, 48), np.float32)
    got = osh.colours(g, block, 3, 3, cam)
    assert got[0, 0] == 0.0 and np.array_equal(got[0, 1:].view(np.uint32), g[0, 5:7].view(np.uint32))   # rest 0, then max(., 0)


def _prepass_inputs(rng, n, eye, rotated: bool):
    g = _records(rng, n)
    V, P = _camera_matrices(eye)
    if rotated:   # rotated about an oblique axis, scaled non-uniformly and translated
        a = np.radians(37.0)
        ax = np.array([1.0, 2.0, -0.5]) / np.linalg.norm([1.0, 2.0, -0.5])
        Kx = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
        R = np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx
        Mr = np.eye(4)
        Mr[:3, :3] = R @ np.diag([1.3, 0.7, 1.1])
        Mr[:3, 3] = (0.2, -0.1, 0.3)
        M = column_major(Mr.astype(np.float32))
    else:
        M = column_major(np.eye(4, dtype=np.float32))
    return g, V, P, M


@pytest.mark.parametrize("mode", [0, 1, 2, 6])
@pytest.mark.parametrize("rotated", [False, True])
def test_prepass_sh_is_the_prepass_with_the_sh_colour(mode, rotated):
    """orc_prepass_sh = orc_prepass except the colour of modes 0 and 6, which is orc_sh_colours of the survivors; modes 1
    and 2 and sh_degree 0 are orc_prepass bit for bit."""
    rng = np.random.default_rng(mode + 10 * rotated)
    n = 3000
    g, V, P, M = _prepass_inputs(rng, n, (0.4, 0.8, 3.0), rotated)
    block = (rng.normal(size=(n, 48)) * 0.4).astype(np.float32)
    args = (V, P, M, (800.0, 600.0), (0.01, 100.0), 1.0, mode)
    base_q, base_d = oracle.prepass(g, *args, fmt=1, ply_has_pbr=0)
    q0, d0 = osh.prepass_sh(g, *args, 0, block, 3, 0)
    assert np.array_equal(q0.view(np.uint32), base_q.view(np.uint32)) and np.array_equal(d0.view(np.uint32), base_d.view(np.uint32))
    q, d = osh.prepass_sh(g, *args, 0, block, 3, 3)
    assert len(q) == len(base_q) > 100 and np.array_equal(d.view(np.uint32), base_d.view(np.uint32))
    other = [c for c in range(24) if not (mode in (0, 6) and c in (8, 9, 10))]
    assert np.array_equal(q[:, other].view(np.uint32), base_q[:, other].view(np.uint32))
    if mode in (0, 6):
        cam = osh.camera(V, M)
        rgb = osh.colours(g, block, 3, 3, cam)
        wpos = g[:, 0:3] @ np.asarray(M, np.float32).reshape(4, 4)[:3, :3] + np.asarray(M, np.float32).reshape(4, 4)[3, :3]
        idx = np.array([np.argmin(np.abs(wpos - w).sum(axis=1)) for w in q[:, 20:23]])
        assert np.array_equal(q[:, 8:11].view(np.uint32), rgb[idx].view(np.uint32))
        assert not np.array_equal(q[:, 8:11], base_q[:, 8:11])


# ---- argument checks without a GPU ------------------------------------------------------------------------------------------
def test_prepass_sh_rejects_bad_arguments_before_any_launch():
    """M2S_E_INVALID for another layout, buffer_degree > 3, sh_degree > buffer_degree, a NULL d_sh with sh_degree > 0 and a
    singular V M; the checks run before the context is used (C.c_void_p(1) stands for it)."""
    L = lib()
    INV = _abi.M2S_E_INVALID
    I4 = np.eye(4, dtype=np.float32).ravel()
    ctx, buf, sh = C.c_void_p(1), C.c_void_p(256), C.c_void_p(512)

    def call(layout=_abi.VIEW_PLY, buffer_degree=3, sh_degree=3, d_sh=sh, V=I4):
        p = _abi.make_prepass_params(V, I4, I4, (64, 64), (0.1, 10.0), 1.0, 0, layout)
        return L.m2s_prepass_sh_enqueue(ctx, buf, 10, None, C.byref(p), d_sh, buffer_degree, sh_degree, buf, buf, buf, None)

    for layout in (_abi.LAYOUT_REF96, _abi.LAYOUT_PACKED56, 99):
        assert call(layout=layout) == INV
    assert b"VIEW_PLY" in L.m2s_last_error()
    assert call(buffer_degree=4, sh_degree=1) == INV
    assert call(buffer_degree=1, sh_degree=2) == INV and b"sh_degree" in L.m2s_last_error()
    assert call(d_sh=None) == INV and b"NULL d_sh" in L.m2s_last_error()
    assert call(d_sh=C.c_void_p(520)) == INV and b"16-byte" in L.m2s_last_error()
    assert call(V=np.zeros(16, np.float32)) == INV and b"singular" in L.m2s_last_error()
    p = _abi.make_prepass_params(I4, I4, I4, (64, 64), (0.1, 10.0), 1.0, 0, _abi.VIEW_PLY)
    v = C.c_uint32(0)
    assert L.m2s_prepass_sh(None, buf, 10, C.byref(p), sh, 3, 3, buf, buf, C.byref(v)) == INV
    assert L.m2s_prepass_sh(ctx, buf, 10, C.byref(p), None, 3, 1, buf, buf, C.byref(v)) == INV


def test_decode_sh_rejects_offsets_outside_the_row():
    rng = np.random.default_rng(3)
    props = _standard_with_rest(rng, 45)
    info = api.ply_parse_header(_header(props))
    L = lib()
    bad = _abi.m2s_ply_info.from_buffer_copy(info)
    bad.f_rest[44] = info.row_stride - 2
    args = (C.c_void_p(1), C.byref(bad), C.c_void_p(16), 1, C.c_void_p(16))
    assert L.m2s_ply_decode_sh_enqueue(*args, C.c_void_p(32), None) == _abi.M2S_E_INVALID
    assert b"f_rest_44" in L.m2s_last_error()
    bad = _abi.m2s_ply_info.from_buffer_copy(info)
    bad.sh_degree = 4
    assert L.m2s_ply_decode_sh_enqueue(C.c_void_p(1), C.byref(bad), C.c_void_p(16), 1, C.c_void_p(16), C.c_void_p(32), None) == _abi.M2S_E_INVALID
    assert L.m2s_ply_decode_sh_enqueue(C.c_void_p(1), C.byref(info), C.c_void_p(16), 1, C.c_void_p(16), C.c_void_p(40), None) == _abi.M2S_E_INVALID
    assert b"16-byte" in L.m2s_last_error()
    assert _abi.m2s_ply_info.f_rest.offset == PREFIX + 4 and C.sizeof(_abi.m2s_ply_info) == 288


def test_file_order_to_block():
    rest = np.arange(2 * 45, dtype=np.float32).reshape(2, 45)
    b = osh.block_from_file_order(rest, 3)
    assert b.shape == (2, 48) and (b[:, 45:] == 0).all()
    # coefficient k (1..15) of channel c is f_rest_{15 c + k - 1}; the block holds it at 3 (k - 1) + c
    for k in range(1, 16):
        for c in range(3):
            assert b[1, 3 * (k - 1) + c] == rest[1, 15 * c + k - 1]
