"""CPU tests of the codec checker (oracle/m2s_codec_oracle.c): its per-value formulas reproduce the fields of the files the
reference's own parsers::savePlyVector wrote (tests/golden/ref_ply_vectors.npz) bit for bit, and the loader's decodings
of those files as the .ply loader's restatement computes them."""
from __future__ import annotations

import os

import numpy as np
import pytest

from mesh2splat_b200 import _abi, api
from oracle import codec, ply_load

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_ply_vectors.npz"))


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return bool(((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))).all())


def _body(fmt):
    data = G[f"ply_format_{fmt}"].tobytes()
    start = data.index(b"end_header\n") + len(b"end_header\n")
    return data, np.frombuffer(data[start:], np.uint8)


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_encodings_equal_the_reference_writer_golden(fmt):
    rec = G["records"].view(np.float32).reshape(-1, 24)
    mult = float(G["scale_multiplier"])
    n = len(rec)
    _, body = _body(fmt)
    stride = {0: 248, 1: 76, 2: 48}[fmt]
    f = np.ascontiguousarray(body.reshape(n, stride)[:, : stride // 4 * 4]).view(np.float32)
    ls = codec.log_scale(rec[:, 8:11], mult)
    if fmt == 2:
        mn = np.where(rec[:, 9] < rec[:, 8], rec[:, 9], rec[:, 8])
        assert _bits_equal(f[:, 8:11], np.stack([ls[:, 0], ls[:, 1], codec.log_scale(mn, mult)], 1))
        return
    sh0, op = codec.sh0(rec[:, 4:7]), codec.logit(rec[:, 7])
    col = {0: (6, 54, 55), 1: (6, 11, 12)}[fmt]
    assert _bits_equal(f[:, col[0]: col[0] + 3], sh0)
    assert _bits_equal(f[:, col[1]], op)
    assert _bits_equal(f[:, col[2]: col[2] + 3], ls)


@pytest.mark.parametrize("fmt", [0, 1])
def test_decodings_equal_the_loader_restatement(fmt):
    data, body = _body(fmt)
    info = api.ply_parse_header(data)
    got = ply_load.load(body, info)
    f = np.ascontiguousarray(body).view(np.float32).reshape(int(info.vertex_count), -1)
    off = {k: int(info.offset[i]) // 4 for i, k in enumerate(_abi.PLY_PROPS)}
    assert _bits_equal(got[:, 7], codec.sigmoid(f[:, off["opacity"]]))
    assert _bits_equal(got[:, 8:11], codec.expf(f[:, [off["scale_0"], off["scale_1"], off["scale_2"]]]))


def test_edge_values():
    """The clamp, the poles and the specials of each formula, as the reference's code gives them."""
    a = np.array([0.0, -0.0, 1.0, -1.0, 2.0, np.inf, -np.inf, np.nan], np.float32)
    lg = codec.logit(a)
    assert np.isposinf(lg[2]) and np.isposinf(lg[4]) and np.isposinf(lg[5])          # alpha >= 1 -> +inf
    assert lg[0] == lg[1] == lg[3] == lg[6] == np.float32(-np.log(np.float32(1e8)))    # alpha <= 0 -> -log(1e8)
    assert np.isnan(lg[7])                                                             # std::clamp keeps NaN
    s = codec.log_scale(np.array([0.0, -0.0, -1.0, np.inf, np.nan, 1.0], np.float32), 1.0)
    assert np.isneginf(s[0]) and np.isneginf(s[1]) and np.isnan(s[2]) and np.isposinf(s[3]) and np.isnan(s[4]) and s[5] == 0.0
    e = codec.expf(np.array([-np.inf, np.inf, 0.0, 89.0, -104.0], np.float32))
    assert e[0] == 0.0 and np.isposinf(e[1]) and e[2] == 1.0 and np.isposinf(e[3]) and e[4] == 0.0
    assert codec.sh0(np.array([0.5], np.float32))[0] == 0.0
