"""The .ply loader's host half (SURVEY 8 f-10): m2s_ply_parse_header against the reference's own loadPlyFile (golden
fixtures made by it, tests/golden/make_golden_ply_load.py), the C restatement of loadPlyFile's arithmetic against the
reference's records, every deliberate deviation, and the header parser on hostile input."""
from __future__ import annotations

import ctypes as C
import mmap
import os
import types

import numpy as np
import pytest

from mesh2splat_b200 import _abi, api
from mesh2splat_b200._lib import M2SError, lib
from oracle import ply_load

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_ply_load_vectors.npz")
Z = np.load(GOLDEN)
NAMES = [str(n) for n in Z["names"]]
ACCEPTED = [n for n in NAMES if int(Z[f"ok_{n}"]) and not int(Z[f"dev_{n}"])]
TYPE_BYTES = {"char": 1, "int8": 1, "uchar": 1, "uint8": 1, "short": 2, "int16": 2, "ushort": 2, "uint16": 2, "int": 4, "int32": 4,
              "uint": 4, "uint32": 4, "float": 4, "float32": 4, "double": 8, "float64": 8}


def _file(name: str) -> bytes:
    return Z[f"file_{name}"].tobytes()


def _format_error(data: bytes, file_size=None) -> str:
    with pytest.raises(M2SError) as e:
        api.ply_parse_header(data, file_size)
    assert e.value.status == _abi.M2S_E_FORMAT, e.value
    return e.value.message


def _same_bits(a, b) -> bool:
    return np.array_equal(np.ascontiguousarray(a, np.float32).view(np.uint32), np.ascontiguousarray(b, np.float32).view(np.uint32))


def _plain_header(data: bytes):
    """An independent reading of a well-formed binary header: (count, body offset, stride, {name: offset}) of 'vertex'."""
    end = data.index(b"end_header") + len(b"end_header")
    body = data.index(b"\n", end) + 1
    elems, skip = [], 0
    for line in data[:end].decode().replace("\r", "").split("\n")[2:]:
        t = line.split()
        if t and t[0] == "element":
            elems.append([t[1], int(t[2]), []])
        elif t and t[0] == "property":
            elems[-1][2].append((t[-1], 0 if t[1] == "list" else TYPE_BYTES[t[1]]))
    for name, count, props in elems:
        if name == "vertex":
            offs, o = {}, 0
            for pn, b in props:
                offs.setdefault(pn, o)
                o += b
            return count, body + skip, o, offs
        skip += count * sum(b for _, b in props)
    raise AssertionError("no vertex element")


@pytest.mark.parametrize("name", [n for n in NAMES if not int(Z[f"dev_{n}"])])   # deviations: test_deviations_...
def test_header_accepts_exactly_what_the_reference_accepts(name):
    data = _file(name)
    if not int(Z[f"ok_{name}"]):
        _format_error(data)
        return
    info = api.ply_parse_header(data)
    rec = Z[f"rec_{name}"]
    assert info.vertex_count == len(rec) and info.has_pbr == int(Z[f"pbr_{name}"])
    count, body, stride, offs = _plain_header(data)
    assert (info.vertex_count, info.body_offset, info.row_stride) == (count, body, stride)
    want = {n: offs[n] for n in _abi.PLY_PROPS if n in offs}
    assert info.offsets() == want


@pytest.mark.parametrize("name", ACCEPTED)
def test_restatement_matches_the_reference_records_bit_for_bit(name):
    data = _file(name)
    info = api.ply_parse_header(data)
    rows = data[info.body_offset: info.body_offset + info.vertex_count * info.row_stride]
    got = ply_load.load(rows, info, info.vertex_count)
    assert _same_bits(got, Z[f"rec_{name}"]), f"{int((got.view(np.uint32) != Z[f'rec_{name}'].view(np.uint32)).sum())} words differ"


def test_zero_vertices_have_pbr_whatever_the_properties():
    info = api.ply_parse_header(_file("zero_vertices"))
    assert info.vertex_count == 0 and info.has_pbr == 1 and int(Z["pbr_zero_vertices"]) == 1
    assert "nx" not in info.offsets()


def test_deviations_are_format_errors_with_their_cause():
    """Files the reference takes (ascii, big-endian, a list element before 'vertex', a truncated body) and the files it
    rejects itself: each M2S_E_FORMAT with a message naming the cause."""
    causes = {"dev_ascii": "ascii", "dev_big_endian": "binary_big_endian", "dev_list_before_vertex": "list property",
              "dev_truncated": "truncated", "writer_fmt2": "'f_dc_0'", "double_required": "'x' is not float",
              "double_optional": "'nx' is not float", "missing_rot3": "'rot_3'"}
    for name, cause in causes.items():
        assert int(Z[f"dev_{name}"]) == (1 if name.startswith("dev_") else 0)
        assert int(Z[f"ok_{name}"]) == (1 if name.startswith("dev_") else 0), name
        msg = _format_error(_file(name))
        assert cause in msg, (name, msg)
    assert "end_header" in _format_error(b"ply\nformat binary_little_endian 1.0\nelement vertex 0\n")
    wide = b"".join(b"property %s %s\n" % (b"float", n.encode()) for n in _abi.PLY_PROPS) + b"".join(b"property double p%d\n" % k for k in range(503))
    assert "rows of 4100 bytes" in _format_error(b"ply\nformat binary_little_endian 1.0\nelement vertex 0\n" + wide + b"end_header\n")


def test_truncated_bodies_and_overflowing_counts():
    data = _file("writer_fmt1")
    info = api.ply_parse_header(data)
    end = info.body_offset + info.vertex_count * info.row_stride
    assert end == len(data)
    for cut in (1, 3, info.row_stride, len(data) - info.body_offset):
        assert "truncated" in _format_error(data[:-cut])
        assert "truncated" in _format_error(data, file_size=len(data) - cut)   # a prefix with the true file size
    api.ply_parse_header(data[: info.body_offset], file_size=len(data))        # the header alone is enough
    hdr = data[: info.body_offset].decode()
    for count in ("18446744073709551615", "-1", str((1 << 64) // info.row_stride + 1), "99999999999999999999999"):
        msg = _format_error(hdr.replace(f"element vertex {info.vertex_count}", f"element vertex {count}").encode())
        assert "overflows" in msg, msg
    big = hdr.replace(f"element vertex {info.vertex_count}", f"element vertex {((1 << 64) - 64) // info.row_stride}").encode()
    assert "truncated" in _format_error(big) or "overflows" in _format_error(big)
    before = hdr.replace("element vertex", "element cam 6148914691236517206\nproperty uchar a\nproperty uchar b\nproperty uchar c\nelement vertex")
    assert "2^64" in _format_error(before.encode()) or "overflows" in _format_error(before.encode())


def test_decode_rejects_rows_it_cannot_take():
    info = api.ply_parse_header(_file("writer_fmt0"))
    L = lib()
    bad = _abi.m2s_ply_info.from_buffer_copy(info)
    bad.row_stride = 4097
    assert L.m2s_ply_decode_enqueue(C.c_void_p(1), C.byref(bad), C.c_void_p(16), 1, C.c_void_p(16), None) == _abi.M2S_E_INVALID
    bad = _abi.m2s_ply_info.from_buffer_copy(info)
    bad.offset[_abi.PLY_PROPS.index("rot_3")] = info.row_stride - 3
    assert L.m2s_ply_decode_enqueue(C.c_void_p(1), C.byref(bad), C.c_void_p(16), 1, C.c_void_p(16), None) == _abi.M2S_E_INVALID
    assert b"outside the row" in L.m2s_last_error()
    assert L.m2s_ply_decode_enqueue(C.c_void_p(1), C.byref(info), C.c_void_p(16), 1, C.c_void_p(8), None) == _abi.M2S_E_INVALID
    assert L.m2s_ply_parse_header(None, 0, 0, None) == _abi.M2S_E_INVALID


class _GuardPages:
    """Bytes placed against an inaccessible page on either side: a read before or past them faults."""

    def __init__(self):
        self.page = mmap.PAGESIZE
        self.m = mmap.mmap(-1, 3 * self.page, prot=mmap.PROT_READ | mmap.PROT_WRITE)
        self.base = C.addressof(C.c_char.from_buffer(self.m))
        libc = C.CDLL(None, use_errno=True)
        libc.mprotect.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
        for off in (0, 2 * self.page):
            assert libc.mprotect(self.base + off, self.page, 0) == 0

    def parse(self, data: bytes, at_end: bool):
        n = len(data)
        assert n <= self.page
        off = self.page + (self.page - n if at_end else 0)
        self.m[off: off + n] = data
        info = _abi.m2s_ply_info()
        return lib().m2s_ply_parse_header(C.c_void_p(self.base + off), n, n, C.byref(info)), info


def test_mutated_headers_never_read_outside_their_bytes():
    """A bounded, seeded mutation of header bytes (flips, deletions, duplications, truncations), each parsed with its bytes
    against an inaccessible page at both ends: the parser returns OK or M2S_E_FORMAT, and an accepted header describes a
    body inside the bytes given."""
    rng = np.random.default_rng(7)
    g = _GuardPages()
    seeds = [_file(n) for n in ("writer_fmt0", "writer_fmt1", "uchar_odd_pbr", "face_after", "fixed_before", "crlf_comments")]
    tokens = [b" ", b"\n", b"\r", b"0", b"9", b"-", b"element vertex ", b"property float ", b"property list uchar int ",
              b"end_header", b"comment", b"double", b"\x00", b"\xff"]
    accepted = 0
    for it in range(1500):
        s = seeds[it % len(seeds)]
        hdr_end = s.index(b"end_header") + 11
        d = bytearray(s[: min(len(s), hdr_end + 300)])
        for _ in range(int(rng.integers(1, 5))):
            k = int(rng.integers(0, max(1, min(hdr_end, len(d)))))
            op = int(rng.integers(0, 4))
            if op == 0 and k < len(d):
                d[k] = int(rng.integers(0, 256))
            elif op == 1:
                del d[k: k + int(rng.integers(1, 12))]
            elif op == 2:
                d[k:k] = tokens[int(rng.integers(0, len(tokens)))]
            elif op == 3:
                d = d[: int(rng.integers(0, len(d) + 1))]
        d = bytes(d[: g.page])
        for at_end in (True, False):
            st, info = g.parse(d, at_end)
            assert st in (_abi.M2S_OK, _abi.M2S_E_FORMAT), st
            if st == _abi.M2S_OK:
                accepted += at_end
                assert 1 <= info.row_stride <= _abi.PLY_MAX_STRIDE
                assert info.body_offset + info.vertex_count * info.row_stride <= len(d)
                assert all(o + 4 <= info.row_stride for o in info.offsets().values())
    assert accepted > 0


def test_scene_manager_load_ply_returns_false_on_a_malformed_file(tmp_path):
    """SceneManager.loadPly checks the header on the host first: a file the loader cannot take returns False and leaves the
    render context as it was (no device is touched)."""
    rc = types.SimpleNamespace(ctx=None, gaussianBuffer="previous", numberOfGaussians=7, format=0, plyHasPbr=False)
    sm = api.SceneManager(rc)
    for name in ("dev_ascii", "dev_truncated", "missing_rot3", "writer_fmt2"):
        p = tmp_path / f"{name}.ply"
        p.write_bytes(_file(name))
        assert sm.loadPly(str(p)) is False
    assert sm.loadPly(str(tmp_path / "missing.ply")) is False
    assert (rc.gaussianBuffer, rc.numberOfGaussians, rc.format, rc.plyHasPbr) == ("previous", 7, 0, False)
