#!/usr/bin/env python3
"""Generates the .ply loader's golden data (SURVEY 8 f-10) from the REFERENCE's own loader and prepass shader.

  ref_ply_load_vectors.npz     small .ply files (key file_<name>, the bytes) and what parsers::loadPlyFile makes of each
                               (ok_<name>: 1 loaded / 0 rejected, rec_<name>: [n, 24] GaussianDataSSBO, pbr_<name>: hasPbr;
                               dev_<name>: 1 for the files this project rejects on purpose, see m2s.h)
  ref_prepass_ply_vectors.npz  the reference's prepass shader with u_format 1, u_plyHasPbr 0 and 1, on records loaded by
                               the reference from .ply files (inputs, camera, survivors)

Needs a checkout of the reference: oracle/build_ply_load.py compiles the reference's
parsers.cpp (happly included) into oracle/_ref/libm2s_refplyload.so, oracle/build.py its .ply writer and prepass shader.

    python tests/golden/make_golden_ply_load.py
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import oracle  # noqa: E402
from oracle import build as obuild  # noqa: E402
from oracle import build_ply_load, ply_load  # noqa: E402

NP_TYPES = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "char": "i1",
            "ushort": "<u2", "short": "<i2", "int": "<i4", "uint": "<u4"}
STANDARD = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2", "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
PBR = ["nx", "ny", "nz", "metallicFactor", "roughnessFactor"]


def values(rng, name, n):
    """Plausible 3DGS values per property."""
    if name in ("x", "y", "z"):
        return (rng.random(n) - 0.5) * 4
    if name.startswith("f_dc") or name.startswith("f_rest"):
        return rng.normal(size=n)
    if name == "opacity":
        return rng.normal(size=n) * 3
    if name.startswith("scale_"):
        return rng.normal(size=n) - 4
    if name.startswith("rot_"):
        return rng.normal(size=n)
    if name in ("nx", "ny", "nz"):
        return rng.normal(size=n)
    return rng.random(n) * 255 if name in ("red", "green", "blue") else rng.random(n)


def vertex_rows(rng, props, n, fill=None):
    """props: [(type, name)] -> bytes of n rows; fill(name, array) may overwrite values."""
    dt = np.dtype([(name, NP_TYPES[t]) for t, name in props])
    a = np.zeros(n, dt)
    for t, name in props:
        v = values(rng, name, n)
        if fill is not None:
            v = fill(name, v)
        a[name] = v
    return a.tobytes()


def ply(elements, fmt="binary_little_endian", lines=(), eol="\n"):
    """elements: [(name, count, [(type, name) or ('list', count type, type, name)], body bytes)]."""
    h = ["ply", f"format {fmt} 1.0", *lines]
    for name, count, props, _ in elements:
        h.append(f"element {name} {count}")
        for p in props:
            h.append(f"property list {p[1]} {p[2]} {p[3]}" if p[0] == "list" else f"property {p[0]} {p[1]}")
    h.append("end_header")
    return (eol.join(h) + eol).encode() + b"".join(body for *_, body in elements)


def fixtures(rng, tmp):
    F = {}   # name -> (bytes, deviation)
    std = [("float", n) for n in STANDARD]
    pbr = [("float", n) for n in ("x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2", "metallicFactor", "roughnessFactor",
                                  "opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3")]
    # the reference writer's own three formats (format 2 has no f_dc_0: rejected)
    g = np.asarray(__import__("make_golden_prepass").gaussians(rng, 40, 0.02), np.float32)
    g[:, 7] = np.clip(g[:, 7], 0.02, 0.98)
    for fmt in (0, 1, 2):
        p = os.path.join(tmp, f"w{fmt}.ply")
        assert oracle.ref_save_ply(p, g, fmt, 0.65 / 256)
        F[f"writer_fmt{fmt}"] = (open(p, "rb").read(), 0)
    # permuted and extra properties (an extra double is never read)
    perm = [("float", n) for n in rng.permutation(STANDARD + PBR[:3])] + [("uchar", "red"), ("double", "confidence"), ("float", "f_rest_0")]
    perm = perm[:5] + perm[-3:] + perm[5:-3]
    F["permuted_extra"] = (ply([("vertex", 37, perm, vertex_rows(rng, perm, 37))]), 0)
    # uchar / ushort properties make the stride and the offsets odd; all PBR properties present
    odd = [("uchar", "red"), ("uchar", "green"), ("uchar", "blue")] + pbr[:7] + [("ushort", "flags")] + pbr[7:]
    F["uchar_odd_pbr"] = (ply([("vertex", 45, odd, vertex_rows(rng, odd, 45))]), 0)
    # a face element after vertex, a fixed-size element before it; comment / obj_info lines; CR LF line ends
    faces = b"".join(bytes([3]) + np.array(rng.integers(0, 20, 3), "<i4").tobytes() for _ in range(6))
    cam = [("float", "fx"), ("uchar", "id"), ("double", "t")]
    F["face_after"] = (ply([("vertex", 20, pbr, vertex_rows(rng, pbr, 20)), ("face", 6, [("list", "uchar", "int", "vertex_indices")], faces)],
                           lines=["comment made by make_golden_ply_load", "obj_info seeded"]), 0)
    F["fixed_before"] = (ply([("camera", 3, cam, vertex_rows(rng, cam, 3)), ("vertex", 21, std, vertex_rows(rng, std, 21))],
                             lines=["comment a camera element first"]), 0)
    F["crlf_comments"] = (ply([("vertex", 9, std, vertex_rows(rng, std, 9))], lines=["comment one", "obj_info two", "comment"], eol="\r\n"), 0)
    # 0 and 1 vertices (0: hasPbr 1 whatever the properties)
    F["zero_vertices"] = (ply([("vertex", 0, std, b"")]), 0)
    F["one_vertex"] = (ply([("vertex", 1, pbr, vertex_rows(rng, pbr, 1))]), 0)
    F["normals_no_pbr"] = (ply([("vertex", 8, std + [("float", "nx"), ("float", "ny"), ("float", "nz")],
                                 vertex_rows(rng, std + [("float", "nx"), ("float", "ny"), ("float", "nz")], 8))]), 0)
    # double required / double optional / missing rot_3: rejected
    dreq = [("double", "x")] + std[1:]
    F["double_required"] = (ply([("vertex", 4, dreq, vertex_rows(rng, dreq, 4))]), 0)
    dopt = std + [("double", "nx"), ("float", "ny"), ("float", "nz"), ("float", "metallicFactor"), ("float", "roughnessFactor")]
    F["double_optional"] = (ply([("vertex", 4, dopt, vertex_rows(rng, dopt, 4))]), 0)
    F["missing_rot3"] = (ply([("vertex", 4, std[:-1], vertex_rows(rng, std[:-1], 4))]), 0)
    # quaternions: unnormalised, zero, NaN, inf, tiny (denormal squares), huge (squares overflow)
    quats = np.array([[2, 0, 0, 0], [0, 0, 0, 0], [-0.0, 0, 0, 0], [np.nan, 1, 0, 0], [0, np.inf, 0, 0], [1e-30, 2e-30, 0, 0],
                      [1e-45, 0, 0, 0], [3e19, 4e19, 0, 0], [1e-20, 1e-20, 1e-20, 1e-20], [-1, -2, -3, -4], [0.5, 0.5, 0.5, 0.5],
                      [1e30, 1, 1, 1]], np.float32)
    nq = len(quats)

    def fill_q(name, v):
        return quats[:, int(name[-1])] if name.startswith("rot_") else v
    F["quaternions"] = (ply([("vertex", nq, pbr, vertex_rows(rng, pbr, nq, fill_q))]), 0)
    # opacity and log-scale extremes: +-inf, NaN, denormals, +-100, the expf overflow / underflow edges
    ext = np.array([np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1e-40, 100, -100, 88.72, 88.73, -87.3, -103.9, -104, 0, -0.0, 20, -20,
                    1.5, -7.25, 0.6931472], np.float32)

    def fill_e(name, v):
        if name == "opacity" or name.startswith("scale_"):
            return np.roll(ext, {"opacity": 0, "scale_0": 3, "scale_1": 7, "scale_2": 11}[name])
        return v
    F["extremes"] = (ply([("vertex", len(ext), std, vertex_rows(rng, std, len(ext), fill_e))]), 0)
    # random values of the standard layout, enough rows for the exp comparison
    many = [("float", n) for n in STANDARD[:3]] + [("float", "nx"), ("float", "ny"), ("float", "nz")] + \
        [("float", n) for n in STANDARD[3:6]] + [("float", f"f_rest_{k}") for k in range(45)] + [("float", n) for n in STANDARD[6:]]
    F["standard_random"] = (ply([("vertex", 300, many, vertex_rows(rng, many, 300))]), 0)
    # files the reference takes and this project rejects on purpose (m2s.h, deviations)
    F["dev_ascii"] = (b"ply\nformat ascii 1.0\nelement vertex 1\n" + "".join(f"property float {n}\n" for n in STANDARD).encode()
                      + b"end_header\n" + (" ".join(["0.5"] * len(STANDARD)) + "\n").encode(), 1)
    be = [(t, n) for t, n in std]
    F["dev_big_endian"] = (ply([("vertex", 2, be, np.frombuffer(vertex_rows(rng, be, 2), "<f4").astype(">f4").tobytes())], fmt="binary_big_endian"), 1)
    F["dev_list_before_vertex"] = (ply([("face", 2, [("list", "uchar", "int", "vertex_indices")], faces[:26]),
                                        ("vertex", 5, std, vertex_rows(rng, std, 5))]), 1)
    F["dev_truncated"] = (ply([("vertex", 10, std, vertex_rows(rng, std, 10))])[:-7], 1)
    return F


def main():
    assert build_ply_load.build_ref_ply_load() is not None and obuild.build_ref_ply() is not None, "needs the reference checkout"
    assert obuild.build_ref_prepass() is not None
    rng = np.random.default_rng(20261016)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        F = fixtures(rng, tmp)
        for name, (data, dev) in F.items():
            p = os.path.join(tmp, name + ".ply")
            with open(p, "wb") as f:
                f.write(data)
            r = ply_load.ref_load(p)
            out[f"file_{name}"] = np.frombuffer(data, np.uint8)
            out[f"dev_{name}"] = np.array(dev)
            out[f"ok_{name}"] = np.array(0 if r is None else 1)
            if r is not None:
                out[f"rec_{name}"], out[f"pbr_{name}"] = r[0], np.array(r[1])
            print(f"{name:24s} {len(data):6d} B  {'rejected' if r is None else f'{len(r[0])} records, hasPbr {r[1]}'}")
    out["names"] = np.array(sorted(F))
    path = os.path.join(HERE, "ref_ply_load_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")

    # the prepass on loaded records: u_format 1 without and with PBR values
    from make_golden_prepass import column_major, look_at, perspective
    rot = np.eye(4, dtype=np.float32)
    c, s = np.cos(0.4), np.sin(0.4)
    rot[:3, :3] = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], np.float32)
    rot[:3, 3] = [0.2, 0.1, -0.3]
    pp = {}
    cases = [(0, 0, np.eye(4, dtype=np.float32), [3.0, 2.0, 4.0]), (0, 2, rot, [-2.0, 1.5, 3.0]),
             (1, 2, np.eye(4, dtype=np.float32), [1.0, -2.0, 3.5]), (1, 0, rot, [2.5, 2.5, 2.5])]
    with tempfile.TemporaryDirectory() as tmp:
        for i, (has_pbr, mode, M, eye) in enumerate(cases):
            props = [("float", n) for n in STANDARD + (PBR if has_pbr else [])]
            n = 300

            def fill(name, v):
                return (rng.random(n) - 0.5) * 4 if name in ("x", "y", "z") else (rng.normal(size=n) - 4.5 if name.startswith("scale_") else v)
            data = ply([("vertex", n, props, vertex_rows(rng, props, n, fill))])
            p = os.path.join(tmp, f"p{i}.ply")
            with open(p, "wb") as f:
                f.write(data)
            recs, pbr = ply_load.ref_load(p)
            assert pbr == has_pbr
            V = look_at(np.array(eye, np.float64), np.zeros(3), np.array([0.0, 1.0, 0.0])).astype(np.float32)
            P = perspective(np.radians(45.0), 16 / 9, 0.01, 100.0)
            quads, depths = oracle.ref_prepass(recs, column_major(V), column_major(P), column_major(M), (1280.0, 720.0), (0.01, 100.0),
                                               0.65 / 512, mode, 1, has_pbr)
            assert 30 < len(quads) < n, len(quads)
            pp[f"g{i}"] = recs
            pp[f"view{i}"] = column_major(V); pp[f"proj{i}"] = column_major(P); pp[f"model{i}"] = column_major(M)
            pp[f"params{i}"] = np.array([1280.0, 720.0, 0.01, 100.0, 0.65 / 512, mode, has_pbr], np.float64)
            pp[f"quads{i}"] = quads; pp[f"depths{i}"] = depths
    pp["ncases"] = np.array(len(cases))
    path = os.path.join(HERE, "ref_prepass_ply_vectors.npz")
    np.savez_compressed(path, **pp)
    print("wrote", path, os.path.getsize(path), "bytes;", [len(pp[f"quads{i}"]) for i in range(len(cases))], "survivors")


if __name__ == "__main__":
    main()
