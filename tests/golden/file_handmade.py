"""Hand-assembled `.ply` / `.splat` fixtures + the level-0 SplatBuffer records expected from them.  TEST INFRASTRUCTURE ONLY.

Every file is written row by row with struct.pack, and every expected record is derived with scalar Python arithmetic straight from the
reference's progressive-load semantics: PlyParserUtils.readVertex (uchar read as u / 255.0), INRIAV1PlyParser.parseToUncompressedSplat
(exp(scale) or 0.01, floor((0.5 + SH_C0 f_dc) 255) or floor(red 255), floor(sigmoid(opacity) 255) or 0, clamp to [0, 255], quaternion
normalised), SplatBuffer.writeSplatDataToSectionBuffer level 0 (normalised again, `|| 0` on scale / colour / SH, Float32Array stores),
SplatParser (.splat rows).  NaN is stored as 0x7fc00000.  Imports neither the product package nor oracle/ -- it is the third party both
are checked against.

`python tests/golden/file_handmade.py` rewrites tests/golden/file_handmade_*.ply / .splat (committed, a few KB each)."""
from __future__ import annotations

import math
import random
import struct
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
PLY, SPLAT = 1, 2
SH_C0 = 0.28209479177387814
FMT = {"double": "d", "int": "i", "uint": "I", "float": "f", "short": "h", "ushort": "H", "uchar": "B"}
INF, NAN = float("inf"), float("nan")
INRIA = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"]
TAIL = ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]


def f32_bits(v: float) -> int:
    """Float32Array element assignment (round to nearest even, overflow to inf), NaN as 0x7fc00000."""
    if v != v:
        return 0x7FC00000
    with np.errstate(over="ignore"):
        return int(np.array([v], np.float64).astype(np.float32).view(np.uint32)[0])


def ply_bytes(props, rows, *, header_lines=()) -> bytes:
    head = ["ply", "format binary_little_endian 1.0", *header_lines, f"element vertex {len(rows)}", *[f"property {t} {n}" for n, t in props], "end_header"]
    fmt = "<" + "".join(FMT[t] for _, t in props)
    body = b"".join(struct.pack(fmt, *[r[n] for n, _ in props]) for r in rows)
    return ("\n".join(head) + "\n").encode("ascii") + body


def normalize(x, y, z, w):
    """three.js Quaternion.normalize: l = sqrt(x x + y y + z z + w w); 0 -> (0, 0, 0, 1); else times 1 / l."""
    ln = math.sqrt(x * x + y * y + z * z + w * w) if all(v == v for v in (x, y, z, w)) else NAN
    if ln == 0:
        return 0.0, 0.0, 0.0, 1.0
    il = 1 / ln if ln == ln else NAN
    return x * il, y * il, z * il, w * il


def floor_clamp(v: float) -> int:
    if v != v:
        return 0
    if v == INF:
        return 255
    if v == -INF:
        return 0
    return max(0, min(255, math.floor(v)))


def sigmoid255(o: float) -> float:
    try:
        e = math.exp(-o)
    except OverflowError:
        e = INF
    return (1 / (1 + e)) * 255 if o == o else NAN


def exp_js(v: float) -> float:
    if v != v:
        return NAN
    try:
        return math.exp(v)
    except OverflowError:
        return INF


def expected_ply(props, rows, sh_degree: int) -> tuple[bytes, int]:
    """Level-0 records of a .ply file, and the output SH degree."""
    types = dict(props)
    nrest = sum(1 for n, _ in props if n.startswith("f_rest"))
    c = nrest // 3
    file_deg = 2 if c >= 8 else (1 if c >= 3 else 0)
    deg = min(sh_degree, file_deg)
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    out = b""
    for r in rows:
        val = lambda n: float(r[n]) / 255.0 if types[n] == "uchar" else float(struct.unpack("<" + FMT[types[n]], struct.pack("<" + FMT[types[n]], r[n]))[0])
        rec = struct.pack("<3I", *(f32_bits(val(k)) for k in "xyz"))
        if "scale_0" in types:
            s = [exp_js(val(f"scale_{k}")) for k in range(3)]
            s = [0.0 if v != v else v for v in s]
        else:
            s = [0.01] * 3
        rec += struct.pack("<3I", *(f32_bits(v) for v in s))
        q = normalize(*normalize(val("rot_0"), val("rot_1"), val("rot_2"), val("rot_3")))
        rec += struct.pack("<4I", *(f32_bits(v) for v in q))
        if "f_dc_0" in types:
            rgb = [(0.5 + SH_C0 * val(f"f_dc_{k}")) * 255 for k in range(3)]
        elif "red" in types:
            rgb = [val(k) * 255 for k in ("red", "green", "blue")]
        else:
            rgb = [0.0] * 3
        a = sigmoid255(val("opacity")) if "opacity" in types else 0.0
        rec += bytes(floor_clamp(v) for v in (*rgb, a))
        for s_ in range(ncomp):
            src = (s_ % 3) + c * (s_ // 3) if s_ < 9 else 3 + (s_ - 9) % 5 + c * ((s_ - 9) // 5)
            v = val(f"f_rest_{src}")
            rec += struct.pack("<I", f32_bits(0.0 if v != v or v == 0 else v))
        out += rec
    return out, deg


def expected_splat(rows) -> bytes:
    out = b""
    for c, s, rgba, q in rows:
        x, y, z, w = normalize((q[1] - 128) / 128, (q[2] - 128) / 128, (q[3] - 128) / 128, (q[0] - 128) / 128)
        out += struct.pack("<6I", *(f32_bits(float(np.float32(v))) for v in (*c, *s)))
        out += struct.pack("<4I", *(f32_bits(v) for v in (w, x, y, z))) + bytes(rgba)
    return out


def splat_bytes(rows) -> bytes:
    return b"".join(struct.pack("<6f4B4B", *c, *s, *rgba, *q) for c, s, rgba, q in rows)


# ---- fixtures ---------------------------------------------------------------------------------------------------------------------
def _inria_rows(rng, n, nrest, *, props):
    rows = []
    for _ in range(n):
        r = {k: 0 for k, _ in props}
        r.update(x=rng.uniform(-3, 3), y=rng.uniform(-3, 3), z=rng.uniform(-3, 3), opacity=rng.uniform(-6, 6))
        for k in range(3):
            r[f"f_dc_{k}"] = rng.uniform(-2, 2)
            r[f"scale_{k}"] = rng.uniform(-7, -1)
        for k in range(4):
            r[f"rot_{k}"] = rng.gauss(0, 1)
        for k in range(nrest):
            r[f"f_rest_{k}"] = rng.uniform(-0.5, 0.5)
        rows.append(r)
    return rows


def _inria(nrest, *, n=5, seed=0, header_lines=(), normals=True):
    props = [(k, "float") for k in (INRIA if normals else [k for k in INRIA if not k.startswith("n")])]
    props += [(f"f_rest_{k}", "float") for k in range(nrest)] + [(k, "float") for k in TAIL]
    rng = random.Random(seed)
    return props, _inria_rows(rng, n, nrest, props=props), header_lines


def fixture_sh0():
    return _inria(0, seed=1, header_lines=("comment Generated by a trainer", "obj_info num_cameras 12", "comment end of comments"), normals=False)


def fixture_sh1():
    return _inria(9, seed=2)


def fixture_sh2():
    return _inria(24, seed=3)


def fixture_sh3():
    return _inria(45, n=6, seed=4)


def fixture_shuffled():
    """Properties out of the usual order, extra properties of other types (one of them an unread double), f_rest of degree 1, short scales."""
    props = [("rot_2", "float"), ("extra_d", "double"), ("f_rest_3", "float"), ("z", "float"), ("scale_1", "short"), ("f_dc_2", "float"),
             ("rot_0", "float"), ("f_rest_0", "float"), ("label", "uchar"), ("x", "float"), ("f_rest_8", "float"), ("f_rest_1", "float"),
             ("scale_0", "short"), ("opacity", "float"), ("f_dc_0", "float"), ("f_rest_2", "float"), ("y", "float"), ("rot_3", "float"),
             ("f_rest_4", "float"), ("f_rest_5", "float"), ("nx", "float"), ("f_rest_6", "float"), ("scale_2", "short"), ("f_dc_1", "float"),
             ("f_rest_7", "float"), ("rot_1", "float"), ("ident", "uint")]
    rng = random.Random(5)
    rows = _inria_rows(rng, 7, 9, props=props)
    for r in rows:
        for k in range(3):
            r[f"scale_{k}"] = rng.randrange(-6, 2)
        r["extra_d"], r["label"], r["ident"] = rng.uniform(-1e300, 1e300), rng.randrange(256), rng.randrange(1 << 32)
    return props, rows, ()


def fixture_uchar_rgb():
    """uchar red/green/blue and no f_dc; no scale (0.01) and no opacity (alpha 0); a zero quaternion; uchar centre and rotation fields."""
    props = [("x", "float"), ("y", "uchar"), ("z", "float"), ("red", "uchar"), ("green", "uchar"), ("blue", "uchar"),
             ("rot_0", "float"), ("rot_1", "float"), ("rot_2", "uchar"), ("rot_3", "float")]
    rng = random.Random(6)
    rows = []
    for i in range(8):
        r = dict(x=rng.uniform(-2, 2), y=rng.randrange(256), z=rng.uniform(-2, 2), red=rng.randrange(256), green=rng.randrange(256),
                 blue=rng.randrange(256), rot_0=rng.gauss(0, 1), rot_1=rng.gauss(0, 1), rot_2=rng.randrange(256), rot_3=rng.gauss(0, 1))
        if i == 0:
            r.update(rot_0=0.0, rot_1=0.0, rot_2=0, rot_3=0.0)           # zero quaternion -> (0, 0, 0, 1)
        if i == 1:
            r.update(red=0, green=255, blue=1)
        rows.append(r)
    return props, rows, ()


def _opacity_typed(t, values, seed):
    props = [(k, "float") for k in ("x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2")] + [("opacity", t)] + \
            [(f"scale_{k}", "float") for k in range(3)] + [(f"rot_{k}", "float") for k in range(4)]
    rng = random.Random(seed)
    rows = _inria_rows(rng, len(values), 0, props=props)
    for r, v in zip(rows, values):
        r["opacity"] = v
    return props, rows, ()


def fixture_uchar_opacity():
    return _opacity_typed("uchar", [0, 1, 127, 128, 200, 255], 7)


def fixture_short_opacity():
    return _opacity_typed("short", [-32768, -6, -1, 0, 1, 6, 32767], 8)


def fixture_nonfinite():
    """NaN and +-inf in every kind of field, and colours that clamp at both ends."""
    props, rows, _ = _inria(9, n=9, seed=9, normals=False)
    rows[0].update(x=NAN, scale_0=NAN, f_dc_0=NAN, opacity=NAN, f_rest_0=NAN)
    rows[1].update(y=INF, scale_1=INF, f_dc_1=INF, opacity=INF, f_rest_4=INF)
    rows[2].update(z=-INF, scale_2=-INF, f_dc_2=-INF, opacity=-INF, f_rest_8=-INF)
    rows[3].update(rot_0=NAN)
    rows[4].update(rot_1=INF)
    rows[5].update(f_dc_0=100.0, f_dc_1=-100.0, f_dc_2=1.7724538509055159, scale_0=200.0)   # 255 / 0 / the 255 boundary / exp overflow
    rows[6].update(f_dc_0=-1.7724538509055159, f_rest_1=-0.0, scale_1=-200.0)
    rows[7].update(rot_0=1e-30, rot_1=0.0, rot_2=0.0, rot_3=0.0)
    rows[8].update(rot_0=3e38, rot_1=3e38, rot_2=3e38, rot_3=3e38)
    return props, rows, ()


def fixture_splat():
    rng = random.Random(10)
    rows = []
    for i in range(9):
        c = [rng.uniform(-4, 4) for _ in range(3)]
        s = [math.exp(rng.uniform(-6, -1)) for _ in range(3)]
        rgba = [rng.randrange(256) for _ in range(4)]
        q = [rng.randrange(256) for _ in range(4)]
        if i == 0:
            q = [128, 128, 128, 128]                                         # zero quaternion -> (0, 0, 0, 1), stored [1, 0, 0, 0]
        if i == 1:
            q = [255, 128, 128, 128]
        if i == 2:
            c[0], s[1] = NAN, INF
        rows.append((c, s, rgba, q))
    return rows


PLY_FIXTURES = {
    "sh0": fixture_sh0, "sh1": fixture_sh1, "sh2": fixture_sh2, "sh3": fixture_sh3, "shuffled": fixture_shuffled, "uchar_rgb": fixture_uchar_rgb,
    "uchar_opacity": fixture_uchar_opacity, "short_opacity": fixture_short_opacity, "nonfinite": fixture_nonfinite,
}
FILE_DEGREE = {"sh0": 0, "sh1": 1, "sh2": 2, "sh3": 2, "shuffled": 1, "uchar_rgb": 0, "uchar_opacity": 0, "short_opacity": 0, "nonfinite": 1}


def ply_fixture(name: str):
    """-> (file bytes, props, rows)"""
    props, rows, header_lines = PLY_FIXTURES[name]()
    return ply_bytes(props, rows, header_lines=header_lines), props, rows


def splat_fixture():
    rows = fixture_splat()
    return splat_bytes(rows), rows


def fixture_files() -> dict:
    """{file name: bytes} of every committed fixture."""
    out = {f"file_handmade_{name}.ply": ply_fixture(name)[0] for name in PLY_FIXTURES}
    out["file_handmade_basic.splat"] = splat_fixture()[0]
    return out


# ---- malformed files: (format, bytes, status, words the message must contain) -----------------------------------------------------------
def _ply_text(lines, body=b"\0" * 4096):
    return ("\n".join(lines) + "\n").encode("utf-8") + body


_GOOD = ["ply", "format binary_little_endian 1.0", "element vertex 2"] + [f"property float {k}" for k in ("x", "y", "z", "rot_0", "rot_1", "rot_2", "rot_3")]
BAD_ARG, CAPACITY = 1, 7
MALFORMED = {
    "no_end_header": (PLY, _ply_text(_GOOD), BAD_ARG, "end_header"),
    "end_header_crlf": (PLY, ("\r\n".join(_GOOD + ["end_header"]) + "\r\n").encode() + b"\0" * 64, BAD_ARG, "end_header"),
    "end_header_at_eof": (PLY, "\n".join(_GOOD + ["end_header"]).encode(), BAD_ARG, "end_header"),
    "non_ascii_header": (PLY, _ply_text(_GOOD[:2] + ["comment café"] + _GOOD[2:] + ["end_header"]), BAD_ARG, "ASCII"),
    "ascii_format": (PLY, _ply_text(["ply", "format ascii 1.0"] + _GOOD[2:] + ["end_header"]), BAD_ARG, "binary_little_endian"),
    "big_endian": (PLY, _ply_text(["ply", "format binary_big_endian 1.0"] + _GOOD[2:] + ["end_header"]), BAD_ARG, "binary_little_endian"),
    "property_list": (PLY, _ply_text(_GOOD + ["property list uchar int vertex_indices", "end_header"]), BAD_ARG, "property list"),
    "unknown_type": (PLY, _ply_text(_GOOD + ["property float32 nx", "end_header"]), BAD_ARG, "float32"),
    "double_read_property": (PLY, _ply_text(_GOOD[:3] + ["property double x"] + _GOOD[4:] + ["end_header"]), BAD_ARG, "double"),
    "missing_xyz": (PLY, _ply_text([g for g in _GOOD if not g.endswith(" z")] + ["end_header"]), BAD_ARG, "x, y or z"),
    "missing_rot": (PLY, _ply_text([g for g in _GOOD if not g.endswith("rot_3")] + ["end_header"]), BAD_ARG, "rot_0"),
    "f_rest_count": (PLY, _ply_text(_GOOD + [f"property float f_rest_{k}" for k in range(12)] + ["end_header"]), BAD_ARG, "f_rest"),
    "playcanvas": (PLY, _ply_text(["ply", "format binary_little_endian 1.0", "element chunk 1", "property float min_x", "element vertex 2",
                                   "property uint packed_position", "end_header"]), BAD_ARG, "PlayCanvas"),
    "inria_v2": (PLY, _ply_text(["ply", "format binary_little_endian 1.0", "element codebook_centers 4", "property float x"] + _GOOD[2:] + ["end_header"]),
                 BAD_ARG, "INRIA v2"),
    "short_body": (PLY, _ply_text(_GOOD + ["end_header"], body=b"\0" * 55), BAD_ARG, "shorter"),
    "splat_not_multiple_of_32": (SPLAT, b"\0" * 33, BAD_ARG, "32-byte"),
}


if __name__ == "__main__":
    for name, data in fixture_files().items():
        (HERE / name).write_bytes(data)
        print(name, len(data), "bytes")
