"""Hand-assembled PlayCanvas-compressed `.ply` fixtures + the level-0 SplatBuffer records expected from them.  TEST INFRASTRUCTURE ONLY.

Every file is written row by row with struct.pack, and every expected record is derived with scalar Python arithmetic straight from the
reference's semantics: PlayCanvasCompressedPlyParser.decompressBaseSplat (11-10-11 / 8888 unorm, lerp(a, b, t) = a (1 - t) + b t
between the chunk's extremes, Math.exp of the scale lerp, 2-10-10-10 smallest-three rotation, Math.round of the colour lerp when the
chunk has both extremes of a channel, else floor), decompressSphericalHarmonics (u8 (8 / 255) - 4 from f_rest_{j readCoeff + k}),
SplatBuffer.writeSplatDataToSectionBuffer level 0 (quaternion normalised once, `|| 0`, Float32Array stores).  NaN is stored as
0x7fc00000.  Imports neither the product package nor oracle/.

A zero-length quaternion cannot be encoded: a, b and c are (k / 1023 - 0.5) sqrt(2), never 0, and m² = 1 - (a² + b² + c²) whenever m
is real.  The rotation fixture covers the other end: patterns whose a² + b² + c² exceeds 1 (m and the stored quaternion are NaN).

`python tests/golden/pcply_handmade.py` rewrites tests/golden/pcply_handmade_*.ply (committed, a few KB each)."""
from __future__ import annotations

import math
import random
import struct
from pathlib import Path

HERE = Path(__file__).resolve().parent
PLY = 1
FMT = {"char": "b", "uchar": "B", "short": "h", "ushort": "H", "int": "i", "uint": "I", "float": "f", "double": "d"}
INF, NAN = float("inf"), float("nan")
POS_SCALE = ["min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y", "min_scale_z",
             "max_scale_x", "max_scale_y", "max_scale_z"]
COLOR = ["min_r", "min_g", "min_b", "max_r", "max_g", "max_b"]
PACKED = [("packed_position", "uint"), ("packed_rotation", "uint"), ("packed_scale", "uint"), ("packed_color", "uint")]
NORM = 1.0 / (math.sqrt(2) * 0.5)
SH_INDEX = [0, 1, 2, 9, 10, 11, 12, 13, 24, 25, 26, 27, 28, 29, 30,
            3, 4, 5, 14, 15, 16, 17, 18, 31, 32, 33, 34, 35, 36, 37,
            6, 7, 8, 19, 20, 21, 22, 23, 38, 39, 40, 41, 42, 43, 44]


def f32_bits(v: float) -> int:
    """Float32Array element assignment (round to nearest even, overflow to inf), NaN as 0x7fc00000."""
    if v != v:
        return 0x7FC00000
    try:
        return struct.unpack("<I", struct.pack("<f", v))[0]
    except OverflowError:
        # struct refuses finite values beyond float32's range: round-to-nearest there is +-inf unless the value rounds down to FLT_MAX
        flt_max = 3.4028234663852886e38
        half_ulp_above = flt_max + 2.0 ** 103
        if abs(v) < half_ulp_above:
            return struct.unpack("<I", struct.pack("<f", math.copysign(flt_max, v)))[0]
        return 0x7F800000 if v > 0 else 0xFF800000


def stored(v: float, t: str) -> float:
    """A chunk property as the reference's typed array holds it."""
    return struct.unpack("<" + FMT[t], struct.pack("<" + FMT[t], v))[0]


def pc_bytes(chunk_props, chunk_rows, vertex_props, vertex_rows, sh_rows=None, nsh=0, *, comments=()) -> bytes:
    head = ["ply", "format binary_little_endian 1.0", *[f"comment {c}" for c in comments], f"element chunk {len(chunk_rows)}",
            *[f"property {t} {n}" for n, t in chunk_props], f"element vertex {len(vertex_rows)}", *[f"property {t} {n}" for n, t in vertex_props]]
    body = b"".join(struct.pack("<" + "".join(FMT[t] for _, t in chunk_props), *[r[n] for n, _ in chunk_props]) for r in chunk_rows)
    body += b"".join(struct.pack("<" + "".join(FMT[t] for _, t in vertex_props), *[r[n] for n, _ in vertex_props]) for r in vertex_rows)
    if sh_rows is not None:
        head += [f"element sh {len(sh_rows)}", *[f"property uchar f_rest_{k}" for k in range(nsh)]]
        body += b"".join(bytes(r) for r in sh_rows)
    return ("\n".join(head + ["end_header"]) + "\n").encode("ascii") + body


def unorm(v: int, bits: int) -> float:
    t = (1 << bits) - 1
    return (v & t) / t


def lerp(a: float, b: float, t: float) -> float:
    return a * (1 - t) + b * t


def js_round(v: float) -> float:
    """Math.round by the spec: the nearest integer, ties towards +inf."""
    if v != v or v in (INF, -INF):
        return v
    r = float(math.floor(v))
    return r + 1 if v - r >= 0.5 else r


def clamp_u8(v: float) -> int:
    """clamp(v, 0, 255) then `|| 0` into a Uint8ClampedArray (v is an integer, +-inf or NaN here)."""
    if v != v:
        return 0
    return int(max(0.0, min(255.0, v)))


def exp_js(v: float) -> float:
    if v != v:
        return NAN
    try:
        return math.exp(v)
    except OverflowError:
        return INF


def mul(a: float, b: float) -> float:
    """IEEE product with JavaScript's inf * 0 = NaN (Python raises nothing here, but keep it explicit)."""
    return a * b


def normalize(x, y, z, w):
    """three.js Quaternion.normalize: l = sqrt(x x + y y + z z + w w); 0 -> (0, 0, 0, 1); else times 1 / l."""
    if any(v != v for v in (x, y, z, w)):
        return NAN, NAN, NAN, NAN
    ln = math.sqrt(x * x + y * y + z * z + w * w)
    if ln == 0:
        return 0.0, 0.0, 0.0, 1.0
    il = 1 / ln
    return x * il, y * il, z * il, w * il


def unpack_rot(v: int):
    a = (unorm(v >> 20, 10) - 0.5) * NORM
    b = (unorm(v >> 10, 10) - 0.5) * NORM
    c = (unorm(v, 10) - 0.5) * NORM
    s = (a * a + b * b) + c * c
    m = math.sqrt(1.0 - s) if 1.0 - s >= 0 else NAN
    return [(m, a, b, c), (a, m, b, c), (a, b, m, c), (a, b, c, m)][v >> 30]


def expected(chunk_props, chunk_rows, vertex_rows, sh_rows, nsh, sh_degree: int) -> tuple[bytes, int]:
    """Level-0 records of a compressed file, and the output SH degree."""
    types = dict(chunk_props)
    file_deg = 3 if nsh >= 45 else (2 if nsh >= 24 else (1 if nsh >= 9 else 0))
    deg = min(sh_degree, file_deg)
    out_coeff, read_coeff = [0, 3, 8][deg], [0, 3, 8, 15][file_deg]
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    out = b""
    for i, r in enumerate(vertex_rows):
        ch = chunk_rows[i // 256]
        e = lambda k: stored(ch[k], types[k])  # noqa: E731
        pos, scl, col = r["packed_position"], r["packed_scale"], r["packed_color"]
        p = [unorm(pos >> 21, 11), unorm(pos >> 11, 10), unorm(pos, 11)]
        s = [unorm(scl >> 21, 11), unorm(scl >> 11, 10), unorm(scl, 11)]
        rec = struct.pack("<3I", *(f32_bits(lerp(e(f"min_{a}"), e(f"max_{a}"), p[k])) for k, a in enumerate("xyz")))
        sc = [exp_js(lerp(e(f"min_scale_{a}"), e(f"max_scale_{a}"), s[k])) for k, a in enumerate("xyz")]
        rec += struct.pack("<3I", *(f32_bits(0.0 if v != v else v) for v in sc))
        rec += struct.pack("<4I", *(f32_bits(v) for v in normalize(*unpack_rot(r["packed_rotation"]))))
        rgba = []
        for k, a in enumerate("rgb"):
            c = unorm(col >> (24 - 8 * k), 8)
            if f"min_{a}" in types and f"max_{a}" in types:
                rgba.append(clamp_u8(js_round(mul(lerp(e(f"min_{a}"), e(f"max_{a}"), c), 255))))
            else:
                rgba.append(clamp_u8(math.floor(c * 255)))
        rgba.append(clamp_u8(math.floor(unorm(col, 8) * 255)))
        rec += bytes(rgba)
        if ncomp:
            frc = [0.0] * 45
            for j in range(3):
                for k in range(15):
                    if k < out_coeff and k < read_coeff:
                        frc[SH_INDEX[j * 15 + k]] = sh_rows[i][j * read_coeff + k] * (8 / 255) - 4
            rec += b"".join(struct.pack("<I", f32_bits(frc[s_] or 0.0)) for s_ in range(ncomp))
        out += rec
    return out, deg


# ---- fixtures -------------------------------------------------------------------------------------------------------------------------
def _chunk(rng, colors: str, types=None):
    """One chunk row: extremes of position (-4..4), log-scale (-7..-1) and, for the channels in `colors`, colour (around 0..1)."""
    r = {}
    for a in "xyz":
        lo = rng.uniform(-4, 0)
        r[f"min_{a}"], r[f"max_{a}"] = lo, lo + rng.uniform(0.5, 4)
        lo = rng.uniform(-7, -4)
        r[f"min_scale_{a}"], r[f"max_scale_{a}"] = lo, lo + rng.uniform(0.5, 3)
    for a in colors:
        lo = rng.uniform(-0.2, 0.4)
        r[f"min_{a}"], r[f"max_{a}"] = lo, lo + rng.uniform(0.3, 1.0)
    return r


def _chunk_props(colors: str, ctype="float"):
    return [(k, "float") for k in POS_SCALE] + [(f"{m}_{a}", ctype) for m in ("min", "max") for a in colors]


def _vertex(rng):
    return {n: rng.randrange(1 << 32) for n, _ in PACKED}


def _build(n, n_chunks, colors, nsh, seed, *, extra=(), comments=(), ctype="float"):
    rng = random.Random(seed)
    chunk_props = _chunk_props(colors, ctype)
    chunk_rows = [_chunk(rng, colors) for _ in range(n_chunks)]
    vertex_props = [*extra, *PACKED]
    vertex_rows = []
    for _ in range(n):
        r = _vertex(rng)
        for name, t in extra:
            r[name] = rng.randrange(256) if t == "uchar" else rng.uniform(-1, 1)
        vertex_rows.append(r)
    sh_rows = [[rng.randrange(256) for _ in range(nsh)] for _ in range(n)] if nsh else None
    return dict(chunk_props=chunk_props, chunk_rows=chunk_rows, vertex_props=vertex_props, vertex_rows=vertex_rows, sh_rows=sh_rows,
                nsh=nsh, comments=comments)


def fixture_sh0():
    """No sh element, colour extremes on every channel, 300 splats over two chunks (the second one partial), comment lines."""
    return _build(300, 2, "rgb", 0, 1, comments=("Generated by the compressor", "vertices 300"))


def fixture_sh1():
    """No colour extremes (floor path), more chunk rows than needed, an extra vertex property ahead of the packed words."""
    return _build(5, 3, "", 9, 2, extra=(("tag", "uchar"), ("weight", "float")))


def fixture_sh2():
    """Only the green channel has extremes; 24 f_rest bytes per splat."""
    return _build(40, 1, "g", 24, 3)


def fixture_sh3():
    """45 f_rest bytes (read as degree 2), 261 splats over two chunks, double colour extremes."""
    return _build(261, 2, "rgb", 45, 4, ctype="double")


def fixture_edges():
    """Chunk 0: every largest-component slot, NaN rotations (a² + b² + c² > 1), colour lerps clamping at 0 and 255 and one landing on
    127.5 (Math.round -> 128).  Chunk 1: NaN and +-inf extremes (NaN centre, exp(inf) scale, inf * 0 in a lerp, -inf colour); a blue lerp
    landing exactly on 0.5 (Math.round -> 1, where round-half-even gives 0) and one on 1.5 - 2^-52 (-> 1).  Colour extremes are double,
    so the lerp can hit those values exactly.  No colour lerp can land on 0.49999999999999994: no double times 255 rounds to it."""
    d = _build(264, 2, "rgb", 0, 5, ctype="double")
    c0, c1 = d["chunk_rows"]
    c0.update(min_r=0.5, max_r=0.75, min_g=-2.0, max_g=-1.0, min_b=1.5, max_b=3.0)
    c1.update(min_x=NAN, max_y=INF, min_z=-INF, max_scale_x=INF, min_scale_y=NAN, min_r=-INF, max_g=INF,
              min_b=0.00196078431372549, max_b=0.00588235294117647)     # times 255: exactly 0.5, and 1.5 - 2^-52
    rows = d["vertex_rows"]
    for s in range(4):   # slot s, a = b = c = 0.5 +- : m real
        rows[s]["packed_rotation"] = (s << 30) | (511 << 20) | (600 << 10) | 400
    for s in range(4):   # all three at the 10-bit extremes: a² + b² + c² = 1.5 -> NaN
        rows[4 + s]["packed_rotation"] = (s << 30) | (0 << 20) | (1023 << 10) | 0
    rows[8]["packed_color"] = 0x00000080                      # r lerp t = 0 -> 0.5 * 255 = 127.5 -> 128; g below 0; b above 1
    rows[9]["packed_color"] = 0xFFFFFFFF
    rows[256]["packed_position"], rows[256]["packed_scale"] = 0, 0
    rows[257]["packed_position"], rows[257]["packed_scale"] = 0xFFFFFFFF, 0xFFFFFFFF
    rows[258]["packed_color"] = 0x12345600                    # blue t = 0: min_b 255 = 0.5
    rows[259]["packed_color"] = 0x1234FF00                    # blue t = 1: max_b 255 = 1.5 - 2^-52
    return d


PC_FIXTURES = {"sh0": fixture_sh0, "sh1": fixture_sh1, "sh2": fixture_sh2, "sh3": fixture_sh3, "edges": fixture_edges}
FILE_DEGREE = {"sh0": 0, "sh1": 1, "sh2": 2, "sh3": 2, "edges": 0}


def pc_fixture(name: str):
    """-> (file bytes, fixture dict)"""
    d = PC_FIXTURES[name]()
    return pc_bytes(d["chunk_props"], d["chunk_rows"], d["vertex_props"], d["vertex_rows"], d["sh_rows"], d["nsh"], comments=d["comments"]), d


def expected_records(name: str, sh_degree: int) -> tuple[bytes, int]:
    d = PC_FIXTURES[name]()
    return expected(d["chunk_props"], d["chunk_rows"], d["vertex_rows"], d["sh_rows"], d["nsh"], sh_degree)


def fixture_files() -> dict:
    """{file name: bytes} of every committed fixture."""
    return {f"pcply_handmade_{name}.ply": pc_fixture(name)[0] for name in PC_FIXTURES}


# ---- malformed compressed files: (bytes, words the message must contain) ---------------------------------------------------------------
BAD_ARG = 1
_CHUNK = ["element chunk 1"] + [f"property float {k}" for k in POS_SCALE]
_VERTEX = ["element vertex 2"] + [f"property uint {k}" for k, _ in PACKED]
_SH = ["element sh 2"] + [f"property uchar f_rest_{k}" for k in range(9)]
_HEAD = ["ply", "format binary_little_endian 1.0"]
_BODY = b"\0" * (48 + 2 * 16 + 2 * 9)


def _text(lines, body=_BODY):
    return ("\n".join(lines + ["end_header"]) + "\n").encode("ascii") + body


PREFIX = ".ply: PlayCanvas compressed .ply:"
MALFORMED = {
    "element_order": (_text(_HEAD + _VERTEX + _CHUNK), "element 'vertex'"),
    "unknown_element": (_text(_HEAD + _CHUNK + _VERTEX + ["element face 0"]), "element 'face'"),
    "no_vertex": (_text(_HEAD + _CHUNK), "vertex element"),
    "obj_info": (_text(_HEAD + ["obj_info generator"] + _CHUNK + _VERTEX), "header keyword 'obj_info'"),
    "empty_line": (_text(_HEAD + [""] + _CHUNK + _VERTEX), "empty header line"),
    "property_list": (_text(_HEAD + _CHUNK + _VERTEX + ["property list uchar int idx"]), "property list"),
    "unknown_type": (_text(_HEAD + _CHUNK + _VERTEX + ["property float32 w"]), "float32"),
    "missing_max_z": (_text(_HEAD + [ln for ln in _CHUNK if not ln.endswith(" max_z")] + _VERTEX), "max_z"),
    "missing_scale": (_text(_HEAD + [ln for ln in _CHUNK if not ln.endswith(" min_scale_y")] + _VERTEX), "min_scale_y"),
    "missing_packed": (_text(_HEAD + _CHUNK + [ln for ln in _VERTEX if not ln.endswith("packed_color")]), "packed_color"),
    "packed_not_uint": (_text(_HEAD + _CHUNK + [ln.replace("uint packed_scale", "int packed_scale") for ln in _VERTEX]), "uint"),
    "too_few_chunks": (_text(_HEAD + ["element chunk 1"] + _CHUNK[1:] + ["element vertex 257"] + _VERTEX[1:], b"\0" * 8192), "chunk rows"),
    "sh_rows": (_text(_HEAD + _CHUNK + _VERTEX + ["element sh 3"] + _SH[1:]), "rows"),
    "sh_count": (_text(_HEAD + _CHUNK + _VERTEX + _SH[:-1]), "8 properties"),
    "sh_names": (_text(_HEAD + _CHUNK + _VERTEX + _SH[:-1] + ["property uchar f_rest_9"]), "f_rest_0 .. f_rest_8"),
    "sh_type": (_text(_HEAD + _CHUNK + _VERTEX + _SH[:-1] + ["property float f_rest_8"]), "uchar"),
    "duplicate": (_text(_HEAD + _CHUNK + ["property float min_x"] + _VERTEX), "declared twice"),
    "short_body": (_text(_HEAD + _CHUNK + _VERTEX + _SH, body=_BODY[:-1]), "shorter"),
    "ascii_format": (_text(["ply", "format ascii 1.0"] + _CHUNK + _VERTEX), "binary_little_endian"),
}


if __name__ == "__main__":
    for name, data in fixture_files().items():
        (HERE / name).write_bytes(data)
        print(name, len(data), "bytes")
