"""Handmade INRIA v2 (codebook) `.ply` fixtures and the level-0 records derived for them here, splat by splat, with scalar arithmetic
(Python floats are JavaScript numbers).  Run this file to rewrite the fixtures: `python tests/golden/inriav2_handmade.py`.

The derivation restates INRIAV2PlyParser.decodeCodeBook + parseToUncompressedSplat + the level-0 writer:
  codebook  fromHalfFloat(entry), 0 when the row lacks the entry; opacity Math.round(sigmoid(v) 255), features_dc
            Math.round((0.5 + SH_C0 v) 255), scaling Math.exp(v), the other pages v
  lookup    codeBook[page][index]; an index outside 0 .. rows - 1 is `undefined`, NaN from then on
  centre    fromHalfFloat(x | y | z)
  scale     codeBook[scaling][scale_k] (0.01 without scale_*), the writer's `|| 0`; all three 0 when the scale_0 index names no row
            (the writer tests scale_0 !== undefined)
  rotation  Quaternion(re[rot_0], im[rot_1], im[rot_2], im[rot_3]) normalised twice; stored x, y, z, w
  colour    clamp(floor(codeBook[features_dc][f_dc_k]), 0, 255), 0 without f_dc_* (red/green/blue are never read); NaN -> 0
  alpha     clamp(floor(codeBook[opacity][opacity]), 0, 255), 0 without opacity
  SH        slot s < 9 from page features_rest_(s % 3) at f_rest_(s % 3 + c (s / 3)), slot 9 + s from features_rest_(3 + s % 5) at
            f_rest_(3 + s % 5 + c (s / 5)), c = f_rest count / 3; min(requested, file degree) read, the image at the requested
            degree with 0 past them; the writer's `|| 0`
"""
from __future__ import annotations

import math
import struct
from pathlib import Path

HERE = Path(__file__).resolve().parent
PLY = 1
BAD_ARG = 1
SH_C0 = 0.28209479177387814
PAGES = ["features_dc"] + [f"features_rest_{k}" for k in range(15)] + ["opacity", "scaling", "rotation_re", "rotation_im"]
_FMT = {"uchar": "B", "short": "h", "ushort": "H", "int": "i", "uint": "I", "float": "f", "double": "d"}
NAN = float("nan")


# ---- scalar derivation -------------------------------------------------------------------------------------------------------------
def _f32_bits(v: float) -> bytes:
    if v != v:
        return struct.pack("<I", 0x7FC00000)
    if abs(v) != math.inf and abs(v) >= 3.4028235677973366e38:     # rounds to f32 infinity
        v = math.copysign(math.inf, v)
    return struct.pack("<f", v)


def _half(h: int) -> float:
    h &= 0xFFFF
    sign = -1.0 if (h >> 15) & 1 else 1.0
    e, m = (h >> 10) & 31, h & 1023
    if e == 0:
        return sign * 2.0 ** -14 * m / 1024
    if e == 31:
        return NAN if m else sign * math.inf
    return sign * 2.0 ** (e - 15) * (1 + m / 1024)


def _exp(v: float) -> float:
    try:
        return math.exp(v)
    except OverflowError:
        return math.inf


def _round(v: float) -> float:
    if v != v or abs(v) == math.inf:
        return v
    r = math.floor(v)
    return r + 1.0 if v - r >= 0.5 else float(r)


def _u8(v: float) -> int:
    if v != v:
        return 0
    if abs(v) == math.inf:
        return 255 if v > 0 else 0
    return min(max(math.floor(v), 0), 255)


def _normalize(x, y, z, w):
    ln = math.sqrt(x * x + y * y + z * z + w * w)
    if ln == 0:
        return 0.0, 0.0, 0.0, 1.0
    il = 1.0 / ln
    return x * il, y * il, z * il, w * il


def page_value(page: int, bits) -> float:
    v = 0.0 if bits is None else _half(bits)
    if PAGES[page] == "opacity":
        return _round((1 / (1 + _exp(-v))) * 255)
    if PAGES[page] == "features_dc":
        return _round((0.5 + SH_C0 * v) * 255)
    if PAGES[page] == "scaling":
        return _exp(v)
    return v


def record(fx: dict, s: dict, sh_degree: int) -> bytes:
    """One splat's level-0 record at the requested SH degree."""
    cb = fx["codebook"]
    names = {k for k, _ in fx["splat_props"]}

    def look(page: int, field: str) -> float:
        i = s.get(field, 0)
        if not 0 <= i < len(cb):
            return NAN
        return page_value(page, cb[i].get(PAGES[page]) if PAGES[page] in {k for k, _ in fx["cb_props"]} else None)

    out = b"".join(_f32_bits(_half(s.get(k, 0))) for k in "xyz")
    scale_read = "scale_0" in names and 0 <= s.get("scale_0", 0) < len(cb)     # the writer: scale_0 !== undefined
    for k in range(3):
        v = (look(17, f"scale_{k}") if scale_read else 0.0) if "scale_0" in names else 0.01
        out += _f32_bits(0.0 if v != v else v)
    q = (look(18, "rot_0"), look(19, "rot_1"), look(19, "rot_2"), look(19, "rot_3"))
    out += b"".join(_f32_bits(v) for v in _normalize(*_normalize(*q)))
    out += bytes(_u8(look(0, f"f_dc_{k}")) if "f_dc_0" in names else 0 for k in range(3))
    out += bytes([_u8(look(16, "opacity")) if "opacity" in names else 0])
    rest = sum(1 for k in names if k.startswith("f_rest"))
    c = rest // 3
    file_deg = 2 if c >= 8 else (1 if c >= 3 else 0)
    nread, ncomp = [0, 9, 24][min(sh_degree, file_deg)], [0, 9, 24][sh_degree]
    for k in range(ncomp):
        v = 0.0
        if k < nread:
            if k < 9:
                v = look(1 + k % 3, f"f_rest_{k % 3 + c * (k // 3)}")
            else:
                v = look(4 + (k - 9) % 5, f"f_rest_{3 + (k - 9) % 5 + c * ((k - 9) // 5)}")
        out += _f32_bits(0.0 if v != v or v == 0 else v)
    return out


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def ply_bytes(fx: dict) -> bytes:
    """Header, then the two elements' rows in header order, written row by row."""
    def element(name, props, rows):
        head = [f"element {name} {len(rows)}", *[f"property {t} {k}" for k, t in props]]
        body = b"".join(b"".join(struct.pack("<" + _FMT[t], r.get(k, 0)) for k, t in props) for r in rows)
        return head, body
    cb = element("codebook_centers", fx["cb_props"], fx["codebook"])
    sp = element("vertex", fx["splat_props"], fx["splats"])
    parts = [cb, sp] if fx.get("codebook_first", True) else [sp, cb]
    head = ["ply", "format binary_little_endian 1.0", "comment INRIA v2 handmade fixture", *parts[0][0], *parts[1][0], "end_header"]
    return ("\n".join(head) + "\n").encode("ascii") + parts[0][1] + parts[1][1]


# float16: +-0, smallest and largest subnormal, smallest normal, 1, -1, 65504, +-inf, NaN (quiet and signalling payloads), 1/3
HALVES = [0x0000, 0x8000, 0x0001, 0x8001, 0x03FF, 0x0400, 0x3C00, 0xBC00, 0x7BFF, 0x7C00, 0xFC00, 0x7E00, 0x7C01, 0xFFFF, 0x3555]
_BASE = [("scale_0", "ushort"), ("scale_1", "ushort"), ("scale_2", "ushort"), ("rot_0", "ushort"), ("rot_1", "ushort"), ("rot_2", "ushort"),
         ("rot_3", "ushort"), ("x", "ushort"), ("y", "ushort"), ("z", "ushort"), ("f_dc_0", "ushort"), ("f_dc_1", "ushort"),
         ("f_dc_2", "ushort"), ("opacity", "ushort")]
_ALL_PAGES = [(k, "ushort") for k in PAGES]


def _codebook(rows: int) -> list[dict]:
    """Rows of distinct, ordinary halves per page (|v| < 4, so every exp is far from overflow); row 0 is all zeros."""
    out = []
    for r in range(rows):
        row = {}
        for p, name in enumerate(PAGES):
            if r == 0:
                row[name] = 0x0000
            else:
                v = ((r * 37 + p * 11) % 61 - 30) / 8.0
                row[name] = struct.unpack("<H", struct.pack("<e", v))[0]
        out.append(row)
    return out


def _splats(n: int, rows: int, rest: int, **fixed) -> list[dict]:
    out = []
    for i in range(n):
        s = {k: (i * 7 + j * 3 + 1) % rows for j, (k, _) in enumerate(_BASE)}
        s.update({k: struct.unpack("<H", struct.pack("<e", ((i * 13 + j * 5) % 41 - 20) / 4.0))[0] for j, k in enumerate("xyz")})
        s.update({f"f_rest_{k}": (i * 5 + k * 2 + 1) % rows for k in range(rest)})
        s.update(fixed)
        out.append(s)
    return out


def _sh_case(rest: int, index_type: str = "ushort", rows: int = 9) -> dict:
    props = [(k, "ushort" if k in "xyz" else index_type) for k, _ in _BASE] + [(f"f_rest_{k}", index_type) for k in range(rest)]
    splats = _splats(12, rows, rest)
    splats[0].update({k: 0 for k in ("rot_0", "rot_1", "rot_2", "rot_3", "f_dc_0", "f_dc_1", "f_dc_2", "opacity")})  # zero rotation, ties
    return dict(cb_props=_ALL_PAGES, codebook=_codebook(rows), splat_props=props, splats=splats)


def _halves_case() -> dict:
    """Every page row r and every centre holds an edge half; the splats read rows in several rotations of the list."""
    rows = len(HALVES)
    cb = [{name: HALVES[(r + p) % rows] for p, name in enumerate(PAGES)} for r in range(rows)]
    rest = 24
    props = list(_BASE) + [(f"f_rest_{k}", "ushort") for k in range(rest)]
    splats = []
    for i in range(2 * rows):
        s = {k: (i + j) % rows for j, (k, _) in enumerate(_BASE)}
        s.update({k: HALVES[(i + 5 * j) % rows] for j, k in enumerate("xyz")})
        s.update({f"f_rest_{k}": (i + k) % rows for k in range(rest)})
        splats.append(s)
    return dict(cb_props=_ALL_PAGES, codebook=cb, splat_props=props, splats=splats)


def _indices_case() -> dict:
    """short, uint, int and uchar indices, with negative and too-large ones: those read NaN."""
    rows = 6
    types = {"scale_0": "short", "scale_1": "uint", "scale_2": "int", "rot_0": "short", "rot_1": "uint", "rot_2": "int", "rot_3": "uchar",
             "f_dc_0": "short", "f_dc_1": "uint", "f_dc_2": "int", "opacity": "short"}
    props = [(k, types.get(k, "ushort")) for k, _ in _BASE] + [(f"f_rest_{k}", "short" if k % 2 else "uint") for k in range(9)]
    bad = {"short": [-1, -32768, 6, 32767], "uint": [6, 7, 65536, 0xFFFFFFFF], "int": [-1, 6, -2147483648, 2147483647], "uchar": [6, 255, 200, 7]}
    splats = _splats(10, rows, 9)
    for i, s in enumerate(splats[:4]):
        for k, t in props:
            if k not in "xyz" and (i + len(k)) % 2 == 0:
                s[k] = bad[t][i]
    splats[4]["scale_0"] = -1                 # only scale_0 names no row: all three scales 0
    splats[5]["scale_1"] = 6                  # only scale_1: that scale alone 0
    splats[6]["scale_2"] = -2147483648        # only scale_2
    splats[7]["scale_0"] = 6                  # scale_0 too large, scale_1 and scale_2 valid
    return dict(cb_props=_ALL_PAGES, codebook=_codebook(rows), splat_props=props, splats=splats)


def _absent_pages_case() -> dict:
    """The codebook lacks opacity, scaling and features_dc: opacity reads 128, scale 1, colour 128 wherever an index is valid."""
    c = _sh_case(9)
    c["cb_props"] = [(k, "ushort") for k in PAGES if k not in ("opacity", "scaling", "features_dc")]
    c["splats"][1]["opacity"] = 50                                                        # invalid all the same
    return c


def _absent_fields_case() -> dict:
    """The splats lack scale_* and f_dc_*: scale 0.01, colour 0 (red/green/blue are present and never read)."""
    c = _sh_case(0)
    drop = {"scale_0", "scale_1", "scale_2", "f_dc_0", "f_dc_1", "f_dc_2"}
    c["splat_props"] = [p for p in c["splat_props"] if p[0] not in drop] + [("red", "uchar"), ("green", "uchar"), ("blue", "uchar")]
    for i, s in enumerate(c["splats"]):
        s.update(red=200, green=100 + i, blue=3)
    return c


def _padding_case() -> dict:
    """Unknown properties of every type in both elements, between the ones read."""
    c = _sh_case(24, "uchar")
    c["cb_props"] = [("pad_a", "double")] + c["cb_props"][:7] + [("nx", "float"), ("pad_b", "uchar")] + c["cb_props"][7:] + [("pad_c", "int")]
    c["splat_props"] = [("nx", "float"), ("ny", "double")] + c["splat_props"][:5] + [("pad", "uchar")] + c["splat_props"][5:] + [("last", "short")]
    for s in c["splats"]:
        s.update(nx=1.5, ny=-2.25, pad=7, last=-3)
    return c


def _codebook_last_case() -> dict:
    c = _sh_case(45, "ushort", rows=11)
    c["codebook_first"] = False
    return c


FIXTURES = {
    "sh0": _sh_case(0),
    "sh1": _sh_case(9, "uchar"),
    "sh2": _sh_case(24, "short"),
    "sh3": _sh_case(45, "uint"),
    "codebook_last": _codebook_last_case(),
    "absent_pages": _absent_pages_case(),
    "absent_fields": _absent_fields_case(),
    "indices": _indices_case(),
    "halves": _halves_case(),
    "padding": _padding_case(),
    "empty": dict(cb_props=_ALL_PAGES, codebook=_codebook(3), splat_props=_sh_case(9)["splat_props"], splats=[]),
}


def file_degree(name: str) -> int:
    rest = sum(1 for k, _ in FIXTURES[name]["splat_props"] if k.startswith("f_rest"))
    return 2 if rest >= 24 else (1 if rest >= 9 else 0)


def fixture(name: str) -> bytes:
    return ply_bytes(FIXTURES[name])


def file_name(name: str) -> str:
    """Not `*_handmade*.ply`: the tests that load every such file in file order (gs_upload_file) do not apply to this flavour."""
    return f"inriav2_codebook_{name}.ply"


def expected_records(name: str, sh_degree: int) -> bytes:
    fx = FIXTURES[name]
    return b"".join(record(fx, s, sh_degree) for s in fx["splats"])


# ---- malformed files: name -> (bytes, words the message must contain) ---------------------------------------------------------------
def _text(lines, body=b"\0" * 4096) -> bytes:
    return ("\n".join(lines) + "\n").encode("ascii") + body


_CB = ["element codebook_centers 4"] + [f"property ushort {k}" for k in PAGES]
_SP = ["element vertex 2"] + [f"property ushort {k}" for k in ("x", "y", "z", "rot_0", "rot_1", "rot_2", "rot_3")]
_HEAD = ["ply", "format binary_little_endian 1.0"]


def _swap(lines, old, new):
    return [new if ln == old else ln for ln in lines]


MALFORMED = {
    "ascii_format": (_text(["ply", "format ascii 1.0"] + _CB + _SP + ["end_header"]), "binary_little_endian"),
    "no_format": (_text(["ply"] + _CB + _SP + ["end_header"]), "no 'format"),
    "property_list": (_text(_HEAD + _CB + _SP + ["property list uchar int vertex_indices", "end_header"]), "property list"),
    "property_list_codebook": (_text(_HEAD + _CB + ["property list uchar int idx"] + _SP + ["end_header"]), "property list"),
    "unknown_type": (_text(_HEAD + _CB + _SP + ["property float32 nx", "end_header"]), "float32"),
    "char_type": (_text(_HEAD + _CB + _SP + ["property char nx", "end_header"]), "'char' unknown"),
    "duplicate": (_text(_HEAD + _CB + _SP + ["property ushort rot_0", "end_header"]), "declared twice"),
    "duplicate_codebook": (_text(_HEAD + _CB + ["property ushort opacity"] + _SP + ["end_header"]), "declared twice"),
    "property_first": (_text(_HEAD + ["property ushort x"] + _CB + _SP + ["end_header"]), "before the first element"),
    "missing_xyz": (_text(_HEAD + _CB + _swap(_SP, "property ushort z", "property ushort w") + ["end_header"]), "x, y or z"),
    "missing_rot": (_text(_HEAD + _CB + _swap(_SP, "property ushort rot_3", "property ushort rot_4") + ["end_header"]), "rot_0"),
    "scale_group": (_text(_HEAD + _CB + _SP + ["property uchar scale_0", "end_header"]), "scale_0..scale_2"),
    "dc_group": (_text(_HEAD + _CB + _SP + ["property uchar f_dc_0", "property uchar f_dc_1", "end_header"]), "f_dc_0..f_dc_2"),
    "f_rest_count": (_text(_HEAD + _CB + _SP + [f"property uchar f_rest_{k}" for k in range(12)] + ["end_header"]), "12 f_rest"),
    "f_rest_names": (_text(_HEAD + _CB + _SP + [f"property uchar f_rest_{k + 1}" for k in range(9)] + ["end_header"]), "f_rest_0 .. f_rest_8"),
    "short_body": (_text(_HEAD + _CB + _SP + ["end_header"], body=b"\0" * (4 * 40 + 2 * 14 - 1)), "shorter"),
    "no_codebook_rows_body": (_text(_HEAD + _CB + _SP + ["end_header"], body=b""), "shorter"),
    "two_codebooks": (_text(_HEAD + _CB + _SP + _CB + ["end_header"]), "exactly one codebook_centers"),
    "two_splat_elements": (_text(_HEAD + _CB + _SP + _SP + ["end_header"]), "exactly one codebook_centers"),
    "codebook_only": (_text(_HEAD + _CB + ["end_header"]), "exactly one codebook_centers"),
    "float_x": (_text(_HEAD + _CB + _swap(_SP, "property ushort x", "property float x") + ["end_header"]), "'x' must be a ushort or short"),
    "uchar_z": (_text(_HEAD + _CB + _swap(_SP, "property ushort z", "property uchar z") + ["end_header"]), "'z' must be a ushort or short"),
    "double_y": (_text(_HEAD + _CB + _swap(_SP, "property ushort y", "property double y") + ["end_header"]), "double"),
    "float_index": (_text(_HEAD + _CB + _swap(_SP, "property ushort rot_2", "property float rot_2") + ["end_header"]), "codebook index"),
    "float_f_rest": (_text(_HEAD + _CB + _SP + [f"property float f_rest_{k}" for k in range(9)] + ["end_header"]), "codebook index"),
    "double_opacity": (_text(_HEAD + _CB + _SP + ["property double opacity", "end_header"]), "double"),
    "float_entry": (_text(_HEAD + _swap(_CB, "property ushort scaling", "property float scaling") + _SP + ["end_header"]),
                    "codebook entry 'scaling' must be a ushort or short"),
    "uchar_entry": (_text(_HEAD + _swap(_CB, "property ushort features_dc", "property uchar features_dc") + _SP + ["end_header"]),
                    "codebook entry 'features_dc'"),
    "too_many_rows": (_text(_HEAD + ["element codebook_centers 1048577", "property ushort opacity"] + _SP + ["end_header"]),
                      "codebook of 1048577 rows (at most 1048576)"),
}
for _v in MALFORMED.values():
    assert _v[0].startswith(b"ply\n")


def fixture_files() -> dict[str, bytes]:
    return {file_name(k): fixture(k) for k in FIXTURES}


if __name__ == "__main__":
    for fname, data in fixture_files().items():
        (HERE / fname).write_bytes(data)
        print(fname, len(data))
