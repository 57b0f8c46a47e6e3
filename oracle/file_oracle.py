"""oracle/file_oracle.py -- TEST INFRASTRUCTURE ONLY.  Imports nothing from the product package.

NumPy restatement of the level-0 `.ksplat` image the reference's progressive loader builds from a `.ply` or `.splat` file (file order,
one compression-level-0 SplatBuffer section, no splat removed):
  .ply    PlyLoader.js:192-206 -> INRIAV1PlyParser.parseToUncompressedSplat (:143-207, readVertex with normalize = true,
          PlyParserUtils.js:278-302) -> SplatBuffer.writeSplatDataToSectionBuffer, level 0 (SplatBuffer.js:1092-1124, 1168-1172)
  .splat  SplatLoader.js:108 -> SplatParser.parseToUncompressedSplatBufferSection (SplatParser.js:13-56)
  header  writeHeaderToBuffer (:856-875) / writeSectionHeaderToBuffer (:944-961) as the loaders call them, with the final counts
Every step is JavaScript-number (f64, unfused) arithmetic; NumPy does not contract.  NaN lands in the image as 0x7fc00000.

Two kinds of value depend on how a libm rounds `exp` (the reference's V8, NumPy and CUDA may each be 1 ulp off): a scale whose f64
exp lies within 2 f64 ulps of an f32 rounding midpoint, and an alpha whose floor(255 * sigmoid) changes when exp(-opacity) moves by
2 f64 ulps (255 * sigmoid within a few ulps of an integer).  `level0_image` flags those splats in its `ambiguous` mask.

Also: vectorised writers for test inputs (`write_ply`: any property order, any of the seven scalar types, extra properties;
`write_splat`).
"""
from __future__ import annotations

import re
import struct

import numpy as np

PLY = 1
SPLAT = 2
SH_C0 = 0.28209479177387814
_TYPES = {"double": "<f8", "int": "<i4", "uint": "<u4", "float": "<f4", "short": "<i2", "ushort": "<u2", "uchar": "u1"}
_CANON_NAN = np.uint32(0x7FC00000)


# ---- writers (test inputs) ---------------------------------------------------------------------------------------------------------
def write_ply(props: list[tuple[str, str]], columns: dict, count: int, *, comments=(), extra_header=()) -> bytes:
    """props: [(name, type)] in file order; columns[name]: values (cast to the property's type; absent = zeros)."""
    dt = np.dtype([(n, _TYPES[t]) for n, t in props])
    rec = np.zeros(count, dt)
    for n, _ in props:
        if n in columns:
            rec[n] = np.asarray(columns[n]).astype(dt[n])
    lines = ["ply", "format binary_little_endian 1.0", *[f"comment {c}" for c in comments], *extra_header, f"element vertex {count}",
             *[f"property {t} {n}" for n, t in props], "end_header"]
    return ("\n".join(lines) + "\n").encode("ascii") + rec.tobytes()


def write_splat(centers, scales, rgba, rot_u8) -> bytes:
    """32-byte rows: centre f32x3, scale f32x3, RGBA u8x4, rotation u8x4 (w, x, y, z around 128)."""
    n = len(centers)
    dt = np.dtype([("c", "<f4", 3), ("s", "<f4", 3), ("rgba", "u1", 4), ("q", "u1", 4)])
    rec = np.zeros(n, dt)
    rec["c"], rec["s"], rec["rgba"], rec["q"] = centers, scales, rgba, rot_u8
    return rec.tobytes()


# ---- .ply header (reference semantics on well-formed INRIA v1 files) -----------------------------------------------------------------
def parse_ply_header(data: bytes) -> dict:
    data = bytes(data)
    end = data.index(b"end_header")
    text = data[:end + 10].decode("ascii")
    lines = [ln.strip() for ln in text.split("\n")]
    count, props, in_first = None, [], False
    for ln in lines:
        if ln.startswith("element"):
            if in_first:
                break
            in_first = True
            count = int(ln.split()[2])
        elif ln.startswith("property") and in_first:
            m = re.match(r"(\w+)\s+(\w+)\s+(\w+)", ln)
            props.append((m.group(3), m.group(2)))
    nrest = sum(1 for n, _ in props if n.startswith("f_rest"))
    cpc = nrest // 3
    degree = 2 if cpc >= 8 else (1 if cpc >= 3 else 0)
    return dict(count=count, props=props, data_offset=end + 11, sh_degree=degree, sh_per_channel=cpc)


def _ply_columns(data: bytes, h: dict) -> dict:
    dt = np.dtype([(n, _TYPES[t]) for n, t in h["props"]])
    rec = np.frombuffer(bytes(data), dt, count=h["count"], offset=h["data_offset"])
    out = {}
    for n, t in h["props"]:
        v = rec[n].astype(np.float64)
        out[n] = v / 255.0 if t == "uchar" else v                      # readVertex(normalize = true)
    return out


def _normalize(x, y, z, w):
    """three.js Quaternion.normalize on JavaScript numbers."""
    ln = np.sqrt(((x * x + y * y) + z * z) + w * w)
    zero = ln == 0
    with np.errstate(divide="ignore", invalid="ignore"):
        il = 1.0 / ln
    x, y, z, w = x * il, y * il, z * il, w * il
    return (np.where(zero, 0.0, x), np.where(zero, 0.0, y), np.where(zero, 0.0, z), np.where(zero, 1.0, w))


def _f32(v) -> np.ndarray:
    """Float32Array assignment, NaN as 0x7fc00000."""
    with np.errstate(over="ignore", invalid="ignore"):
        f = np.asarray(v, np.float64).astype(np.float32)
    b = f.view(np.uint32).copy()
    b[np.isnan(f)] = _CANON_NAN
    return b.view(np.float32)


def _u8_floor(v) -> np.ndarray:
    """clamp(Math.floor(v), 0, 255), then `|| 0` (NaN -> 0)."""
    c = np.clip(np.floor(v), 0.0, 255.0)
    return np.where(np.isnan(c), 0.0, c).astype(np.uint8)


def _exp_band(e: np.ndarray):
    """exp results 2 f64 ulps below / above e: what another libm's exp (each within 1 ulp) may return."""
    lo = np.nextafter(np.nextafter(e, -np.inf), -np.inf)
    hi = np.nextafter(np.nextafter(e, np.inf), np.inf)
    return np.where(np.isfinite(e) & (e > 0), lo, e), np.where(np.isfinite(e), hi, e)


def _header(count: int, sh_degree: int) -> bytes:
    h = bytearray(4096)
    struct.pack_into("<BB", h, 0, 0, 1)                                 # version 0.1
    struct.pack_into("<4I", h, 4, 1, 1, count, count)                  # max sections, sections, max splats, splats
    struct.pack_into("<H", h, 20, 0)                                    # compression level 0
    struct.pack_into("<5f", h, 24, 0.0, 0.0, 0.0, -1.5, 1.5)            # scene centre, default 8-bit SH range
    s = bytearray(1024)
    struct.pack_into("<2I", s, 0, count, count)
    struct.pack_into("<H", s, 40, sh_degree)
    return bytes(h) + bytes(s)


def level0_records(fmt: int, data: bytes, sh_degree: int = 0):
    """-> (records u8[n, 44 | 80 | 140], output SH degree, ambiguous bool[n])."""
    with np.errstate(all="ignore"):         # inf / NaN fields are part of the input domain
        return _level0_records(fmt, data, sh_degree)


def _level0_records(fmt: int, data: bytes, sh_degree: int):
    if fmt == SPLAT:
        data = bytes(data)
        n = len(data) // 32
        row = np.frombuffer(data, np.uint8).reshape(n, 32)
        rec = np.zeros((n, 44), np.uint8)
        rec[:, 0:24] = _f32(row[:, 0:24].copy().view(np.float32).astype(np.float64)).view(np.uint8).reshape(n, 24)
        q = (row[:, 28:32].astype(np.float64) - 128) / 128
        x, y, z, w = _normalize(q[:, 1], q[:, 2], q[:, 3], q[:, 0])
        rec[:, 24:40] = _f32(np.stack([w, x, y, z], 1)).view(np.uint8).reshape(n, 16)
        rec[:, 40:44] = row[:, 24:28]
        return rec, 0, np.zeros(n, bool)
    h = parse_ply_header(data)
    n = h["count"]
    col = _ply_columns(data, h)
    deg = min(sh_degree, h["sh_degree"])
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    rec = np.zeros((n, 44 + 4 * ncomp), np.uint8)
    ambiguous = np.zeros(n, bool)
    rec[:, 0:12] = _f32(np.stack([col["x"], col["y"], col["z"]], 1)).view(np.uint8).reshape(n, 12)
    if "scale_0" in col:
        with np.errstate(over="ignore", invalid="ignore"):
            e = np.stack([np.exp(col[f"scale_{k}"]) for k in range(3)], 1)
            lo, hi = _exp_band(e)
            ambiguous |= (_f32(lo).view(np.uint32) != _f32(hi).view(np.uint32)).any(1)               # within 2 ulps of an f32 rounding midpoint
        e = np.where(np.isnan(e), 0.0, e)                                # `|| 0`
    else:
        e = np.full((n, 3), 0.01)
    rec[:, 12:24] = _f32(e).view(np.uint8).reshape(n, 12)
    x, y, z, w = col["rot_0"], col["rot_1"], col["rot_2"], col["rot_3"]
    x, y, z, w = _normalize(*_normalize(x, y, z, w))                    # parser, then writer
    rec[:, 24:40] = _f32(np.stack([x, y, z, w], 1)).view(np.uint8).reshape(n, 16)
    with np.errstate(over="ignore", invalid="ignore"):
        if "f_dc_0" in col:
            rgb = [(0.5 + SH_C0 * col[f"f_dc_{k}"]) * 255 for k in range(3)]
        elif "red" in col:
            rgb = [col[c] * 255 for c in ("red", "green", "blue")]
        else:
            rgb = [np.zeros(n)] * 3
        if "opacity" in col:
            e = np.exp(-col["opacity"])
            a = (1 / (1 + e)) * 255
            lo, hi = _exp_band(e)
            ambiguous |= _u8_floor((1 / (1 + lo)) * 255) != _u8_floor((1 / (1 + hi)) * 255)   # an exp 2 ulps off moves the alpha byte
        else:
            a = np.zeros(n)
    rec[:, 40:44] = np.stack([_u8_floor(v) for v in (*rgb, a)], 1)
    if ncomp:
        c = h["sh_per_channel"]
        src = [(s % 3) + c * (s // 3) for s in range(9)] + [3 + (s % 5) + c * (s // 5) for s in range(15)]
        sh = np.stack([col[f"f_rest_{src[s]}"] for s in range(ncomp)], 1)
        sh = np.where(np.isnan(sh) | (sh == 0), 0.0, sh)                 # `|| 0`
        rec[:, 44:] = _f32(sh).view(np.uint8).reshape(n, 4 * ncomp)
    return rec, deg, ambiguous


def level0_image(fmt: int, data: bytes, sh_degree: int = 0):
    """-> (level-0 .ksplat bytes, ambiguous bool[n]).  sh_degree = the Viewer's sphericalHarmonicsDegree (.splat: always 0)."""
    rec, deg, ambiguous = level0_records(fmt, data, sh_degree)
    return _header(rec.shape[0], deg) + rec.tobytes(), ambiguous
