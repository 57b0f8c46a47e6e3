"""oracle/pcply_oracle.py -- TEST INFRASTRUCTURE ONLY.  Imports nothing from the product package.

NumPy restatement of the level-0 `.ksplat` image the reference builds from a PlayCanvas-compressed `.ply` (file order, one
compression-level-0 SplatBuffer section):
  header  PlayCanvasCompressedPlyParser.decodeHeaderText (:74-157); blocks chunk, vertex, sh read in that order (readPly :297-313)
  splat   decompressBaseSplat (:379-432), decompressSphericalHarmonics (:434-460), parseToUncompressedSplatBuffer (:547-585)
  writer  SplatBuffer.writeSplatDataToSectionBuffer, level 0 (normalise once, `|| 0`, Float32Array / Uint8ClampedArray stores)
Every step is JavaScript-number (f64, unfused) arithmetic; NumPy does not contract.  NaN lands in the image as 0x7fc00000.  The only
libm call is `exp` in the scale: a splat is flagged `ambiguous` when an `exp` 2 f64 ulps away would give another f32 scale.

Also: writers for test inputs -- `write_pcply` (chunk table, packed words and SH bytes given) and `quantize` (float splats in, a
realistic compressed file out, the way the PlayCanvas tools pack one: per-256-splat extremes, real unit quaternions).
"""
from __future__ import annotations

import numpy as np

from oracle.file_oracle import _exp_band, _f32, _header, _normalize

_TYPES = {"char": "i1", "uchar": "u1", "short": "<i2", "ushort": "<u2", "int": "<i4", "uint": "<u4", "float": "<f4", "double": "<f8"}
EXTREMES = ["min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y", "min_scale_z",
            "max_scale_x", "max_scale_y", "max_scale_z", "min_r", "min_g", "min_b", "max_r", "max_g", "max_b"]
PACKED = ["packed_position", "packed_rotation", "packed_scale", "packed_color"]
NORM = 1.0 / (np.sqrt(2.0) * 0.5)
# level-0 slot s -> (channel j, coefficient k): the layout the INRIA path writes (shIndexMap inverted)
_SLOT_JK = [(s // 3, s % 3) for s in range(9)] + [((s - 9) // 5, 3 + (s - 9) % 5) for s in range(9, 24)]


# ---- writers (test inputs) ---------------------------------------------------------------------------------------------------------
def _block(props, cols, count) -> bytes:
    dt = np.dtype([(n, _TYPES[t]) for n, t in props])
    rec = np.zeros(count, dt)
    for n, _ in props:
        if n in cols:
            rec[n] = np.asarray(cols[n]).astype(dt[n])
    return rec.tobytes()


def write_pcply(chunk_props, chunk_cols, n_chunks, vertex_props, vertex_cols, n, sh=None, *, comments=()) -> bytes:
    """chunk_props / vertex_props: [(name, type)] in file order; *_cols[name]: values.  sh: u8[n, 9 | 24 | 45] or None."""
    lines = ["ply", "format binary_little_endian 1.0", *[f"comment {c}" for c in comments], f"element chunk {n_chunks}",
             *[f"property {t} {k}" for k, t in chunk_props], f"element vertex {n}", *[f"property {t} {k}" for k, t in vertex_props]]
    body = _block(chunk_props, chunk_cols, n_chunks) + _block(vertex_props, vertex_cols, n)
    if sh is not None:
        sh = np.ascontiguousarray(sh, np.uint8)
        lines += [f"element sh {n}", *[f"property uchar f_rest_{k}" for k in range(sh.shape[1])]]
        body += sh.tobytes()
    return ("\n".join(lines + ["end_header"]) + "\n").encode("ascii") + body


def _unit(v, bits):
    q = (1 << bits) - 1
    return np.clip(np.rint(v * q), 0, q).astype(np.uint32)


def quantize(centers, log_scales, quats_xyzw, rgba, sh=None, *, color_extremes=True) -> bytes:
    """Float splats -> a PlayCanvas-compressed file.  rgba in [0, 1]; sh: f[n, 9 | 24 | 45] (channel-major, as f_rest_*)."""
    centers, log_scales, rgba = (np.asarray(a, np.float64) for a in (centers, log_scales, rgba))
    n = len(centers)
    nc = (n + 255) // 256
    pad = nc * 256 - n

    def extremes(v):
        w = np.concatenate([v, np.repeat(v[-1:], pad, 0)]) if pad else v
        w = w.reshape(nc, 256, -1)
        return w.min(1).astype(np.float32).astype(np.float64), w.max(1).astype(np.float32).astype(np.float64)

    def rel(v, lo, hi):
        ch = np.arange(n) // 256
        span = hi[ch] - lo[ch]
        return np.where(span > 0, (v - lo[ch]) / np.where(span > 0, span, 1), 0.0)

    cols = {}
    words = {}
    for key, v in (("", centers), ("scale_", log_scales)):
        lo, hi = extremes(v)
        for i, a in enumerate("xyz"):
            cols[f"min_{key}{a}"], cols[f"max_{key}{a}"] = lo[:, i], hi[:, i]
        t = rel(v, lo, hi)
        words[key] = (_unit(t[:, 0], 11) << 21) | (_unit(t[:, 1], 10) << 11) | _unit(t[:, 2], 11)
    q = np.asarray(quats_xyzw, np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    big = np.argmax(np.abs(q), 1)
    q = q * np.where(q[np.arange(n), big] < 0, -1.0, 1.0)[:, None]
    rest = q[np.arange(4)[None, :] != big[:, None]].reshape(n, 3)
    r = _unit(rest / NORM + 0.5, 10)
    rot = (big.astype(np.uint32) << 30) | (r[:, 0] << 20) | (r[:, 1] << 10) | r[:, 2]
    c = rgba[:, :3]
    if color_extremes:
        lo, hi = extremes(c)
        for i, a in enumerate("rgb"):
            cols[f"min_{a}"], cols[f"max_{a}"] = lo[:, i], hi[:, i]
        c = rel(c, lo, hi)
    cb = _unit(np.concatenate([c, rgba[:, 3:4]], 1), 8)
    color = (cb[:, 0] << 24) | (cb[:, 1] << 16) | (cb[:, 2] << 8) | cb[:, 3]
    chunk_props = [(k, "float") for k in EXTREMES if k in cols]
    vcols = dict(packed_position=words[""], packed_rotation=rot, packed_scale=words["scale_"], packed_color=color)
    shu = None if sh is None else np.clip(np.rint((np.asarray(sh, np.float64) + 4) * (255 / 8)), 0, 255).astype(np.uint8)
    return write_pcply(chunk_props, cols, nc, [(k, "uint") for k in PACKED], vcols, n, shu)


# ---- reader (reference semantics on well-formed files) -------------------------------------------------------------------------------
def parse_header(data: bytes) -> dict:
    data = bytes(data)
    end = data.index(b"\nend_header\n")
    els = []
    for ln in data[:end].decode("ascii").split("\n")[1:]:
        w = ln.split()
        if w[0] == "element":
            els.append(dict(name=w[1], count=int(w[2]), props=[]))
        elif w[0] == "property":
            els[-1]["props"].append((w[2], w[1]))
    at = end + len(b"\nend_header\n")
    for e in els:
        e["dtype"] = np.dtype([(k, _TYPES[t]) for k, t in e["props"]])
        e["offset"] = at
        at += e["dtype"].itemsize * e["count"]
    return {e["name"]: e for e in els}


def _read(data: bytes, e: dict) -> np.ndarray:
    return np.frombuffer(bytes(data), e["dtype"], count=e["count"], offset=e["offset"])


def _unorm(v, bits):
    t = (1 << bits) - 1
    return (v & np.uint32(t)).astype(np.float64) / t


def _lerp(a, b, t):
    return a * (1 - t) + b * t


def _js_round(v):
    """Math.round: nearest integer, ties towards +inf (v - floor(v) is exact for v >= 0; below 0 the result clamps to 0)."""
    r = np.floor(v)
    return np.where(v - r >= 0.5, r + 1, r)


def _u8(v):
    """clamp(v, 0, 255), then `|| 0` (NaN -> 0) and the Uint8ClampedArray store of an integer."""
    c = np.clip(v, 0.0, 255.0)
    return np.where(np.isnan(c), 0.0, c).astype(np.uint8)


def level0_records(data: bytes, sh_degree: int = 0):
    """-> (records u8[n, 44 | 80 | 140], output SH degree, ambiguous bool[n])."""
    with np.errstate(all="ignore"):         # NaN / inf extremes and NaN rotations are part of the input domain
        return _level0_records(data, sh_degree)


def _level0_records(data: bytes, sh_degree: int):
    h = parse_header(data)
    chunk, vert = _read(data, h["chunk"]), _read(data, h["vertex"])
    n = h["vertex"]["count"]
    ch = np.arange(n) // 256
    ext = {k: chunk[k].astype(np.float64)[ch] for k in chunk.dtype.names}
    nsh = len(h["sh"]["props"]) if "sh" in h else 0
    file_deg = 3 if nsh >= 45 else (2 if nsh >= 24 else (1 if nsh >= 9 else 0))
    deg = min(sh_degree, file_deg)
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    rec = np.zeros((n, 44 + 4 * ncomp), np.uint8)
    pos, scl = vert["packed_position"], vert["packed_scale"]
    t = [(pos >> 21, 11), (pos >> 11, 10), (pos, 11)]
    ts = [(scl >> 21, 11), (scl >> 11, 10), (scl, 11)]
    xyz = [_lerp(ext[f"min_{a}"], ext[f"max_{a}"], _unorm(*t[i])) for i, a in enumerate("xyz")]
    rec[:, 0:12] = _f32(np.stack(xyz, 1)).view(np.uint8).reshape(n, 12)
    e = np.stack([np.exp(_lerp(ext[f"min_scale_{a}"], ext[f"max_scale_{a}"], _unorm(*ts[i]))) for i, a in enumerate("xyz")], 1)
    lo, hi = _exp_band(e)
    ambiguous = (_f32(lo).view(np.uint32) != _f32(hi).view(np.uint32)).any(1)
    e = np.where(np.isnan(e), 0.0, e)                                    # `|| 0`
    rec[:, 12:24] = _f32(e).view(np.uint8).reshape(n, 12)
    rot = vert["packed_rotation"]
    a, b, c = ((_unorm(rot >> s, 10) - 0.5) * NORM for s in (20, 10, 0))
    m = np.sqrt(1.0 - ((a * a + b * b) + c * c))
    slot = rot >> 30
    q = [np.where(slot == 0, m, a), np.where(slot == 0, a, np.where(slot == 1, m, b)),
         np.where(slot <= 1, b, np.where(slot == 2, m, c)), np.where(slot <= 2, c, m)]
    rec[:, 24:40] = _f32(np.stack(_normalize(*q), 1)).view(np.uint8).reshape(n, 16)
    col = vert["packed_color"]
    rgba = []
    for k, a_ in enumerate("rgb"):
        ck = _unorm(col >> (24 - 8 * k), 8)
        if f"min_{a_}" in ext and f"max_{a_}" in ext:
            rgba.append(_u8(_js_round(_lerp(ext[f"min_{a_}"], ext[f"max_{a_}"], ck) * 255)))
        else:
            rgba.append(_u8(np.floor(ck * 255)))
    rgba.append(_u8(np.floor(_unorm(col, 8) * 255)))
    rec[:, 40:44] = np.stack(rgba, 1)
    if ncomp:
        read = {1: 3, 2: 8, 3: 15}[file_deg]
        shb = _read(data, h["sh"])
        sh = np.stack([shb[f"f_rest_{j * read + k}"].astype(np.float64) * (8 / 255) - 4 for j, k in _SLOT_JK[:ncomp]], 1)
        sh = np.where(sh == 0, 0.0, sh)                                  # `|| 0`
        rec[:, 44:] = _f32(sh).view(np.uint8).reshape(n, 4 * ncomp)
    return rec, deg, ambiguous


def level0_image(data: bytes, sh_degree: int = 0):
    """-> (level-0 .ksplat bytes, ambiguous bool[n]).  sh_degree = the Viewer's sphericalHarmonicsDegree."""
    rec, deg, ambiguous = level0_records(data, sh_degree)
    return _header(rec.shape[0], deg) + rec.tobytes(), ambiguous
