"""tests/spz_oracle.py -- TEST INFRASTRUCTURE ONLY.  Imports nothing from the product package.

NumPy restatement of what the reference's SpzLoader builds from a `.spz` file:
  stream  Compression.decompressGzipped, then deserializePackedGaussians (SpzLoader.js:255-342): a 16-byte header (magic, version,
          numPoints u32; shDegree, fractionalBits, flags, reserved u8), then the planes positions, alphas, colours, scales, rotations, SH
  splat   unpackGaussians (:160-250) + unpackedSplatToUncompressedSplat (:84-145)
  writer  SplatBuffer.writeSplatDataToSectionBuffer, level 0 (normalise a second time, Float32Array stores), one section in file order
          (optimizeSplatData off); `generator_inputs` gives what SplatBufferGenerator reads for the optimizeSplatData path
Every step is exact JavaScript-number arithmetic except the scale's `exp`: a splat is flagged `ambiguous` when an `exp` 2 f64 ulps away
would give another f32 scale.

Also: `write_spz` (planes given, optionally gzipped) and `quantize` (float splats in, a realistic v2 file out, the way Niantic's
spz library packs one).
"""
from __future__ import annotations

import gzip
import struct

import numpy as np

from oracle.file_oracle import SH_C0, _exp_band, _f32, _header, _normalize, _u8_floor
from oracle.pcply_oracle import _SLOT_JK

MAGIC = 0x5053474E
SPZ = 4
DIM = {0: 0, 1: 3, 2: 8, 3: 15}
COLOR_SCALE = 0.15


# ---- writers (test inputs) ---------------------------------------------------------------------------------------------------------
def write_spz(positions, alphas, colors, scales, rotations, sh=None, *, version=2, sh_degree=0, fractional_bits=12, flags=0,
              count=None, compress=False) -> bytes:
    """Planes as given: positions u8[n, 9] (v2, 24-bit little-endian fixed point) or u16[n, 3] (v1, float16 bits); alphas u8[n];
    colors, scales, rotations u8[n, 3]; sh u8[n, 3 * dim] (coefficient-major, channel-minor).  count overrides the header's numPoints."""
    n = len(alphas)
    pos = np.ascontiguousarray(positions, np.uint8 if version != 1 else "<u2")
    sh = np.zeros((n, 3 * DIM[sh_degree]), np.uint8) if sh is None else np.ascontiguousarray(sh, np.uint8)
    head = struct.pack("<3I4B", MAGIC, version, n if count is None else count, sh_degree, fractional_bits, flags, 0)
    body = b"".join(np.ascontiguousarray(a, np.uint8).tobytes() for a in (alphas, colors, scales, rotations))
    data = head + pos.tobytes() + body + sh.tobytes()
    return gzip.compress(data, mtime=0) if compress else data


def quantize(centers, log_scales, quats_xyzw, rgba, sh=None, *, sh_degree=0, fractional_bits=12, compress=False) -> bytes:
    """Float splats -> a v2 stream.  rgba in [0, 1] (colour as displayed, alpha as opacity); sh: f[n, 3, dim] (channel, coefficient)."""
    centers, log_scales, rgba = (np.asarray(a, np.float64) for a in (centers, log_scales, rgba))
    n = len(centers)
    fixed = np.clip(np.rint(centers * (1 << fractional_bits)), -(1 << 23), (1 << 23) - 1).astype(np.int64) & 0xFFFFFF
    pos = np.stack([(fixed >> (8 * b)) & 0xFF for b in range(3)], 2).reshape(n, 9)
    scales = np.clip(np.rint((log_scales + 10) * 16), 0, 255)
    q = np.asarray(quats_xyzw, np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    q = q * np.where(q[:, 3:4] < 0, -1.0, 1.0)
    rot = np.clip(np.rint((q[:, :3] + 1) * 127.5), 0, 255)
    colors = np.clip(np.rint(((rgba[:, :3] - 0.5) / SH_C0 * COLOR_SCALE + 0.5) * 255), 0, 255)
    alphas = np.clip(np.rint(rgba[:, 3] * 255), 0, 255)
    shq = None
    if sh_degree:
        s = np.asarray(sh, np.float64).transpose(0, 2, 1).reshape(n, -1)             # [i][k][j]
        shq = np.clip(np.rint(s * 128 + 128), 0, 255)
    return write_spz(pos, alphas, colors, scales, rot, shq, sh_degree=sh_degree, fractional_bits=fractional_bits, compress=compress)


# ---- reader (reference semantics on well-formed streams) -----------------------------------------------------------------------------
def packed(data) -> bytes:
    """The packed stream of a `.spz` file as stored (gzip) or of an already inflated stream."""
    data = bytes(data)
    return gzip.decompress(data) if data[:2] == b"\x1f\x8b" else data


def parse(data) -> dict:
    data = packed(data)
    magic, version, n, deg, fb, flags, _ = struct.unpack_from("<3I4B", data, 0)
    assert magic == MAGIC and version in (1, 2) and deg <= 3
    at = 16
    planes = {}
    for name, width in (("positions", 6 if version == 1 else 9), ("alphas", 1), ("colors", 3), ("scales", 3), ("rotations", 3),
                        ("sh", 3 * DIM[deg])):
        planes[name] = np.frombuffer(data, np.uint8, n * width, at).reshape(n, width)
        at += n * width
    assert at == len(data)
    return dict(version=version, count=n, sh_degree=deg, fractional_bits=fb, flags=flags, **planes)


def position_scale(fractional_bits: int) -> float:
    """1.0 / (1 << fractionalBits) with JavaScript's int32 shift (count mod 32; 1 << 31 is -2^31)."""
    p = 1 << (fractional_bits & 31)
    return 1.0 / (p - (1 << 32) if p >= 1 << 31 else p)


def centers_f64(p: dict) -> np.ndarray:
    n = p["count"]
    if p["version"] == 1:
        return p["positions"].copy().view("<u2").view(np.float16).astype(np.float64).reshape(n, 3)   # halfToFloat is exact
    b = p["positions"].reshape(n, 3, 3).astype(np.int64)
    v = b[:, :, 0] | (b[:, :, 1] << 8) | (b[:, :, 2] << 16)
    v = (v ^ 0x800000) - 0x800000
    return v.astype(np.float64) * position_scale(p["fractional_bits"])


def scale_values(b) -> np.ndarray:
    return np.exp(np.asarray(b, np.float64) / 16.0 - 10.0)


def flagged_scale_bytes() -> np.ndarray:
    """bool[256]: scale bytes whose f32 scale depends on how `exp` rounds (within 2 f64 ulps of an f32 rounding midpoint)."""
    lo, hi = _exp_band(scale_values(np.arange(256)))
    return _f32(lo).view(np.uint32) != _f32(hi).view(np.uint32)


def level0_records(data, sh_degree: int = 0):
    """-> (records u8[n, 44 | 80 | 140], output SH degree, ambiguous bool[n]).  sh_degree = the Viewer's sphericalHarmonicsDegree."""
    p = parse(data)
    n = p["count"]
    deg = min(sh_degree, p["sh_degree"], 2)
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    rec = np.zeros((n, 44 + 4 * ncomp), np.uint8)
    with np.errstate(all="ignore"):
        rec[:, 0:12] = _f32(centers_f64(p)).view(np.uint8).reshape(n, 12)
    rec[:, 12:24] = _f32(scale_values(p["scales"])).view(np.uint8).reshape(n, 12)
    ambiguous = flagged_scale_bytes()[p["scales"]].any(1) if n else np.zeros(0, bool)
    x, y, z = (p["rotations"][:, k].astype(np.float64) / 127.5 - 1.0 for k in range(3))
    w = np.sqrt(np.maximum(0.0, 1.0 - ((x * x + y * y) + z * z)))
    q = _normalize(*_normalize(w, x, y, z))                              # Quaternion.set(w, x, y, z).normalize(), then the writer's
    rec[:, 24:40] = _f32(np.stack(q, 1)).view(np.uint8).reshape(n, 16)
    c = p["colors"].astype(np.float64)
    rec[:, 40:43] = _u8_floor(np.floor(((((c / 255.0) - 0.5) / COLOR_SCALE) * SH_C0 + 0.5) * 255))
    rec[:, 43] = p["alphas"][:, 0]
    if ncomp:
        sh = p["sh"]
        v = np.stack([(sh[:, 3 * k + j].astype(np.float64) - 128.0) / 128.0 for j, k in _SLOT_JK[:ncomp]], 1)
        rec[:, 44:] = _f32(v).view(np.uint8).reshape(n, 4 * ncomp)
    return rec, deg, ambiguous


def level0_image(data, sh_degree: int = 0):
    """-> (level-0 .ksplat bytes, ambiguous bool[n]): what SpzLoader gives with optimizeSplatData off."""
    rec, deg, ambiguous = level0_records(data, sh_degree)
    return _header(rec.shape[0], deg) + rec.tobytes(), ambiguous


def generator_inputs(data, sh_degree: int = 0):
    """-> (records, centres f64[n, 3], raw SH f64[n, ncomp], SH degree, ambiguous) for oracle.generate_oracle.generate: what
    SplatBufferGenerator reads from SpzLoader's UncompressedSplatArray (optimizeSplatData on)."""
    rec, deg, amb = level0_records(data, sh_degree)
    p = parse(data)
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    sh = np.zeros((p["count"], 0))
    if ncomp:
        sh = np.stack([(p["sh"][:, 3 * k + j].astype(np.float64) - 128.0) / 128.0 for j, k in _SLOT_JK[:ncomp]], 1)
    return rec, centers_f64(p), sh, deg, amb
