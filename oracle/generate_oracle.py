"""NumPy / scalar restatement of SplatBufferGenerator.getStandardGenerator (test infrastructure; imports nothing from the product).

  SplatPartitioner.getStandardPartitioner (SplatPartitioner.js:46-99)
  SplatBuffer.generateFromUncompressedSplatArrays (SplatBuffer.js:1177-1326) and computeBucketsForUncompressedSplatArray (:1328-1399)
  SplatBuffer.writeSplatDataToSectionBuffer (:1069-1172), toHalfFloat (three r160), toUint8 (SplatBuffer.js:21-25)

Inputs are what the generator reads per splat: the level-0 record its writer would produce, the centre as a JavaScript number and the
raw SH values (`generator_inputs`).  The order-dependent parts (the SH range scan, bucket filling, object-key order) are scalar loops.
Ties in the partition order keep file order (the reference leaves them to V8's sort; DESIGN.md section 2).
"""
from __future__ import annotations

import math
import struct

import numpy as np

from . import file_oracle as FO
from . import pcply_oracle as PC

HALF_RANGE = 1.5
SCALE_RANGE = 32767


def _is_pcply(data: bytes) -> bool:
    head = bytes(data[:bytes(data[:65536]).find(b"end_header")])
    return b"element chunk" in head or b"packed_" in head


def _pcply_inputs(data: bytes, sh_degree: int):
    """PlayCanvas-compressed .ply: the f64 lerp centres and the raw u8 * 8 / 255 - 4 SH beside the level-0 records."""
    rec, deg, amb = PC.level0_records(data, sh_degree)
    h = PC.parse_header(data)
    chunk, vert = PC._read(data, h["chunk"]), PC._read(data, h["vertex"])
    n = h["vertex"]["count"]
    ext = {k: chunk[k].astype(np.float64)[np.arange(n) // 256] for k in chunk.dtype.names}
    pos = vert["packed_position"]
    t = [(pos >> 21, 11), (pos >> 11, 10), (pos, 11)]
    with np.errstate(all="ignore"):
        c64 = np.stack([PC._lerp(ext[f"min_{a}"], ext[f"max_{a}"], PC._unorm(*t[i])) for i, a in enumerate("xyz")], 1)
    ncomp = {0: 0, 1: 9, 2: 24}[deg]
    sh = np.zeros((n, 0))
    if ncomp:
        nsh = len(h["sh"]["props"])
        read = {9: 3, 24: 8, 45: 15}[9 if nsh < 24 else (24 if nsh < 45 else 45)]
        shb = PC._read(data, h["sh"])
        sh = np.stack([shb[f"f_rest_{j * read + k}"].astype(np.float64) * (8 / 255) - 4 for j, k in PC._SLOT_JK[:ncomp]], 1)
    return rec, c64, sh, deg, amb


def generator_inputs(fmt: int, data: bytes, sh_degree: int = 0):
    """-> (records u8[n, 44 | 80 | 140], centres f64[n, 3], raw SH f64[n, ncomp], SH degree, ambiguous bool[n]) for a .ply (INRIA or
    PlayCanvas-compressed) or .splat."""
    if fmt != FO.SPLAT and _is_pcply(data):
        return _pcply_inputs(data, sh_degree)
    rec, deg, amb = FO.level0_records(fmt, data, sh_degree)
    rec = rec.copy()
    n = rec.shape[0]
    with np.errstate(all="ignore"):
        if fmt == FO.SPLAT:
            row = np.frombuffer(bytes(data), np.uint8).reshape(n, 32)
            c64 = row[:, 0:12].copy().view(np.float32).astype(np.float64)
            s = row[:, 12:24].copy().view(np.float32).astype(np.float64)
            s = np.where(np.isnan(s) | (s == 0), 0.0, s)                                 # the writer's `|| 0`
            rec[:, 12:24] = FO._f32(s).view(np.uint8).reshape(n, 12)
            q = (row[:, 28:32].astype(np.float64) - 128) / 128
            x, y, z, w = FO._normalize(q[:, 1], q[:, 2], q[:, 3], q[:, 0])             # parser
            w, x, y, z = FO._normalize(w, x, y, z)                                     # writer: Quaternion(w, x, y, z).normalize()
            rec[:, 24:40] = FO._f32(np.stack([w, x, y, z], 1)).view(np.uint8).reshape(n, 16)
            return rec, c64, np.zeros((n, 0)), 0, amb
        h = FO.parse_ply_header(data)
        col = FO._ply_columns(data, h)
        c64 = np.stack([col["x"], col["y"], col["z"]], 1)
        ncomp = {0: 0, 1: 9, 2: 24}[deg]
        c = h["sh_per_channel"]
        src = [(s % 3) + c * (s // 3) for s in range(9)] + [3 + (s % 5) + c * (s // 5) for s in range(15)]
        sh = np.stack([col[f"f_rest_{src[s]}"] for s in range(ncomp)], 1) if ncomp else np.zeros((n, 0))
    return rec, c64, sh, deg, amb


def _falsy(v: float) -> bool:
    return v != v or v == 0.0


def sh_range(sh_in_order) -> tuple[float, float]:
    """`if (!min || v < min) min = v` (and max) over FRC0..FRC22 of every splat in partition order, then `|| +-1.5`."""
    lo = hi = None
    for row in sh_in_order:
        for v in row[:23]:
            v = float(v)
            if lo is None or _falsy(lo) or v < lo:
                lo = v
            if hi is None or _falsy(hi) or v > hi:
                hi = v
    lo = -HALF_RANGE if lo is None or _falsy(lo) else lo
    hi = HALF_RANGE if hi is None or _falsy(hi) else hi
    return lo, hi


def partition_order(c64, center=(0.0, 0.0, 0.0)) -> np.ndarray:
    """Ascending lengthSq(floor((c - centre) / 0.5) * 0.5); ties in file order, NaN keys last."""
    with np.errstate(all="ignore"):
        v = np.floor((c64 - np.asarray(center, np.float64)) / 0.5) * 0.5
        d = (v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]
    nan = np.isnan(d)
    return np.lexsort((np.arange(len(d)), np.where(nan, 0.0, d), nan))


def _key(bid: float):
    """JS object key identity and enumeration class of String(bucketId)."""
    if bid == bid and 0 <= bid <= 4294967294 and bid == math.floor(bid):
        return (0, int(bid))
    return (1, "NaN" if bid != bid else repr(bid))


def buckets(centers, block: float, bucket_size: int):
    """computeBucketsForUncompressedSplatArray -> [(member rows, f64 centre)] in output order (full, then partial buckets)."""
    n = len(centers)
    if n == 0:
        return []
    mn = [float(v) for v in centers[0]]
    mx = list(mn)
    for i in range(1, n):
        for k in range(3):
            c = float(centers[i][k])
            if c < mn[k]:
                mn[k] = c
            if c > mx[k]:
                mx[k] = c
    yb = math.ceil((mx[1] - mn[1]) / block) if (mx[1] - mn[1]) == (mx[1] - mn[1]) and abs(mx[1] - mn[1]) != math.inf else (mx[1] - mn[1]) / block
    zb = math.ceil((mx[2] - mn[2]) / block) if (mx[2] - mn[2]) == (mx[2] - mn[2]) and abs(mx[2] - mn[2]) != math.inf else (mx[2] - mn[2]) / block
    yb, zb = float(yb), float(zb)
    half = block / 2.0
    full, partial = [], {}
    for i in range(n):
        b = []
        for k in range(3):
            q = (float(centers[i][k]) - mn[k]) / block
            b.append(float(math.floor(q)) if q == q and abs(q) != math.inf else q)
        center = [b[k] * block + mn[k] + half for k in range(3)]
        with np.errstate(all="ignore"):
            bid = float(np.float64(b[0]) * (np.float64(yb) * np.float64(zb)) + np.float64(b[1]) * np.float64(zb) + np.float64(b[2]))
        key = _key(bid)
        bucket = partial.get(key)
        if bucket is None:
            bucket = ([], center)
            partial[key] = bucket
        bucket[0].append(i)
        if len(bucket[0]) >= bucket_size:
            full.append(bucket)
            partial[key] = None
    index = sorted(k for k in partial if k[0] == 0)
    other = [k for k in partial if k[0] == 1]
    return full + [partial[k] for k in index + other if partial[k] is not None]


def _half(v) -> np.ndarray:
    """three's toHalfFloat: clamp to +-65504 (NaN passes), Float32Array store, truncating table lookup."""
    f = FO._f32(np.clip(np.asarray(v, np.float64), -65504.0, 65504.0)).view(np.uint32).astype(np.int64)
    sign = (f >> 16) & 0x8000
    mant = f & 0x7FFFFF
    e = ((f >> 23) & 0xFF) - 127
    base = np.select([e < -27, e < -14, e <= 15, e < 128], [0, 0x400 >> np.clip(-e - 14, 0, 31), (e + 15) << 10, 0x7C00], 0x7C00)
    shift = np.select([e < -27, e < -14, e <= 15, e < 128], [24, -e - 1, 13, 24], 13)
    return ((base | sign) + (mant >> shift)).astype(np.uint16)


def _u8(v, lo, hi) -> np.ndarray:
    with np.errstate(all="ignore"):
        c = np.maximum(np.minimum(v, hi), lo)
        q = np.floor((c - lo) / (hi - lo) * 255)
        q = np.maximum(np.minimum(q, 255.0), 0.0)
    return np.where(np.isnan(q), 0, q).astype(np.uint8)


def _js_round(v):
    r = np.floor(v)
    return np.where(v - r >= 0.5, r + 1, r)


def generate(rec, c64, sh, deg: int, *, level: int = 1, minimum_alpha: int = 1, section_size: int = 0, scene_center=(0.0, 0.0, 0.0),
             block_size: float = 5.0, bucket_size: int = 256, loose=None):
    """The .ksplat image of generateFromUncompressedSplatArrays for one parsed file.  loose (bool[n], optional): splats whose scale and
    alpha bytes may differ with libm's exp; then -> (image, bool mask of those bytes in the image)."""
    n = rec.shape[0]
    ncomp = sh.shape[1]
    order = partition_order(c64, scene_center)
    size = n if section_size <= 0 else min(n, section_size)
    nsec = 0 if n == 0 else -(-n // size)
    lo, hi = sh_range(sh[order] if ncomp else [])
    bps = {0: 44 + 4 * ncomp, 1: 24 + 2 * ncomp, 2: 24 + ncomp}[level]
    sf = SCALE_RANGE / (block_size * 0.5)
    headers, bodies, total, loose_at = [], [], 0, []
    for s in range(nsec):
        rows = order[s * size:(s + 1) * size]
        rows = rows[rec[rows, 43] >= minimum_alpha]
        bl = buckets(c64[rows], block_size, bucket_size)
        nfull = sum(1 for b in bl if len(b[0]) >= bucket_size)
        lens = [len(b[0]) for b in bl[nfull:]]
        out = [rows[i] for b in bl for i in b[0]]
        bc = np.array([b[1] for b in bl for _ in b[0]], np.float64).reshape(-1, 3)
        out = np.asarray(out, np.int64)
        if level == 0:
            data = rec[out].tobytes()
            meta = b""
        else:
            r = np.zeros((len(out), bps), np.uint8)
            with np.errstate(all="ignore"):
                v = _js_round((c64[out] - bc) * sf) + SCALE_RANGE
                v = np.maximum(np.minimum(v, 2 * SCALE_RANGE + 1), 0)
            cq = np.where(np.isnan(v), 0, v).astype(np.uint16)
            f = rec[out, 12:40].copy().view(np.float32).astype(np.float64)
            h = np.concatenate([cq, _half(f)], 1)
            r[:, 0:20] = h.view(np.uint8).reshape(len(out), 20)
            r[:, 20:24] = rec[out, 40:44]
            if ncomp and level == 1:
                r[:, 24:] = _half(rec[out, 44:].copy().view(np.float32).astype(np.float64)).view(np.uint8).reshape(len(out), 2 * ncomp)
            elif ncomp:
                x = sh[out]
                r[:, 24:] = _u8(np.where(np.isnan(x) | (x == 0), 0.0, x), lo, hi)
            data = r.tobytes()
            meta = np.asarray(lens, "<u4").tobytes() + FO._f32(np.array([b[1] for b in bl], np.float64).reshape(-1, 3)).tobytes()
        body = meta + data
        if loose is not None:
            at = len(meta) + bps * np.nonzero(loose[out])[0] if len(out) else np.zeros(0, np.int64)
            cols = list(range(12, 24)) + [43] if level == 0 else list(range(6, 12)) + [23]
            loose_at.append((s, (at[:, None] + np.asarray(cols)[None, :]).ravel() if len(at) else np.zeros(0, np.int64)))
        hd = bytearray(1024)
        struct.pack_into("<2I", hd, 0, len(out), len(out))
        if level >= 1:
            struct.pack_into("<2If", hd, 8, bucket_size, len(bl), block_size)
            struct.pack_into("<HxxI", hd, 20, 12, SCALE_RANGE)
            struct.pack_into("<2I", hd, 32, nfull, len(lens))
        struct.pack_into("<I", hd, 28, len(body))
        struct.pack_into("<H", hd, 40, deg)
        headers.append(bytes(hd))
        bodies.append(body)
        total += len(out)
    h = bytearray(4096)
    struct.pack_into("<BB", h, 0, 0, 1)
    struct.pack_into("<4I", h, 4, nsec, nsec, total, total)
    struct.pack_into("<H", h, 20, level)
    struct.pack_into("<3f", h, 24, *[float(v) for v in scene_center])
    struct.pack_into("<2f", h, 36, lo, hi)
    img = bytes(h) + b"".join(headers) + b"".join(bodies)
    if loose is None:
        return img
    mask = np.zeros(len(img), bool)
    base = 4096 + 1024 * nsec
    for s, at in loose_at:
        mask[base + at] = True
        base += len(bodies[s])
    return img, mask
