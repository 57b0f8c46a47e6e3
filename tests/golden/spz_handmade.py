"""Handmade `.spz` fixtures and the level-0 records derived for them here, splat by splat, with scalar arithmetic (Python floats are
JavaScript numbers).  Run this file to rewrite the fixtures: `python tests/golden/spz_handmade.py`.  Each fixture is the packed stream
gzipped with mtime 0; the committed files are compared after gunzip (deflate output may differ between zlib versions).

The derivation restates SpzLoader.unpackGaussians + unpackedSplatToUncompressedSplat + the level-0 writer:
  position  v2: the 24-bit value sign-extended, times 1.0 / (1 << fractionalBits) with JavaScript's int32 shift; v1: halfToFloat
  scale     Math.exp(b / 16 - 10)
  rotation  xyz = b / 127.5 - 1, w = sqrt(max(0, 1 - ((x x + y y) + z z))); Quaternion(w, x, y, z) normalised twice; stored w, x, y, z
  colour    clamp(floor(((c / 255 - 0.5) / 0.15 * SH_C0 + 0.5) * 255), 0, 255); alpha the byte
  SH        (b - 128) / 128 of file coefficient k, channel j (byte 3k + j) into FRC 3j + k (k < 3) or 9 + 5j + (k - 3) (k < 8)
"""
from __future__ import annotations

import gzip
import math
import struct
from pathlib import Path

HERE = Path(__file__).resolve().parent
SPZ = 4
BAD_ARG = 1
MAGIC = 0x5053474E
DIM = [0, 3, 8, 15]
SH_C0 = 0.28209479177387814


# ---- scalar derivation -------------------------------------------------------------------------------------------------------------
def _f32_bits(v: float) -> bytes:
    if v != v:
        return struct.pack("<I", 0x7FC00000)
    return struct.pack("<f", v)


def _half(h: int) -> float:
    sign = -1.0 if (h >> 15) & 1 else 1.0
    e, m = (h >> 10) & 31, h & 1023
    if e == 0:
        return sign * 2.0 ** -14 * m / 1024
    if e == 31:
        return math.nan if m else sign * math.inf
    return sign * 2.0 ** (e - 15) * (1 + m / 1024)


def _scale_of_shift(fb: int) -> float:
    p = 1 << (fb % 32)
    if p >= 1 << 31:
        p -= 1 << 32
    return 1.0 / p


def _normalize(x, y, z, w):
    ln = math.sqrt(x * x + y * y + z * z + w * w)
    if ln == 0:
        return 0.0, 0.0, 0.0, 1.0
    il = 1.0 / ln
    return x * il, y * il, z * il, w * il


def _frc_slot(j: int, k: int) -> int:
    return 3 * j + k if k < 3 else 9 + 5 * j + (k - 3)


def record(s: dict, version: int, fb: int, file_deg: int, sh_degree: int) -> bytes:
    """One splat's level-0 record at output degree min(sh_degree, file degree, 2)."""
    out = b""
    for k in range(3):
        if version == 1:
            out += _f32_bits(_half(s["pos"][k]))
        else:
            v = s["pos"][k]
            if v & 0x800000:
                v -= 1 << 24
            out += _f32_bits(v * _scale_of_shift(fb))
    for k in range(3):
        out += _f32_bits(math.exp(s["scale"][k] / 16.0 - 10.0))
    x, y, z = (b / 127.5 - 1.0 for b in s["rot"])
    w = math.sqrt(max(0.0, 1.0 - (x * x + y * y + z * z)))
    q = _normalize(*_normalize(w, x, y, z))
    out += b"".join(_f32_bits(v) for v in q)
    for c in s["color"]:
        v = math.floor(((((c / 255.0) - 0.5) / 0.15) * SH_C0 + 0.5) * 255)
        out += bytes([min(max(v, 0), 255)])
    out += bytes([s["alpha"]])
    deg = min(sh_degree, file_deg, 2)
    ncomp = [0, 9, 24][deg]
    slots = [0.0] * ncomp
    for j in range(3):
        for k in range(DIM[deg]):
            slots[_frc_slot(j, k)] = (s["sh"][3 * k + j] - 128) / 128
    out += b"".join(_f32_bits(v) for v in slots)
    return out


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def stream(splats: list[dict], *, version=2, fb=12, sh_degree=0, flags=0, count=None) -> bytes:
    n = len(splats)
    head = struct.pack("<3I4B", MAGIC, version, n if count is None else count, sh_degree, fb, flags, 0)
    if version == 1:
        pos = b"".join(struct.pack("<3H", *s["pos"]) for s in splats)
    else:
        pos = b"".join(bytes(b for v in s["pos"] for b in (v & 0xFF, (v >> 8) & 0xFF, v >> 16)) for s in splats)
    planes = [bytes([s["alpha"]]) for s in splats], [bytes(s["color"]) for s in splats], [bytes(s["scale"]) for s in splats], \
             [bytes(s["rot"]) for s in splats], [bytes(s["sh"]) for s in splats]
    return head + pos + b"".join(b"".join(p) for p in planes)


def _splat(i: int, deg: int, **kw) -> dict:
    """A splat whose bytes vary with i; SH bytes distinct per (coefficient, channel) so any mix-up of the layout shows."""
    s = dict(pos=[(0x012345 * (i + 1)) & 0xFFFFFF, (0x7F00FF + 977 * i) & 0xFFFFFF, (0xF0F0F0 - 4099 * i) & 0xFFFFFF],
             alpha=(37 * i + 200) % 256, color=[(53 * i + 7) % 256, (29 * i + 100) % 256, (71 * i + 50) % 256],
             scale=[(11 * i + 60) % 256, (13 * i + 90) % 256, (17 * i + 120) % 256], rot=[(31 * i + 5) % 256, (47 * i + 60) % 256, (59 * i + 200) % 256],
             sh=[(7 * m + 19 * i + 3) % 256 for m in range(3 * DIM[deg])])
    s.update(kw)
    return s


def _sh_case(deg: int) -> list[dict]:
    d = 3 * DIM[deg]
    return [
        _splat(0, deg, pos=[0x000000, 0x7FFFFF, 0x800000], alpha=255, color=[0, 128, 255], scale=[0, 160, 255], rot=[0, 127, 128],
               sh=[128] * d),                                                            # SH exactly 0 (the generator's `!min ||` quirk)
        _splat(1, deg, pos=[0xFFFFFF, 0x000001, 0x123456], alpha=0, color=[255, 0, 100], scale=[100, 101, 102], rot=[255, 255, 255],
               sh=[0] * d),                                                              # w clamps at max(0, 1 - 3)
        _splat(2, deg, rot=[128, 128, 128], sh=[255] * d),
        _splat(3, deg, rot=[127, 127, 127], alpha=1),
        _splat(4, deg, rot=[0, 0, 0], color=[1, 254, 127]),                              # w clamps again; colour just inside the clamps
        _splat(5, deg, rot=[255, 0, 128]),
        *[_splat(i, deg) for i in range(6, 19)],
    ]


# float16: +-0, smallest and largest subnormal, smallest normal, 1, 65504, +-inf, NaN (quiet and signalling payloads)
_HALVES = [0x0000, 0x8000, 0x0001, 0x8001, 0x03FF, 0x0400, 0x3C00, 0xBC00, 0x7BFF, 0x7C00, 0xFC00, 0x7E00, 0x7C01, 0xFFFF, 0x3555]


def _v1_case() -> list[dict]:
    h = _HALVES
    return [_splat(i, 0, pos=[h[i % len(h)], h[(i + 5) % len(h)], h[(i + 10) % len(h)]]) for i in range(len(h))]


def _fb_case() -> list[dict]:
    edge = [0x000000, 0x000001, 0x7FFFFF, 0x800000, 0x800001, 0xFFFFFF, 0x400000, 0xC00000]
    return [_splat(i, 0, pos=[edge[i % 8], edge[(i + 3) % 8], edge[(i + 6) % 8]]) for i in range(8)]


def _scale_case() -> list[dict]:
    return [_splat(b, 1, scale=[b, (b + 85) % 256, (b + 170) % 256]) for b in range(256)]


# name -> (splats, header keywords)
FIXTURES = {
    "sh0": (_sh_case(0), dict(sh_degree=0)),
    "sh1": (_sh_case(1), dict(sh_degree=1, flags=1)),                                   # the antialiased flag is ignored
    "sh2": (_sh_case(2), dict(sh_degree=2)),
    "sh3": (_sh_case(3), dict(sh_degree=3, fb=16)),
    "v1": (_v1_case(), dict(version=1)),
    "fb0": (_fb_case(), dict(fb=0)),
    "fb31": (_fb_case(), dict(fb=31)),                                                   # 1 << 31 = -2^31: every coordinate flips sign
    "fb32": (_fb_case(), dict(fb=32)),                                                   # 1 << 32 = 1
    "fb33": (_fb_case(), dict(fb=33)),                                                   # 1 << 33 = 2
    "scales": (_scale_case(), dict(sh_degree=1, fb=8)),
    "empty": ([], dict(sh_degree=3)),
}


def header_kw(name: str) -> dict:
    kw = dict(version=2, fb=12, sh_degree=0, flags=0)
    kw.update(FIXTURES[name][1])
    return kw


def packed_fixture(name: str) -> bytes:
    splats, kw = FIXTURES[name]
    return stream(splats, **kw)


def file_name(name: str) -> str:
    return f"spz_handmade_{name}.spz"


def expected_records(name: str, sh_degree: int) -> tuple[bytes, int]:
    splats, _ = FIXTURES[name]
    kw = header_kw(name)
    deg = min(sh_degree, kw["sh_degree"], 2)
    return b"".join(record(s, kw["version"], kw["fb"], kw["sh_degree"], sh_degree) for s in splats), deg


# ---- malformed streams: name -> (bytes, words the message must contain) --------------------------------------------------------------
def _malformed() -> dict:
    good = packed_fixture("sh1")
    bad = {
        "short_header": (good[:15], "shorter than the 16-byte header"),
        "empty_buffer": (b"", "shorter than the 16-byte header"),
        "magic": (struct.pack("<I", 0x5053474F) + good[4:], "magic"),
        "version0": (good[:4] + struct.pack("<I", 0) + good[8:], "version 0 not supported"),
        "version3": (good[:4] + struct.pack("<I", 3) + good[8:], "version 3 not supported"),
        "too_many_points": (stream([], count=10_000_001), "more than 10000000"),
        "sh_degree4": (good[:12] + bytes([4]) + good[13:], "SH degree 4"),
        "truncated": (good[:-1], "take exactly"),
        "trailing": (good + b"\0", "take exactly"),
        "count_mismatch": (stream(_sh_case(1), sh_degree=1, count=18), "take exactly"),
        "gzip": (gzip.compress(good, mtime=0), "decompress it first"),
    }
    return bad


MALFORMED = _malformed()


def fixture_files() -> dict[str, bytes]:
    """file name -> gzipped bytes as written."""
    return {file_name(k): gzip.compress(packed_fixture(k), mtime=0) for k in FIXTURES}


if __name__ == "__main__":
    for fname, data in fixture_files().items():
        (HERE / fname).write_bytes(data)
        print(fname, len(data))
