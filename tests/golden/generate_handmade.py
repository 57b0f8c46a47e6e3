"""Hand-derived .ksplat images of SplatBufferGenerator.getStandardGenerator for small `.splat` files.  Every byte below comes from the
layout worked out by hand in the comments (no product or oracle code).  Coordinates are multiples of 0.25, so every f64 step is exact.

Scene (file order P4, P2, P6, P0, P5, P3, P1; block 1.0, bucket size 2, scene centre 0):
  point  centre              partition key   xB yB zB   id = xB * (yBlocks * zBlocks) + yB * zBlocks + zB
  P0     (0.25, 0.25, 0.25)  0               0  0  0    0
  P1     (1.00, 0.75, 0.75)  1.5             0  0  0    0
  P2     (1.25, 0.25, 0.25)  1               1  0  0    2
  P3     (1.25, 0.75, 0.25)  1.25            1  0  0    2
  P4     (0.25, 1.75, 0.25)  2.25            0  1  0    1
  P5     (2.25, 0.25, 0.25)  4               2  0  0    4
  P6     (2.25, 1.75, 1.25)  7.25            2  1  1    6
  min (0.25, 0.25, 0.25), max (2.25, 1.75, 1.25): yBlocks = ceil(1.5) = 2, zBlocks = ceil(1.0) = 1.
Partition order P0 P2 P3 P1 P4 P5 P6.  Filling: id 2 fills first (P2, P3), then id 0 (P0, P1): full buckets in completion order, not
id order.  Partial buckets in ascending id: 1 (P4), 4 (P5), 6 (P6).  Output P2 P3 P0 P1 P4 P5 P6.
Bucket centres xB + 0.75, yB + 0.75, zB + 0.75 of the creator: id2 (1.75, 0.75, 0.75), id0 (0.75, 0.75, 0.75), id1 (0.75, 1.75, 0.75),
id4 (2.75, 0.75, 0.75), id6 (2.75, 1.75, 1.75).
Level 1 centres: Math.round((c - centre) * 65534) + 32767: a delta of -0.5 gives 0, 0 gives 32767, and P1's x delta 0.25 gives
16383.5, a tie that Math.round takes up: 16384 + 32767 = 49151.
Every splat: scale (0.5, 0.25, 1.0) -> halves 0x3800 0x3400 0x3C00; rotation bytes (255, 128, 128, 128) -> (127/128, 0, 0, 0), normalised
twice -> w = 1 -> halves 0x3C00 0 0 0; colour (10 i, 20, 30, 200) for file index i.
"""
import struct

CENTERS = {"P0": (0.25, 0.25, 0.25), "P1": (1.0, 0.75, 0.75), "P2": (1.25, 0.25, 0.25), "P3": (1.25, 0.75, 0.25), "P4": (0.25, 1.75, 0.25),
           "P5": (2.25, 0.25, 0.25), "P6": (2.25, 1.75, 1.25)}
FILE_ORDER = ["P4", "P2", "P6", "P0", "P5", "P3", "P1"]
OUT_ORDER = ["P2", "P3", "P0", "P1", "P4", "P5", "P6"]
Q_LEVEL1 = {"P2": (0, 0, 0), "P3": (0, 32767, 0), "P0": (0, 0, 0), "P1": (49151, 32767, 32767), "P4": (0, 32767, 0), "P5": (0, 0, 0),
            "P6": (0, 32767, 0)}
BUCKET_CENTERS = [(1.75, 0.75, 0.75), (0.75, 0.75, 0.75), (0.75, 1.75, 0.75), (2.75, 0.75, 0.75), (2.75, 1.75, 1.75)]
OPTIONS = dict(block_size=1.0, bucket_size=2)


def splat_file() -> bytes:
    out = b""
    for i, p in enumerate(FILE_ORDER):
        out += struct.pack("<3f3f4B4B", *CENTERS[p], 0.5, 0.25, 1.0, 10 * i, 20, 30, 200, 255, 128, 128, 128)
    return out


def _rgba(p):
    return bytes((10 * FILE_ORDER.index(p), 20, 30, 200))


def _header(sections, splats, level):
    h = bytearray(4096)
    struct.pack_into("<BB", h, 0, 0, 1)
    struct.pack_into("<4I", h, 4, sections, sections, splats, splats)
    struct.pack_into("<H", h, 20, level)
    struct.pack_into("<5f", h, 24, 0.0, 0.0, 0.0, -1.5, 1.5)       # no SH: the 8-bit range is the default
    return bytes(h)


def _section(count, level, buckets, full, partial, storage):
    s = bytearray(1024)
    struct.pack_into("<2I", s, 0, count, count)
    if level >= 1:
        struct.pack_into("<2If", s, 8, 2, buckets, 1.0)
        struct.pack_into("<H", s, 20, 12)
        struct.pack_into("<I", s, 24, 32767)
        struct.pack_into("<2I", s, 32, full, partial)
    struct.pack_into("<I", s, 28, storage)
    return bytes(s)


def image_level1() -> bytes:
    body = struct.pack("<3I", 1, 1, 1) + b"".join(struct.pack("<3f", *c) for c in BUCKET_CENTERS)
    for p in OUT_ORDER:
        body += struct.pack("<3H3H4H", *Q_LEVEL1[p], 0x3800, 0x3400, 0x3C00, 0x3C00, 0, 0, 0) + _rgba(p)
    return _header(1, 7, 1) + _section(7, 1, 5, 2, 3, len(body)) + body


def image_level0() -> bytes:
    body = b"".join(struct.pack("<3f3f4f", *CENTERS[p], 0.5, 0.25, 1.0, 1.0, 0.0, 0.0, 0.0) + _rgba(p) for p in OUT_ORDER)
    return _header(1, 7, 0) + _section(7, 0, 0, 0, 0, len(body)) + body


def image_all_removed(level) -> bytes:
    """minimum alpha 201 > every alpha (200): one section that keeps no splat."""
    return _header(1, 0, level) + _section(0, level, 0, 0, 0, 0)


def cases():
    """-> [(name, .splat bytes, generator options, expected image)]"""
    f = splat_file()
    out = []
    for alpha in (0, 1, 128):
        out.append((f"level1_alpha{alpha}", f, dict(OPTIONS, compression_level=1, minimum_alpha=alpha), image_level1()))
    out.append(("level0", f, dict(OPTIONS, compression_level=0, minimum_alpha=1), image_level0()))
    for level in (0, 1):
        out.append((f"all_removed_level{level}", f, dict(OPTIONS, compression_level=level, minimum_alpha=201), image_all_removed(level)))
    out.append(("empty", b"", dict(OPTIONS, compression_level=1, minimum_alpha=1), _header(0, 0, 1)))
    return out
