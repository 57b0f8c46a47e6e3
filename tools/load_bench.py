"""Load throughput of gs_upload_file: a seeded garden-sized INRIA `.ply` (5.8 M splats, 45 f_rest, about 1.4 GB), `.splat`,
PlayCanvas-compressed `.ply` (5.8 M splats, 45 SH bytes, about 0.36 GB), `.spz` (5.8 M splats, SH degree 3, version 2, 64 bytes per
splat before gzip) or INRIA v2 (codebook) `.ply` (5.8 M splats, SH degree 3, 62 bytes per splat: half x/y/z and uchar indices into a
256-row codebook of all 20 entries) built in memory, then loaded with sphericalHarmonicsDegree 2 a few times.  For `.spz` each run also times the host
gunzip (gzip.decompress of the file as stored) on its own, before the load of the packed stream it returns.

Prints one JSON line per run and a summary: wall clock around the whole call (it ends in a stream synchronise), device time of the
conversion and decode kernels from the engine's CUDA-event timeline (gs_set_profiling), the time the copy stream segments took, and
file GB/s.  The card name and power limit are printed in the same run.

With --optimize the file goes through SplatBufferGenerator on the GPU (gs_upload_file_optimized) at compression level --level; the
generation's phases appear in the timeline as gen_* segments.  INRIA v2 loads only that way, so --format inriav2 implies --optimize.

    python tools/load_bench.py [--splats 5800000] [--repeats 3] [--format ply|splat|pcply|spz|inriav2] [--optimize --level 0|1|2]
"""
from __future__ import annotations

import argparse
import ctypes as C
import gzip
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from gaussiansplats3d_b200 import Engine, _native as N  # noqa: E402


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def garden_ply(n: int, seed: int = 0) -> bytes:
    """INRIA property order: x y z nx ny nz f_dc_0..2 f_rest_0..44 opacity scale_0..2 rot_0..3, all float (248 bytes per splat)."""
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{k}" for k in range(45)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    rng = np.random.default_rng(seed)
    rec = np.empty((n, len(names)), np.float32)
    for k, nm in enumerate(names):
        if nm in ("x", "y", "z"):
            rec[:, k] = rng.uniform(-20, 20, n)
        elif nm.startswith("scale"):
            rec[:, k] = rng.uniform(-7, -2, n)
        elif nm.startswith("n"):
            rec[:, k] = 0
        else:
            rec[:, k] = rng.standard_normal(n, np.float32) * (0.2 if nm.startswith("f_rest") else 1.0)
    head = "\n".join(["ply", "format binary_little_endian 1.0", f"element vertex {n}", *[f"property float {nm}" for nm in names], "end_header"]) + "\n"
    return head.encode("ascii") + rec.tobytes()


def splat_file(n: int, seed: int = 0) -> bytes:
    rng = np.random.default_rng(seed)
    rec = np.empty((n, 8), np.float32)
    rec[:, 0:3] = rng.uniform(-20, 20, (n, 3))
    rec[:, 3:6] = np.exp(rng.uniform(-7, -2, (n, 3)))
    rec[:, 6:8] = rng.integers(0, 256, (n, 8), dtype=np.uint8).view(np.float32)
    return rec.tobytes()


def pcply_file(n: int, seed: int = 0) -> bytes:
    """PlayCanvas-compressed: chunk rows of 18 float extremes, vertex rows of 4 packed uints, sh rows of 45 uchar f_rest."""
    rng = np.random.default_rng(seed)
    nc = (n + 255) // 256
    ext = ["min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y", "min_scale_z",
           "max_scale_x", "max_scale_y", "max_scale_z", "min_r", "min_g", "min_b", "max_r", "max_g", "max_b"]
    lo = np.concatenate([rng.uniform(-20, 0, (nc, 3)), rng.uniform(-7, -4, (nc, 3)), rng.uniform(-0.2, 0.3, (nc, 3))], 1)
    hi = lo + np.concatenate([rng.uniform(1, 20, (nc, 3)), rng.uniform(0.5, 3, (nc, 3)), rng.uniform(0.5, 1, (nc, 3))], 1)
    chunk = np.empty((nc, 18), np.float32)
    chunk[:, [0, 1, 2, 6, 7, 8, 12, 13, 14]], chunk[:, [3, 4, 5, 9, 10, 11, 15, 16, 17]] = lo, hi
    vertex = rng.integers(0, 1 << 32, (n, 4), dtype=np.uint64).astype(np.uint32)
    sh = rng.integers(0, 256, (n, 45), dtype=np.uint8)
    head = "\n".join(["ply", "format binary_little_endian 1.0", f"element chunk {nc}", *[f"property float {k}" for k in ext],
                      f"element vertex {n}", *[f"property uint packed_{k}" for k in ("position", "rotation", "scale", "color")],
                      f"element sh {n}", *[f"property uchar f_rest_{k}" for k in range(45)], "end_header"]) + "\n"
    return head.encode("ascii") + chunk.tobytes() + vertex.tobytes() + sh.tobytes()


def spz_file(n: int, seed: int = 0) -> bytes:
    """A gzipped v2 stream at SH degree 3: positions within +-20 at 12 fractional bits, random bytes in every other plane."""
    rng = np.random.default_rng(seed)
    fixed = (rng.uniform(-20, 20, (n, 3)) * 4096).astype(np.int64) & 0xFFFFFF
    pos = np.stack([(fixed >> (8 * b)) & 0xFF for b in range(3)], 2).astype(np.uint8)
    planes = rng.integers(0, 256, (n, 1 + 3 + 3 + 3 + 45), dtype=np.uint8)
    head = np.array([0x5053474E, 2, n], "<u4").tobytes() + bytes([3, 12, 0, 0])
    alphas, colors, scales, rotations, sh = (np.ascontiguousarray(planes[:, a:b]) for a, b in ((0, 1), (1, 4), (4, 7), (7, 10), (10, 55)))
    body = b"".join(a.tobytes() for a in (pos, alphas, colors, scales, rotations, sh))
    return gzip.compress(head + body, compresslevel=6, mtime=0)


def inriav2_file(n: int, seed: int = 0) -> bytes:
    """INRIA v2: a 256-row codebook of the 20 half entries, then splat rows of half x y z and uchar scale, rot, f_dc, opacity, f_rest."""
    rng = np.random.default_rng(seed)
    pages = ["features_dc"] + [f"features_rest_{k}" for k in range(15)] + ["opacity", "scaling", "rotation_re", "rotation_im"]
    cb = rng.standard_normal((256, 20)).astype(np.float16)
    cb[:, 17] = rng.uniform(-7, -2, 256)
    fields = ["scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3", "f_dc_0", "f_dc_1", "f_dc_2", "opacity"] + \
        [f"f_rest_{k}" for k in range(45)]
    rec = np.empty(n, np.dtype([("xyz", "<f2", 3), ("idx", "u1", len(fields))]))
    rec["xyz"] = rng.uniform(-20, 20, (n, 3))
    rec["idx"] = rng.integers(0, 256, (n, len(fields)), dtype=np.uint8)
    head = "\n".join(["ply", "format binary_little_endian 1.0", "element codebook_centers 256", *[f"property ushort {k}" for k in pages],
                      f"element vertex {n}", *[f"property ushort {k}" for k in "xyz"], *[f"property uchar {k}" for k in fields],
                      "end_header"]) + "\n"
    return head.encode("ascii") + cb.tobytes() + rec.tobytes()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--splats", type=int, default=5_800_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--format", choices=("ply", "splat", "pcply", "spz", "inriav2"), default="ply")
    ap.add_argument("--optimize", action="store_true", help="load through SplatBufferGenerator (gs_upload_file_optimized)")
    ap.add_argument("--level", type=int, default=0, choices=(0, 1, 2), help="compression level of --optimize")
    a = ap.parse_args()
    a.optimize = a.optimize or a.format == "inriav2"
    fmt = {"splat": N.GS_FILE_SPLAT, "spz": N.GS_FILE_SPZ}.get(a.format, N.GS_FILE_PLY)
    data = {"ply": garden_ply, "splat": splat_file, "pcply": pcply_file, "spz": spz_file, "inriav2": inriav2_file}[a.format](a.splats)
    print(json.dumps(dict(card=card(), format=a.format, splats=a.splats, file_bytes=len(data), optimize=a.optimize, level=a.level)))
    lib = N.load()
    e = Engine(a.splats, max_width=1920, max_height=1080)

    def load(stream):
        if a.optimize:
            e.upload_file_optimized(fmt, stream, sh_degree=2, compression_level=a.level)
        else:
            e.upload_file(fmt, stream, sh_degree=2)
    packed = gzip.decompress(data) if a.format == "spz" else data
    load(packed)                                    # warm-up: first-touch allocations of the engine's SH / covariance buffers
    runs = []
    for r in range(a.repeats):
        gunzip = None
        if a.format == "spz":
            t0 = time.perf_counter()
            packed = gzip.decompress(data)
            gunzip = time.perf_counter() - t0
        e.set_profiling(True)
        t0 = time.perf_counter()
        load(packed)
        wall = time.perf_counter() - t0
        buf = (N.gs_kernel_time * 4096)()
        cnt = C.c_uint32(0)
        N.check(lib.gs_kernel_timings(e._h, buf, 4096, C.byref(cnt)), "gs_kernel_timings")
        e.set_profiling(False)
        per = {}
        for i in range(min(cnt.value, 4096)):
            per[buf[i].name.decode()] = per.get(buf[i].name.decode(), 0.0) + buf[i].ms
        kernels = sum(v for k, v in per.items() if k.startswith("k_") or k.startswith("gen_"))
        run = dict(run=r, wall_ms=wall * 1e3, kernels_ms=kernels, **{f"{k}_ms": v for k, v in per.items()}, file_GBps=len(packed) / wall / 1e9)
        if gunzip is not None:
            run["host_gunzip_ms"] = gunzip * 1e3
        runs.append(run)
        print(json.dumps(run))
    med = lambda k: float(np.median([x[k] for x in runs]))  # noqa: E731
    extra = dict(host_gunzip_ms=med("host_gunzip_ms"), packed_bytes=len(packed)) if a.format == "spz" else {}
    print(json.dumps(dict(summary=True, card=card(), format=a.format, splats=a.splats, file_bytes=len(data), wall_ms=med("wall_ms"),
                          kernels_ms=med("kernels_ms"), file_GBps=med("file_GBps"), **extra)))
    e.close()


if __name__ == "__main__":
    main()
