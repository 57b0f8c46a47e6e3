"""Time gs_compute_bounding_box (SplatMesh.computeBoundingBox on the GPU) on bonsai-, garden- and 16 M-sized scenes.

    python tools/bounds_bench.py [--workloads bonsai,garden,synth16m] [--calls 50]

Each workload is bench.py's synthetic scene, held three ways, each timed without and with scene transforms:
  records   a .splat file of the scene decoded on an engine with ray records, under a static scene transform: the box reads the 56-byte
            records (getSplatCenter's f64 centre) and applies the transform in f64 when asked
  packed    the scene host-packed on a static engine: the box reads the 16-byte centre-colour texels, the identity applied when asked
  dynamic   the same on a dynamic engine: the scene's transform applied per splat when asked
For each, `calls` calls are timed on the host around the call, which ends in a stream synchronise (the box is on the host when it
returns); the median is reported with the bytes of splat data read per second at that median.  One JSON line per workload and way, each
with the card's name and power limit read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

WORKLOADS = {"bonsai": (1_200_000, 0, "bonsai"), "garden": (5_800_000, 2, "garden"), "synth16m": (16_000_000, 0, "bonsai")}


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def splat_file(raw) -> bytes:
    """The scene as a .splat file (SplatParser's 32-byte rows: centre, scale, rgba, rotation bytes)."""
    n = raw.count
    rec = np.zeros((n, 8), np.float32)
    rec[:, 0:3] = raw.centers
    rec[:, 3:6] = raw.scales
    b = rec.view(np.uint8).reshape(n, 32)
    b[:, 24:28] = np.asarray(raw.colors, np.uint8)
    q = np.asarray(raw.rotations, np.float32)            # x y z w -> the file's w x y z bytes
    b[:, 28:32] = np.clip(np.round(q[:, [3, 0, 1, 2]] * 128 + 128), 0, 255).astype(np.uint8)
    return rec.tobytes()


def time_calls(fn, calls: int) -> float:
    fn()                                                  # warm: the kernels' first load, the call's buffers
    ts = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="bonsai,garden,synth16m")
    ap.add_argument("--calls", type=int, default=50)
    args = ap.parse_args()
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import synthetic_scene
    gpu = card()
    xf = TM.compose((0.5, -1.25, 2.0), (0.3, -0.5, 0.2, 0.7874007874011811), (1.5, 0.75, 1.25))
    for name in args.workloads.split(","):
        n, seed, kind = WORKLOADS[name]
        raw = synthetic_scene(n, seed=seed, kind=kind)
        cc = np.empty((n, 4), np.uint32)
        cc[:, 0] = np.asarray(raw.colors, np.uint32)[:, 3] << 24
        cc[:, 1:] = np.ascontiguousarray(raw.centers, np.float32).view(np.uint32)
        cov = np.zeros((n, 6), np.float16)
        ways = []
        e = Engine(n, ray_records=True, max_width=64, max_height=64)
        e.upload_file(N.GS_FILE_SPLAT, splat_file(raw), transform16=xf)
        ways.append(("records", e, 56, [dict(apply_scene_transforms=False), dict(apply_scene_transforms=True)]))
        e = Engine(n, max_width=64, max_height=64)
        e.upload_splat_data(cc, cov)
        ways.append(("packed", e, 16, [dict(apply_scene_transforms=False), dict(apply_scene_transforms=True)]))
        e = Engine(n, dynamic_mode=True, max_width=64, max_height=64)
        e.upload_splat_data(cc, cov)
        ways.append(("dynamic", e, 16, [dict(apply_scene_transforms=False), dict(apply_scene_transforms=True, scene_transforms=[xf])]))
        for way, e, rec_bytes, calls in ways:
            for kw in calls:
                ms = time_calls(lambda: e.compute_bounding_box(-1, **kw), args.calls)
                lo, hi = e.compute_bounding_box(-1, **kw)
                print(json.dumps(dict(workload=name, splats=n, way=way, scene_transforms=kw["apply_scene_transforms"], calls=args.calls,
                                      median_ms=round(ms, 4), read_gb_per_s=round(n * rec_bytes / (ms * 1e-3) / 1e9, 1),
                                      box_min=[float(v) for v in lo], box_max=[float(v) for v in hi], gpu=gpu)), flush=True)
            e.close()


if __name__ == "__main__":
    main()
