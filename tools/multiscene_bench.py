"""Time a dynamic multi-scene mesh the shape of the reference's demo/dynamic_scenes.html.

    python tools/multiscene_bench.py [--frames 120] [--scale 1.0]

Three .ksplat images generated from seeds as bench.py's scenes are: a garden-sized scene (5.8 M splats, SH2) and two bonsai-sized
scenes (1.2 M splats each), all at compression level 1.  They go into one Viewer(dynamicScene=True) through addSplatScenes, and the
two bonsai scenes move on orbits every frame at 1920 x 1080, as in the demo.  --scale multiplies every splat count.  One JSON line with
  load_ms           the host time of addSplatScenes (every image through one gs_upload_scenes)
  dynamic_frame_ms  the median device time of one frame (sort + render) between CUDA events on the engine's stream, transforms moving
  static_frame_ms   the same for the same splats in a static mesh (the transforms baked at load, nothing applied per frame)
and the card's name and power limit, read in the same run.  Dynamic mode adds a 4x4 product per splat in k_depth and a product plus an
inverse per splat in k_project; this reports that cost.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import math
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

W, H = 1920, 1080
SCENES = ((5_800_000, 2, "garden", 2), (1_200_000, 2, "bonsai", 1), (1_200_000, 2, "bonsai", 4))   # (splats, SH degree, kind, seed)


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def images(scale: float) -> list[bytes]:
    from gaussiansplats3d_b200 import ksplat
    from gaussiansplats3d_b200.scenes import synthetic_scene
    out = []
    for n, sh, kind, seed in SCENES:
        r = synthetic_scene(max(int(n * scale), 1), seed=seed, kind=kind, sh_degree=sh)
        out.append(ksplat.write(r.centers, r.scales, r.rotations, r.colors, r.sh, r.sh_degree, compression_level=1))
    return out


def orbit(t: float):
    """Positions of the two moving scenes at time t (radians)."""
    return (6.0 * math.cos(t), 1.0, 6.0 * math.sin(t)), (-6.0 * math.cos(0.7 * t), 2.0, -6.0 * math.sin(0.7 * t))


def measure(imgs, dynamic: bool, frames: int):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.viewer import Viewer
    v = Viewer(dict(width=W, height=H, sphericalHarmonicsDegree=2, dynamicScene=dynamic, initialCameraPosition=(0, 8, 22)))
    p1, p2 = orbit(0.0)
    opts = [dict(format=3, data=imgs[0]), dict(format=3, data=imgs[1], position=p1, scale=(0.4, 0.4, 0.4)),
            dict(format=3, data=imgs[2], position=p2, scale=(0.4, 0.4, 0.4))]
    t0 = time.perf_counter()
    v.addSplatScenes(opts)
    v.engine.synchronize()
    load_ms = (time.perf_counter() - t0) * 1e3
    ev0, ev1 = v.engine.event(), v.engine.event()
    times = []
    for k in range(frames + 10):
        if dynamic:
            p1, p2 = orbit(0.02 * k)
            v.getSplatScene(1).position, v.getSplatScene(2).position = p1, p2
        ev0.record()
        v.frame(frame_format=N.GS_FRAME_RGBA8, download=False)
        ev1.record()
        v.engine.synchronize()
        if k >= 10:   # the first frames capture the frame graph
            times.append(ev0.elapsed_ms(ev1))
    n = v.splatMesh.getSplatCount()
    v.dispose()
    return load_ms, statistics.median(times), min(times), n


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    gpu = card()
    imgs = images(args.scale)
    load_ms, dyn_ms, dyn_min, n = measure(imgs, True, args.frames)
    _, static_ms, static_min, _ = measure(imgs, False, args.frames)
    print(json.dumps(dict(scenes=len(imgs), splats=n, width=W, height=H, frames=args.frames, load_ms=round(load_ms, 2),
                          dynamic_frame_ms=round(dyn_ms, 4), dynamic_frame_ms_min=round(dyn_min, 4), static_frame_ms=round(static_ms, 4),
                          static_frame_ms_min=round(static_min, 4), dynamic_vs_static=round(dyn_ms / static_ms, 3), gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
