"""Time the binning kernels that bench.py's workloads never launch: the radix binning of frames above 256 coarse tiles
(k_tile_count, k_tile_emit, the k_radix_*[tile,*] passes) and the sharded sort's subset compaction (k_subset_count, k_subset_emit).

    python tools/binning_bench.py [--splats 5800000] [--width 7680] [--height 4320] [--seconds 1.0]

The scene is bench.py's synthetic garden (seed 2, garden camera) at SH degree 0, since binning does not read the harmonics.  Two engines
render it at the given size: a single-GPU one, and rank 0 of a two-rank group on the same device with GS_SUBSET_MIN=1, whose frame sorts
only the splats that reach its own coarse tiles and bins the sharded way.  Each renders warm-up frames, then profiled frames
(gs_set_profiling, one CUDA event after every kernel) until about `seconds` of frames are collected.  One JSON line per engine with the
median, minimum and maximum of every binning kernel over those frames, the frame's instance count, and the card's name and power limit
read in the same run.  Without a GPU the engine cannot be created and the tool fails."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

KERNELS = ("k_tile_count", "k_tile_emit", "k_subset_count", "k_subset_emit")


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def measure(raw, width: int, height: int, seconds: float, world: int) -> dict:
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["garden"]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=width, height=height,
                    sphericalHarmonicsDegree=0, rank=0, world_size=world))
    v.addSplatScene(raw)
    v.camera.update()
    v.updateSplatMesh()
    e, n = v.engine, raw.count
    prepared = e.prepare_frame(v.mvp_matrix().astype(np.float32), v.uniforms(), width, height, n)
    ev0, ev1 = e.event(), e.event()
    for _ in range(3):                                    # warm-up: module load, first allocations, the frame's graph
        ev0.record()
        e.frame_async(None, None, width, height, n, prepared=prepared)
        ev1.record()
        e.synchronize()
    frames = max(5, int(seconds * 1e3 / ev0.elapsed_ms(ev1)))
    e.set_profiling(True)
    acc: dict[str, list[float]] = {}
    for _ in range(frames):
        for _ in range(10):      # queued work that lets the host enqueue the whole frame ahead of the device, so that the gaps
            e.flush_l2()         # between events are kernel time; the last one leaves L2 cold, as in bench.py's timeline
        e.frame_async(None, None, width, height, n, prepared=prepared)
        e.synchronize()
        for name, ms in e.kernel_timings():
            if name in KERNELS or "[tile," in name:
                acc.setdefault(name, []).append(ms)
    e.set_profiling(False)
    line = dict(world_size=world, frames=frames, tile_instances=int(e.timings()["tile_instances"]),
                kernels_ms={k: dict(median=round(statistics.median(t), 4), min=round(min(t), 4), max=round(max(t), 4)) for k, t in acc.items()})
    v.dispose()
    return line


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--splats", type=int, default=5_800_000)
    ap.add_argument("--width", type=int, default=7680)
    ap.add_argument("--height", type=int, default=4320)
    ap.add_argument("--seconds", type=float, default=1.0, help="profiled frames per engine, in seconds of frame time")
    args = ap.parse_args()
    from gaussiansplats3d_b200.scenes import synthetic_scene
    gpu = card()
    raw = synthetic_scene(args.splats, seed=2, kind="garden", sh_degree=0)
    os.environ["GS_SUBSET_MIN"] = "1"                     # read when a sharded frame is enqueued; single-GPU frames never sort a subset
    for world in (1, 2):
        line = dict(splats=args.splats, width=args.width, height=args.height, **measure(raw, args.width, args.height, args.seconds, world), gpu=gpu)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
