"""Time gs_build_splat_tree (the SplatTree built on the GPU at load) on bench.py's bonsai, garden and 16 M synthetic scenes.

    python tools/tree_build_bench.py [--workloads bonsai,garden,synth16m] [--repeats 7] [--host]

Each workload uploads the scene's centres and alphas (GS_BUF_CENTERS_COLORS is all the build reads), builds the tree once to warm up,
then `repeats` times at the Viewer's values (depth 8, 1000 centres per node, alpha >= 1).  Two clocks per build: the device time the call
reports (CUDA events on the engine's stream around all of its kernels) and the wall clock around the call, which ends synchronised and so
includes its allocations, its per-level read-backs and the release of its scratch.  One JSON line per workload with the median and the
spread of both, the tree's sizes, the scratch the build allocated, and the card's name and power limit read in the same run.
`--host` also times the host build (splat_tree.SplatTree.processSplatMesh) beside it and checks that both give the same leaves; it takes
tens of seconds at 16 M splats.  Without a GPU the engine cannot be created and the tool fails."""
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


def centers_colors(raw) -> np.ndarray:
    cc = np.empty((raw.count, 4), np.uint32)
    c = np.asarray(raw.colors, np.uint32)
    cc[:, 0] = c[:, 0] | (c[:, 1] << 8) | (c[:, 2] << 16) | (c[:, 3] << 24)
    cc[:, 1:] = np.ascontiguousarray(raw.centers, np.float32).view(np.uint32)
    return cc


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="bonsai,garden,synth16m")
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--host", action="store_true", help="also time the host build and compare the leaves")
    args = ap.parse_args()
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.splat_tree import SplatTree
    gpu = card()
    for name in args.workloads.split(","):
        n, seed, kind = WORKLOADS[name]
        raw = synthetic_scene(n, seed=seed, kind=kind)
        e = Engine(n, max_width=64, max_height=64)
        e.upload_splat_data(centers_colors(raw), np.zeros((n, 6), np.float32))
        e.build_splat_tree()                                  # warm-up: module load, first allocations
        device_ms, wall_ms = [], []
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            info = e.build_splat_tree()
            wall_ms.append((time.perf_counter() - t0) * 1e3)
            device_ms.append(info["build_ms"])
        line = dict(workload=name, splats=n, leaves=info["leaf_count"], nodes=info["node_count"], indexes=info["index_count"], levels=info["level_count"],
                    max_leaf_depth=info["max_leaf_depth"], max_level_memberships=info["max_level_memberships"],
                    scratch_mb=round(info["scratch_bytes"] / 2**20, 1), scratch_bytes_per_splat=round(info["scratch_bytes"] / n, 1), repeats=args.repeats,
                    device_ms_median=round(statistics.median(device_ms), 3), device_ms_min=round(min(device_ms), 3), device_ms_max=round(max(device_ms), 3),
                    wall_ms_median=round(statistics.median(wall_ms), 3), wall_ms_min=round(min(wall_ms), 3), wall_ms_max=round(max(wall_ms), 3), gpu=gpu)
        if args.host:
            t0 = time.perf_counter()
            want = SplatTree().processSplatMesh(raw.centers, raw.colors[:, 3], 1)
            line["host_build_s"] = round(time.perf_counter() - t0, 2)
            got = e.read_splat_tree()
            line["equals_host_tree"] = bool(all(np.array_equal(getattr(got, k), getattr(want, k)) for k in
                                                ("node_min", "node_max", "offsets", "indexes", "depth", "all_min", "all_max", "all_parent", "leaf_node")))
        print(json.dumps(line), flush=True)
        e.close()


if __name__ == "__main__":
    main()
