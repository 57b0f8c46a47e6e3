"""Time gs_raycast on bonsai-, garden- and 16 M-sized SplatTrees.

    python tools/raycast_bench.py [--workloads bonsai,garden,synth16m] [--calls 20] [--ellipsoid]

Each workload is bench.py's synthetic scene with a static mesh (the decompose of S R T runs per candidate splat) and the SplatTree the
Viewer builds.  For each of 64 screen positions (8 x 8 grid, bench.py's camera) the wall-clock time of `calls` gs_raycast calls with
capacity 1 is taken around the call, which ends in a stream synchronise; the median over all calls is reported together with the reached
leaves, candidate splats and hits per ray.  One JSON line per workload."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

WORKLOADS = {"bonsai": (1_200_000, 0, "bonsai"), "garden": (5_800_000, 2, "garden"), "synth16m": (16_000_000, 0, "bonsai")}
CAMERA = dict(position=(1.54163, 2.68515, -6.37228), look_at=(0.45622, 1.95338, 1.51278), up=(0.01933, -0.7583, -0.65161))


def reached_leaves(leaves, o, d) -> np.ndarray:
    """bool[m]: Ray.intersectBox (Ray.js:26-82) on every node, vectorised in its operation order, ANDed up each leaf's ancestor chain."""
    mn, mx = leaves.all_min, leaves.all_max
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    eps = 0.0001

    def inside(p):
        return ~((p < mn - eps) | (p > mx + eps)).any(1)

    hit = inside(np.broadcast_to(o, mn.shape))
    for a in range(3):
        if d[a] == 0:
            continue
        plane = mx[:, a] if d[a] < 0 else mn[:, a]
        to_side = plane - o[a]
        ok = to_side * -np.sign(d[a]) < 0
        p = np.empty_like(mn)
        p[:, a] = plane
        for b in ((a + 1) % 3, (a + 2) % 3):
            p[:, b] = d[b] / d[a] * to_side + o[b]
        hit |= ok & inside(p)
    node = leaves.leaf_node.astype(np.int64)
    out = hit[node]
    par = leaves.all_parent
    while (node >= 0).any():
        node = np.where(node >= 0, par[np.maximum(node, 0)], -1)
        out &= np.where(node >= 0, hit[np.maximum(node, 0)], True)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="bonsai,garden,synth16m")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--ellipsoid", action="store_true")
    args = ap.parse_args()
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.raycaster import Raycaster, ray_records_from_raw
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.splat_tree import SplatTree
    w, h = 1920, 1080
    for name in args.workloads.split(","):
        n, seed, kind = WORKLOADS[name]
        raw = synthetic_scene(n, seed=seed, kind=kind)
        t0 = time.perf_counter()
        leaves = SplatTree().processSplatMesh(raw.centers, raw.colors[:, 3], 1)
        build_s = time.perf_counter() - t0
        e = Engine(n, ray_records=True)
        e.upload_ray_records(ray_records_from_raw(raw))
        e.upload_splat_tree(leaves)
        e.upload_splat_tree_nodes(leaves)
        cam = TM.PerspectiveCamera(50, w / h, 0.1, 1000.0)
        cam.position = np.array(CAMERA["position"])
        cam.up = np.array(CAMERA["up"]) / np.linalg.norm(CAMERA["up"])
        cam.look_at(CAMERA["look_at"])
        rc = Raycaster()
        times, hits, reached, cand = [], [], [], []
        offsets = leaves.offsets.astype(np.int64)
        for iy in range(8):
            for ix in range(8):
                rc.setFromCameraAndScreenPosition(cam, ((ix + 0.5) * w / 8, (iy + 0.5) * h / 8), (w, h))
                for c in range(args.calls + 2):
                    t = time.perf_counter()
                    _, total = e.raycast(rc.ray.origin, rc.ray.direction, None, ellipsoid=args.ellipsoid, capacity=1)
                    if c >= 2:
                        times.append((time.perf_counter() - t) * 1e3)
                hits.append(total)
                r = reached_leaves(leaves, rc.ray.origin, rc.ray.direction)
                reached.append(int(r.sum()))
                cand.append(int((np.diff(offsets) * r).sum()))
        print(json.dumps(dict(workload=name, splats=n, leaves=leaves.count, nodes=int(leaves.all_parent.shape[0]), tree_build_s=round(build_s, 2),
                              mode="ellipsoid" if args.ellipsoid else "sphere", median_ms=round(statistics.median(times), 4),
                              p90_ms=round(float(np.percentile(times, 90)), 4), reached_leaves_median=int(np.median(reached)),
                              candidates_median=int(np.median(cand)), candidates_max=int(max(cand)), hits_median=int(np.median(hits)),
                              hits_max=int(max(hits)))), flush=True)
        e.close()


if __name__ == "__main__":
    main()
