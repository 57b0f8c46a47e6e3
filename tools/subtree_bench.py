"""Time the SplatTree forest of a dynamic multi-scene mesh: tools/multiscene_bench.py's mesh (a garden-sized scene and two bonsai-sized
scenes, the two small ones moving) with one sub-tree per scene.

    python tools/subtree_bench.py [--frames 120] [--scale 1.0]

One JSON line with
  forest_build_ms       device time of gs_build_splat_tree on the dynamic mesh (one sub-tree per scene)
  static_build_ms       the same splats in a static mesh: one tree over all of them
  gather_us             device time of one gs_gather_for_sort_subtrees (cull + layout + copy), median over the moving orbit
  frame_ms_tree / frame_ms_no_tree   median time between CUDA events around Viewer.update + render over the moving orbit (the host
                        gaps of the gather's read-back included) with splatTree on (gather, then sort only the gathered splats) and
                        off (sort every splat); render_count_tree / render_count_no_tree: the mean splats sorted and drawn per frame
  raycast_us            host time of one Raycaster.intersectSplatMesh through the screen centre (returns synchronised), median
and the card's name and power limit, read in the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from multiscene_bench import H, W, card, images, orbit  # noqa: E402


def viewer(imgs, dynamic: bool, tree: bool):
    from gaussiansplats3d_b200.viewer import Viewer
    v = Viewer(dict(width=W, height=H, sphericalHarmonicsDegree=2, dynamicScene=dynamic, initialCameraPosition=(0, 8, 22), splatTree=tree,
                    raycast=tree))
    p1, p2 = orbit(0.0)
    v.addSplatScenes([dict(format=3, data=imgs[0]), dict(format=3, data=imgs[1], position=p1, scale=(0.4, 0.4, 0.4)),
                      dict(format=3, data=imgs[2], position=p2, scale=(0.4, 0.4, 0.4))])
    v.engine.synchronize()
    return v


def frames(v, count: int, gather: bool):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.splat_tree import fov_cosines
    ev0, ev1 = v.engine.event(), v.engine.event()
    times, gathers, rendered = [], [], []
    for k in range(count + 10):
        p1, p2 = orbit(0.02 * k)
        v.getSplatScene(1).position, v.getSplatScene(2).position = p1, p2
        if gather:
            mesh = v.splatMesh
            mesh.fillTransformsArray()
            base = TM.invert(v.camera.matrixWorld)
            views = [TM.multiply(base, mesh.getSceneTransform(s)) for s in range(mesh.getSceneCount())]
            cx, cy = fov_cosines(v.renderWidth, v.renderHeight, v.camera.fov)
            ev0.record()
            v.engine.gather_for_sort_subtrees(views, cx, cy)
            ev1.record()
            v.engine.synchronize()
            if k >= 10:
                gathers.append(ev0.elapsed_ms(ev1) * 1e3)
        ev0.record()
        v.update()                    # runSplatSort: the gather (with a tree), then the sort of what it gathered
        v.render(frame_format=N.GS_FRAME_RGBA8, download=False)
        ev1.record()
        v.engine.synchronize()
        if k >= 10:   # warm-up
            times.append(ev0.elapsed_ms(ev1))
            rendered.append(v.splatRenderCount)
    return statistics.median(times), statistics.mean(rendered), (statistics.median(gathers) if gathers else None)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--scale", type=float, default=1.0)
    args = ap.parse_args()
    gpu = card()
    imgs = images(args.scale)

    v = viewer(imgs, True, True)
    n = v.splatMesh.getSplatCount()
    info = v.engine.build_splat_tree(8, 1000, 1)      # again, warm: the build the viewer ran at load included first launches
    forest_ms, sub_trees = info["build_ms"], info["sub_tree_count"]
    frame_tree, count_tree, gather_us = frames(v, args.frames, True)
    casts = []
    for _ in range(25):
        t0 = time.perf_counter()
        v.raycaster.setFromCameraAndScreenPosition(v.camera, (W / 2, H / 2), (W, H))
        v.raycaster.intersectSplatMesh(v.splatMesh, capacity=1)
        casts.append((time.perf_counter() - t0) * 1e6)
    v.dispose()

    v = viewer(imgs, True, False)
    frame_plain, count_plain, _ = frames(v, args.frames, False)
    v.dispose()

    v = viewer(imgs, False, True)
    v.engine.build_splat_tree(8, 1000, 1)
    static_ms = v.engine.build_splat_tree(8, 1000, 1)["build_ms"]
    v.dispose()

    print(json.dumps(dict(scenes=len(imgs), splats=n, sub_trees=sub_trees, width=W, height=H, frames=args.frames,
                          forest_build_ms=round(forest_ms, 3), static_build_ms=round(static_ms, 3), gather_us=round(gather_us, 1),
                          frame_ms_tree=round(frame_tree, 4), render_count_tree=round(count_tree), frame_ms_no_tree=round(frame_plain, 4),
                          render_count_no_tree=round(count_plain), raycast_us=round(statistics.median(casts), 1), gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
