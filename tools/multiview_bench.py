"""Time multi-view frames (gs_frame_views) against the mono frames they replace.

    python tools/multiview_bench.py [--workloads bonsai,garden] [--views 1,2,4,8] [--frames 60] [--rounds 3]

For each of bench.py's bonsai (1.2 M splats) and garden (5.8 M splats, SH2) workloads, V cameras on a circle around the scene's target,
the first at bench.py's first camera, 1920 x 1080 per view.  Three cases, each frame after an L2 flush:
  views   one V-view frame: one batched sort of the V cameras, every view projected, binned and blended in shared launches
  mono_V  V mono gs_frame_async calls, one per camera: what the V views cost without this feature
  mono    one mono frame of the first camera
The mono cases are timed between two CUDA events on the engine's stream around their frame graphs; a multi-view frame returns only once
its status has been read back, so it is timed by the engine's own events around its frame graph (gs_timings.render_total_ms of a graph
frame).  The cases take turns in blocks of frames / rounds frames, each after five warm-up frames (a change of view count captures a new
frame graph).  One JSON line per workload, view count and case with the median and minimum, and the card's name and power limit read in
the same run.  Needs a GPU."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

W, H = 1920, 1080


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def ring(viewer, count):
    """`count` cameras around the viewer camera's target, the first the viewer camera itself."""
    from gaussiansplats3d_b200 import three_math as TM
    cam = viewer.camera
    out = [cam]
    for i in range(1, count):
        c = TM.PerspectiveCamera(cam.fov, cam.aspect, cam.near, cam.far)
        c.up = cam.up
        c.position = cam.target + TM.rotate_about_axis(cam.position - cam.target, cam.up, 2.0 * np.pi * i / count)
        c.look_at(cam.target)
        c.update()
        out.append(c)
    return out


def measure(workload: str, view_counts, frames: int, rounds: int, gpu: str):
    import dataclasses

    import bench
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    n, sh, kind, seed, cam, _, _, _ = bench.WORKLOADS[workload]
    c = CAMERAS[cam]
    vmax = max(view_counts)
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=W, height=H,
                    sphericalHarmonicsDegree=sh))
    v.addSplatScene(synthetic_scene(n, seed=seed, kind=kind, sh_degree=sh))
    v.camera.update()
    v.updateSplatMesh()
    # the stacked frame of vmax views: an engine as tall as that
    from gaussiansplats3d_b200.engine import Engine
    e = Engine(n, max_width=W, max_height=vmax * H)
    p = v.splatMesh.packed
    e.upload_splat_data(p.centers_colors, p.covariances, p.sh, p.sh_degree)
    e.upload_centers(p.int_centers)
    u = v.uniforms()
    cams = ring(v, vmax)
    views = [v.viewFor(x) for x in cams]
    fmt = dict(frame_format=N.GS_FRAME_RGBA8, flip_y=True)
    mono = [e.prepare_frame(x.model_view_proj, dataclasses.replace(u, model_view=x.model_view, projection=x.projection,
                                                                     camera_position=x.camera_position, focal=x.focal),
                            W, H, n, **fmt) for x in views]
    ev0, ev1 = e.event(), e.event()

    def run(case, count):
        if case == "views":
            e.flush_l2()
            e.frame_views(views[:count], u, W, H, n, download=False, **fmt)
            return e.timings()["render_total_ms"]
        e.flush_l2()
        ev0.record()
        for prepared in mono[:count if case == "mono_V" else 1]:
            e.frame_async(None, None, 0, 0, 0, prepared=prepared)
        ev1.record()
        e.synchronize()
        return ev0.elapsed_ms(ev1)

    for count in view_counts:
        cases = ["views", "mono_V", "mono"]
        times = {k: [] for k in cases}
        for _ in range(rounds):
            for k in cases:
                for _ in range(5):
                    run(k, count)
                for _ in range(max(frames // rounds, 1)):
                    times[k].append(run(k, count))
        med = {k: statistics.median(t) for k, t in times.items()}
        for k, t in times.items():
            line = dict(workload=workload, splats=n, view_width=W, view_height=H, views=count, case=k, frames=len(t),
                        frame_ms=round(med[k], 4), frame_ms_min=round(min(t), 4))
            if k == "views":
                line["vs_mono_V_pct"] = round(100.0 * (med["views"] / med["mono_V"] - 1.0), 2)
                line["per_view_ms"] = round(med["views"] / count, 4)
            line["gpu"] = gpu
            print(json.dumps(line), flush=True)
    e.close()
    v.dispose()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="bonsai,garden")
    ap.add_argument("--views", default="1,2,4,8")
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    gpu = card()
    for wl in args.workloads.split(","):
        measure(wl, [int(x) for x in args.views.split(",")], args.frames, args.rounds, gpu)


if __name__ == "__main__":
    main()
