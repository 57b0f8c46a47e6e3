"""Time frames that render their view depth (gs_render_params.depth) against the same frames without it.

    python tools/depth_bench.py [--workloads bonsai,garden] [--frames 60]

For each of bench.py's bonsai (1.2 M splats, 1080p) and garden (5.8 M splats, SH2, 1080p) workloads, from its first camera, the frame
with depth off and on, the two cases alternating within one run so that clock and neighbour drift hit both alike (in blocks of
frames: the depth bit is part of the frame graph's key, so each switch captures the graph again, in an untimed frame):
  frame     gs_frame_async between two CUDA events on the engine's stream (the captured frame graph: device time per frame)
  blend     k_blend alone, from profiled frames (one event after every kernel, no graph)
and one multi-view case: 4 cameras around the workload's first one, at a quarter of the frame each (gs_frame_views), timed on the device
from profiled frames: the views' k_blend, and the sum of every kernel of the frame (host work and launch gaps excluded).  The depth stays on the device (no depth_out), as the picture does.  One JSON line per workload and case with
the medians and the change of depth on against off, and the card's name and power limit read in the same run.  Needs a GPU and torch."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
ROUNDS = 6      # blocks per case, alternating
sys.path.insert(0, str(ROOT))


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def _line(gpu, base, **kw):
    off, on = kw.pop("off"), kw.pop("on")
    line = dict(kw)
    for k in off:
        line[f"{k}_off"] = round(statistics.median(off[k]), 4)
        line[f"{k}_on"] = round(statistics.median(on[k]), 4)
        line[f"{k}_depth_pct"] = round(100.0 * (line[f"{k}_on"] / line[f"{k}_off"] - 1.0), 2)
    line.update(base, gpu=gpu)
    print(json.dumps(line), flush=True)


def measure(workload: str, frames: int, gpu: str):
    import bench
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.viewer import Viewer
    v, raw = bench.build_viewer(workload, 0, 1, 0)
    e = v.engine
    n, _, _, _, _, w, h, _ = bench.WORKLOADS[workload]
    v.frame(frame_format=N.GS_FRAME_RGBA8, flip_y=True, download=False)
    mvp = v.mvp_matrix().astype(np.float32)
    prepared = {d: e.prepare_frame(mvp, v.uniforms(), w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=True, depth=d) for d in (False, True)}
    ev0, ev1 = e.event(), e.event()
    for _ in range(5):
        for d in (False, True):
            e.frame_async(None, None, w, h, n, prepared=prepared[d])
    e.synchronize()
    t = {False: dict(frame_ms=[]), True: dict(frame_ms=[])}
    for _ in range(ROUNDS):
        for d in (False, True):
            e.frame_async(None, None, w, h, n, prepared=prepared[d])
            e.synchronize()
            for _ in range(-(-frames // ROUNDS)):
                e.flush_l2()
                ev0.record()
                e.frame_async(None, None, w, h, n, prepared=prepared[d])
                ev1.record()
                e.synchronize()
                t[d]["frame_ms"].append(ev0.elapsed_ms(ev1))
    e.set_profiling(True)
    for d in (False, True):
        t[d]["blend_ms"] = []
    for _ in range(frames):
        for d in (False, True):
            e.flush_l2()
            e.frame_async(None, None, w, h, n, prepared=prepared[d])
            e.synchronize()
            t[d]["blend_ms"] += [ms for name, ms in e.kernel_timings() if name == "k_blend"]
    e.set_profiling(False)
    _line(gpu, dict(frames=frames), workload=workload, splats=n, width=w, height=h, case="mono", off=t[False], on=t[True])
    v.dispose()

    # 4 views of a quarter of the frame each, on a ring around the first camera's target
    from gaussiansplats3d_b200.scenes import CAMERAS
    V, vw, vh = 4, w // 2, h // 2
    c0 = CAMERAS[bench.WORKLOADS[workload][4]]
    mv = Viewer(dict(width=vw, height=vh, maxViews=V, sphericalHarmonicsDegree=raw.sh_degree, cameraUp=c0["up"],
                     initialCameraPosition=c0["position"], initialCameraLookAt=c0["look_at"]))
    mv.addSplatScene(raw)
    mv.update()
    target, up = np.asarray(c0["look_at"], np.float64), np.asarray(c0["up"], np.float64) / np.linalg.norm(c0["up"])
    off = np.asarray(c0["position"], np.float64) - target
    cams = []
    for i in range(V):
        c = TM.PerspectiveCamera(50.0, vw / vh, 0.1, 1000.0)
        c.position = target + TM.rotate_about_axis(off, up, 0.25 * np.pi * i)
        c.up = up
        c.look_at(target)
        c.update()
        cams.append(c)
    me = mv.engine
    me.set_profiling(True)
    for _ in range(3):
        for d in (False, True):
            mv.frameViews(cams, download=False, depth=d)
    t = {False: dict(kernels_ms=[], blend_ms=[]), True: dict(kernels_ms=[], blend_ms=[])}
    for _ in range(frames):
        for d in (False, True):
            me.flush_l2()
            mv.frameViews(cams, download=False, depth=d)
            kt = me.kernel_timings()
            t[d]["kernels_ms"].append(sum(ms for _, ms in kt))
            t[d]["blend_ms"] += [ms for name, ms in kt if name == "k_blend"]
    me.set_profiling(False)
    _line(gpu, dict(frames=frames), workload=workload, splats=n, width=vw, height=vh, views=V, case="multi-view", off=t[False], on=t[True])
    mv.dispose()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="bonsai,garden")
    ap.add_argument("--frames", type=int, default=60)
    args = ap.parse_args()
    gpu = card()
    print(json.dumps(dict(gpu=gpu)), flush=True)
    for wl in args.workloads.split(","):
        measure(wl, args.frames, gpu)


if __name__ == "__main__":
    main()
