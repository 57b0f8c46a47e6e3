"""Time WebXR stereo frames (gs_render_params.eyes) against the mono frames they replace.

    python tools/stereo_bench.py [--workloads bonsai,garden] [--frames 150] [--rounds 3]

For each of bench.py's bonsai (1.2 M splats) and garden (5.8 M splats, SH2) workloads, from its first camera, a Viewer in WebXR mode with
two eyes 64 mm apart around that camera and 1920 x 1080 per eye (a 3840 x 1080 XR framebuffer).  Three cases, each through gs_frame_async
from pre-marshalled arguments, between two CUDA events on the engine's stream (device time of the frame graphs):
  mono    one eye's mono frame (1920 x 1080): depth sort + projection + binning + blend
  stereo  the stereo frame: one sort, both eyes projected, binned and blended (3840 x 1080)
  two     two mono gs_frame calls, one per eye: what a stereo frame costs without this feature
Each frame follows an L2 flush.  The cases take turns in blocks of frames / rounds frames, each block after five warm-up frames: a switch
between mono and stereo captures a new frame graph, and its host time must not fall between the events.  One JSON line per workload and
case with the median and minimum, stereo and two also against mono, and the card's name and power limit read in the same run.  Needs a
GPU."""
from __future__ import annotations

import argparse
import dataclasses
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

IPD = 0.064
EYE_W, EYE_H = 1920, 1080


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def eye_cameras(viewer):
    from gaussiansplats3d_b200 import three_math as TM
    cam = viewer.camera
    right = cam.matrixWorld[0:3]
    out = []
    for s in (-0.5, 0.5):
        c = TM.PerspectiveCamera(cam.fov, cam.aspect, cam.near, cam.far)
        c.position, c.up = cam.position + s * IPD * right, cam.up
        c.look_at(cam.target + s * IPD * right)
        c.update()
        out.append(c)
    return out


def measure(workload: str, frames: int, rounds: int, gpu: str):
    import bench
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer, WebXRMode
    n, sh, kind, seed, cam, _, _, _ = bench.WORKLOADS[workload]
    c = CAMERAS[cam]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=2 * EYE_W, height=EYE_H,
                    sphericalHarmonicsDegree=sh, webXRMode=WebXRMode.VR))
    v.addSplatScene(synthetic_scene(n, seed=seed, kind=kind, sh_degree=sh))
    v.camera.update()
    v.updateSplatMesh()
    e = v.engine
    mvp, u = v.mvp_matrix().astype(np.float32), v.uniforms()
    eyes = v.xrEyes(eye_cameras(v))
    fmt = dict(frame_format=N.GS_FRAME_RGBA8, flip_y=True)
    mono = [e.prepare_frame(mvp, dataclasses.replace(u, model_view=eye.model_view, projection=eye.projection, camera_position=eye.camera_position),
                            EYE_W, EYE_H, n, **fmt) for eye in eyes]
    stereo = e.prepare_frame(mvp, u, 2 * EYE_W, EYE_H, n, eyes=eyes, **fmt)
    cases = {"mono": [mono[0]], "stereo": [stereo], "two": mono}
    ev0, ev1 = e.event(), e.event()
    times = {k: [] for k in cases}
    for _ in range(rounds):
        for k, prepared in cases.items():
            # a switch between mono and stereo frames captures a new frame graph: the warm-up frames take it, not the timed ones
            for _ in range(5):
                for p in prepared:
                    e.frame_async(None, None, 0, 0, 0, prepared=p)
            e.synchronize()
            for _ in range(frames // rounds):
                e.flush_l2()
                ev0.record()
                for p in prepared:
                    e.frame_async(None, None, 0, 0, 0, prepared=p)
                ev1.record()
                e.synchronize()
                times[k].append(ev0.elapsed_ms(ev1))
    med = {k: statistics.median(t) for k, t in times.items()}
    for k, t in times.items():
        line = dict(workload=workload, splats=n, eye_width=EYE_W, eye_height=EYE_H, case=k, frames=frames,
                    frame_ms=round(med[k], 4), frame_ms_min=round(min(t), 4))
        if k != "mono":
            line["vs_mono"] = round(med[k] / med["mono"], 3)
        if k == "stereo":
            line["vs_two_pct"] = round(100.0 * (med["stereo"] / med["two"] - 1.0), 2)
        line["gpu"] = gpu
        print(json.dumps(line), flush=True)
    v.dispose()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="bonsai,garden")
    ap.add_argument("--frames", type=int, default=150)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    gpu = card()
    for wl in args.workloads.split(","):
        measure(wl, args.frames, args.rounds, gpu)


if __name__ == "__main__":
    main()
