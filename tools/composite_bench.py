"""Time frames composited into an opaque pass (gs_render_params dest_color / dest_depth) against the plain frame.

    python tools/composite_bench.py [--workloads bonsai,garden] [--frames 50]

For each of bench.py's bonsai (1.2 M splats, 1080p) and garden (5.8 M splats, SH2, 1080p) workloads, from its first camera, four cases:
  none      no inputs (the plain frame, the k_blend<.., false> kernel)
  noop      depth 1 and colour 0 everywhere: the composite kernel with nothing to hide
  half      the left half of the screen behind a wall at the median window depth of the drawn splats, patterned colour there
  occluded  depth 0 everywhere: every splat hidden
The inputs are CUDA tensors (device pointers), so no host copy enters the frame.  Per case: warm-up frames, then `frames` frames through
gs_frame_async, each between two CUDA events on the engine's stream (the captured frame graph: device time per frame), and as many
profiled frames (one event after every kernel, no graph) for the blend kernel alone.  One JSON line per workload and case with the
medians and the change against `none`, and the card's name and power limit read in the same run.  Needs a GPU and torch."""
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


def card() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def inputs(case: str, w: int, h: int, median_zw: float):
    import torch
    if case == "none":
        return {}
    depth = torch.ones((h, w), dtype=torch.float32)
    color = torch.zeros((h, w, 4), dtype=torch.uint8)
    if case == "half":
        depth[:, : w // 2] = median_zw
        yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
        check = (((yy >> 3) + (xx >> 3)) & 1).to(torch.uint8)
        color[..., 0], color[..., 1], color[..., 2] = 40 + 160 * check, 120, 200 - 160 * check
        color[..., 3] = 255
        color[:, w // 2:] = 0
    elif case == "occluded":
        depth.zero_()
        color[..., 3] = 255
    out = dict(dest_color=color.cuda(), dest_depth=depth.cuda())
    torch.cuda.synchronize()
    return out


def measure(workload: str, frames: int, gpu: str):
    import bench
    from gaussiansplats3d_b200 import _native as N
    v, raw = bench.build_viewer(workload, 0, 1, 0)
    e = v.engine
    n, _, _, _, _, w, h, _ = bench.WORKLOADS[workload]
    v.frame(frame_format=N.GS_FRAME_RGBA8, flip_y=True, download=False)
    proj = e.read_projected(n)
    drawn = proj["valid"] == 1
    median_zw = float(np.median(np.float32(0.5) * proj["ndc_z"][drawn] + np.float32(0.5)))
    mvp = v.mvp_matrix().astype(np.float32)
    ev0, ev1 = e.event(), e.event()
    base = None
    for case in ("none", "noop", "half", "occluded"):
        kw = inputs(case, w, h, median_zw)
        prepared = e.prepare_frame(mvp, v.uniforms(), w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=True, **kw)
        for _ in range(5):
            e.frame_async(None, None, w, h, n, prepared=prepared)
        e.synchronize()
        frame_ms = []
        for _ in range(frames):
            e.flush_l2()
            ev0.record()
            e.frame_async(None, None, w, h, n, prepared=prepared)
            ev1.record()
            e.synchronize()
            frame_ms.append(ev0.elapsed_ms(ev1))
        e.set_profiling(True)
        blend_ms = []
        for _ in range(frames):
            e.flush_l2()
            e.frame_async(None, None, w, h, n, prepared=prepared)
            e.synchronize()
            blend_ms += [ms for name, ms in e.kernel_timings() if name == "k_blend"]
        e.set_profiling(False)
        line = dict(workload=workload, splats=n, width=w, height=h, case=case, frames=frames,
                    frame_ms=round(statistics.median(frame_ms), 4), frame_ms_min=round(min(frame_ms), 4),
                    blend_ms=round(statistics.median(blend_ms), 4), blend_ms_min=round(min(blend_ms), 4))
        if base is None:
            base = line
        else:
            line["frame_vs_none_pct"] = round(100.0 * (line["frame_ms"] / base["frame_ms"] - 1.0), 2)
            line["blend_vs_none_pct"] = round(100.0 * (line["blend_ms"] / base["blend_ms"] - 1.0), 2)
        line["gpu"] = gpu
        print(json.dumps(line), flush=True)
    v.dispose()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="bonsai,garden")
    ap.add_argument("--frames", type=int, default=50)
    args = ap.parse_args()
    gpu = card()
    for wl in args.workloads.split(","):
        measure(wl, args.frames, gpu)


if __name__ == "__main__":
    main()
