"""Streamed load of a garden-sized INRIA `.ply` (5.8 M splats, 45 f_rest, about 1.4 GB, built in memory as tools/load_bench.py builds it)
through gs_stream_append in 256 KiB, 4 MiB and 64 MiB appends, loaded with sphericalHarmonicsDegree 2.  For each append size it reports
the time from the first append to the first renderable frame (the first append that committed splats, then one frame of them), the
total load time (first append to close) against gs_upload_file of the whole file, the median append cost, and the frame time of the
half-loaded scene (median of 20 gs_frame calls at 1920x1080).  The card name and power limit are printed in the same run.

    python tools/progressive_bench.py [--splats 5800000] [--appends 262144,4194304,67108864]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))

from gaussiansplats3d_b200 import Engine, _native as N  # noqa: E402
from gaussiansplats3d_b200.engine import Uniforms  # noqa: E402
from load_bench import card, garden_ply  # noqa: E402

W, H = 1920, 1080


def frame_args(n: int):
    """A camera looking at the scene's centre from 60 units away (the seeded scene spans [-20, 20]^3)."""
    f = 1.0 / np.tan(np.radians(25.0))
    proj = np.array([f * H / W, 0, 0, 0, 0, f, 0, 0, 0, 0, -1.0002, -1, 0, 0, -0.20002, 0], np.float32)
    mv = np.eye(4, dtype=np.float32)
    mv[3, 2] = -60.0
    mv = mv.reshape(16)
    mvp = (proj.reshape(4, 4).T @ mv.reshape(4, 4).T).T.reshape(16).astype(np.float32)
    u = Uniforms(model_view=mv, projection=proj, camera_position=np.array([0, 0, 60], np.float32), focal=(proj[0] * 0.5 * W, proj[5] * 0.5 * H),
                 viewport=(float(W), float(H)), sh_degree=2)
    return mvp, u


def frame_ms(e: Engine, n: int, reps: int = 20) -> float:
    mvp, u = frame_args(n)
    e.frame(mvp, u, W, H, n, download=False)
    N.check(e._lib.gs_synchronize(e._h), "gs_synchronize")
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        e.frame(mvp, u, W, H, n, download=False)
        N.check(e._lib.gs_synchronize(e._h), "gs_synchronize")
        ts.append((time.perf_counter() - t) * 1e3)
    return float(np.median(ts))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--splats", type=int, default=5_800_000)
    ap.add_argument("--appends", default="262144,4194304,67108864")
    a = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    data = garden_ply(a.splats)
    mv = memoryview(data)
    e = Engine(a.splats, max_width=W, max_height=H)
    e.upload_file(N.GS_FILE_PLY, data, sh_degree=2)   # warm-up: module load and first allocations
    t = time.perf_counter()
    e.upload_file(N.GS_FILE_PLY, data, sh_degree=2)
    whole_s = time.perf_counter() - t
    for size in map(int, a.appends.split(",")):
        s = e.open_stream(N.GS_FILE_PLY, sh_degree=2)
        costs, first_frame_s, half_ms = [], None, None
        t0 = time.perf_counter()
        for k in range(0, len(data), size):
            t = time.perf_counter()
            loaded = s.append(mv[k:k + size])
            costs.append(time.perf_counter() - t)
            if first_frame_s is None and loaded:
                mvp, u = frame_args(loaded)
                e.frame(mvp, u, W, H, loaded, download=False)
                N.check(e._lib.gs_synchronize(e._h), "gs_synchronize")
                first_frame_s = time.perf_counter() - t0
            if half_ms is None and loaded >= a.splats // 2:
                pause = time.perf_counter()
                half_ms = frame_ms(e, loaded)
                t0 += time.perf_counter() - pause   # the half-loaded frames are not part of the load
        info = s.close()
        total_s = time.perf_counter() - t0
        assert info["splat_count"] == a.splats
        print(json.dumps({"append_bytes": size, "appends": len(costs), "first_frame_ms": round(first_frame_s * 1e3, 2),
                          "load_s": round(total_s, 3), "upload_file_s": round(whole_s, 3), "median_append_ms": round(float(np.median(costs)) * 1e3, 3),
                          "half_loaded_frame_ms": round(half_ms, 3), "splats": a.splats, "file_bytes": len(data)}), flush=True)


if __name__ == "__main__":
    main()
