"""GPU parity at BASELINE.json's full sizes (configs[2], [3]; configs[1] lives in test_raster_gpu.test_full_hd_bonsai_frame, configs[4] in
test_sort_gpu), held to the f64 restatements by tests/frame_f64.py: the draw order each gs_frame used bit-exact against the compiled
reference sorter (oracle/_ref; the C restatement where that is absent), every splat's projection within its per-splat f64 bounds, the
tile-instance count, and the blend within its per-pixel f64 bounds -- over the whole frame for the three garden orbit frames, and over
windows covering more than a quarter of the 16 M / 4K frame, whose whole-frame restatement costs several CPU-minutes.  Both configs
draw more than 2 097 152 splats, so k_bin_scan carries its running offset across more than one 1024-chunk block."""
import numpy as np
import pytest

import frame_f64 as FF

pytestmark = pytest.mark.gpu


def orbit_camera(cam: dict, k: int, degrees_per_frame: float = 3.0):
    """Frame k of the orbit SURVEY 8(d) specifies for configs[2]: the demo camera (demo/garden.html:39-41) rotated about cameraUp through
    the look-at point by 3 degrees per frame."""
    up = np.asarray(cam["up"], np.float64)
    up /= np.linalg.norm(up)
    a = np.deg2rad(degrees_per_frame * k)
    d = np.asarray(cam["position"], np.float64) - np.asarray(cam["look_at"], np.float64)
    rot = d * np.cos(a) + np.cross(up, d) * np.sin(a) + up * np.dot(up, d) * (1.0 - np.cos(a))     # Rodrigues
    return np.asarray(cam["look_at"], np.float64) + rot


def test_config3_garden_5p8m_sh2_orbit(gs, oracle_mod):
    """BASELINE configs[2]: 5.8 M splats, SH degree 2, 1920x1080, orbiting camera: three orbit angles (frames 0, 40, 80 of the 120)."""
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    n, w, h = 5_800_000, 1920, 1080
    raw = synthetic_scene(n, seed=2, kind="garden", sh_degree=2)
    cam = CAMERAS["garden"]
    v = Viewer(dict(cameraUp=cam["up"], initialCameraPosition=cam["position"], initialCameraLookAt=cam["look_at"], width=w, height=h, sphericalHarmonicsDegree=2))
    v.addSplatScene(raw)
    for k in (0, 40, 80):
        v.camera.position = orbit_camera(cam, k)
        v.camera.look_at(cam["look_at"])
        got = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
        FF.check_viewer_frame(f"garden orbit frame {k}", v, got=got, min_compared=n // 4)
        print(f"garden orbit frame {k}: timings {v.engine.timings()}")
    v.dispose()


def test_config4_16m_sh0_4k(gs, oracle_mod):
    """BASELINE configs[3]: 16 M splats SH0 at 3840x2160 on one GPU (the 8-GPU tiling of the same frame is compared with this one in
    test_multi_gpu / bench.py).  Runs the 32-px-tile path (255 coarse tiles of 256x128 px).  The blend is checked on nine 640x368-px
    windows, 25.6 % of the frame; the projection of every splat."""
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    n, w, h = 16_000_000, 3840, 2160
    raw = synthetic_scene(n, seed=3, kind="bonsai", sh_degree=0)
    cam = CAMERAS["bonsai"]
    v = Viewer(dict(cameraUp=cam["up"], initialCameraPosition=cam["position"], initialCameraLookAt=cam["look_at"], width=w, height=h))
    v.addSplatScene(raw)
    got = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
    wins = FF.windows(w, h, 640, 368)       # corners, edge midpoints and centre; the last ones run to the frame's right and bottom edges
    share = sum(ww * wh for _, _, ww, wh in wins) / (w * h)
    assert share >= 0.25 and max(x + ww for x, _, ww, _ in wins) == w and max(y + wh for _, y, _, wh in wins) == h
    FF.check_viewer_frame("16M @4K", v, got=got, windows=wins, min_compared=n // 4)
    print(f"16M @4K: blend checked on {len(wins)} windows, {100 * share:.1f} % of the frame; timings {v.engine.timings()}")
    v.dispose()
