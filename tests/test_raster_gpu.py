"""GPU frames end to end: depth sort, CUDA projection, tile binning and the front-to-back blend, each frame held to the f64
restatements by tests/frame_f64.py.  The draw order the frame actually used (the engine's sorted indexes, or the order passed in)
must equal the reference sorter's bit for bit when the engine sorted; every drawn splat's projection must lie within its per-splat
f64 bounds (tests/projection_f64.py: centre, ndc z, colour, alpha and the quad's B1 B1^T + B2 B2^T; `valid` equal on every
unambiguous splat); the tile-instance count must match the host's count; and every channel of every pixel must lie within its f64
blend bound (tests/blend_f64.py), in RGBA32F and, where the test renders it, RGBA8.  The CPU oracle's projection is held to the same
per-splat bounds."""
import numpy as np
import pytest

import frame_f64 as FF

pytestmark = pytest.mark.gpu


def _viewer(gs, raw, width, height, cam="bonsai", **opts):
    from gaussiansplats3d_b200.viewer import Viewer
    from gaussiansplats3d_b200.scenes import CAMERAS
    c = CAMERAS[cam]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=width, height=height, **opts))
    v.addSplatScene(raw)
    return v


@pytest.mark.parametrize("sh_degree,fmt", [(0, "f16"), (1, "f16"), (2, "f16"), (2, "u8"), (2, "f32")])
def test_projection_matches_vertex_shader(gs, oracle_mod, sh_degree, fmt):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    raw = synthetic_scene(60_000, seed=4, kind="bonsai", sh_degree=sh_degree)
    v = Viewer(dict(width=640, height=360, sphericalHarmonicsDegree=sh_degree, initialCameraPosition=(1.5, 2.7, -6.4), initialCameraLookAt=(0.4, 0.3, 0.2), cameraUp=(0, -1, -0.6)))
    v.splatMesh = None
    from gaussiansplats3d_b200.viewer import SplatMesh
    v.addSplatScene(raw)
    if fmt != "f16" and sh_degree:
        from gaussiansplats3d_b200.scenes import pack_scene
        v.splatMesh.packed = pack_scene(raw, sh_format=fmt)
        v.splatMesh.setRenderer(v.engine)
    v.update()
    v.render(download=False)
    got = v.engine.read_projected(raw.count)
    p = v.splatMesh.packed
    import projection_f64 as PF
    h = PF.project(v.uniforms(), p.centers_colors, p.covariances, p.sh, p.sh_degree)
    rep = PF.compare(got, h)
    print("\n" + PF.format_report(f"vertex shader sh{sh_degree} {fmt}", rep))
    PF.assert_within("GPU", rep, min_compared=1000)
    want = oracle_mod.project(v.uniforms(), p.centers_colors, p.covariances, p.sh, p.sh_degree)
    PF.assert_within("oracle", PF.compare(want, h), min_compared=1000)


@pytest.mark.parametrize("n,w,h,sh_degree", [(20_000, 320, 200, 0), (200_000, 1000, 600, 1), (150_000, 801, 455, 2)])
def test_frame_matches_reference_blend(gs, oracle_mod, n, w, h, sh_degree):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(n, seed=7, kind="bonsai", sh_degree=sh_degree)
    v = _viewer(gs, raw, w, h, sphericalHarmonicsDegree=sh_degree)
    v.update()
    got = v.render(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
    assert got[..., 3].max() > 0.5, "frame is empty"
    # canvas format + image orientation: the flipped RGBA8 frame, read bottom-up, is the same picture
    got8 = v.render(frame_format=gs._native.GS_FRAME_RGBA8, flip_y=True).copy()
    FF.check_viewer_frame(f"{n} splats {w}x{h} sh{sh_degree}", v, got=got, got8=got8[::-1], min_compared=n // 4)
    t = v.engine.timings()
    assert t["tile_instances"] > 0 and t["visible_splats"] > 0
    v.dispose()


def test_full_hd_bonsai_frame(gs, oracle_mod):
    """BASELINE configs[1]: 1.2M splats, SH0, 1920x1080, bonsai camera, gs_frame in RGBA32F and RGBA8: the draw order it used, every
    splat's projection and the whole frame against the f64 restatements."""
    from gaussiansplats3d_b200.scenes import synthetic_scene
    n = 1_200_000
    raw = synthetic_scene(n, seed=1, kind="bonsai", sh_degree=0)
    v = _viewer(gs, raw, 1920, 1080)
    got = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
    got8 = v.frame(frame_format=gs._native.GS_FRAME_RGBA8, flip_y=False).copy()
    FF.check_viewer_frame("1080p bonsai", v, got=got, got8=got8, min_compared=n // 4)
    print(f"1080p bonsai timings {v.engine.timings()}")
    v.dispose()


def test_explicit_sorted_indexes_and_worker_topology(gs, oracle_mod):
    """updateRenderIndexes(sortedIndexes) path: order comes from the host (separate sort worker), as in the reference."""
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    raw = synthetic_scene(50_000, seed=12, kind="uniform")
    v = Viewer(dict(width=400, height=300, sharedMemoryForWorkers=True))
    v.addSplatScene(raw, separate_sort_worker=True)
    v.update()
    assert v.splatMesh.renderIndexes is not None and not v.sortRunning
    order = v.splatMesh.renderIndexes.copy()
    got = v.render(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
    FF.check_viewer_frame("host-sorted order", v, got=got, order=order, sort=None, min_compared=1000)
    # a deliberately different (front-to-back) order must give a different picture: order is honoured
    rev = order[::-1].copy()
    got_rev = v.engine.render(v.uniforms(), 400, 300, raw.count, rev, flip_y=False)
    FF.check_viewer_frame("reversed order", v, got=got_rev, order=rev, sort=None, min_compared=1000)
    assert np.abs(got_rev - got).max() > 0.05
    v.dispose()


def test_render_options(gs, oracle_mod):
    """antialiased compensation, point-cloud mode, half covariances, splatScale, fade-in."""
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(40_000, seed=3, kind="bonsai")
    for opts, tweak in ((dict(antialiased=True), None), (dict(halfPrecisionCovariancesOnGPU=True), None), (dict(), "point"), (dict(), "scale"), (dict(), "fade")):
        v = _viewer(gs, raw, 480, 270, **opts)
        if tweak == "point":
            v.splatMesh.pointCloudModeEnabled = True
        if tweak == "scale":
            v.splatMesh.splatScale = 0.6
        if tweak == "fade":
            v.splatMesh.fadeInComplete = False
            v.splatMesh.visibleRegionFadeStartRadius = 2.0
        v.update()
        got = v.render(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
        FF.check_viewer_frame(f"render options {opts or tweak}", v, got=got, min_compared=1000)
        v.dispose()


def test_dynamic_scenes_and_optional_effects(gs, oracle_mod):
    """SURVEY 8f N3: per-scene transforms in the vertex stage (SplatMaterial.js:136-146, :181-183), scene opacity / visibility
    (SplatMaterial.js:124-133, SplatMaterial3D.js:198-202), 3 scenes, SH1 so the per-scene camera transform matters."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Engine, Uniforms
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    n, w, h = 60_000, 512, 300
    raw = synthetic_scene(n, seed=6, kind="uniform", sh_degree=1)
    p = pack_scene(raw)
    rng = np.random.default_rng(3)
    scene_idx = rng.integers(0, 3, n, dtype=np.uint32)
    transforms = np.tile(np.eye(4, dtype=np.float64).T.reshape(16), (32, 1))
    transforms[1] = TM.compose((1.5, 0.0, -1.0), (0.0, np.sin(0.3), 0.0, np.cos(0.3)), (1.2, 1.2, 1.2))
    transforms[2] = TM.compose((-2.0, 0.5, 0.5), (np.sin(0.2), 0.0, 0.0, np.cos(0.2)), (0.7, 0.7, 0.7))
    cam = TM.PerspectiveCamera(50, w / h, 0.1, 1000)
    cam.position = np.array([0.0, 4.0, 12.0]); cam.look_at((0, 0, 0))
    opacity = np.ones(32, np.float32); opacity[1] = 0.6
    vis = np.ones(32, np.int32)
    for effects, hide in ((0, False), (1, False), (1, True)):
        v = vis.copy()
        if hide:
            v[2] = 0
        u = Uniforms(model_view=cam.matrixWorldInverse.astype(np.float32), projection=cam.projectionMatrix.astype(np.float32),
                     camera_position=cam.position.astype(np.float32), focal=(cam.projectionMatrix[0] * 0.5 * w, cam.projectionMatrix[5] * 0.5 * h),
                     viewport=(w, h), sh_degree=1, scene_count=3, scene_transforms=transforms.astype(np.float32), view_matrix=cam.matrixWorldInverse.astype(np.float32),
                     scene_opacity=opacity, scene_visibility=v, enable_optional_effects=effects, dynamic_mode=1)
        order = rng.permutation(n).astype(np.uint32)     # any order: the blend must honour it
        with Engine(n, max_width=w, max_height=h, dynamic_mode=True) as e:
            e.upload_splat_data(p.centers_colors, p.covariances, p.sh, p.sh_degree, scene_indexes=scene_idx)
            got = e.render(u, w, h, n, order, flip_y=False)
            FF.check_frame(f"3 dynamic scenes, effects {effects}, scene 2 hidden {hide}", e, u, w, h, n, p.centers_colors, p.covariances,
                           p.sh, p.sh_degree, scene_idx, got=got, order=order, min_compared=1000)
            proj = e.read_projected(n)
        if hide:
            assert (proj["valid"][scene_idx == 2] == 0).all()


def test_precision_20bit_and_float_sort_feed_the_same_frame(gs, oracle_mod):
    """splatSortDistanceMapPrecision 20 (3 radix passes) and the float sort mode drive the renderer like the default."""
    from gaussiansplats3d_b200.scenes import synthetic_scene
    raw = synthetic_scene(80_000, seed=13, kind="bonsai")
    for opts in (dict(splatSortDistanceMapPrecision=20), dict(integerBasedSort=False, splatSortDistanceMapPrecision=22)):
        v = _viewer(gs, raw, 480, 270, **opts)
        got = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
        FF.check_viewer_frame(f"sort {opts}", v, got=got, min_compared=1000)
        v.dispose()


@pytest.mark.parametrize("name", ["bonsai-sh0-160x100", "bonsai-sh2-128x96", "garden-sh1-200x120"])
def test_frame_and_order_match_committed_fixture(gs, name):
    """Against tests/golden/raster_golden.npz (no oracle call at run time): the order the Viewer-driven frame drew must reproduce the
    stored draw order bit for bit (that order is the compiled reference sorter's), and the frame must pass the f64 checks."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
    import raster_cases
    from gaussiansplats3d_b200.scenes import synthetic_scene
    gold = np.load(Path(__file__).resolve().parent / "golden" / "raster_golden.npz")
    n, seed, kind, sh, w, h, cam = raster_cases.CASES[name]
    raw = synthetic_scene(n, seed=seed, kind=kind, sh_degree=sh)
    v = _viewer(gs, raw, w, h, cam=cam, sphericalHarmonicsDegree=sh)
    v.update()
    got = v.render(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
    assert np.array_equal(v.engine.read_buffer(gs._native.GS_BUF_SORTED_INDEXES, np.uint32, n), gold[name + "|order"])
    FF.check_viewer_frame(f"fixture {name}", v, got=got, sort=None, min_compared=100)
    v.dispose()


@pytest.mark.parametrize("w,h", [(1000, 600), (2600, 1500)])
def test_frame_matches_reference_blend_at_both_tile_sizes(gs, oracle_mod, w, h):
    """Counting-sort binning and the block blend, held to the f64 restatements, at both fine-tile sizes: 1000x600 has at most 256 coarse tiles of
    128x64 px and runs with 16-px tiles (4 warps per tile), 2600x1500 exceeds that and runs with 32-px tiles (16 warps per tile)."""
    from gaussiansplats3d_b200.scenes import synthetic_scene
    n = 200_000
    raw = synthetic_scene(n, seed=7, kind="bonsai", sh_degree=1)
    v = _viewer(gs, raw, w, h, sphericalHarmonicsDegree=1)
    v.update()
    got = v.render(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False)
    assert FF.BF.tile_px(w, h) == (16 if w == 1000 else 32)
    FF.check_viewer_frame(f"{w}x{h}", v, got=got, min_compared=n // 4)
    v.dispose()


def test_dynamic_scene_applies_its_transform(gs, oracle_mod):
    """Viewer(dynamicScene=True).addSplatScene(position, rotation, scale): the transform is NOT baked; the sorter (sorter.cpp:44-50) and the
    vertex stage (SplatMaterial.js:136-146) apply it every frame.  Both frames -- the dynamic one and the static viewer's, which bakes the
    same transform at load -- pass the f64 checks on their own (each draw order against the reference sorter run the viewer's way), and
    they show the same picture up to the sort's tie-breaking."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    n, w, h = 60_000, 480, 270
    raw = synthetic_scene(n, seed=21, kind="bonsai", sh_degree=0)
    q = np.array([0.1, 0.35, -0.2, 0.9]); q /= np.linalg.norm(q)
    kw = dict(position=(0.6, -0.4, 0.8), rotation=tuple(q), scale=(1.4, 1.4, 1.4))
    c = CAMERAS["bonsai"]
    frames = {}
    for dynamic in (False, True):
        v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h, dynamicScene=dynamic))
        v.addSplatScene(raw, **kw)
        frames[dynamic] = v.frame(frame_format=gs._native.GS_FRAME_RGBA32F, flip_y=False).copy()
        if dynamic:
            u = v.uniforms()
            assert u.dynamic_mode == 1 and not np.allclose(u.scene_transforms[0], TM.identity())
        FF.check_viewer_frame(f"dynamic={dynamic}", v, got=frames[dynamic], min_compared=1000)
        v.dispose()
    assert frames[True][..., 3].max() > 0.5
    d = np.abs(frames[True] - frames[False])
    assert (d <= 2.0 / 255).mean() >= 0.995, (d <= 2.0 / 255).mean()          # same picture; ties in the two sorts may resolve differently


def test_pipelined_frames_equal_blocking_frames(gs):
    """gs_frame_begin / gs_frame_end (two or three frames in flight, alternating device frame buffers, copies on a second stream) must deliver
    exactly the pictures gs_frame delivers, in order, for a moving camera."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import synthetic_scene
    n, w, h = 150_000, 640, 360
    raw = synthetic_scene(n, seed=8, kind="bonsai", sh_degree=1)
    v = _viewer(gs, raw, w, h, sphericalHarmonicsDegree=1)
    e = v.engine
    cams = []
    for k in range(6):
        v.camera.position = np.asarray(v.initialCameraPosition) + np.array([0.15 * k, -0.05 * k, 0.1 * k])
        v.camera.look_at(v.initialCameraLookAt)
        v.camera.update(); v.updateSplatMesh()
        cams.append(e.prepare_frame(v.mvp_matrix().astype(np.float32), v.uniforms(), w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=True))
    want = []
    for prep in cams:
        out = N.pinned_empty((h, w, 4), np.uint8)
        e.frame_prepared(prep, out)
        want.append(out.copy())
    bufs = [N.pinned_empty((h, w, 4), np.uint8) for _ in range(2)]
    got = []
    e.frame_begin(cams[0], bufs[0])
    for i in range(len(cams)):
        if i + 1 < len(cams):
            e.frame_begin(cams[i + 1], bufs[(i + 1) & 1])
        e.frame_end()
        got.append(bufs[i & 1].copy())
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), f"pipelined frame {i} differs"
    assert not np.array_equal(want[0], want[-1])
    with pytest.raises(RuntimeError):
        e.frame_end()                                   # nothing in flight any more
    # three frames in flight over the two device buffers (begin(i+2) before end(i)); each needs its own host buffer; statistics of the
    # frame that ended come from the blend kernel's status snapshot
    bufs = [N.pinned_empty((h, w, 4), np.uint8) for _ in range(3)]
    got = []
    e.frame_begin(cams[0], bufs[0])
    e.frame_begin(cams[1], bufs[1])
    for i in range(len(cams)):
        if i + 2 < len(cams):
            e.frame_begin(cams[i + 2], bufs[(i + 2) % 3])
        e.frame_end()
        assert e.timings()["visible_splats"] > 0 and e.timings()["tile_instances"] > 0
        got.append(bufs[i % 3].copy())
    for i, (a, b) in enumerate(zip(got, want)):
        assert np.array_equal(a, b), f"3-deep pipelined frame {i} differs"
    e.frame_begin(cams[0], bufs[0]); e.frame_begin(cams[1], bufs[1]); e.frame_begin(cams[2], bufs[2])
    with pytest.raises(RuntimeError):
        e.frame_begin(cams[3], bufs[0])                 # a fourth frame in flight is refused
    with pytest.raises(RuntimeError):
        e.frame_async(None, None, w, h, n, prepared=cams[3])   # so is anything else that would overwrite a frame buffer being copied out
    for _ in range(3):
        e.frame_end()
    v.dispose()
