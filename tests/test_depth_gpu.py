"""GPU: the view depth beside the colour (gs_render_params.depth).  Mono frames against the f64 restatement (tests/depth_f64.py) fed
the GPU's own raw records and draw order, every pixel within its bound; the colour bit-identical with and without depth; a wall of
opaque splats at a known depth; stereo halves and multi-view bands bit-identical to the mono depth of their eye or camera; composited
frames; every frame path; refusals and callers built before the fields."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import blend_f64 as BF
import depth_f64 as DF
import frame_f64 as FF

pytestmark = pytest.mark.gpu

_scenes = {}


def _raw(n, sh_degree=1, seed=7):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    key = (n, sh_degree, seed)
    if key not in _scenes:
        _scenes[key] = synthetic_scene(n, seed=seed, kind="bonsai", sh_degree=sh_degree)
    return _scenes[key]


def _viewer(w, h, n=200_000, sh_degree=1, **opts):
    from gaussiansplats3d_b200.scenes import CAMERAS
    from gaussiansplats3d_b200.viewer import Viewer
    c = CAMERAS["bonsai"]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h,
                    sphericalHarmonicsDegree=sh_degree, **opts))
    v.addSplatScene(_raw(n, sh_degree))
    v.update()
    return v


def _check_mono(label, v, fmt, flip_y, windows=None, dest_depth=None):
    """Render with depth; hold the depth to the restatement of the GPU's records and order; return (colour, depth)."""
    e, n = v.engine, v.splatMesh.getSplatCount()
    w, h = v.renderWidth, v.renderHeight
    rgba, depth = v.render(frame_format=fmt, flip_y=flip_y, depth=True, dest_depth=dest_depth)
    assert depth.shape == (h, w) and depth.dtype == np.float32
    order = e.read_buffer(0, np.uint32, v.splatMesh.instanceCount)   # the draw order the frame used (GS_BUF_SORTED_INDEXES)
    rec = BF.read_records(e, n)
    P = v.uniforms().projection
    for win in ([(0, 0, w, h)] if windows is None else windows):
        res = DF.restate(rec, order, w, h, P, window=win, dest_depth=dest_depth, flip_y=flip_y)
        DF.check(f"{label} {win}", res, DF.crop(depth, win, flip_y))
    return rgba, depth


@pytest.mark.parametrize("w,h", [(1000, 600), (2600, 1500)])       # 16-px and 32-px fine tiles
@pytest.mark.parametrize("fmt_name", ["rgba8", "rgba32f"])
@pytest.mark.parametrize("flip_y", [False, True])
def test_mono_depth_within_the_restatement_and_colour_unchanged(gs, w, h, fmt_name, flip_y):
    N = gs._native
    fmt = N.GS_FRAME_RGBA8 if fmt_name == "rgba8" else N.GS_FRAME_RGBA32F
    v = _viewer(w, h)
    plain = v.render(frame_format=fmt, flip_y=flip_y)
    rgba, depth = _check_mono(f"{w}x{h} {fmt_name} flip_y={flip_y}", v, fmt, flip_y, windows=FF.windows(w, h) if w > 1000 else None)
    assert np.array_equal(rgba.view(np.uint8), plain.view(np.uint8)), "the colour with depth must be the colour without it, bit for bit"
    if fmt_name == "rgba32f":     # +inf exactly where no splat reached: 1 - T == 0 (an RGBA8 alpha of 0 may hide a faint 1 - T)
        assert np.array_equal(np.isposinf(depth), plain[..., 3] == 0)
    v.dispose()


def test_radix_binning_and_options(gs):
    """More coarse tiles than the counting sort takes (radix binning), SH0, point-cloud mode and the optional effects."""
    N = gs._native
    v = _viewer(4100, 2100, n=60_000, sh_degree=0)
    _check_mono("radix binning", v, N.GS_FRAME_RGBA32F, True, windows=FF.windows(4100, 2100))
    v.dispose()
    for what in ("point cloud", "optional effects"):
        v = _viewer(800, 480, n=60_000, **({"enableOptionalEffects": True} if what == "optional effects" else {}))
        if what == "point cloud":
            v.splatMesh.pointCloudModeEnabled = True
        plain = v.render(frame_format=N.GS_FRAME_RGBA8)
        rgba, _ = _check_mono(what, v, N.GS_FRAME_RGBA8, True)
        assert np.array_equal(rgba, plain)
        v.dispose()


def _check_engine(label, e, u, w, h, n, order, fmt, flip_y, windows=None):
    """An engine's render of `order` with depth: the colour bit-identical to the render without it, the depth within the restatement
    of the GPU's records and that order."""
    plain = e.render(u, w, h, n, order, frame_format=fmt, flip_y=flip_y)
    rgba, depth = e.render(u, w, h, n, order, frame_format=fmt, flip_y=flip_y, depth=True)
    assert np.array_equal(rgba.view(np.uint8), plain.view(np.uint8)), f"{label}: the colour changed with depth"
    rec = BF.read_records(e, n)
    for win in ([(0, 0, w, h)] if windows is None else windows):
        DF.check(f"{label} {win}", DF.restate(rec, order, w, h, u.projection, window=win, flip_y=flip_y), DF.crop(depth, win, flip_y))
    return depth


@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160)])
def test_baseline_sizes(gs, w, h):
    """The BASELINE frame sizes: bonsai's 1.2 M splats (SH0) at 1080p, and at synth16m's 3840x2160 (16-px tiles by counting sort,
    32-px tiles)."""
    N = gs._native
    v = _viewer(w, h, n=1_200_000, sh_degree=0)
    plain = v.render(frame_format=N.GS_FRAME_RGBA8)
    rgba, _ = _check_mono(f"BASELINE {w}x{h}", v, N.GS_FRAME_RGBA8, True, windows=FF.windows(w, h))
    assert np.array_equal(rgba, plain)
    v.dispose()


def test_orthographic_frame(gs):
    """An orthographic projection: d = (P[14] - ndc) / P[10], through the mono frame's own ProjParams block."""
    import test_multi_view_gpu as M
    from gaussiansplats3d_b200 import _native as N
    w, h = 600, 400
    raw, packed = M._scene(60_000)
    n = packed.count
    cam = M._ring(1, w, h)[0]
    P = np.zeros(16)
    P[0], P[5], P[10], P[14], P[15] = 1.0 / (4.0 * w / h), 1.0 / 4.0, -2.0 / 999.9, -1000.1 / 999.9, 1.0
    u = dataclasses.replace(M._substituted(M._shared(w, h, orthographic_mode=1), M._view(cam, w, h)), projection=P.astype(np.float32),
                            focal=(P[0] * 0.5 * w, P[5] * 0.5 * h))
    order = np.random.default_rng(4).permutation(n).astype(np.uint32)
    with M._engine(packed, raw, w, h) as e:
        for fmt, flip_y in ((N.GS_FRAME_RGBA32F, False), (N.GS_FRAME_RGBA8, True)):
            depth = _check_engine(f"orthographic flip_y={flip_y}", e, u, w, h, n, order, fmt, flip_y)
            assert np.isfinite(depth).sum() > 1000       # pixels the splats reach, each held to its bound above


def test_dynamic_scenes_moving(gs):
    """A dynamic mesh of three scenes with optional effects, the scenes moving between frames: each frame's depth within the
    restatement, its colour unchanged."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Engine, Uniforms
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    n, w, h = 60_000, 512, 300
    p = pack_scene(synthetic_scene(n, seed=6, kind="uniform", sh_degree=1))
    rng = np.random.default_rng(3)
    scene_idx = rng.integers(0, 3, n, dtype=np.uint32)
    cam = TM.PerspectiveCamera(50, w / h, 0.1, 1000)
    cam.position = np.array([0.0, 4.0, 12.0]); cam.look_at((0, 0, 0))
    opacity = np.ones(32, np.float32); opacity[1] = 0.6
    order = rng.permutation(n).astype(np.uint32)
    with Engine(n, max_width=w, max_height=h, dynamic_mode=True) as e:
        e.upload_splat_data(p.centers_colors, p.covariances, p.sh, p.sh_degree, scene_indexes=scene_idx)
        for t in (0.0, 0.5, 1.0):      # the scenes move
            xf = np.tile(np.eye(4, dtype=np.float64).T.reshape(16), (32, 1))
            xf[1] = TM.compose((1.5 + t, 0.0, -1.0 - 2 * t), (0.0, np.sin(0.3 + t), 0.0, np.cos(0.3 + t)), (1.2, 1.2, 1.2))
            xf[2] = TM.compose((-2.0, 0.5 + t, 0.5 + 3 * t), (np.sin(0.2), 0.0, 0.0, np.cos(0.2)), (0.7, 0.7, 0.7))
            u = Uniforms(model_view=cam.matrixWorldInverse.astype(np.float32), projection=cam.projectionMatrix.astype(np.float32),
                         camera_position=cam.position.astype(np.float32), focal=(cam.projectionMatrix[0] * 0.5 * w, cam.projectionMatrix[5] * 0.5 * h),
                         viewport=(w, h), sh_degree=1, scene_count=3, scene_transforms=xf.astype(np.float32),
                         view_matrix=cam.matrixWorldInverse.astype(np.float32), scene_opacity=opacity, scene_visibility=np.ones(32, np.int32),
                         enable_optional_effects=1, dynamic_mode=1)
            _check_engine(f"dynamic t={t}", e, u, w, h, n, order, N.GS_FRAME_RGBA32F, False)


def _wall_scene(depth_world, n_side=64, extent=None, grow=1.0):
    """Opaque round splats tiling the plane z = -depth_world in front of a camera at the origin looking down -z."""
    from gaussiansplats3d_b200.scenes import RawScene
    extent = depth_world if extent is None else extent
    xs = np.linspace(-extent, extent, n_side)
    X, Y = np.meshgrid(xs, xs)
    n = X.size
    centers = np.stack([X.ravel(), Y.ravel(), np.full(n, -depth_world)], 1).astype(np.float32)
    s = 2.0 * extent / (n_side - 1) * 1.5 * grow
    scales = np.tile(np.float32([s, s, s * 1e-3]), (n, 1))
    rot = np.tile(np.float32([0, 0, 0, 1]), (n, 1))
    colors = np.tile(np.uint8([200, 100, 50, 255]), (n, 1))
    return RawScene(centers, scales, rot, colors, None, 0)


def _wall_frame(P, w, h, raw, orthographic=False):
    from gaussiansplats3d_b200.engine import Engine, Uniforms
    from gaussiansplats3d_b200.scenes import pack_scene
    packed = pack_scene(raw)
    n = packed.count
    eye = np.eye(4, dtype=np.float32).reshape(16)
    u = Uniforms(model_view=eye, projection=np.asarray(P, np.float32), camera_position=np.zeros(3, np.float32),
                 focal=(P[0] * 0.5 * w, P[5] * 0.5 * h), viewport=(w, h), orthographic_mode=1 if orthographic else 0)
    with Engine(n, max_width=w, max_height=h) as e:
        e.upload_splat_data(packed.centers_colors, packed.covariances, packed.sh, packed.sh_degree)
        e.upload_centers(packed.int_centers)
        mvp = np.asarray(P, np.float32)
        rgba, depth = e.frame(mvp, u, w, h, n, depth=True)
    return rgba, depth


def _assert_wall(inner, d, tol):
    """Most of the frame's middle is wall, and every pixel a splat reaches reads the wall's depth (pixels between splats are +inf)."""
    hit = np.isfinite(inner)
    assert hit.mean() > 0.3 and np.isposinf(inner[~hit]).all(), hit.mean()
    assert np.abs(inner[hit] - d).max() <= tol, (np.abs(inner[hit] - d).max(), tol)


@pytest.mark.parametrize("d", [2.0, 10.0, 100.0])
def test_wall_at_a_known_depth(gs, d):
    """A fronto-parallel wall of opaque splats reads its depth within the conversion bound, perspective and orthographic."""
    from gaussiansplats3d_b200 import three_math as TM
    w, h = 320, 240
    P = TM.make_perspective(50.0, w / h, 0.1, 1000.0)
    rgba, depth = _wall_frame(P, w, h, _wall_scene(d))
    inner = depth[h // 4:3 * h // 4, w // 4:3 * w // 4]
    tol = 4.0 * DF.conversion_bound(d, 0.1, 1000.0) + 2e-5 * d
    _assert_wall(inner, d, tol)
    P = TM.make_orthographic(-4.0, 4.0, 3.0, -3.0, 0.1, 1000.0)
    rgba, depth = _wall_frame(P, w, h, _wall_scene(d, extent=5.0, grow=4.0), orthographic=True)
    inner = depth[h // 4:3 * h // 4, w // 4:3 * w // 4]
    tol = 4.0 * DF.conversion_bound(d, 0.1, 1000.0, orthographic=True) + 2e-5 * d
    _assert_wall(inner, d, tol)


def test_stereo_halves_are_the_eyes_mono_depth(gs):
    import test_stereo_gpu as S
    from gaussiansplats3d_b200 import _native as N
    eye_w, h = 640, 480
    raw, packed = S._scene(60_000)
    n = packed.count
    viewer, cams = S._rig(eye_w, h)
    u, eyes = S._shared(viewer, eye_w, h), S._eyes(cams)
    from gaussiansplats3d_b200 import three_math as TM
    mvp = TM.multiply(viewer.projectionMatrix, viewer.matrixWorldInverse).astype(np.float32)
    with S._engine(n, 2 * eye_w, h, packed) as e:
        plain = e.frame(mvp, u, 2 * eye_w, h, n, frame_format=N.GS_FRAME_RGBA32F, eyes=eyes)
        rgba, depth = e.frame(mvp, u, 2 * eye_w, h, n, frame_format=N.GS_FRAME_RGBA32F, eyes=eyes, depth=True)
        order = e.read_buffer(0, np.uint32, n)
    assert np.array_equal(rgba, plain)
    with S._engine(n, eye_w, h, packed) as ref:
        for i, eye in enumerate(eyes):
            _, want = ref.render(S._substituted(u, eye), eye_w, h, n, order, frame_format=N.GS_FRAME_RGBA32F, flip_y=True, depth=True)
            assert np.array_equal(depth[:, i * eye_w:(i + 1) * eye_w].view(np.uint32), want.view(np.uint32)), f"eye {i}"


@pytest.mark.parametrize("count", [1, 2, 4, 16])
def test_multi_view_bands_are_the_cameras_mono_depth(gs, count):
    import test_multi_view_gpu as M
    from gaussiansplats3d_b200 import _native as N
    w, h = 160, 96
    raw, packed = M._scene(30_000)
    n = packed.count
    views = [M._view(c, w, h) for c in M._ring(count, w, h, fovs=[50.0, 35.0, 70.0])]
    u = M._shared(w, h)
    with M._engine(packed, raw, w, count * h) as e:
        plain = e.frame_views(views, u, w, h, n)
        frames, depths = e.frame_views(views, u, w, h, n, depth=True)
    assert np.array_equal(frames, plain) and depths.shape == (count, h, w)
    with M._engine(packed, raw, w, h) as ref:
        for i, v in enumerate(views):
            sp = ref._sort_params(v.model_view_proj, n, n, None, None, None)
            want = np.empty((h, w), np.float32)
            rp, _ = ref._render_params(w, h, n, None, N.GS_FRAME_RGBA8, True, depth=True, depth_out=want)
            uc = M._substituted(u, v).to_c()
            frame = np.empty((h, w, 4), np.uint8)
            N.check(ref._lib.gs_frame(ref._h, C.byref(sp), C.byref(uc), C.byref(rp), None, N.ptr(frame)), "gs_frame")
            assert np.array_equal(depths[i].view(np.uint32), want.view(np.uint32)), f"view {i} of {count}"


def test_composite_depth(gs):
    N = gs._native
    w, h = 1000, 600
    v = _viewer(w, h)
    n = v.splatMesh.getSplatCount()
    _, plain_depth = v.render(frame_format=N.GS_FRAME_RGBA8, depth=True)
    _, ones = v.render(frame_format=N.GS_FRAME_RGBA8, depth=True, dest_depth=np.ones((h, w), np.float32))
    assert np.array_equal(ones.view(np.uint32), plain_depth.view(np.uint32))
    _, zeros = v.render(frame_format=N.GS_FRAME_RGBA8, depth=True, dest_depth=np.zeros((h, w), np.float32))
    assert np.isposinf(zeros).all()
    proj = v.engine.read_projected(n)
    zw = (np.float32(0.5) * proj["ndc_z"][proj["valid"] == 1] + np.float32(0.5)).astype(np.float32)
    lo, hi = np.quantile(zw, 0.05), np.quantile(zw, 0.95)
    plane = np.broadcast_to((lo + (hi - lo) * (np.arange(w, dtype=np.float32) + 0.5) / w).astype(np.float32), (h, w)).copy()
    _check_mono("composite tilted plane", v, N.GS_FRAME_RGBA8, True, dest_depth=plane)
    # the composited colour is the same with and without depth, over a colour and a depth input
    bg = np.full((h, w, 4), 90, np.uint8)
    bg[..., 3] = 255
    plain = v.render(frame_format=N.GS_FRAME_RGBA8, dest_color=bg, dest_depth=plane)
    rgba, _ = v.render(frame_format=N.GS_FRAME_RGBA8, dest_color=bg, dest_depth=plane, depth=True)
    assert np.array_equal(rgba, plain)
    v.dispose()


def test_depth_buffer_follows_pipelined_and_async_frames(gs):
    """GS_BUF_DEPTH after pipelined frames of different cameras without depth_out, whose graphs replay on alternating planes, and after a
    gs_frame_async that follows them: always the last frame's own depth."""
    import test_multi_view_gpu as M
    from gaussiansplats3d_b200 import _native as N
    w, h = 320, 200
    raw, packed = M._scene(30_000)
    n = packed.count
    views = [M._view(c, w, h) for c in M._ring(5, w, h)]
    u0 = M._shared(w, h)
    with M._engine(packed, raw, w, h) as ref:
        want = []
        for v in views:
            _, d = ref.frame(v.model_view_proj, M._substituted(u0, v), w, h, n, depth=True)
            want.append(d)
    assert not np.array_equal(want[0], want[2])

    def dev_depth(e):
        ptr, nbytes = e.buffer_dev(N.GS_BUF_DEPTH)
        assert ptr and nbytes == w * h * 4
        return e.read_buffer(N.GS_BUF_DEPTH, np.float32, w * h).reshape(h, w)

    with M._engine(packed, raw, w, h) as e:
        e.set_graph_enabled(True)
        assert e.buffer_dev(N.GS_BUF_DEPTH) == (0, 0)
        for rounds in range(2):          # the second round replays both parities' graphs
            frames = [np.empty((h, w, 4), np.uint8) for _ in range(3)]
            for i in range(3):
                e.frame_begin(e.prepare_frame(views[i].model_view_proj, M._substituted(u0, views[i]), w, h, n, depth=True), frames[i])
            for _ in range(3):
                e.frame_end()
            assert np.array_equal(dev_depth(e).view(np.uint32), want[2].view(np.uint32)), f"round {rounds}: not the third frame's depth"
            e.frame_async(views[3].model_view_proj, M._substituted(u0, views[3]), w, h, n, depth=True)
            e.synchronize()
            assert np.array_equal(dev_depth(e).view(np.uint32), want[3].view(np.uint32)), f"round {rounds}: not the async frame's depth"
        # a plain frame leaves the last depth where it was
        e.frame(views[4].model_view_proj, M._substituted(u0, views[4]), w, h, n)
        assert np.array_equal(dev_depth(e).view(np.uint32), want[3].view(np.uint32))


def test_frame_paths_agree(gs):
    """Graph, eager, async + GS_BUF_DEPTH (host read and torch view), pipelined frames with their own depth_out, a projection changed
    between graph replays, and one engine switching between depth and plain frames, against fresh engines."""
    import torch
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.parallel import _DevicePointer
    w, h = 640, 400
    v = _viewer(w, h, n=80_000)
    e, n, u = v.engine, v.splatMesh.getSplatCount(), v.uniforms()
    mvp = v.mvp_matrix().astype(np.float32)
    e.set_graph_enabled(True)
    _, graph = e.frame(mvp, u, w, h, n, depth=True)
    _, graph2 = e.frame(mvp, u, w, h, n, depth=True)          # replay
    e.set_graph_enabled(False)
    _, eager = e.frame(mvp, u, w, h, n, depth=True)
    assert np.array_equal(graph.view(np.uint32), eager.view(np.uint32)) and np.array_equal(graph2.view(np.uint32), eager.view(np.uint32))
    e.set_graph_enabled(True)
    e.frame_async(mvp, u, w, h, n, depth=True)
    e.synchronize()
    host = e.read_buffer(N.GS_BUF_DEPTH, np.float32, w * h).reshape(h, w)
    ptr, nbytes = e.buffer_dev(N.GS_BUF_DEPTH)
    assert nbytes == w * h * 4
    dev = torch.as_tensor(_DevicePointer(ptr, nbytes), device="cuda").view(torch.float32).view(h, w).cpu().numpy()
    assert np.array_equal(host.view(np.uint32), eager.view(np.uint32)) and np.array_equal(dev.view(np.uint32), host.view(np.uint32))
    # pipelined: three frames in flight, each with its own depth_out
    prepared = e.prepare_frame(mvp, u, w, h, n, depth=True)
    outs = [np.full((h, w), np.nan, np.float32) for _ in range(3)]
    frames = [np.empty((h, w, 4), np.uint8) for _ in range(3)]
    for i in range(3):
        e.frame_begin(prepared, frames[i], depth_out=outs[i])
    for _ in range(3):
        e.frame_end()
    for o in outs:
        assert np.array_equal(o.view(np.uint32), eager.view(np.uint32))
    # a changed projection (narrower fov, other near / far) between graph replays: the fresh engine's depth
    from gaussiansplats3d_b200 import three_math as TM
    P2 = TM.make_perspective(40.0, w / h, 0.5, 200.0).astype(np.float32)
    u2 = dataclasses.replace(u, projection=P2, focal=(P2[0] * 0.5 * w, P2[5] * 0.5 * h))
    mvp2 = TM.multiply(P2, np.asarray(u.model_view, np.float64)).astype(np.float32)
    _, moved = e.frame(mvp2, u2, w, h, n, depth=True)
    plain_after = e.frame(mvp, u, w, h, n)
    _, back = e.frame(mvp, u, w, h, n, depth=True)
    assert np.array_equal(back.view(np.uint32), eager.view(np.uint32))
    fresh = _viewer(w, h, n=80_000)
    fe = fresh.engine
    _, want = fe.frame(mvp2, u2, w, h, n, depth=True)
    assert np.array_equal(moved.view(np.uint32), want.view(np.uint32)) and not np.array_equal(moved, eager)
    assert np.array_equal(plain_after, fe.frame(mvp, u, w, h, n))
    fresh.dispose()
    v.dispose()


def test_refusals_and_old_callers(gs):
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    w, h = 320, 200
    v = _viewer(w, h, n=20_000)
    e, n, u = v.engine, v.splatMesh.getSplatCount(), v.uniforms()
    mvp = v.mvp_matrix().astype(np.float32)
    plain = e.frame(mvp, u, w, h, n)
    sp = e._sort_params(mvp, n, n, None, None, None)
    uc = u.to_c()
    rp, _ = e._render_params(w, h, n, None, N.GS_FRAME_RGBA8, True)
    rp.depth = 2
    out = np.empty((h, w, 4), np.uint8)
    assert e._lib.gs_frame(e._h, C.byref(sp), C.byref(uc), C.byref(rp), None, N.ptr(out)) == N.GS_ERR_BAD_ARG
    # a caller built before the depth fields: depth and depth_out lie past its struct_size and are never read
    rp.depth, rp.struct_size = 1, N.gs_render_params.depth.offset
    rp.depth_out = C.cast(C.c_void_p(16), C.POINTER(C.c_float))
    assert e._lib.gs_frame(e._h, C.byref(sp), C.byref(uc), C.byref(rp), None, N.ptr(out)) == 0
    assert np.array_equal(out, plain)
    # a peer-attached engine (world 2) refuses depth and still renders its next plain frame
    from gaussiansplats3d_b200.scenes import pack_scene
    packed = pack_scene(_raw(20_000))
    root = Engine(n, max_width=w, max_height=h, rank=0, world_size=2)
    peer = Engine(n, max_width=w, max_height=h, rank=1, world_size=2)
    for x in (root, peer):
        x.upload_splat_data(packed.centers_colors, packed.covariances, packed.sh, packed.sh_degree)
        x.upload_centers(packed.int_centers)
    peer.peer_attach_local(root)
    with pytest.raises(RuntimeError, match="single-GPU"):
        peer.frame(mvp, u, w, h, n, depth=True)
    peer.frame_async(mvp, u, w, h, n)       # the peers' frames go first, then rank 0's releases them
    root.frame(mvp, u, w, h, n)
    peer.synchronize()
    peer.close(); root.close()
    v.dispose()


def test_viewer_returns_rgba_and_depth(gs):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import CAMERAS
    w, h = 320, 200
    v = _viewer(w, h, n=20_000, maxViews=2)
    for rgba, depth in (v.render(depth=True), v.frame(depth=True)):
        assert rgba.shape == (h, w, 4) and depth.shape == (h, w) and np.isfinite(depth).any()
    cams = [v.camera, TM.PerspectiveCamera(40.0, w / h, 0.1, 1000.0)]
    c = CAMERAS["bonsai"]
    cams[1].position = np.asarray(c["position"], np.float64) * 1.2
    cams[1].up = np.asarray(c["up"], np.float64) / np.linalg.norm(c["up"])
    cams[1].look_at(c["look_at"])
    cams[1].update()
    rgba, depth = v.frameViews(cams, depth=True)
    assert rgba.shape == (2, h, w, 4) and depth.shape == (2, h, w)
    v.dispose()
    vr = _viewer(2 * 320, 200, n=20_000, webXRMode=1)
    viewer_cam = vr.camera
    eyes = [TM.PerspectiveCamera(50.0, 320 / 200, 0.1, 1000.0) for _ in range(2)]
    for s, cam in zip((-1.0, 1.0), eyes):
        cam.position = np.asarray(viewer_cam.position, np.float64) + s * 0.032 * np.asarray(viewer_cam.matrixWorld[0:3])
        cam.up = np.asarray(c["up"], np.float64) / np.linalg.norm(c["up"])
        cam.look_at(np.asarray(c["look_at"]) + s * 0.032 * np.asarray(viewer_cam.matrixWorld[0:3]))
        cam.update()
    rgba, depth = vr.frame(xrCameras=eyes, depth=True)
    assert rgba.shape == (200, 640, 4) and depth.shape == (200, 640) and np.isfinite(depth).any()
    vr.dispose()
