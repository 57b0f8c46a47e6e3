"""GPU: multi-view frames (gs_frame_views).  Several cameras of one mesh in one frame, each with its own depth sort, the views stacked
top to bottom.  The contract is exact: each band is byte for byte what gs_frame renders for that camera alone on an engine that never
saw a multi-view frame, and each view's block of sorted_out is what gs_sort returns for its matrix.  The mono frames are held to the
f64 projection and blend bounds elsewhere, so identity carries those bounds over."""
import ctypes as C
import dataclasses
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

_scenes = {}


def _scene(n, sh_degree=1, half=False, seed=31):
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    key = (n, sh_degree, half, seed)
    if key not in _scenes:
        raw = synthetic_scene(n, seed=seed, kind="bonsai", sh_degree=sh_degree)
        _scenes[key] = (raw, pack_scene(raw, half_covariances=half))
    return _scenes[key]


def _camera(pos, look, up, aspect, fov=50.0):
    from gaussiansplats3d_b200 import three_math as TM
    cam = TM.PerspectiveCamera(fov, aspect, 0.1, 1000.0)
    cam.position = np.asarray(pos, np.float64)
    cam.up = np.asarray(up, np.float64) / np.linalg.norm(up)
    cam.look_at(look)
    cam.update()
    return cam


def _ring(count, w, h, *, radius_scale=1.0, fovs=None):
    """`count` cameras on a circle around the bonsai camera's target, the first at the bonsai camera (radius scaled)."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.scenes import CAMERAS
    c = CAMERAS["bonsai"]
    look, up = np.asarray(c["look_at"]), np.asarray(c["up"])
    off = (np.asarray(c["position"]) - look) * radius_scale
    cams = []
    for i in range(count):
        pos = look + TM.rotate_about_axis(off, up, 2.0 * np.pi * i / max(count, 1))
        cams.append(_camera(pos, look, up, w / h, fovs[i % len(fovs)] if fovs else 50.0))
    return cams


def _view(cam, w, h, dynamic=False, ortho_zoom=1.0):
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import View
    P = cam.projectionMatrix
    return View(model_view_proj=TM.multiply(P, cam.matrixWorldInverse).astype(np.float32), model_view=cam.matrixWorldInverse.astype(np.float32),
                projection=P.astype(np.float32), camera_position=np.asarray(cam.position, np.float32), focal=(P[0] * 0.5 * w, P[5] * 0.5 * h),
                ortho_zoom=ortho_zoom, view_matrix=cam.matrixWorldInverse.astype(np.float32) if dynamic else None)


def _shared(w, h, sh_degree=1, **kw):
    """The uniforms every view shares; the camera fields are placeholders that each view replaces."""
    from gaussiansplats3d_b200.engine import Uniforms
    return Uniforms(model_view=np.eye(4, dtype=np.float32), projection=np.eye(4, dtype=np.float32), camera_position=np.zeros(3, np.float32),
                    focal=(1.0, 1.0), viewport=(w, h), sh_degree=sh_degree, **kw)


def _substituted(u, v):
    return dataclasses.replace(u, model_view=v.model_view, projection=v.projection, camera_position=v.camera_position, focal=v.focal,
                               ortho_zoom=v.ortho_zoom, view_matrix=v.view_matrix if u.dynamic_mode else u.view_matrix)


def _engine(packed, raw, w, h, *, dynamic=False, integer=True, distance_map_range=1 << 16, scene_indexes=None):
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import float_centers
    n = packed.count
    e = Engine(n, max_width=w, max_height=h, dynamic_mode=dynamic, integer_based_sort=integer, distance_map_range=distance_map_range)
    e.upload_splat_data(packed.centers_colors, packed.covariances, packed.sh, packed.sh_degree, scene_indexes=scene_indexes)
    si = scene_indexes if scene_indexes is not None else (np.zeros(n, np.uint32) if dynamic else None)
    e.upload_centers(packed.int_centers if integer else float_centers(raw.centers), si)
    return e


def _mono(e, v, u, w, h, n, *, sort_count=None, indexes=None, transforms=None, fmt=None, flip_y=True):
    """gs_frame of one view alone: (frame, sorted indexes)."""
    from gaussiansplats3d_b200 import _native as N
    fmt = N.GS_FRAME_RGBA8 if fmt is None else fmt
    sp = e._sort_params(v.model_view_proj, n if sort_count is None else sort_count, n, indexes, transforms, None)
    rp, _ = e._render_params(w, h, n, None, fmt, flip_y)
    uc = _substituted(u, v).to_c()
    shape, dt = e._frame_shape(w, h, fmt)
    frame, order = np.empty(shape, dt), np.empty(n, np.uint32)
    N.check(e._lib.gs_frame(e._h, C.byref(sp), C.byref(uc), C.byref(rp), N.ptr(order), N.ptr(frame)), "gs_frame")
    return frame, order


def _check(views, u, packed, raw, w, h, *, what, fmt=None, flip_y=True, sort_count=None, indexes=None, transforms=None, engine_kw=None):
    """Renders `views` as one multi-view frame and each view alone on a second engine, and compares band by band and block by block."""
    from gaussiansplats3d_b200 import _native as N
    fmt = N.GS_FRAME_RGBA8 if fmt is None else fmt
    n, V = packed.count, len(views)
    kw = engine_kw or {}
    order = np.empty((V, n), np.uint32)
    with _engine(packed, raw, w, V * h, **kw) as e:
        frames = e.frame_views(views, u, w, h, n, indexes, sort_count=sort_count, frame_format=fmt, flip_y=flip_y, sorted_out=order,
                               transforms=transforms)
    with _engine(packed, raw, w, h, **kw) as ref:
        for i, v in enumerate(views):
            want, want_order = _mono(ref, v, u, w, h, n, sort_count=sort_count, indexes=indexes, transforms=transforms, fmt=fmt, flip_y=flip_y)
            assert np.array_equal(order[i], want_order), f"{what}: view {i} of {V}: its draw order differs from gs_sort's"
            assert np.array_equal(frames[i].view(np.uint8), want.view(np.uint8)), f"{what}: view {i} of {V}: its band differs from gs_frame's"
    return frames


@pytest.mark.parametrize("V", [1, 2, 3, 8, 16])
@pytest.mark.parametrize("fmt_name,flip_y", [("rgba8", True), ("rgba32f", False)])
def test_bands_are_the_mono_frames(gs, V, fmt_name, flip_y):
    N = gs._native
    fmt = N.GS_FRAME_RGBA8 if fmt_name == "rgba8" else N.GS_FRAME_RGBA32F
    w, h = 330, 190
    raw, packed = _scene(40_000)
    views = [_view(c, w, h) for c in _ring(V, w, h, fovs=[50.0, 65.0, 40.0])]
    frames = _check(views, _shared(w, h), packed, raw, w, h, what=f"V={V} {fmt_name} flip_y={flip_y}", fmt=fmt, flip_y=flip_y)
    assert frames[0][..., 3].max() > 0
    if V > 1:
        assert not np.array_equal(frames[0], frames[1]), "two cameras gave the same picture: the test would not notice swapped views"


@pytest.mark.parametrize("fmt_name,flip_y", [("rgba8", False), ("rgba32f", True)])
def test_formats_with_the_other_row_order(gs, fmt_name, flip_y):
    N = gs._native
    fmt = N.GS_FRAME_RGBA8 if fmt_name == "rgba8" else N.GS_FRAME_RGBA32F
    w, h = 256, 144
    raw, packed = _scene(30_000)
    views = [_view(c, w, h) for c in _ring(3, w, h)]
    _check(views, _shared(w, h), packed, raw, w, h, what=f"{fmt_name} flip_y={flip_y}", fmt=fmt, flip_y=flip_y)


# (SH degree, f16 covariances, integer sort, distance map range, sort count as a fraction of the render count, a caller's index list)
CONFIGS = [
    (0, False, True, 1 << 16, 1.0, False), (2, False, True, 1 << 16, 1.0, False), (2, True, True, 1 << 16, 1.0, False),
    (1, False, False, 1 << 16, 1.0, False), (1, True, False, 1 << 20, 1.0, False), (1, False, True, 1 << 12, 1.0, False),
    (1, False, True, 1 << 16, 0.4, False), (1, False, False, 1 << 20, 0.3, True), (2, True, True, 1 << 16, 1.0, True),
]


@pytest.mark.parametrize("sh,half,integer,R,frac,caller", CONFIGS)
def test_storage_sort_modes_and_partial_sorts(gs, sh, half, integer, R, frac, caller):
    w, h = 300, 170
    raw, packed = _scene(35_000, sh_degree=sh, half=half)
    n = packed.count
    views = [_view(c, w, h) for c in _ring(3, w, h, fovs=[50.0, 70.0])]
    indexes = np.random.default_rng(5).permutation(n).astype(np.uint32) if caller else None
    _check(views, _shared(w, h, sh_degree=sh), packed, raw, w, h, what=f"sh{sh} half={half} int={integer} R={R} frac={frac} caller={caller}",
           sort_count=int(n * frac), indexes=indexes, engine_kw=dict(integer=integer, distance_map_range=R))


@pytest.mark.parametrize("dynamic", [False, True])
def test_multi_scene_meshes(gs, dynamic):
    N = gs._native
    from gaussiansplats3d_b200 import three_math as TM
    w, h = 280, 160
    raw, packed = _scene(30_000)
    n = packed.count
    scene_idx = (np.arange(n) % 2).astype(np.uint32)
    xf = np.tile(np.eye(4, dtype=np.float32).reshape(16), N.GS_MAX_SCENES)
    xf[16:32] = TM.compose((0.4, -0.2, 0.3), (0.0, 0.1305262, 0.0, 0.9914449), (1.0, 1.0, 1.0)).astype(np.float32)
    opacity = np.ones(N.GS_MAX_SCENES, np.float32)
    opacity[1] = 0.5
    kw = dict(scene_count=2, enable_optional_effects=1, scene_opacity=opacity)
    if dynamic:
        kw.update(dynamic_mode=1, scene_transforms=xf)
    u = _shared(w, h, **kw)
    views = [_view(c, w, h, dynamic=dynamic) for c in _ring(4, w, h)]
    _check(views, u, packed, raw, w, h, what=f"two scenes dynamic={dynamic}", transforms=xf if dynamic else None,
           engine_kw=dict(dynamic=dynamic, scene_indexes=scene_idx))


@pytest.mark.parametrize("w,h", [(1920, 1080), (4100, 2100)])
def test_both_binning_paths(gs, w, h):
    """1920x1080 per view: at most 255 coarse tiles (counting-sort binning); 4100x2100: more than 256 at 32 px (radix binning)."""
    raw, packed = _scene(60_000)
    views = [_view(c, w, h) for c in _ring(2, w, h)]
    _check(views, _shared(w, h), packed, raw, w, h, what=f"{w}x{h}")


def test_odd_cameras(gs):
    """Cameras of different fov, one with nothing in view (looking away from the cloud) and one inside the cloud."""
    from gaussiansplats3d_b200.scenes import CAMERAS
    w, h = 320, 200
    raw, packed = _scene(40_000)
    c = CAMERAS["bonsai"]
    look = np.asarray(c["look_at"])
    pos = np.asarray(c["position"])
    cams = [_camera(pos, look, c["up"], w / h, 50.0), _camera(pos, look, c["up"], w / h, 90.0),
            _camera(pos, 2 * pos - look, c["up"], w / h, 50.0), _camera((0.05, 0.02, 0.0), look, c["up"], w / h, 60.0)]
    frames = _check([_view(x, w, h) for x in cams], _shared(w, h), packed, raw, w, h, what="odd cameras")
    assert frames[2][..., 3].max() == 0, "the camera looking away from the cloud sees splats"
    assert frames[3][..., 3].max() > 0


def test_orthographic_views(gs):
    """An orthographic set: the shared uniforms in orthographic mode, each view with its own orthographic projection and zoom."""
    from gaussiansplats3d_b200 import three_math as TM
    w, h = 300, 180
    raw, packed = _scene(30_000)
    views = []
    for i, cam in enumerate(_ring(3, w, h)):
        half = 4.0 + i
        P = np.zeros(16)
        P[0], P[5], P[10], P[14], P[15] = 1.0 / (half * w / h), 1.0 / half, -2.0 / 999.9, -1000.1 / 999.9, 1.0
        v = _view(cam, w, h, ortho_zoom=1.0 + 0.5 * i)
        views.append(dataclasses.replace(v, projection=P.astype(np.float32), focal=(P[0] * 0.5 * w, P[5] * 0.5 * h),
                                         model_view_proj=TM.multiply(P, cam.matrixWorldInverse).astype(np.float32)))
    _check(views, _shared(w, h, orthographic_mode=1), packed, raw, w, h, what="orthographic")


def test_one_view_is_the_mono_frame(gs):
    from gaussiansplats3d_b200 import three_math as TM
    w, h = 400, 240
    raw, packed = _scene(40_000)
    n = packed.count
    cam = _ring(1, w, h)[0]
    v = _view(cam, w, h)
    u = _substituted(_shared(w, h), v)
    with _engine(packed, raw, w, h) as a, _engine(packed, raw, w, h) as b:
        order = np.empty((1, n), np.uint32)
        got = a.frame_views([v], _shared(w, h), w, h, n, sorted_out=order)
        mono_order = np.empty(n, np.uint32)
        want = b.frame(TM.multiply(cam.projectionMatrix, cam.matrixWorldInverse).astype(np.float32), u, w, h, n, sorted_out=mono_order)
    assert np.array_equal(got[0], want) and np.array_equal(order[0], mono_order)


@pytest.mark.parametrize("graphs", [True, False])
def test_one_engine_across_mono_stereo_and_multi_view(gs, graphs):
    """Mono, stereo, multi-view at several view counts and mono again on one engine: every frame equals a fresh engine's."""
    from gaussiansplats3d_b200.engine import Eye
    w, h = 240, 150
    raw, packed = _scene(30_000)
    n = packed.count
    cams = _ring(8, w, h, fovs=[50.0, 60.0])
    views = [_view(c, w, h) for c in cams]
    u = _shared(w, h)
    mvp0 = views[0].model_view_proj
    eyes = tuple(Eye(model_view=v.model_view, projection=v.projection, camera_position=v.camera_position) for v in views[:2])
    stereo_u = dataclasses.replace(_substituted(u, views[0]), viewport=(w, h))

    def fresh(kind, arg):
        with _engine(packed, raw, 2 * w, 8 * h) as f:
            f.set_graph_enabled(graphs)
            return run(f, kind, arg)

    def run(e, kind, arg):
        if kind == "mono":
            return e.frame(mvp0, _substituted(u, views[0]), w, h, n).copy()
        if kind == "stereo":
            return e.frame(mvp0, stereo_u, 2 * w, h, n, eyes=eyes).copy()
        return e.frame_views(views[:arg], u, w, h, n).copy()

    seq = [("mono", 0), ("stereo", 0), ("multi", 3), ("multi", 8), ("mono", 0), ("multi", 2), ("multi", 3), ("stereo", 0), ("mono", 0)]
    with _engine(packed, raw, 2 * w, 8 * h) as e:
        e.set_graph_enabled(graphs)
        for i, (kind, arg) in enumerate(seq):
            got = run(e, kind, arg)
            assert np.array_equal(got, fresh(kind, arg)), f"frame {i} ({kind} {arg}) differs from a fresh engine's"


def test_overflow_in_one_view(gs):
    """An instance-list overflow in one view only is GS_ERR_CAPACITY with the counts; the engine's next frame is a fresh engine's.
    GS_INSTANCE_FACTOR=0 leaves the lists 4 instances per 16-px tile plus 65536: the bonsai view of 150k splats needs more (every
    visible splat is at least one instance), a camera looking away needs none, and 20k splats fit."""
    N = gs._native
    from gaussiansplats3d_b200.scenes import CAMERAS
    w, h = 640, 400
    raw, packed = _scene(150_000)
    n = packed.count
    c = CAMERAS["bonsai"]
    pos, look = np.asarray(c["position"]), np.asarray(c["look_at"])
    seen, away = (_view(_camera(pos, look, c["up"], w / h), w, h), _view(_camera(pos, 2 * pos - look, c["up"], w / h), w, h))
    u = _shared(w, h)
    old = os.environ.get("GS_INSTANCE_FACTOR")
    os.environ["GS_INSTANCE_FACTOR"] = "0"
    try:
        e = _engine(packed, raw, w, 3 * h)
        fresh = _engine(packed, raw, w, 3 * h)
    finally:
        if old is None:
            del os.environ["GS_INSTANCE_FACTOR"]
        else:
            os.environ["GS_INSTANCE_FACTOR"] = old
    with e, fresh:
        ok = [seen, _view(_ring(2, w, h)[1], w, h)]
        want = fresh.frame_views(ok, u, w, h, 20_000).copy()
        assert want[..., 3].max() > 0
        with pytest.raises(N.GsError) as ei:
            e.frame_views([away, seen, away], u, w, h, n)
        assert ei.value.code == N.GS_ERR_CAPACITY and "instances needed" in str(ei.value), str(ei.value)
        assert np.array_equal(e.frame_views(ok, u, w, h, 20_000), want), "the frame after an overflow differs from a fresh engine's"


def test_refusals(gs):
    N = gs._native
    from gaussiansplats3d_b200.engine import Engine, Eye
    w, h = 200, 120
    raw, packed = _scene(20_000)
    n = packed.count
    views = [_view(c, w, h) for c in _ring(3, w, h)]
    u = _shared(w, h)

    def call(e, vs, count=None, *, sp_kw=None, rp_kw=None, height=h):
        sp = e._sort_params(np.zeros(16, np.float32), n, n, None, None, None)
        for k, v in (sp_kw or {}).items():
            setattr(sp, k, v)
        rp, _ = e._render_params(w, height, n, None, N.GS_FRAME_RGBA8, True, **(rp_kw or {}))
        arr = (N.gs_view * max(len(vs), 1))(*[v.to_c() for v in vs])
        uc = u.to_c()
        rc = e._lib.gs_frame_views(e._h, C.byref(sp), C.byref(uc), C.byref(rp), arr, len(vs) if count is None else count, None, None)
        return rc, e._lib.gs_last_error_message().decode()

    with _engine(packed, raw, w, 3 * h) as e:
        pre = np.zeros(n, np.int32)
        cases = [
            (dict(count=0), "view_count 0"),
            (dict(count=N.GS_MAX_VIEWS + 1), f"view_count {N.GS_MAX_VIEWS + 1}"),
            (dict(rp_kw=dict(eyes=tuple(Eye(v.model_view, v.projection, v.camera_position) for v in views[:2]))), "eyes"),
            (dict(rp_kw=dict(dest_depth=np.ones((h, w), np.float32))), "composited"),
            (dict(sp_kw=dict(use_precomputed_distances=1, precomputed_distances=pre.ctypes.data)), "precomputed distances"),
            (dict(height=h + 1), "max_height"),
        ]
        for kw, msg in cases:
            rc, text = call(e, views, **kw)
            assert rc == N.GS_ERR_BAD_ARG and msg in text, (kw, rc, text)
        # the engine still renders after every refusal
        e.frame_views(views, u, w, h, n)
    with Engine(n, max_width=w, max_height=3 * h, rank=0, world_size=2) as e2:
        e2.upload_splat_data(packed.centers_colors, packed.covariances, packed.sh, packed.sh_degree)
        e2.upload_centers(packed.int_centers)
        rc, text = call(e2, views)
        assert rc == N.GS_ERR_BAD_ARG and "single-GPU" in text, (rc, text)


def test_viewer_frame_views_of_its_camera_is_its_frame(gs):
    from gaussiansplats3d_b200.scenes import synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    w, h = 360, 220
    raw = synthetic_scene(30_000, seed=9, kind="bonsai", sh_degree=1)
    v = Viewer(dict(width=w, height=h, sphericalHarmonicsDegree=1, cameraUp=(0.01933, -0.7583, -0.65161), devicePixelRatio=1.0, maxViews=2,
                    initialCameraPosition=(1.54163, 2.68515, -6.37228), initialCameraLookAt=(0.45622, 1.95338, 1.51278)))
    try:
        v.addSplatScene(raw)
        want = v.frame().copy()
        got = v.frameViews([v.camera])
        assert got.shape == (1, h, w, 4) and np.array_equal(got[0], want)
        other = _camera((-1.0, 2.0, -6.5), (0.45622, 1.95338, 1.51278), (0.01933, -0.7583, -0.65161), w / h, 70.0)
        both = v.frameViews([v.camera, other])
        assert np.array_equal(both[0], want) and not np.array_equal(both[1], want)
    finally:
        v.dispose()
