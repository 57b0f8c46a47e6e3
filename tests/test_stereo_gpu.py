"""GPU: WebXR stereo frames (gs_render_params.eyes).  Both eyes of an XR framebuffer side by side in one frame, from one draw order, as
three.js draws the splat mesh once per sub-camera of the XR ArrayCamera with the order of the viewer camera's sort.  The contract is
exact: each half of a stereo frame is bit-identical to the mono frame of one eye's size with the same draw order and uniforms and that
eye's four gs_eye fields substituted."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

IPD = 0.064   # metres between the eyes
# eye sizes: 16-px tiles, 32-px tiles binned by counting sort, more than kBinTiles coarse tiles at 32 px (radix binning); no eye width
# is a multiple of its tile edge
EYE_SIZES = [(810, 600), (2600, 1500), (4100, 2100)]

_scenes = {}


def _scene(n, sh_degree=1):
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    key = (n, sh_degree)
    if key not in _scenes:
        raw = synthetic_scene(n, seed=31, kind="bonsai", sh_degree=sh_degree)
        _scenes[key] = (raw, pack_scene(raw))
    return _scenes[key]


def _camera(pos, look, up, aspect):
    from gaussiansplats3d_b200 import three_math as TM
    cam = TM.PerspectiveCamera(50.0, aspect, 0.1, 1000.0)
    cam.position = np.asarray(pos, np.float64)
    cam.up = np.asarray(up, np.float64) / np.linalg.norm(up)
    cam.look_at(look)
    cam.update()
    return cam


def _rig(eye_w, h, head=(0.0, 0.0, 0.0)):
    """The bonsai viewer camera (moved by `head`) and two eye cameras IPD apart along its right axis, looking the same way."""
    from gaussiansplats3d_b200.scenes import CAMERAS
    c = CAMERAS["bonsai"]
    pos, look = np.add(c["position"], head), np.add(c["look_at"], head)
    viewer = _camera(pos, look, c["up"], eye_w / h)
    right = viewer.matrixWorld[0:3]
    eyes = [_camera(pos + s * 0.5 * IPD * right, look + s * 0.5 * IPD * right, c["up"], eye_w / h) for s in (-1.0, 1.0)]
    return viewer, eyes


def _shared(viewer, eye_w, h, sh_degree=1, dynamic=None):
    """gs_uniforms as Viewer.updateSplatMesh + uniforms() build them for an eye-sized render dimension (viewer camera fields)."""
    from gaussiansplats3d_b200.engine import Uniforms
    P = viewer.projectionMatrix
    kw = {} if dynamic is None else dict(dynamic_mode=1, scene_transforms=dynamic, view_matrix=viewer.matrixWorldInverse.astype(np.float32), scene_count=1)
    return Uniforms(model_view=viewer.matrixWorldInverse.astype(np.float32), projection=P.astype(np.float32),
                    camera_position=viewer.position.astype(np.float32), focal=(P[0] * 0.5 * eye_w, P[5] * 0.5 * h), viewport=(eye_w, h),
                    sh_degree=sh_degree, **kw)


def _eyes(cams, dynamic=False):
    from gaussiansplats3d_b200.engine import Eye
    return tuple(Eye(model_view=c.matrixWorldInverse.astype(np.float32), projection=c.projectionMatrix.astype(np.float32),
                     camera_position=np.asarray(c.matrixWorld[12:15], np.float32),
                     view_matrix=c.matrixWorldInverse.astype(np.float32) if dynamic else None) for c in cams)


def _substituted(u, eye):
    """The mono uniforms of one eye: the shared ones with that eye's four fields."""
    import dataclasses
    return dataclasses.replace(u, model_view=eye.model_view, projection=eye.projection, camera_position=eye.camera_position,
                               view_matrix=eye.view_matrix if u.dynamic_mode else u.view_matrix)


def _engine(n, w, h, packed, *, dynamic=False):
    from gaussiansplats3d_b200.engine import Engine
    e = Engine(n, max_width=w, max_height=h, dynamic_mode=dynamic)
    e.upload_splat_data(packed.centers_colors, packed.covariances, packed.sh, packed.sh_degree)
    e.upload_centers(packed.int_centers, np.zeros(n, np.uint32) if dynamic else None)
    return e


def _order(e, viewer, n, transforms=None):
    from gaussiansplats3d_b200 import three_math as TM
    mvp = TM.multiply(viewer.projectionMatrix, viewer.matrixWorldInverse).astype(np.float32)
    order, _ = e.sort(mvp, n, n, None, transforms=transforms)
    return order, mvp


def _assert_halves(frame, left, right, what):
    eye_w = left.shape[1]
    assert frame.shape == (left.shape[0], 2 * eye_w, 4), (what, frame.shape, left.shape)
    assert np.array_equal(frame[:, :eye_w].view(np.uint8), left.view(np.uint8)), f"{what}: the left half differs from the left eye's mono frame"
    assert np.array_equal(frame[:, eye_w:].view(np.uint8), right.view(np.uint8)), f"{what}: the right half differs from the right eye's mono frame"


@pytest.mark.parametrize("eye_w,h", EYE_SIZES)
@pytest.mark.parametrize("fmt_name", ["rgba8", "rgba32f"])
@pytest.mark.parametrize("flip_y", [False, True])
def test_halves_are_the_mono_eye_frames(gs, eye_w, h, fmt_name, flip_y):
    N = gs._native
    fmt = N.GS_FRAME_RGBA8 if fmt_name == "rgba8" else N.GS_FRAME_RGBA32F
    n = 120_000
    _, packed = _scene(n)
    viewer, cams = _rig(eye_w, h)
    u, eyes = _shared(viewer, eye_w, h), _eyes(cams)
    with _engine(n, 2 * eye_w, h, packed) as e:
        order, _ = _order(e, viewer, n)
        stereo = e.render(u, 2 * eye_w, h, n, order, frame_format=fmt, flip_y=flip_y, eyes=eyes).copy()
        mono = [e.render(_substituted(u, eye), eye_w, h, n, order, frame_format=fmt, flip_y=flip_y).copy() for eye in eyes]
    assert mono[0][..., 3].max() > 0 and mono[1][..., 3].max() > 0
    assert not np.array_equal(mono[0], mono[1]), "the eyes see the same picture: the test would not notice swapped eyes"
    _assert_halves(stereo, mono[0], mono[1], f"{eye_w}x{h} {fmt_name} flip_y={flip_y}")


def test_camera_position_and_dynamic_view_matrix_are_per_eye(gs):
    """SH degree 1 colours depend on each eye's camera_position; a dynamic mesh places splats with each eye's view matrix."""
    N = gs._native
    from gaussiansplats3d_b200 import three_math as TM
    n, eye_w, h = 60_000, 640, 480
    raw, packed = _scene(n)
    viewer, cams = _rig(eye_w, h)
    # the camera positions alone change the picture (same matrices, eyes swapped only in camera_position)
    u, eyes = _shared(viewer, eye_w, h), _eyes(cams)
    swapped = (eyes[0].__class__(eyes[0].model_view, eyes[0].projection, eyes[1].camera_position), eyes[1])
    with _engine(n, 2 * eye_w, h, packed) as e:
        order, _ = _order(e, viewer, n)
        a = e.render(u, 2 * eye_w, h, n, order, eyes=eyes).copy()
        b = e.render(u, 2 * eye_w, h, n, order, eyes=swapped).copy()
        _assert_halves(b, e.render(_substituted(u, swapped[0]), eye_w, h, n, order), e.render(_substituted(u, swapped[1]), eye_w, h, n, order), "sh1")
    assert not np.array_equal(a[:, :eye_w], b[:, :eye_w]), "camera_position did not reach the SH colours"
    # dynamic mode: per-scene transform in the vertex stage, view matrix per eye
    xf = np.tile(np.eye(4, dtype=np.float32).reshape(16), N.GS_MAX_SCENES)
    xf[:16] = TM.compose((0.1, -0.05, 0.2), (0.0, 0.0871557, 0.0, 0.9961947), (1.0, 1.0, 1.0)).astype(np.float32)
    u = _shared(viewer, eye_w, h, dynamic=xf)
    eyes = _eyes(cams, dynamic=True)
    with _engine(n, 2 * eye_w, h, packed, dynamic=True) as e:
        order, _ = _order(e, viewer, n, transforms=xf)
        stereo = e.render(u, 2 * eye_w, h, n, order, frame_format=N.GS_FRAME_RGBA32F, eyes=eyes).copy()
        mono = [e.render(_substituted(u, eye), eye_w, h, n, order, frame_format=N.GS_FRAME_RGBA32F).copy() for eye in eyes]
        still = e.render(_substituted(u, eyes[0]), eye_w, h, n, order, frame_format=N.GS_FRAME_RGBA32F).copy()
        import dataclasses
        moved = e.render(dataclasses.replace(_substituted(u, eyes[0]), view_matrix=eyes[1].view_matrix), eye_w, h, n, order,
                         frame_format=N.GS_FRAME_RGBA32F)
    _assert_halves(stereo, mono[0], mono[1], "dynamic")
    assert not np.array_equal(still, moved), "the view matrix does not place splats in dynamic mode"


def test_frame_sorts_once_with_the_viewer_camera(gs):
    N = gs._native
    n, eye_w, h = 100_000, 960, 540
    _, packed = _scene(n)
    viewer, cams = _rig(eye_w, h)
    u, eyes = _shared(viewer, eye_w, h), _eyes(cams)
    with _engine(n, 2 * eye_w, h, packed) as e:
        order, mvp = _order(e, viewer, n)
        got_order = np.empty(n, np.uint32)
        frame = e.frame(mvp, u, 2 * eye_w, h, n, sorted_out=got_order, eyes=eyes).copy()
        assert np.array_equal(got_order, order), "gs_frame with eyes must sort exactly as gs_sort with the same MVP"
        mono = [e.render(_substituted(u, eye), eye_w, h, n, order, frame_format=N.GS_FRAME_RGBA8, flip_y=True).copy() for eye in eyes]
    _assert_halves(frame, mono[0], mono[1], "gs_frame")


def test_graph_eager_and_pipelined_frames_agree(gs):
    """The frame graph and the eager path give the same stereo frame; pipelined stereo frames with a moving head equal gs_frame's."""
    N = gs._native
    n, eye_w, h = 100_000, 800, 600
    _, packed = _scene(n)
    heads = [(0.03 * i, -0.01 * i, 0.02 * i) for i in range(6)]
    with _engine(n, 2 * eye_w, h, packed) as e:
        args = []
        for head in heads:
            viewer, cams = _rig(eye_w, h, head)
            _, mvp = _order(e, viewer, n)
            args.append((mvp, _shared(viewer, eye_w, h), _eyes(cams)))
        want = [e.frame(mvp, u, 2 * eye_w, h, n, eyes=eyes).copy() for mvp, u, eyes in args]
        assert not np.array_equal(want[0], want[-1])
        e.set_graph_enabled(False)
        eager = [e.frame(mvp, u, 2 * eye_w, h, n, eyes=eyes).copy() for mvp, u, eyes in args]
        e.set_graph_enabled(True)
        for i, (a, b) in enumerate(zip(want, eager)):
            assert np.array_equal(a, b), f"frame {i}: the eager stereo frame differs from the graph's"
        bufs = [N.pinned_empty((h, 2 * eye_w, 4), np.uint8) for _ in range(3)]
        prepared = [e.prepare_frame(mvp, u, 2 * eye_w, h, n, eyes=eyes) for mvp, u, eyes in args]
        got = []
        e.frame_begin(prepared[0], bufs[0])
        e.frame_begin(prepared[1], bufs[1])
        for i in range(len(heads)):
            if i + 2 < len(heads):
                e.frame_begin(prepared[i + 2], bufs[(i + 2) % 3])
            e.frame_end()
            got.append(bufs[i % 3].copy())
        for i, (a, b) in enumerate(zip(want, got)):
            assert np.array_equal(a, b), f"pipelined stereo frame {i} differs from gs_frame's"
        # gs_frame_async leaves the same frame on the device
        e.frame_async(args[2][0], args[2][1], 2 * eye_w, h, n, eyes=args[2][2])
        e.synchronize()
        dev = e.read_buffer(N.GS_BUF_FRAME, np.uint8, h * 2 * eye_w * 4).reshape(h, 2 * eye_w, 4)
        assert np.array_equal(dev, want[2])


def test_mono_and_stereo_frames_do_not_leak_into_each_other(gs):
    """One engine renders mono -> stereo -> mono -> stereo at different sizes (16- and 32-px tiles); each frame equals a fresh engine's.
    The 2048x1024 eyes have 256 coarse tiles each at 16 px, the most a frame at 16-px tiles can have, and more than the engine's
    5200x1500 maximum has at 32 px (252)."""
    n = 80_000
    _, packed = _scene(n)
    W, H = 5200, 1500
    seq = [(False, 1000, 600), (True, 800, 600), (False, 640, 480), (True, 2600, 1500), (False, 1000, 600), (True, 800, 600),
           (True, 2048, 1024)]

    def one(e, stereo, w, h):
        viewer, cams = _rig(w, h)
        u, eyes = _shared(viewer, w, h), _eyes(cams)
        _, mvp = _order(e, viewer, n)
        if stereo:
            return e.frame(mvp, u, 2 * w, h, n, eyes=eyes).copy()
        u = _shared(viewer, w, h)
        return e.frame(mvp, u, w, h, n).copy()

    with _engine(n, W, H, packed) as e:
        got = [one(e, *s) for s in seq]
    for i, s in enumerate(seq):
        with _engine(n, W, H, packed) as f:
            want = one(f, *s)
        assert np.array_equal(got[i], want), f"frame {i} {s}: differs from the same frame on a fresh engine"


def test_overflow_in_a_stereo_frame_is_reported_and_the_engine_recovers(gs, monkeypatch):
    import re
    N = gs._native
    from gaussiansplats3d_b200.engine import Engine
    monkeypatch.setenv("GS_INSTANCE_FACTOR", "0.05")
    n, eye_w, h = 300_000, 1920, 1080
    _, packed = _scene(n, sh_degree=0)
    viewer, cams = _rig(eye_w, h)
    u, eyes = _shared(viewer, eye_w, h, sh_degree=0), _eyes(cams)

    def fresh_fit(fit):
        with Engine(n, max_width=2 * eye_w, max_height=h) as f:
            f.upload_splat_data(packed.centers_colors, packed.covariances)
            return f.render(u, 2 * eye_w, h, len(fit), fit, eyes=eyes).copy()

    e = Engine(n, max_width=2 * eye_w, max_height=h)
    e.upload_splat_data(packed.centers_colors, packed.covariances)
    e.upload_centers(packed.int_centers)
    order, mvp = _order(e, viewer, n)
    fit = order[-50:]
    want_fit = fresh_fit(fit)
    for path in ("render", "frame"):
        with pytest.raises(N.GsError) as ei:
            if path == "render":
                e.render(u, 2 * eye_w, h, n, order, eyes=eyes)
            else:
                e.frame(mvp, u, 2 * eye_w, h, n, eyes=eyes)
        assert ei.value.code == N.GS_ERR_CAPACITY, str(ei.value)
        mt = re.search(r"(\d+) instances needed, capacity (\d+)", str(ei.value))
        assert mt and int(mt.group(1)) > int(mt.group(2)), str(ei.value)
        assert e.timings()["tile_instances"] == int(mt.group(1))
        got = e.render(u, 2 * eye_w, h, len(fit), fit, eyes=eyes)
        assert np.array_equal(got, want_fit), f"{path}: the stereo frame after the overflow differs from a fresh engine's"
    e.close()


def test_refusals_and_old_callers(gs):
    N = gs._native
    from gaussiansplats3d_b200.engine import Engine
    n, eye_w, h = 20_000, 320, 240
    _, packed = _scene(n)
    viewer, cams = _rig(eye_w, h)
    u, eyes = _shared(viewer, eye_w, h), _eyes(cams)

    def refused(e, match, **kw):
        args = dict(width=2 * eye_w, uniforms=u)
        args.update(kw)
        with pytest.raises(N.GsError) as ei:
            e.render(args["uniforms"], args["width"], h, n, np.arange(n, dtype=np.uint32), eyes=eyes,
                     **{k: v for k, v in kw.items() if k.startswith("dest_")})
        assert ei.value.code == N.GS_ERR_BAD_ARG and match in str(ei.value), str(ei.value)

    import dataclasses
    with _engine(n, 2 * eye_w + 2, h, packed) as e:
        refused(e, "even width", width=2 * eye_w + 1, uniforms=dataclasses.replace(u, viewport=((2 * eye_w + 1) // 2, h)))
        refused(e, "composited", dest_depth=np.ones((h, 2 * eye_w), np.float32))
        refused(e, "viewport uniform", uniforms=dataclasses.replace(u, viewport=(2 * eye_w, h)))
        # a caller built before `eyes` (smaller struct_size) renders the mono frame of the whole width, whatever the field holds
        order = np.arange(n, dtype=np.uint32)
        mono = e.render(u, 2 * eye_w, h, n, order).copy()
        p, keep = e._render_params(2 * eye_w, h, n, order, N.GS_FRAME_RGBA32F, False, eyes=eyes)
        p.struct_size = N.gs_render_params.eyes.offset
        out = np.empty((h, 2 * eye_w, 4), np.float32)
        N.check(e._lib.gs_render(e._h, C.byref(u.to_c()), C.byref(p), N.ptr(out)), "gs_render")
        assert np.array_equal(out, mono)
    with Engine(n, max_width=2 * eye_w, max_height=h, rank=0, world_size=2) as e:
        e.upload_splat_data(packed.centers_colors, packed.covariances, packed.sh, packed.sh_degree)
        refused(e, "single-GPU")
