"""GPU: frames composited into a caller's opaque pass (gs_render_params dest_color / dest_depth): every splat depth-tested against the
pass's depth (LessEqualDepth, no depth writes) and blended over its colour, as the reference's Viewer draws the splat mesh after its
threeScene (Viewer.js:1599-1620).  Against the plain frame, the background, and the f64 restatement of the composite
(tests/blend_f64.py) fed the GPU's own raw records and draw order: the depth decision is the same f32 comparison on both sides, and every
channel of every pixel must lie within its own bound (RGBA8: the f64 value rounded, or a neighbour where the bound straddles a step)."""
import ctypes as C

import numpy as np
import pytest

import blend_f64 as BF

pytestmark = pytest.mark.gpu

SIZES = [(1000, 600), (2600, 1500)]      # 16-px fine tiles (4 warps per tile) and 32-px fine tiles (16 warps per tile)
FORMATS = ["rgba8", "rgba32f"]


def _fmt(N, name):
    return N.GS_FRAME_RGBA8 if name == "rgba8" else N.GS_FRAME_RGBA32F


_scenes = {}


def _viewer(w, h, n=200_000):
    from gaussiansplats3d_b200.scenes import CAMERAS, synthetic_scene
    from gaussiansplats3d_b200.viewer import Viewer
    if n not in _scenes:
        _scenes[n] = synthetic_scene(n, seed=7, kind="bonsai", sh_degree=1)
    c = CAMERAS["bonsai"]
    v = Viewer(dict(cameraUp=c["up"], initialCameraPosition=c["position"], initialCameraLookAt=c["look_at"], width=w, height=h,
                    sphericalHarmonicsDegree=1))
    v.addSplatScene(_scenes[n])
    v.update()
    return v


def _pattern(h, w, fmt_name, seed=0):
    """An opaque, patterned background: 8-px checks of two colours with some noise, alpha 1."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    check = (((yy >> 3) + (xx >> 3)) & 1).astype(np.float32)[..., None]
    c = check * np.float32([0.9, 0.3, 0.1, 1.0]) + (1 - check) * np.float32([0.1, 0.5, 0.8, 1.0])
    c[..., :3] += rng.random((h, w, 3), dtype=np.float32) * 0.1
    c = np.clip(c, 0, 1).astype(np.float32)
    return np.floor(c * 255 + 0.5).astype(np.uint8) if fmt_name == "rgba8" else c


def _zw(proj):
    drawn = proj["valid"] == 1
    return (np.float32(0.5) * proj["ndc_z"][drawn] + np.float32(0.5)).astype(np.float32)


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("fmt_name", FORMATS)
def test_noop_inputs_and_full_occlusion(gs, w, h, fmt_name):
    N = gs._native
    fmt = _fmt(N, fmt_name)
    v = _viewer(w, h)
    plain = v.render(frame_format=fmt, flip_y=False)
    assert plain[..., 3].max() > 0
    zero = np.zeros((h, w, 4), plain.dtype)
    noop = v.render(frame_format=fmt, flip_y=False, dest_color=zero, dest_depth=np.ones((h, w), np.float32))
    assert np.array_equal(noop.view(np.uint8), plain.view(np.uint8)), "depth 1 over a zero background must be the plain frame, bit for bit"
    proj = v.engine.read_projected(v.splatMesh.getSplatCount())
    assert (_zw(proj) > 0).all()         # no splat on the near plane, so depth 0 hides every one
    bg = _pattern(h, w, fmt_name)
    occluded = v.render(frame_format=fmt, flip_y=False, dest_color=bg, dest_depth=np.zeros((h, w), np.float32))
    assert np.array_equal(occluded, bg)
    # NaN depth passes nothing; depth alone (no colour) composites over (0, 0, 0, 0)
    nan = v.render(frame_format=fmt, flip_y=False, dest_color=bg, dest_depth=np.full((h, w), np.nan, np.float32))
    assert np.array_equal(nan, bg)
    depth_only = v.render(frame_format=fmt, flip_y=False, dest_depth=np.ones((h, w), np.float32))
    assert np.array_equal(depth_only.view(np.uint8), plain.view(np.uint8))
    v.dispose()


def _tilted_plane(proj, w, h, cover=0.75):
    """Depth of a plane that rises across x from the 5th to the 95th percentile of the splats' window depths, over the left `cover`
    of the frame; the rest is the cleared depth buffer (1.0)."""
    z = _zw(proj)
    lo, hi = np.quantile(z, 0.05), np.quantile(z, 0.95)
    xs = (np.arange(w, dtype=np.float32) + 0.5) / w
    row = (lo + (hi - lo) * xs / cover).astype(np.float32)
    d = np.broadcast_to(row, (h, w)).copy()
    d[:, xs >= cover] = 1.0
    return d, xs >= cover


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("fmt_name", FORMATS)
def test_tilted_plane_matches_the_composite_oracle(gs, w, h, fmt_name):
    N = gs._native
    fmt = _fmt(N, fmt_name)
    v = _viewer(w, h)
    n = v.splatMesh.getSplatCount()
    plain = v.render(frame_format=fmt, flip_y=False)
    proj = v.engine.read_projected(n)
    order, _ = v.engine.sort(v.mvp_matrix().astype(np.float32), n, n, None)
    depth, uncovered = _tilted_plane(proj, w, h)
    bg = _pattern(h, w, fmt_name, seed=1)
    bg[:, uncovered] = 0                 # the opaque pass covers only where its depth was written
    got = v.render(frame_format=fmt, flip_y=False, dest_color=bg, dest_depth=depth)
    res = BF.restate(BF.read_records(v.engine, n), order, w, h, dest_color=bg, dest_depth=depth)
    BF.check(f"tilted plane {w}x{h} {fmt_name}", res, None if fmt_name == "rgba8" else got, got if fmt_name == "rgba8" else None)
    # the plane hides some splats and shows others: under it, some pixels are the background (every splat hidden), some are what the
    # same background shows with no depth test (every splat drawn), and many are neither
    covered = ~uncovered
    all_pass = v.render(frame_format=fmt, flip_y=False, dest_color=bg)
    hidden = np.all(got[:, covered] == bg[:, covered], axis=-1).mean()
    drawn = np.all(got[:, covered] == all_pass[:, covered], axis=-1).mean()
    assert hidden > 0.001 and drawn > 0.001 and hidden + drawn < 0.99, (hidden, drawn)
    # where the plane does not reach and the background is zero, the frame is the plain frame bit for bit: in every 8x8 block that lies
    # wholly there (a warp composites until ALL of its block's pixels are saturated, so a block that straddles the plane's edge keeps
    # adding below-cutoff contributions where the plain frame had stopped)
    x0 = -(-int(np.argmax(uncovered)) // 8) * 8
    assert uncovered[x0:].all() and x0 < w
    assert np.array_equal(got[:, x0:].view(np.uint8), plain[:, x0:].view(np.uint8))
    v.dispose()


def test_host_and_device_inputs_and_row_order(gs):
    import torch
    N = gs._native
    w, h = 1000, 600
    v = _viewer(w, h)
    n = v.splatMesh.getSplatCount()
    v.render(frame_format=N.GS_FRAME_RGBA8, flip_y=False)
    depth, _ = _tilted_plane(v.engine.read_projected(n), w, h)
    for fmt_name in FORMATS:
        fmt = _fmt(N, fmt_name)
        bg = _pattern(h, w, fmt_name, seed=2)
        host = v.render(frame_format=fmt, flip_y=False, dest_color=bg, dest_depth=depth)
        dev = v.render(frame_format=fmt, flip_y=False, dest_color=torch.from_numpy(bg).cuda(), dest_depth=torch.from_numpy(depth).cuda())
        assert np.array_equal(host, dev)
        mixed = v.render(frame_format=fmt, flip_y=False, dest_color=bg, dest_depth=torch.from_numpy(depth).cuda())
        assert np.array_equal(host, mixed)
        flipped = v.render(frame_format=fmt, flip_y=True, dest_color=bg[::-1].copy(), dest_depth=depth[::-1].copy())
        assert np.array_equal(flipped, host[::-1])
        with pytest.raises(ValueError):     # the colour of an RGBA8 frame is bytes, of an RGBA32F frame floats
            v.render(frame_format=fmt, flip_y=False, dest_color=bg.astype(np.float32 if fmt_name == "rgba8" else np.uint8))
        with pytest.raises(ValueError):
            v.render(frame_format=fmt, flip_y=False, dest_depth=depth[:, :-1])
    v.dispose()


def test_pipelined_and_async_frames_use_their_own_inputs(gs):
    """frame_begin / frame_end (two and three frames in flight) and frame_async, with a different depth and colour per frame and plain
    frames in between, deliver exactly what the blocking frame delivers for the same inputs."""
    N = gs._native
    w, h = 640, 360
    v = _viewer(w, h, n=150_000)
    e = v.engine
    n = v.splatMesh.getSplatCount()
    v.render(frame_format=N.GS_FRAME_RGBA8, flip_y=False)
    base, _ = _tilted_plane(e.read_projected(n), w, h, cover=1.0)
    preps = []
    for k in range(6):
        v.camera.position = np.asarray(v.initialCameraPosition) + np.array([0.1 * k, -0.04 * k, 0.08 * k])
        v.camera.look_at(v.initialCameraLookAt)
        v.camera.update(); v.updateSplatMesh()
        kw = {}
        if k % 3 != 1:        # frames 1 and 4 are plain
            kw = dict(dest_color=_pattern(h, w, "rgba8", seed=10 + k), dest_depth=(base if k % 2 else base[:, ::-1].copy()) + np.float32(0.01 * k))
        preps.append(e.prepare_frame(v.mvp_matrix().astype(np.float32), v.uniforms(), w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=True, **kw))
    want = []
    for prep in preps:
        out = N.pinned_empty((h, w, 4), np.uint8)
        e.frame_prepared(prep, out)
        want.append(out.copy())
    assert len({x.tobytes() for x in want}) == len(want)
    for depth_in_flight in (2, 3):
        bufs = [N.pinned_empty((h, w, 4), np.uint8) for _ in range(depth_in_flight)]
        got = []
        for i in range(depth_in_flight - 1):
            e.frame_begin(preps[i], bufs[i])
        for i in range(len(preps)):
            j = i + depth_in_flight - 1
            if j < len(preps):
                e.frame_begin(preps[j], bufs[j % depth_in_flight])
            e.frame_end()
            got.append(bufs[i % depth_in_flight].copy())
        for i, (a, b) in enumerate(zip(got, want)):
            assert np.array_equal(a, b), f"{depth_in_flight}-deep pipelined frame {i} differs"
    for k in range(len(preps)):        # asynchronous frames: the last one enqueued is the one left in the frame buffer
        e.frame_async(None, None, w, h, n, prepared=preps[(k + 3) % len(preps)])
        e.frame_async(None, None, w, h, n, prepared=preps[k])
        e.synchronize()
        got = e.read_buffer(N.GS_BUF_FRAME, np.uint8, h * w * 4).reshape(h, w, 4)
        assert np.array_equal(got, want[k]), f"asynchronous frame {k} differs"
    v.dispose()


def test_bad_arguments(gs):
    N = gs._native
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    w, h, n = 320, 200, 20_000
    v = _viewer(w, h, n=n)
    e = v.engine
    unif = v.uniforms()
    u = unif.to_c()
    depth = np.ones((h, w), np.float32)
    color = np.zeros((h, w, 4), np.float32)
    order = np.arange(n, dtype=np.uint32)
    for host_field, host_arr in (("dest_depth", depth), ("dest_color", color)):
        p, keep = e._render_params(w, h, n, order, N.GS_FRAME_RGBA32F, False)
        setattr(p, host_field, N.ptr(host_arr))
        setattr(p, host_field + "_dev", e.buffer_dev(N.GS_BUF_FRAME)[0])
        rc = e._lib.gs_render(e._h, C.byref(u), C.byref(p), None)
        assert rc == N.GS_ERR_BAD_ARG, (host_field, rc)
        assert b"not both" in e._lib.gs_last_error_message()
    v.dispose()
    p = pack_scene(synthetic_scene(n, seed=7, kind="bonsai"))
    with Engine(n, max_width=w, max_height=h, rank=0, world_size=2) as e2:
        e2.upload_splat_data(p.centers_colors, p.covariances)
        for kw in (dict(dest_depth=depth), dict(dest_color=color)):
            with pytest.raises(N.GsError) as ei:
                e2.render(unif, w, h, n, order, **kw)
            assert ei.value.code == N.GS_ERR_BAD_ARG and "single-GPU" in str(ei.value)


def test_viewer_render_and_frame_reach_the_engine(gs):
    N = gs._native
    w, h = 480, 270
    v = _viewer(w, h, n=50_000)
    bg = _pattern(h, w, "rgba8", seed=3)
    zero_depth = np.zeros((h, w), np.float32)
    assert np.array_equal(v.render(frame_format=N.GS_FRAME_RGBA8, flip_y=True, dest_color=bg, dest_depth=zero_depth), bg)
    assert np.array_equal(v.frame(frame_format=N.GS_FRAME_RGBA8, flip_y=True, dest_color=bg, dest_depth=zero_depth), bg)
    plain = v.frame(frame_format=N.GS_FRAME_RGBA8, flip_y=True)
    over = v.frame(frame_format=N.GS_FRAME_RGBA8, flip_y=True, dest_color=bg)
    assert not np.array_equal(plain, over) and not np.array_equal(over, bg)
    v.dispose()
