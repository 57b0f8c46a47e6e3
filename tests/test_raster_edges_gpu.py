"""GPU: the rasteriser's edge paths, compared with the oracle's blend of the GPU's OWN projected records (Engine.read_projected ->
oracle.blend / blend_crop in the same draw order).  The projection is tested on its own (test_raster_gpu.test_projection_matches_vertex_shader);
taking it out of the comparison leaves binning and blend, whose only legitimate differences from the f32 oracle are ex2.approx / log2f
against expf, the order of the FMAs, front-to-back against back-to-front compositing, the 1/512 transmittance cutoff (< 0.5/255) and
coverage flips where q = A/8 is within rounding of 1.  Hence the blend-only tolerance, stated once here:
  * every channel of a pixel OUTSIDE the oracle's coverage-boundary map within 1/255 (RGBA32F), and within one step of the oracle's
    frame rounded to 8 bits (RGBA8).  The map (blend(..., flags=True)) marks pixels where splats with a >= 1/255 and |A/8 - 1| <= 4e-3
    could move the pixel by more than 1/4 step if their coverage flipped (transmittance in front x a x e^-4, summed);
  * channels of flagged pixels within 8/255 (9 steps in RGBA8);
  * at most 10 % of the covered pixels flagged, so that the exemption cannot swallow the comparison.  (Every layer of splats puts about
    0.8 % of the pixels it covers within 4e-3 of its q = 1 contour, so a cap of 1 % would only admit scenes one layer deep.)
A dropped splat, a block skipped by the ellipse mask, a missing fine-tile column or an early stop moves unflagged channels by more.
Every test also asserts, from the exported records, that the branch it is about really ran.  Each case prints its worst unflagged and
flagged error (pytest -s)."""
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

UNFLAGGED, FLAGGED, MAX_FLAGGED_FRAC = 1.0 / 255, 8.0 / 255, 0.10
UNFLAGGED8, FLAGGED8 = 1, 9


# ---- scenes and cameras -------------------------------------------------------------------------------------------------------------
def _splats(centers, scales, alpha, rng):
    """centres_colours + covariances of splats with the given centres, per-axis scales and 8-bit alphas; random rotations and colours."""
    from gaussiansplats3d_b200.scenes import compute_covariances, pack_centers_colors
    n = centers.shape[0]
    q = rng.normal(0, 1, (n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    colors = np.empty((n, 4), np.uint8)
    colors[:, :3] = rng.integers(0, 256, (n, 3))
    colors[:, 3] = alpha
    centers = np.asarray(centers, np.float32)
    return pack_centers_colors(centers, colors), compute_covariances(np.asarray(scales, np.float32), q.astype(np.float32)), centers


def _cloud(n, seed, sigma=3.0):
    from gaussiansplats3d_b200.scenes import pack_scene, synthetic_scene
    raw = synthetic_scene(n, seed=seed, kind="uniform")
    raw.centers *= np.float32(sigma / 3.0)
    p = pack_scene(raw)
    return p.centers_colors, p.covariances, raw.centers


def _cat(*scenes):
    return tuple(np.concatenate(parts, 0) for parts in zip(*scenes))


def _camera(w, h, pos, look, up=(0.0, 1.0, 0.0), fov=50.0, near=0.1, far=1000.0, **kw):
    """Uniforms of a three.js PerspectiveCamera (as Viewer.uniforms builds them), its model-view matrix and MVP (column-major)."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    cam = TM.PerspectiveCamera(fov, w / h, near, far)
    cam.position = np.asarray(pos, np.float64)
    cam.up = np.asarray(up, np.float64)
    cam.look_at(look)
    P, mv = cam.projectionMatrix, cam.matrixWorldInverse
    u = Uniforms(model_view=mv.astype(np.float32), projection=P.astype(np.float32), camera_position=cam.position.astype(np.float32),
                 focal=(P[0] * 0.5 * w, P[5] * 0.5 * h), viewport=(w, h), **kw)
    return u, mv, TM.multiply(P, mv).astype(np.float32)


def _view_z(centers, mv):
    m = np.asarray(mv, np.float64).reshape(4, 4).T
    return centers.astype(np.float64) @ m[2, :3] + m[2, 3]


def _back_to_front(centers, mv, idx=None):
    """Draw order: farthest (most negative view z) first."""
    idx = np.arange(centers.shape[0]) if idx is None else np.asarray(idx)
    return idx[np.argsort(_view_z(centers[idx], mv), kind="stable")].astype(np.uint32)


def _engine(n, w, h, cc, cov):
    from gaussiansplats3d_b200.engine import Engine
    e = Engine(n, max_width=w, max_height=h)
    e.upload_splat_data(cc, cov)
    return e


# ---- what the GPU binned: host restatement of k_project's pixel rects ---------------------------------------------------------------
def _tile_shift(w, h):
    """frame_tile_shift: 16-px tiles while the frame has at most 256 coarse tiles of 128x64 px, else 32 px."""
    return 4 if -(-w // 128) * -(-h // 64) <= 256 else 5


def _pixel_rects(ps, w, h):
    """Pixel rect [x0, x1] x [y0, y1] of every splat's AABB clipped to the frame, and whether it is non-empty (k_project's rect)."""
    b1x, b1y, b2x, b2y = (ps[k].astype(np.float32) for k in ("b1x", "b1y", "b2x", "b2y"))
    hx = np.sqrt(b1x * b1x + b2x * b2x) * np.float32(1.0005) + np.float32(0.01)
    hy = np.sqrt(b1y * b1y + b2y * b2y) * np.float32(1.0005) + np.float32(0.01)
    cx, cy = ps["cx"].astype(np.float32), ps["cy"].astype(np.float32)
    fx0, fx1 = np.ceil(cx - hx - np.float32(0.5)), np.floor(cx + hx - np.float32(0.5))
    fy0, fy1 = np.ceil(cy - hy - np.float32(0.5)), np.floor(cy + hy - np.float32(0.5))
    ok = (ps["valid"] == 1) & (fx1 >= 0) & (fy1 >= 0) & (fx0 <= w - 1) & (fy0 <= h - 1) & (fx0 <= fx1) & (fy0 <= fy1)
    r = np.stack([np.clip(fx0, 0, w - 1), np.clip(fy0, 0, h - 1), np.clip(fx1, 0, w - 1), np.clip(fy1, 0, h - 1)], 1)
    return np.where(ok[:, None], r, 0).astype(np.int64), ok


def _coarse_spans(ps, w, h, tile_shift):
    """Coarse tiles (8 x 4 fine tiles) each splat's rect touches: the tile-instance count of the binning."""
    r, ok = _pixel_rects(ps, w, h)
    t = r >> tile_shift
    n = ((t[:, 2] >> 3) - (t[:, 0] >> 3) + 1) * ((t[:, 3] >> 2) - (t[:, 1] >> 2) + 1)
    return np.where(ok, n, 0)


# ---- blend-only comparison ----------------------------------------------------------------------------------------------------------
def _windows(w, h, ww=256, wh=128):
    """Corners (including the last, possibly partial, tile row and column) and centre of a large frame."""
    ww, wh = min(ww, w), min(wh, h)
    xs, ys = (0, (w - ww) // 2 // 8 * 8, w - ww), (0, (h - wh) // 2 // 8 * 8, h - wh)
    return sorted({(x, y, ww, wh) for x in xs for y in ys})


def _check_blend(oracle_mod, label, got, ps, order, w, h, *, got8=None, windows=None):
    """Compare a GPU frame (rows bottom-up) with the oracle's blend of the GPU's records at the blend-only tolerance.  Returns the
    number of covered pixels compared."""
    regions = [(0, 0, w, h)] if windows is None else windows
    wu = wf = 0.0
    w8u = w8f = 0
    nflag = ncov = 0
    for (x0, y0, ww, wh) in regions:
        if windows is None:
            want, flags = oracle_mod.blend(ps, order, w, h, flags=True)
        else:
            want, flags = oracle_mod.blend_crop(ps, order, w, h, x0, y0, ww, wh, flags=True)
        g = got[y0:y0 + wh, x0:x0 + ww].astype(np.float64)
        err = np.abs(g - want)
        fl = np.broadcast_to(flags[..., None], err.shape)
        wu, wf = max(wu, float(err[~fl].max(initial=0.0))), max(wf, float(err[fl].max(initial=0.0)))
        covered = (want[..., 3] > 0) | (g[..., 3] > 0)
        nflag += int((flags & covered).sum())
        ncov += int(covered.sum())
        if got8 is not None:
            want8 = np.floor(np.clip(want, 0.0, 1.0) * 255.0 + 0.5).astype(np.int32)
            d8 = np.abs(got8[y0:y0 + wh, x0:x0 + ww].astype(np.int32) - want8)
            w8u, w8f = max(w8u, int(d8[~fl].max(initial=0))), max(w8f, int(d8[fl].max(initial=0)))
    frac = nflag / max(ncov, 1)
    print(f"\n[{label}] worst unflagged {wu * 255:.3f}/255, worst flagged {wf * 255:.3f}/255, flagged {100 * frac:.3f} % of {ncov} covered px"
          + (f"; RGBA8 worst unflagged {w8u}, flagged {w8f} steps" if got8 is not None else ""))
    assert wu <= UNFLAGGED, f"{label}: unflagged channel off by {wu * 255:.3f}/255"
    assert wf <= FLAGGED, f"{label}: flagged channel off by {wf * 255:.3f}/255"
    assert frac <= MAX_FLAGGED_FRAC, f"{label}: {100 * frac:.2f} % of covered pixels flagged"
    assert w8u <= UNFLAGGED8 and w8f <= FLAGGED8, (label, w8u, w8f)
    return ncov


def _render_both(e, u, w, h, order, n_records):
    """RGBA32F and RGBA8 frames (rows bottom-up) of one render, and the records of the RGBA32F one."""
    from gaussiansplats3d_b200 import _native as N
    rc = len(order)
    got = e.render(u, w, h, rc, order, frame_format=N.GS_FRAME_RGBA32F, flip_y=False).copy()
    ps = e.read_projected(n_records)
    got8 = e.render(u, w, h, rc, order, frame_format=N.GS_FRAME_RGBA8, flip_y=False).copy()
    return got, got8, ps


# ---- cases --------------------------------------------------------------------------------------------------------------------------
def test_huge_splats_and_size_clamp(gs, oracle_mod):
    """~2 K splats 0.3-3 units in front of the camera over a background cloud.  Splats whose rect spans more than 32 coarse tiles are
    walked by the whole warp in round_instances; at maxScreenSpaceSplatSize = 48 most near splats are clamped."""
    rng = np.random.default_rng(101)
    w, h = 1280, 720
    pos = np.array([0.0, 0.0, 10.0])
    m = 2000
    d = rng.uniform(0.3, 3.0, m)
    nx, ny = rng.uniform(-0.9, 0.9, m), rng.uniform(-0.9, 0.9, m)
    t = np.tan(np.deg2rad(25.0))
    near = np.stack([nx * t * (w / h) * d, ny * t * d, pos[2] - d], 1)
    s = np.exp(rng.uniform(np.log(0.004), np.log(0.3), m))[:, None] * np.exp(rng.uniform(-0.3, 0.3, (m, 3)))
    scene = _cat(_cloud(3000, seed=102), _splats(near, s, rng.integers(5, 121, m), rng))
    cc, cov, centers = scene
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    for max_size in (1024.0, 48.0):
        u, mv, _ = _camera(w, h, pos, (0.0, 0.0, 0.0), max_screen_space_splat_size=max_size)
        order = _back_to_front(centers, mv)
        got, got8, ps = _render_both(e, u, w, h, order, n)
        spans = _coarse_spans(ps, w, h, 4)
        vis = _pixel_rects(ps, w, h)[1]
        semi = np.hypot(ps["b1x"], ps["b1y"])
        if max_size > 100:
            assert (spans > 32).sum() >= 100, f"only {(spans > 32).sum()} splats span more than 32 coarse tiles"
        else:
            clamped = vis & (semi >= 48.0 * (1 - 1e-4))
            assert clamped.sum() >= 0.2 * vis.sum(), (clamped.sum(), vis.sum())
            assert semi[vis].max() <= 48.0 * (1 + 1e-4)
        _check_blend(oracle_mod, f"huge splats, max size {max_size:g}", got, ps, order, w, h, got8=got8)
    e.close()


def test_near_plane_and_guard_band(gs, oracle_mod):
    """Camera inside a uniform cloud, plus splats just behind and just beyond the near plane: splats behind the camera or in front of
    the near plane are culled, splats in the 1.2x guard band outside the frustum still draw their part of the ellipse."""
    rng = np.random.default_rng(201)
    w, h = 960, 540
    pos, look = np.zeros(3), np.array([1.0, 0.3, -2.0])
    u, mv, _ = _camera(w, h, pos, look)
    fwd = (look - pos) / np.linalg.norm(look - pos)
    m = np.asarray(mv, np.float64).reshape(4, 4).T
    right, up = m[0, :3], m[1, :3]
    t = np.tan(np.deg2rad(25.0))

    def in_frustum(k, d0, d1):
        d = rng.uniform(d0, d1, k)
        return pos + d[:, None] * (fwd + rng.uniform(-0.9, 0.9, (k, 1)) * t * (w / h) * right + rng.uniform(-0.9, 0.9, (k, 1)) * t * up)

    pts = np.concatenate([in_frustum(300, 0.1, 0.115), in_frustum(200, 0.03, 0.099)], 0)
    s = np.exp(rng.normal(-5.0, 0.5, (pts.shape[0], 3)))
    cc, cov, centers = _cat(_cloud(40_000, seed=202), _splats(pts, s, rng.integers(20, 256, pts.shape[0]), rng))
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    order = _back_to_front(centers, mv)
    got, got8, ps = _render_both(e, u, w, h, order, n)
    vz = _view_z(centers, mv)
    behind = vz > 0
    assert behind.sum() >= 50 and (ps["valid"][behind] == 0).all()
    before_near = (vz < 0) & (vz > -0.099)
    assert before_near.sum() >= 50 and (ps["valid"][before_near] == 0).all()
    valid = ps["valid"] == 1
    assert (valid & (ps["ndc_z"] < -0.9)).sum() >= 50, (valid & (ps["ndc_z"] < -0.9)).sum()
    ndcx, ndcy = ps["cx"] / (0.5 * w) - 1.0, ps["cy"] / (0.5 * h) - 1.0
    band = valid & ((np.abs(ndcx) > 1.0) | (np.abs(ndcy) > 1.0)) & (np.abs(ndcx) <= 1.2) & (np.abs(ndcy) <= 1.2)
    reach = band & _pixel_rects(ps, w, h)[1]
    assert reach.sum() >= 50, f"only {reach.sum()} guard-band splats reach the frame"
    _check_blend(oracle_mod, "near plane / guard band", got, ps, order, w, h, got8=got8)
    e.close()


SHAPES = [  # (w, h, fine-tile px, coarse tiles): what the frame must select
    (1, 1, 16, 1), (7, 5, 16, 1), (8, 8, 16, 1), (17, 9, 16, 1), (129, 65, 16, 4),
    (2048, 1024, 16, 256),          # the last 16-px frame of that shape
    (2049, 1024, 32, 72),           # the first 32-px frame
    (4096, 2048, 32, 256),          # the last frame of the counting-sort binning at 32 px
    (4097, 2049, 32, 289),          # radix-sorted binning + 32-px blend
    (7680, 4320, 32, 1020),
    (8192, 64, 16, 64),             # 512 fine tiles per row: k_bin_place without its compaction (pack_ok = 0)
]


@pytest.mark.parametrize("w,h,tile_px,ncoarse", SHAPES, ids=[f"{s[0]}x{s[1]}" for s in SHAPES])
def test_frame_shapes(gs, oracle_mod, w, h, tile_px, ncoarse):
    """Tiny and odd frames, both sides of the 16 / 32-px and counting-sort / radix switches, and a frame wider than 256 fine tiles.
    The GPU's tile-instance count must equal the host's count of coarse tiles touched at that tile size."""
    shift = _tile_shift(w, h)
    assert 1 << shift == tile_px
    tpx = 1 << shift
    assert -(-w // (8 * tpx)) * -(-h // (4 * tpx)) == ncoarse
    cc, cov, centers = _cloud(20_000, seed=301)
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    # tiny frames look through a narrow field of view: at 50 degrees every splat would be below the shader's size floor and culled
    u, mv, _ = _camera(w, h, (0.0, 0.0, 14.0), (0.0, 0.0, 0.0), fov=50.0 if min(w, h) >= 64 else 0.5)
    order = _back_to_front(centers, mv)
    got, got8, ps = _render_both(e, u, w, h, order, n)
    inst = e.timings()["tile_instances"]
    want_inst = int(_coarse_spans(ps, w, h, shift).sum())
    assert abs(inst - want_inst) <= 1e-3 * want_inst + 2, (inst, want_inst)
    big = w * h > 2_200_000
    ncov = _check_blend(oracle_mod, f"{w}x{h}", got, ps, order, w, h, got8=got8, windows=_windows(w, h) if big else None)
    assert ncov >= min(w * h // 2, 1000)
    assert got[..., 3].max() > 0
    e.close()


@pytest.mark.parametrize("count", [1, 2, 31, 33, 2047, 2048, 2049, 4097])
def test_render_counts(gs, oracle_mod, count):
    """Small and odd render counts around a warp (32), the binning's 2048-rank chunk and two chunks, drawn from 50 K uploaded splats."""
    rng = np.random.default_rng(400 + count)
    w, h = 640, 360
    cc, cov, centers = _cloud(50_000, seed=401, sigma=2.0)
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    u, mv, _ = _camera(w, h, (0.0, 0.0, 9.0), (0.0, 0.0, 0.0))
    vis = np.flatnonzero(np.abs(_view_z(centers, mv) + 9.0) < 4.0)
    order = _back_to_front(centers, mv, rng.choice(vis, count, replace=False))
    got, got8, ps = _render_both(e, u, w, h, order, n)
    assert (ps["valid"][order] == 1).sum() >= max(1, count // 2)
    ncov = _check_blend(oracle_mod, f"render count {count}", got, ps, order, w, h, got8=got8)
    assert ncov > 0
    e.close()


def test_subset_order_zero_count_and_culled_view(gs, oracle_mod):
    """A render order that is a random strict subset (60 %) of the uploaded splats; render_count = 0 and a view that culls everything
    give all-zero frames in both formats."""
    from gaussiansplats3d_b200 import _native as N
    rng = np.random.default_rng(501)
    w, h = 800, 450
    cc, cov, centers = _cloud(50_000, seed=502)
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    u, mv, _ = _camera(w, h, (0.0, 0.0, 14.0), (0.0, 0.0, 0.0))
    sub = rng.choice(n, int(0.6 * n), replace=False)
    order = _back_to_front(centers, mv, sub)
    got, got8, ps = _render_both(e, u, w, h, order, n)
    assert len(np.unique(order)) == len(order) < n
    _check_blend(oracle_mod, "60 % subset", got, ps, order, w, h, got8=got8)
    dummy = np.zeros(1, np.uint32)
    for fmt in (N.GS_FRAME_RGBA32F, N.GS_FRAME_RGBA8):
        assert not e.render(u, w, h, 0, dummy, frame_format=fmt, flip_y=False).any()
    away, mv_away, _ = _camera(w, h, (0.0, 0.0, 14.0), (0.0, 0.0, 28.0))
    for fmt in (N.GS_FRAME_RGBA32F, N.GS_FRAME_RGBA8):
        assert not e.render(away, w, h, n, _back_to_front(centers, mv_away), frame_format=fmt, flip_y=False).any()
    assert e.timings()["visible_splats"] == 0 and (e.read_projected(n)["valid"] == 0).all()
    e.close()


@pytest.mark.parametrize("zoom", [1.0, 2.5])
def test_orthographic(gs, oracle_mod, zoom):
    """orthographic_mode = 1 (three.js OrthographicCamera with a pixel-sized frustum, zoom 1 and 2.5): the projection stage against
    oracle.project at the tolerances of test_projection_matches_vertex_shader, and the frame at the blend-only tolerance."""
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    rng = np.random.default_rng(601)
    w, h = 800, 600
    m = 8000
    centers = np.stack([rng.normal(0, 150, m), rng.normal(0, 110, m), rng.normal(0, 80, m)], 1)
    s = np.exp(rng.uniform(np.log(0.4), np.log(6.0), (m, 1))) * np.exp(rng.uniform(-0.5, 0.5, (m, 3)))
    cc, cov, centers = _splats(centers, s, rng.integers(10, 256, m), rng)
    cam = TM.PerspectiveCamera(50, w / h, 0.1, 1000)
    cam.position = np.array([30.0, -20.0, 400.0])
    cam.look_at((0.0, 0.0, 0.0))
    proj = TM.make_orthographic(-w / 2, w / 2, h / 2, -h / 2, 0.1, 1000.0, zoom)
    u = Uniforms(model_view=cam.matrixWorldInverse.astype(np.float32), projection=proj.astype(np.float32), camera_position=cam.position.astype(np.float32),
                 focal=(1.0, 1.0), viewport=(w, h), ortho_zoom=zoom, orthographic_mode=1)
    e = _engine(m, w, h, cc, cov)
    order = _back_to_front(centers, cam.matrixWorldInverse)
    got, got8, ps = _render_both(e, u, w, h, order, m)
    want = oracle_mod.project(u, cc, cov)
    assert (ps["valid"] != want["valid"]).mean() < 1e-4
    ok = (ps["valid"] == 1) & (want["valid"] == 1)
    assert ok.sum() > 1000
    for k in ("cx", "cy"):
        assert np.abs(ps[k][ok] - want[k][ok]).max() < 2e-3, k

    def outer(p):
        return np.stack([p["b1x"] ** 2 + p["b2x"] ** 2, p["b1x"] * p["b1y"] + p["b2x"] * p["b2y"], p["b1y"] ** 2 + p["b2y"] ** 2], 1)[ok]
    qg, qw = outer(ps), outer(want)
    rel = np.abs(qg - qw).max(1) / np.maximum(np.abs(qw).max(1), 1e-6)
    assert np.quantile(rel, 0.999) < 2e-3 and rel.max() < 5e-2, (np.quantile(rel, 0.999), rel.max())
    for k in ("r", "g", "b", "a"):
        assert np.abs(ps[k][ok] - want[k][ok]).max() < 5e-4, k
    assert np.abs(ps["ndc_z"][ok] - want["ndc_z"][ok]).max() < 1e-4
    semi = np.sqrt(qw[:, 0] + qw[:, 2])
    assert np.median(semi) > 2.0 * zoom       # the zoom reaches the footprint (pixel-sized world units)
    _check_blend(oracle_mod, f"orthographic zoom {zoom:g}", got, ps, order, w, h, got8=got8)
    e.close()


def test_opaque_stacks(gs, oracle_mod):
    """3 K splats stacked over a 64x64-px region, opaque (alpha 255) interleaved with faint ones: blocks saturate partway through their
    lists, so the 1/512 cutoff decides where compositing stops; blocks get both odd and even record counts (null-record pairing)."""
    rng = np.random.default_rng(701)
    w, h = 320, 240
    u, mv, _ = _camera(w, h, (0.0, 0.0, 10.0), (0.0, 0.0, 0.0))
    f = 0.5 * h / np.tan(np.deg2rad(25.0))
    m = 3000
    px, py, d = rng.uniform(128, 192, m), rng.uniform(88, 152, m), rng.uniform(8.0, 12.0, m)
    r = rng.uniform(3.0, 12.0, m)
    centers = np.stack([(px - 0.5 * w) * d / f, (py - 0.5 * h) * d / f, 10.0 - d], 1)
    s = (r * d / f / np.sqrt(8.0))[:, None] * np.exp(rng.uniform(-0.2, 0.2, (m, 3)))
    alpha = np.where(np.arange(m) % 2 == 0, 255, rng.integers(2, 13, m))
    cc, cov, centers = _splats(centers, s, alpha, rng)
    e = _engine(m, w, h, cc, cov)
    order = _back_to_front(centers, mv)
    got, got8, ps = _render_both(e, u, w, h, order, m)
    # coverage of the region's 8x8-px blocks (pixel centres with q <= 1), per splat
    y, x = np.mgrid[80:160, 120:200].astype(np.float64) + 0.5
    b1 = np.stack([ps["b1x"], ps["b1y"]], 1).astype(np.float64)
    b2 = np.stack([ps["b2x"], ps["b2y"]], 1).astype(np.float64)
    dx, dy = x[None] - ps["cx"][:, None, None], y[None] - ps["cy"][:, None, None]
    qq = ((dx * b1[:, 0, None, None] + dy * b1[:, 1, None, None]) / (b1 * b1).sum(1)[:, None, None]) ** 2 + \
         ((dx * b2[:, 0, None, None] + dy * b2[:, 1, None, None]) / (b2 * b2).sum(1)[:, None, None]) ** 2
    touch = (qq <= 1.0).reshape(m, 10, 8, 10, 8).any(axis=(2, 4))       # [splat, block row, block col]
    counts = touch.sum(0)
    assert (counts % 2 == 1).any() and (counts[counts > 0] % 2 == 0).any(), counts
    # the nearer half of the draw order alone saturates some block below 1/512, and farther splats still reach it
    half = len(order) // 2
    front = oracle_mod.blend_crop(ps, order[half:], w, h, 120, 80, 80, 80)
    tmax = (1.0 - front[..., 3]).reshape(10, 8, 10, 8).max(axis=(1, 3))
    behind = touch[order[:half]].any(0)
    assert ((tmax < 1.0 / 512) & behind).any(), "no block saturates partway through its list"
    _check_blend(oracle_mod, "opaque stacks", got, ps, order, w, h, got8=got8)
    e.close()


@pytest.mark.parametrize("env,w,h", [
    ({"GS_BIN_COMPACT": "0"}, 1920, 1080), ({"GS_BIN_COMPACT": "0"}, 3840, 2160), ({"GS_BIN_COMPACT": "0"}, 8192, 64),
    ({"GS_BINCFG": "1"}, 1920, 1080), ({"GS_BINCFG": "1"}, 3840, 2160),
    ({"GS_BIN": "1"}, 1920, 1080), ({"GS_BIN": "1"}, 3840, 2160),
], ids=lambda v: "-".join(f"{k}={x}" for k, x in v.items()) if isinstance(v, dict) else str(v))
def test_binning_switches_are_bit_identical(gs, monkeypatch, env, w, h):
    """The binning A/B switches build the same per-tile lists in the same order as the default, so the frames (default blend) must be
    bit-identical in both formats."""
    from gaussiansplats3d_b200 import _native as N
    cc, cov, centers = _cloud(150_000, seed=801)
    n = centers.shape[0]
    u, mv, _ = _camera(w, h, (0.0, 0.0, 14.0), (0.0, 0.0, 0.0))
    order = _back_to_front(centers, mv)
    frames = {}
    for name, extra in (("default", {}), ("switched", env)):
        for k in ("GS_BIN_COMPACT", "GS_BINCFG", "GS_BIN", "GS_BLEND", "GS_BLEND_TMA", "GS_BLEND_ROUNDS", "GS_INSTANCE_FACTOR"):
            monkeypatch.delenv(k, raising=False)
        for k, v in extra.items():
            monkeypatch.setenv(k, v)
        e = _engine(n, w, h, cc, cov)
        frames[name] = [e.render(u, w, h, n, order, frame_format=fmt, flip_y=False).copy() for fmt in (N.GS_FRAME_RGBA8, N.GS_FRAME_RGBA32F)]
        frames[name].append(e.timings()["tile_instances"])
        e.close()
    assert frames["default"][0][..., 3].max() > 0
    assert frames["switched"][2] == frames["default"][2]
    assert np.array_equal(frames["switched"][0], frames["default"][0]), "RGBA8 frames differ"
    assert np.array_equal(frames["switched"][1], frames["default"][1]), "RGBA32F frames differ"


def _screen_fillers(m, seed, center=(0.0, 0.0, -2.0)):
    """m large splats in a ball of radius 0.2 about `center`: seen from 2 units away each covers (nearly) the whole frame."""
    rng = np.random.default_rng(seed)
    c = rng.normal(0, 1, (m, 3))
    c = 0.2 * c / np.linalg.norm(c, axis=1, keepdims=True) * rng.uniform(0, 1, (m, 1)) ** (1 / 3) + np.asarray(center)
    return _splats(c, rng.uniform(0.5, 1.0, (m, 3)), rng.integers(3, 40, m), rng)


def _needed(err):
    mt = re.search(r"(\d+) instances needed, capacity (\d+)", str(err))
    assert mt, str(err)
    return int(mt.group(1)), int(mt.group(2))


@pytest.mark.parametrize("scene", ["screen-filling", "small-factor"])
@pytest.mark.parametrize("env", [{}, {"GS_BIN": "1"}, {"GS_BLEND_TMA": "1"}], ids=["bin2", "bin1", "tma"])
def test_instance_overflow_reports_capacity_and_engine_recovers(gs, oracle_mod, monkeypatch, scene, env):
    """More tile instances than the list holds: (a) 1 000 screen-filling splats at the default capacity, (b) GS_INSTANCE_FACTOR=0.05 on
    an ordinary scene.  gs_render, gs_frame and gs_frame_begin/end each raise GsError(GS_ERR_CAPACITY) with the needed count, read only
    inside the list, and the same engine then renders a fitting frame exactly as a fresh engine does."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import integer_centers
    for k in ("GS_BIN", "GS_BLEND", "GS_BLEND_TMA", "GS_INSTANCE_FACTOR"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    w, h = 1920, 1080
    if scene == "screen-filling":
        cc, cov, centers = _screen_fillers(1000, seed=901)
        u, mv, mvp = _camera(w, h, (0.0, 0.0, 0.0), (0.0, 0.0, -1.0))
    else:
        monkeypatch.setenv("GS_INSTANCE_FACTOR", "0.05")
        cc, cov, centers = _cloud(300_000, seed=902)
        u, mv, mvp = _camera(w, h, (0.0, 0.0, 12.0), (0.0, 0.0, 0.0))
    n = centers.shape[0]
    order = _back_to_front(centers, mv)
    fit = order[-50:]                  # the 50 nearest splats fit any capacity

    def fresh_fit():
        with Engine(n, max_width=w, max_height=h) as f:
            f.upload_splat_data(cc, cov)
            return f.render(u, w, h, len(fit), fit, flip_y=False).copy()
    want_fit = fresh_fit()
    e = Engine(n, max_width=w, max_height=h)
    e.upload_splat_data(cc, cov)
    e.upload_centers(integer_centers(centers))
    buf = N.pinned_empty((h, w, 4), np.uint8)
    for path in ("render", "frame", "frame_begin"):
        with pytest.raises(N.GsError) as ei:
            if path == "render":
                e.render(u, w, h, n, order, flip_y=False)
            elif path == "frame":
                e.frame(mvp, u, w, h, n)
            else:
                e.frame_begin(e.prepare_frame(mvp, u, w, h, n), buf)
                e.frame_end()
        assert ei.value.code == N.GS_ERR_CAPACITY, str(ei.value)
        needed, cap = _needed(ei.value)
        assert needed > cap, (path, needed, cap)
        assert e.timings()["tile_instances"] == needed
        got = e.render(u, w, h, len(fit), fit, flip_y=False)
        assert np.array_equal(got, want_fit), f"{path}: the frame after the overflow differs from a fresh engine's"
    print(f"\n[overflow {scene} {env}] {needed} instances needed, capacity {cap}")
    if not env:
        _check_blend(oracle_mod, f"after overflow ({scene})", want_fit, e.read_projected(n), fit, w, h)
    e.close()


def test_engine_reuse_matches_fresh_engines(gs, monkeypatch):
    """One engine renders 4K RGBA8 -> 720p RGBA32F -> render_count 0 -> an overflowing frame -> a 1080p subset -> 1x1; every frame that
    succeeds is bit-identical to the same frame on a fresh engine (nothing of an earlier frame, or of the overflow, leaks)."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    for k in ("GS_BIN", "GS_BLEND", "GS_BLEND_TMA", "GS_INSTANCE_FACTOR", "GS_BIN_COMPACT", "GS_BINCFG"):
        monkeypatch.delenv(k, raising=False)
    rng = np.random.default_rng(1001)
    cloud = _cloud(50_000, seed=1002)
    fill = _screen_fillers(4000, seed=1003, center=(0.0, 0.0, -40.0))
    cc, cov, centers = _cat(cloud, fill)
    n, nc = centers.shape[0], cloud[2].shape[0]
    W, H = 3840, 2160
    frames = []
    for (w, h, fmt, pos, look, idx) in (
            (3840, 2160, N.GS_FRAME_RGBA8, (0.0, 0.0, 14.0), (0.0, 0.0, 0.0), np.arange(nc)),
            (1280, 720, N.GS_FRAME_RGBA32F, (3.0, 1.0, 13.0), (0.0, 0.0, 0.0), np.arange(nc)),
            (1920, 1080, N.GS_FRAME_RGBA8, (0.0, 0.0, 14.0), (0.0, 0.0, 0.0), np.arange(0)),
            (3840, 2160, N.GS_FRAME_RGBA8, (0.0, 0.0, -38.0), (0.0, 0.0, -40.0), np.arange(nc, n)),
            (1920, 1080, N.GS_FRAME_RGBA32F, (-2.0, 0.5, 12.0), (0.0, 0.0, 0.0), rng.choice(nc, int(0.6 * nc), replace=False)),
            (1, 1, N.GS_FRAME_RGBA32F, (0.0, 0.0, 14.0), (0.0, 0.0, 0.0), np.arange(nc))):
        u, mv, _ = _camera(w, h, pos, look)
        order = _back_to_front(centers, mv, idx) if len(idx) else np.zeros(1, np.uint32)
        frames.append((u, w, h, len(idx), order, fmt))
    e = Engine(n, max_width=W, max_height=H)
    e.upload_splat_data(cc, cov)
    got = []
    for i, (u, w, h, rc, order, fmt) in enumerate(frames):
        if i == 3:
            with pytest.raises(N.GsError) as ei:
                e.render(u, w, h, rc, order, frame_format=fmt, flip_y=False)
            assert ei.value.code == N.GS_ERR_CAPACITY and _needed(ei.value)[0] > _needed(ei.value)[1]
            got.append(None)
        else:
            got.append(e.render(u, w, h, rc, order, frame_format=fmt, flip_y=False).copy())
    e.close()
    assert got[0][..., 3].max() > 0 and not got[2].any()
    for i, (u, w, h, rc, order, fmt) in enumerate(frames):
        if got[i] is None:
            continue
        with Engine(n, max_width=W, max_height=H) as f:
            f.upload_splat_data(cc, cov)
            assert np.array_equal(f.render(u, w, h, rc, order, frame_format=fmt, flip_y=False), got[i]), f"frame {i} differs from a fresh engine's"
