"""GPU: the rasteriser's edge paths, held against the f64 restatement of the blend of the GPU's OWN raw projected records
(tests/blend_f64.py, Engine.read_buffer(GS_BUF_SPLAT_RECORDS) in the same draw order).  The projection is tested on its own
(test_projection_gpu.py, test_raster_gpu.test_projection_matches_vertex_shader); taking it out of the comparison leaves binning and blend.
The restatement finds which splats reach each 8x8 block from its own f64 extents, so a record lost by the rects, the half-precision
extents, the tile masks or the block masks is an error.  The tolerance, stated once here: every channel of every pixel within its own
bound (rounding of the kernel's operation sequence, terms whose q is within rounding of 1, and the early stop below the 1/512
transmittance cutoff), nothing exempt; in RGBA8 the byte is the f64 value rounded, or either neighbour where the bound straddles a
rounding boundary.  Every test also asserts, from the exported records, that the branch it is about really ran.  Each case prints its
worst |error|/bound and its share of pixels with an ambiguous term (pytest -s)."""
import re

import numpy as np
import pytest

import blend_f64 as BF
import frame_f64 as FF

pytestmark = pytest.mark.gpu


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


# ---- frames ------------------------------------------------------------------------------------------------------------------------
def _tile_shift(w, h):
    """frame_tile_shift: 16-px tiles while the frame has at most 256 coarse tiles of 128x64 px, else 32 px."""
    return 4 if -(-w // 128) * -(-h // 64) <= 256 else 5


def _render_both(e, u, w, h, order, n_records, flip_y=False):
    """RGBA32F and RGBA8 frames of one render, and the exported (read_projected) and raw records of the RGBA32F one."""
    from gaussiansplats3d_b200 import _native as N
    rc = len(order)
    got = e.render(u, w, h, rc, order, frame_format=N.GS_FRAME_RGBA32F, flip_y=flip_y).copy()
    ps, rec = e.read_projected(n_records), BF.read_records(e, n_records)
    got8 = e.render(u, w, h, rc, order, frame_format=N.GS_FRAME_RGBA8, flip_y=flip_y).copy()
    return got, got8, ps, rec


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
        got, got8, ps, rec = _render_both(e, u, w, h, order, n)
        spans = FF.coarse_spans(ps, w, h, 4)
        vis = FF.pixel_rects(ps, w, h)[1]
        semi = np.hypot(ps["b1x"], ps["b1y"])
        if max_size > 100:
            assert (spans > 32).sum() >= 100, f"only {(spans > 32).sum()} splats span more than 32 coarse tiles"
        else:
            clamped = vis & (semi >= 48.0 * (1 - 1e-4))
            assert clamped.sum() >= 0.2 * vis.sum(), (clamped.sum(), vis.sum())
            assert semi[vis].max() <= 48.0 * (1 + 1e-4)
        FF.check_blend(f"huge splats, max size {max_size:g}", got, rec, order, w, h, got8=got8)
    e.close()


def _extents(rec):
    """Exact half extents of each record's ellipse q <= 1, from its g1, g2 (f64)."""
    g1x, g1y, g2x, g2y = (rec[k].astype(np.float64) for k in ("g1x", "g1y", "g2x", "g2y"))
    det = (g1x * g2y - g1y * g2x) ** 2
    return np.sqrt((g1y ** 2 + g2y ** 2) / det), np.sqrt((g1x ** 2 + g2x ** 2) / det)


def test_axis_aligned_edges_on_pixel_centres(gs):
    """Axis-aligned splats (orthographic, 1 world unit = 1 px) whose AABB edge lies within 1e-3 px outside a column or row of pixel
    centres, at the first or last column / row of a 32-px fine tile, with the splat's centre on the perpendicular row / column: the
    edge pixel is covered with q just below 1 and is the only pixel of its tile and block the splat reaches, so a rect, a
    half-precision extent or a block mask that comes up short drops it.  Also three ~600-px-wide splats whose f32 extent plus margin lies less than half a half-precision step
    above a half value, with the edge pixel 0.05 px inside: only the round-up of hx to half precision keeps that pixel's block."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.engine import Uniforms
    from gaussiansplats3d_b200.scenes import compute_covariances, pack_centers_colors
    w, h = 7680, 4320
    rng = np.random.default_rng(1801)
    cam = TM.PerspectiveCamera(50, w / h, 0.1, 1000)
    cam.position = np.array([0.0, 0.0, 400.0])
    cam.look_at((0.0, 0.0, 0.0))
    u = Uniforms(model_view=cam.matrixWorldInverse.astype(np.float32), projection=TM.make_orthographic(-w / 2, w / 2, h / 2, -h / 2, 0.1, 1000.0, 1.0).astype(np.float32),
                 camera_position=cam.position.astype(np.float32), focal=(1.0, 1.0), viewport=(w, h), ortho_zoom=1.0, orthographic_mode=1)
    # small splats on a grid of 32-px tiles in the upper part of the frame; kind: 0 right, 1 left, 2 top, 3 bottom edge
    m = 160
    kind = np.arange(m) % 4
    tx, ty = 4 + 5 * (np.arange(m) % 46), 55 + 3 * (np.arange(m) // 46)
    sx = np.exp(rng.uniform(np.log(1.0), np.log(8.0), m))
    sy = sx * np.exp(rng.uniform(0.05, 0.7, m))                       # sy > sx: k_project's eigenbasis stays axis-aligned
    eps = rng.uniform(1e-4, 6e-4, m)                                  # the edge this far outside the pixel centre
    # three wide splats: f32 extent + margin t = G + 0.41 above a half value G (spacing 0.5 there), exact extent h = G + 0.1
    G = np.array([520.0, 600.0, 700.0])
    hw = G + 0.1
    sxw = np.sqrt(hw ** 2 / 8.0 - 0.3)
    scales = np.concatenate([np.stack([sx, sy, np.ones(m)], 1), np.stack([sxw, sxw * 1.1, np.ones(3)], 1)])
    n = m + 3
    pos = np.zeros((n, 3))
    q = np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)).astype(np.float32)
    colors = np.empty((n, 4), np.uint8)
    colors[:, :3] = rng.integers(60, 256, (n, 3))
    colors[:, 3] = 255
    cov = compute_covariances(scales.astype(np.float32), q)
    e = _engine(n, w, h, pack_centers_colors(pos.astype(np.float32), colors), cov)
    order = np.arange(n, dtype=np.uint32)
    for _ in range(3):            # place each edge: pixel offsets move the record's centre one to one (orthographic, zoom 1)
        e.render(u, w, h, n, order)
        rec = BF.read_records(e, n)
        hx, hy = _extents(rec)
        want = np.empty((n, 2))
        for i in range(m):
            x0, y0 = 32 * tx[i], 32 * ty[i]
            if kind[i] == 0:   want[i] = (x0 + 0.5 + eps[i] - hx[i], y0 + 16.5)          # right edge at the tile's first column
            elif kind[i] == 1: want[i] = (x0 + 31.5 - eps[i] + hx[i], y0 + 16.5)         # left edge at the tile's last column
            elif kind[i] == 2: want[i] = (x0 + 16.5, y0 + 0.5 + eps[i] - hy[i])          # top edge at the tile's first row
            else:              want[i] = (x0 + 16.5, y0 + 31.5 - eps[i] + hy[i])         # bottom edge at the tile's last row
        for j in range(3):                                                              # right edge pixel 0.05 px inside
            want[m + j] = (32 * (40 + 60 * j) + 0.5 + 0.05 - hx[m + j], 700.5)
        pos[:, :2] += want - np.stack([rec["cx"], rec["cy"]], 1)
        e.upload_splat_data(pack_centers_colors(pos.astype(np.float32), colors), cov)
    got, got8, ps, rec = _render_both(e, u, w, h, order, n)
    hx, hy = _extents(rec)
    assert (ps["valid"] == 1).all() and np.abs(rec["g1x"] * rec["g1y"]).max() == 0.0     # drawn, axis-aligned
    edge = np.where(kind == 0, rec["cx"][:m] + hx[:m], np.where(kind == 1, rec["cx"][:m] - hx[:m],
                    np.where(kind == 2, rec["cy"][:m] + hy[:m], rec["cy"][:m] - hy[:m])))
    off = np.abs(edge - (np.round(edge - 0.5) + 0.5))
    assert (off <= 1e-3).all(), off.max()
    across = np.where(kind < 2, rec["cy"][:m], rec["cx"][:m])
    assert np.abs(across - 0.5 - np.round(across - 0.5)).max() <= 1e-3
    # the wide ones: the edge pixel lies beyond the f32 extent + margin rounded DOWN to half precision, inside the one rounded up
    t = (hx[m:].astype(np.float32) * np.float32(1.0005) + np.float32(0.01)).astype(np.float32)
    rd = np.float16(t).astype(np.float32)
    rd = np.where(rd > t, np.nextafter(np.float16(t), np.float16(-np.inf)).astype(np.float32), rd)
    dist = np.floor(rec["cx"][m:] + hx[m:] - 0.5) + 0.5 - rec["cx"][m:]
    assert (rd < dist).all() and (dist < hx[m:]).all(), (rd, dist, hx[m:])
    wins = [(int(x) // 8 * 8 - 16, int(y) // 8 * 8 - 16, 40, 40) for x, y in
            np.stack([np.where(kind < 2, edge, rec["cx"][:m]), np.where(kind < 2, rec["cy"][:m], edge)], 1)]
    wins += [(int(rec["cx"][m + j] + hx[m + j]) // 8 * 8 - 16, 688, 40, 40) for j in range(3)]
    FF.check_blend("axis-aligned edges on pixel centres", got, rec, order, w, h, got8=got8, windows=wins)
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
    got, got8, ps, rec = _render_both(e, u, w, h, order, n)
    vz = _view_z(centers, mv)
    behind = vz > 0
    assert behind.sum() >= 50 and (ps["valid"][behind] == 0).all()
    before_near = (vz < 0) & (vz > -0.099)
    assert before_near.sum() >= 50 and (ps["valid"][before_near] == 0).all()
    valid = ps["valid"] == 1
    assert (valid & (ps["ndc_z"] < -0.9)).sum() >= 50, (valid & (ps["ndc_z"] < -0.9)).sum()
    ndcx, ndcy = ps["cx"] / (0.5 * w) - 1.0, ps["cy"] / (0.5 * h) - 1.0
    band = valid & ((np.abs(ndcx) > 1.0) | (np.abs(ndcy) > 1.0)) & (np.abs(ndcx) <= 1.2) & (np.abs(ndcy) <= 1.2)
    reach = band & FF.pixel_rects(ps, w, h)[1]
    assert reach.sum() >= 50, f"only {reach.sum()} guard-band splats reach the frame"
    FF.check_blend("near plane / guard band", got, rec, order, w, h, got8=got8)
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
    """Tiny and odd frames, both sides of the 16 / 32-px and counting-sort / radix switches, and a frame wider than 256 fine tiles, with
    the frame's rows in either order.  The GPU's tile-instance count must equal the host's count of coarse tiles touched at that tile
    size; the coarse-tile count (asserted) selects the binning (radix above 256 coarse tiles)."""
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
    for flip_y in (False, True):
        got, got8, ps, rec = _render_both(e, u, w, h, order, n, flip_y)
        inst = e.timings()["tile_instances"]
        want_inst = int(FF.coarse_spans(ps, w, h, shift).sum())
        assert abs(inst - want_inst) <= 1e-3 * want_inst + 2, (inst, want_inst)
        big = w * h > 2_200_000
        ncov = FF.check_blend(f"{w}x{h} flip_y={flip_y}", got, rec, order, w, h, got8=got8, windows=FF.windows(w, h) if big else None, flip_y=flip_y)[0]
        assert ncov >= min(w * h // 2, 1000)
        assert got[..., 3].max() > 0
    e.close()


SCAN_BLOCK = 1024 * 2048       # k_bin_scan: chunks of 2048 draw ranks, scanned in blocks of 1024 threads with a running offset


@pytest.mark.parametrize("count", [1, 2, 31, 33, 2047, 2048, 2049, 4097, SCAN_BLOCK, SCAN_BLOCK + 1, 2_150_000])
def test_render_counts(gs, oracle_mod, count):
    """Small and odd render counts around a warp (32), the binning's 2048-rank chunk and two chunks, drawn from 50 K uploaded splats;
    and the last render count k_bin_scan covers with one block of 1024 chunks, the first that needs a second block (the running
    offset carried between blocks), and one whose second block holds 26 chunks, drawn from the 2.2 M splats in front of the camera."""
    rng = np.random.default_rng(400 + count)
    w, h = 640, 360
    cc, cov, centers = _cloud(50_000 if count < SCAN_BLOCK else 2_200_000, seed=401, sigma=2.0)
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    u, mv, _ = _camera(w, h, (0.0, 0.0, 9.0), (0.0, 0.0, 0.0))
    vis = np.flatnonzero(np.abs(_view_z(centers, mv) + 9.0) < (4.0 if count < SCAN_BLOCK else 9.0))
    order = _back_to_front(centers, mv, rng.choice(vis, count, replace=False))
    got, got8, ps, rec = _render_both(e, u, w, h, order, n)
    assert (ps["valid"][order] == 1).sum() >= max(1, count // 2)
    FF.check_frame(f"render count {count}", e, u, w, h, count, cc, cov, got=got, got8=got8, order=order)
    e.close()


def test_engine_sorted_frame_past_the_scan_block(gs, oracle_mod):
    """gs_frame over 2.2 M splats (more than one k_bin_scan block of 1024 x 2048 draw ranks) at 320x180: the order the frame drew is
    the reference sorter's, and the frame, in RGBA32F and RGBA8, passes the f64 checks."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.scenes import integer_centers
    w, h = 320, 180
    cc, cov, centers = _cloud(2_200_000, seed=401, sigma=2.0)
    n = centers.shape[0]
    assert n > SCAN_BLOCK
    e = _engine(n, w, h, cc, cov)
    ic = integer_centers(centers)
    e.upload_centers(ic)
    u, mv, mvp = _camera(w, h, (0.0, 0.0, 9.0), (0.0, 0.0, 0.0))
    got = e.frame(mvp, u, w, h, n, frame_format=N.GS_FRAME_RGBA32F, flip_y=False).copy()
    got8 = e.frame(mvp, u, w, h, n, frame_format=N.GS_FRAME_RGBA8, flip_y=False).copy()
    FF.check_frame("gs_frame 2.2 M splats", e, u, w, h, n, cc, cov, got=got, got8=got8, sort=dict(centers=ic, mvp=mvp), min_compared=n // 2)
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
    got, got8, ps, rec = _render_both(e, u, w, h, order, n)
    assert len(np.unique(order)) == len(order) < n
    FF.check_blend("60 % subset", got, rec, order, w, h, got8=got8)
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
    """orthographic_mode = 1 (three.js OrthographicCamera with a pixel-sized frustum, zoom 1 and 2.5): the projection stage (and
    oracle.project) within the per-splat f64 bounds of tests/projection_f64.py, and the frame within the f64 blend bounds."""
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
    got, got8, ps, rec = _render_both(e, u, w, h, order, m)
    import projection_f64 as PF
    hres = PF.project(u, cc, cov)
    rep = PF.compare(ps, hres)
    print("\n" + PF.format_report(f"orthographic zoom {zoom:g}", rep))
    PF.assert_within("GPU", rep, min_compared=1000)
    PF.assert_within("oracle", PF.compare(oracle_mod.project(u, cc, cov), hres), min_compared=1000)
    ok = hres["valid"] & ~hres["ambiguous"]
    semi = np.sqrt(hres["qxx"][ok] + hres["qyy"][ok])
    assert np.median(semi) > 2.0 * zoom       # the zoom reaches the footprint (pixel-sized world units)
    FF.check_blend(f"orthographic zoom {zoom:g}", got, rec, order, w, h, got8=got8)
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
    got, got8, ps, rec = _render_both(e, u, w, h, order, m)
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
    FF.check_blend("opaque stacks", got, rec, order, w, h, got8=got8)
    e.close()


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
@pytest.mark.parametrize("w,h", [(1920, 1080), (3840, 2160), (4097, 2049)], ids=["1920x1080", "3840x2160", "4097x2049"])
def test_instance_overflow_reports_capacity_and_engine_recovers(gs, oracle_mod, monkeypatch, scene, w, h):
    """More tile instances than the list holds: (a) 1 000 screen-filling splats at the default capacity, (b) GS_INSTANCE_FACTOR=0.05 on
    an ordinary scene.  gs_render, gs_frame and gs_frame_begin/end each raise GsError(GS_ERR_CAPACITY) with the needed count, read only
    inside the list, and the same engine then renders a fitting frame exactly as a fresh engine does.  1920x1080 (16-px tiles) and
    3840x2160 (32 px) bin by counting sort, 4097x2049 (289 coarse tiles) by the radix sort of the instances."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    from gaussiansplats3d_b200.scenes import integer_centers
    monkeypatch.delenv("GS_INSTANCE_FACTOR", raising=False)
    if scene == "screen-filling":
        cc, cov, centers = _screen_fillers(1000, seed=901)
        # without the default 1024-px size clamp the splats fill 4K frames too, not only 1080p ones
        u, mv, mvp = _camera(w, h, (0.0, 0.0, 0.0), (0.0, 0.0, -1.0), max_screen_space_splat_size=4096.0)
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
    print(f"\n[overflow {scene} {w}x{h}] {needed} instances needed, capacity {cap}")
    FF.check_blend(f"after overflow ({scene} {w}x{h})", want_fit, BF.read_records(e, n), fit, w, h)   # 50 splats: the whole frame is cheap
    e.close()


def test_engine_reuse_matches_fresh_engines(gs, monkeypatch):
    """One engine renders 4K RGBA8 -> 720p RGBA32F -> render_count 0 -> an overflowing frame -> a 1080p subset -> 1x1; every frame that
    succeeds is bit-identical to the same frame on a fresh engine (nothing of an earlier frame, or of the overflow, leaks)."""
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.engine import Engine
    monkeypatch.delenv("GS_INSTANCE_FACTOR", raising=False)
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
