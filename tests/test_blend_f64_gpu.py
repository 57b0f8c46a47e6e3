"""GPU: the blend pixel by pixel against the f64 restatement of its raw records (tests/blend_f64.py), every channel within its own bound,
in RGBA32F and RGBA8.  Cases: small splats far from the frame origin (where quad coordinates taken from the origin would round q by
up to ~4e-3 near its contour, the first-order bound), tile lists longer than one 512-entry batch, a field of faint splats, and
composites over every kind of destination depth.  Frame shapes, both tile sizes and binnings, both row orders and the constructed
edge cases are in tests/test_raster_edges_gpu.py, checked against the same bounds.  Each case asserts from the records and timings that its branch ran
and prints its worst |error|/bound and its share of ambiguous pixels (pytest -s)."""
import numpy as np
import pytest

import blend_f64 as BF
import frame_f64 as FF
from test_raster_edges_gpu import _back_to_front, _camera, _cat, _cloud, _engine, _render_both, _splats

pytestmark = pytest.mark.gpu


def test_small_splats_far_from_the_origin(gs):
    """kernel2DSize 0.1 and splatScale 0.25 at 7680x4320: splats of a pixel or less, |g| up to ~3 px^-1, thousands of pixels from the
    frame origin.  With quad coordinates taken from the origin the first-order bound on q's rounding near its contour is ~4e-3 there
    (~2e-3 emulated), far beyond the tile-relative bound."""
    w, h = 7680, 4320
    cc, cov, centers = _cloud(200_000, seed=1401, sigma=6.0)
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    u, mv, _ = _camera(w, h, (0.0, 0.0, 16.0), (0.0, 0.0, 0.0), kernel_2d_size=0.1, splat_scale=0.25)
    order = _back_to_front(centers, mv)
    got, got8, ps, rec = _render_both(e, u, w, h, order, n)
    vis = FF.pixel_rects(ps, w, h)[1]
    g = np.hypot(rec["g1x"], rec["g1y"])
    far = vis & (rec["cx"] > 4096) & (rec["cy"] > 2048)
    assert (far & (g > 1.0)).sum() >= 500 and g[vis].max() > 1.5 and far.sum() > 10_000, ((far & (g > 1.0)).sum(), g[vis].max(), far.sum())
    wins = [(w - 256, h - 128, 256, 128), (6528, 3664, 256, 128), (5120, 2816, 256, 128), (0, 0, 256, 128)]
    ncov = FF.check_blend("small splats far from the origin", got, rec, order, w, h, got8=got8, windows=wins)[0]
    assert ncov >= 20_000
    e.close()


@pytest.mark.parametrize("w,h,tile", [(640, 360, 16), (2600, 1500, 32)])
def test_long_tile_lists(gs, w, h, tile):
    """A dense knot of splats in front of a cloud: fine tiles whose list is longer than one 512-entry batch, and at 16-px tiles more
    than 128 survivors in one batch, so the staging loop runs more than once."""
    assert BF.tile_px(w, h) == tile
    rng = np.random.default_rng(1501)
    m = 6000
    knot = rng.normal(0, 0.25, (m, 3)) + np.array([0.3, 0.2, 2.0])
    scene = _cat(_cloud(30_000, seed=1502), _splats(knot, np.exp(rng.uniform(np.log(0.005), np.log(0.03), (m, 3))), rng.integers(10, 200, m), rng))
    cc, cov, centers = scene
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    u, mv, _ = _camera(w, h, (0.0, 0.0, 10.0), (0.0, 0.0, 0.0))
    order = _back_to_front(centers, mv)
    got, got8, ps, rec = _render_both(e, u, w, h, order, n)
    r, ok = FF.pixel_rects(ps, w, h)
    t = r[ok] // tile
    fine = np.zeros((-(-h // tile), -(-w // tile)), np.int64)
    for (x0, y0, x1, y1) in t:
        fine[y0:y1 + 1, x0:x1 + 1] += 1
    coarse = np.zeros((-(-fine.shape[0] // 4), -(-fine.shape[1] // 8)), np.int64)     # coarse tiles: 8 x 4 fine tiles
    for (x0, y0, x1, y1) in t:
        coarse[y0 // 4:y1 // 4 + 1, x0 // 8:x1 // 8 + 1] += 1
    ty, tx = np.unravel_index(np.argmax(fine), fine.shape)
    batches = -(-coarse[ty // 4, tx // 8] // 512)
    assert fine[ty, tx] > 512 and batches >= 2, (fine[ty, tx], batches)
    if tile == 16:       # some batch of that tile has more than 128 survivors: the 128-thread staging loop runs twice
        assert fine[ty, tx] / batches > 128, (fine[ty, tx], batches)
    FF.check_blend(f"long tile lists {w}x{h}", got, rec, order, w, h, got8=got8)
    e.close()


def test_faint_splats(gs):
    """A field of faint splats (alpha bytes 1-3, a in [1/255, 3/255]) over a background cloud: dropping any record or rim block moves
    pixels by more than their bounds."""
    rng = np.random.default_rng(1601)
    w, h = 960, 540
    m = 4000
    pts = np.stack([rng.uniform(-4, 4, m), rng.uniform(-2.5, 2.5, m), rng.uniform(-1, 1, m)], 1)
    scene = _cat(_cloud(5_000, seed=1602), _splats(pts, np.exp(rng.uniform(np.log(0.05), np.log(0.3), (m, 3))), rng.integers(1, 4, m), rng))
    cc, cov, centers = scene
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    u, mv, _ = _camera(w, h, (0.0, 0.0, 12.0), (0.0, 0.0, 0.0))
    order = _back_to_front(centers, mv)
    for flip_y in (False, True):
        got, got8, ps, rec = _render_both(e, u, w, h, order, n, flip_y)
        faint = FF.pixel_rects(ps, w, h)[1] & (rec["a"] <= 3.5 / 255)
        assert faint.sum() >= 1000, faint.sum()
        FF.check_blend(f"faint splats flip_y={flip_y}", got, rec, order, w, h, got8=got8, flip_y=flip_y)
    e.close()


@pytest.mark.parametrize("flip_y", [False, True])
@pytest.mark.parametrize("dest", ["rgba32f", "rgba8"])
def test_composite(gs, dest, flip_y):
    """Over a destination colour and depth: depths equal to a splat's f32 window depth at the pixels round its centre and one ulp below
    it, +inf and NaN patches, 8x8 blocks nearer than every splat (the block-maximum skip), and no depth at all."""
    rng = np.random.default_rng(1701)
    w, h = 640, 360
    cc, cov, centers = _cloud(40_000, seed=1702)
    n = centers.shape[0]
    e = _engine(n, w, h, cc, cov)
    u, mv, _ = _camera(w, h, (0.0, 0.0, 12.0), (0.0, 0.0, 0.0))
    order = _back_to_front(centers, mv)
    e.render(u, w, h, n, order)
    rec = BF.read_records(e, n)
    drawn = np.flatnonzero((rec["ndc_z"] >= -1) & (rec["ndc_z"] <= 1) & (rec["cx"] >= 1) & (rec["cx"] < w - 1) & (rec["cy"] >= 1) & (rec["cy"] < h - 1))
    zw = (np.float32(0.5) * rec["ndc_z"] + np.float32(0.5)).astype(np.float32)
    lo, hi = np.quantile(zw[drawn], [0.2, 0.8])
    depth = rng.uniform(lo, hi, (h, w)).astype(np.float32)          # rows bottom-up here
    pick = rng.choice(drawn, 3000, replace=False)
    for k, i in enumerate(pick):                                    # the splat's own zw (or one ulp below) at its centre's 3x3 pixels
        x, y = int(rec["cx"][i]), int(rec["cy"][i])
        depth[y - 1:y + 2, x - 1:x + 2] = zw[i] if k % 2 else np.nextafter(zw[i], np.float32(-np.inf))
    depth[:, 96:128] = np.inf
    depth[64:96, :] = np.nan
    depth[200:264, 200:264] = 0.0                                   # 8x8 blocks nearer than every splat
    color = rng.random((h, w, 4)).astype(np.float32)
    if dest == "rgba8":
        color = np.floor(color * 255 + 0.5).astype(np.uint8)
    dcol, ddep = (color[::-1].copy(), depth[::-1].copy()) if flip_y else (color, depth)
    from gaussiansplats3d_b200 import _native as N
    fmt = N.GS_FRAME_RGBA8 if dest == "rgba8" else N.GS_FRAME_RGBA32F
    got = e.render(u, w, h, n, order, frame_format=fmt, flip_y=flip_y, dest_color=dcol, dest_depth=ddep).copy()
    assert np.array_equal(BF.read_records(e, n), rec)
    res = BF.restate(rec, order, w, h, dest_color=dcol, dest_depth=ddep, flip_y=flip_y)
    rows = got[::-1] if flip_y else got
    assert np.array_equal(rows[200:264, 200:264], color[200:264, 200:264] if dest == "rgba8" else color[200:264, 200:264])
    BF.check(f"composite over {dest} flip_y={flip_y}", res, None if dest == "rgba8" else rows, rows if dest == "rgba8" else None)
    # and without a depth: every fragment passes
    got = e.render(u, w, h, n, order, frame_format=fmt, flip_y=flip_y, dest_color=dcol).copy()
    res = BF.restate(rec, order, w, h, dest_color=dcol, flip_y=flip_y)
    rows = got[::-1] if flip_y else got
    BF.check(f"composite over {dest}, no depth, flip_y={flip_y}", res, None if dest == "rgba8" else rows, rows if dest == "rgba8" else None)
    e.close()
