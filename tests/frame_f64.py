"""One check of a GPU frame against the f64 restatements, for every frame test: the draw order the frame used, every drawn splat's
projection (tests/projection_f64.py), the binning's tile-instance count, and the blend of the GPU's own raw records, every channel of
every pixel within its bound (tests/blend_f64.py).  TEST INFRASTRUCTURE ONLY.

check_frame() after a render or frame of engine `e`:
  * drawn order: the order the caller passed to the render, else the engine's sorted indexes (GS_BUF_SORTED_INDEXES).  When the
    engine sorted (`sort` given), that order must equal the reference sorter's bit for bit (the compiled reference where oracle/_ref
    has it, else oracle/sort_oracle.c);
  * projection: every drawn splat's exported record within its per-splat f64 bounds and `valid` equal (PF.assert_within), projected
    in chunks of at most 1 M splats (the projection is per splat, so the chunks are exact);
  * tile instances: timings()["tile_instances"] equal to the host's count of coarse tiles the drawn records' rects touch (1e-3 + 2);
  * blend: the frame (RGBA32F and / or RGBA8) within the f64 bounds over the whole frame, or over the given 8-px-aligned windows.
It prints the worst |GPU - f64| / bound of the projection and of the blend (pytest -s) and returns them."""
from __future__ import annotations

import time

import numpy as np

import blend_f64 as BF
import projection_f64 as PF

PROJECT_CHUNK = 1 << 20


# ---- what the GPU binned: host restatement of k_project's pixel rects ---------------------------------------------------------------
def pixel_rects(ps, w, h):
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


def coarse_spans(ps, w, h, tile_shift):
    """Coarse tiles (8 x 4 fine tiles) each splat's rect touches: the tile-instance count of the binning."""
    r, ok = pixel_rects(ps, w, h)
    t = r >> tile_shift
    n = ((t[:, 2] >> 3) - (t[:, 0] >> 3) + 1) * ((t[:, 3] >> 2) - (t[:, 1] >> 2) + 1)
    return np.where(ok, n, 0)


# ---- blend ----------------------------------------------------------------------------------------------------------------------------
def windows(w, h, ww=256, wh=128):
    """Corners (including the last, possibly partial, tile row and column), edge midpoints and centre of a large frame."""
    ww, wh = min(ww, w), min(wh, h)
    xs, ys = (0, (w - ww) // 2 // 8 * 8, (w - ww) // 8 * 8), (0, (h - wh) // 2 // 8 * 8, (h - wh) // 8 * 8)
    # windows start on the 8x8 block grid; the last ones run to the frame's edge
    return sorted({(x, y, ww if x < (w - ww) // 8 * 8 else w - x, wh if y < (h - wh) // 8 * 8 else h - y) for x in xs for y in ys})


def check_blend(label, got, rec, order, w, h, *, got8=None, windows=None, flip_y=False, dest_color=None, dest_depth=None):
    """Hold a GPU frame (and its RGBA8 twin) to the f64 restatement of the blend of the GPU's raw records `rec` in draw order `order`,
    over the whole frame or the given 8-px-aligned windows; dest_color / dest_depth: the composite inputs the frame was given, in its
    row order.  Returns (covered pixels compared, worst RGBA32F |err| / bound)."""
    ncov, worst = 0, 0.0
    for win in ([(0, 0, w, h)] if windows is None else windows):
        res = BF.restate(rec, order, w, h, window=win, dest_color=dest_color, dest_depth=dest_depth, flip_y=flip_y)
        rep = BF.check(f"{label} {win}", res, None if got is None else BF.crop(got, win, flip_y), None if got8 is None else BF.crop(got8, win, flip_y))
        ncov += rep["covered"]
        worst = max(worst, rep.get("worst32", 0.0))
    return ncov, worst


# ---- draw order -----------------------------------------------------------------------------------------------------------------------
def reference_order(centers, mvp, render_count, *, indexes=None, sort_count=None, splat_count=None, precision=16, integer=True,
                    scene_indexes=None, transforms=None, dynamic=False):
    """The reference sorter's sortIndexes() (the compiled reference where oracle/_ref has it, else oracle/sort_oracle.c)."""
    import oracle
    sorter = oracle.ref_sort_indexes if oracle.have_ref() else oracle.port_sort_indexes
    n = centers.shape[0] if splat_count is None else splat_count
    idx = np.arange(render_count, dtype=np.uint32) if indexes is None else indexes
    return sorter(idx, centers, None, np.asarray(mvp, np.float32), scene_indexes, transforms, 1 << precision,
                  render_count if sort_count is None else sort_count, render_count, n, False, integer, dynamic)


# ---- projection -----------------------------------------------------------------------------------------------------------------------
def check_projection(label, u, ps, drawn, centers_colors, covariances, sh=None, sh_degree=0, scene_indexes=None, min_compared=1):
    """Every splat in `drawn` (splat ids): its exported record `ps[id]` within the f64 bounds of the vertex stage.  Returns the merged
    report (PF.compare's, summed over chunks of at most PROJECT_CHUNK splats)."""
    tot = dict(valid_mismatch=0, compared=0, ambiguous=0, worst={k: 0.0 for k in PF.FIELDS}, outside={k: 0 for k in PF.FIELDS})
    for i in range(0, len(drawn), PROJECT_CHUNK):
        ids = drawn[i:i + PROJECT_CHUNK]
        want = PF.project(u, centers_colors[ids], covariances[ids], None if sh is None else sh[ids], sh_degree,
                          None if scene_indexes is None else scene_indexes[ids])
        rep = PF.compare(ps[ids], want)
        for k in ("valid_mismatch", "compared", "ambiguous"):
            tot[k] += rep[k]
        for k in PF.FIELDS:
            tot["worst"][k] = max(tot["worst"][k], rep["worst"][k])
            tot["outside"][k] += rep["outside"][k]
    print("\n" + PF.format_report(label, tot))
    PF.assert_within(label, tot, min_compared=min_compared)
    return tot


# ---- the whole frame ------------------------------------------------------------------------------------------------------------------
def check_frame(label, e, u, w, h, render_count, centers_colors, covariances, sh=None, sh_degree=0, scene_indexes=None, *, got=None,
                got8=None, order=None, sort=None, windows=None, flip_y=False, min_compared=1, dest_color=None, dest_depth=None):
    """Check the last frame engine `e` drew with uniforms `u` into a w x h frame from render_count splats of the scene it holds
    (centers_colors, covariances, sh, sh_degree, scene_indexes: what it was uploaded from).  got / got8: that frame in RGBA32F / RGBA8
    (either may be None; both must come from the same draw).  order: the draw order the caller passed in, else the engine's sorted
    indexes are read.  sort: the reference_order() keywords (centers, mvp, ...) when the engine sorted.  windows: 8-px-aligned windows
    (x0, y0, w, h) of the blend check, None for the whole frame.  dest_color / dest_depth: the composite inputs of a composited frame,
    as the engine was given them (host arrays).  Returns (worst projection ratio, worst blend ratio)."""
    from gaussiansplats3d_b200 import _native as N
    t0 = time.time()
    if order is None:
        order = e.read_buffer(N.GS_BUF_SORTED_INDEXES, np.uint32, render_count)
    order = np.asarray(order, np.uint32)
    assert order.shape == (render_count,), (order.shape, render_count)
    if sort is not None:
        want = reference_order(render_count=render_count, **sort)
        assert np.array_equal(order, want), f"{label}: the draw order differs from the reference sorter's at {np.flatnonzero(order != want)[:5].tolist()}"
    nrec = int(order.max()) + 1 if render_count else 0
    ps = e.read_projected(nrec)
    rec = BF.read_records(e, nrec)
    timings = e.timings()
    drawn = np.unique(order)
    assert len(drawn) == render_count, f"{label}: the draw order repeats splats"
    prep = check_projection(f"{label} projection", u, ps, drawn, centers_colors, covariances, sh, sh_degree, scene_indexes, min_compared)
    shift = 4 if BF.tile_px(w, h) == 16 else 5
    want_inst = int(coarse_spans(ps[order], w, h, shift).sum())
    inst = timings["tile_instances"]
    assert abs(inst - want_inst) <= 1e-3 * want_inst + 2, f"{label}: {inst} tile instances, host count {want_inst}"
    t1 = time.time()
    ncov, worst = check_blend(label, got, rec, order, w, h, got8=got8, windows=windows, flip_y=flip_y, dest_color=dest_color, dest_depth=dest_depth)
    assert ncov > 0, f"{label}: nothing covered"
    pworst = max(prep["worst"].values())
    area = w * h if windows is None else sum(win[2] * win[3] for win in windows)
    print(f"[{label}] {render_count} splats drawn, {w}x{h}, {100 * area / (w * h):.1f} % of the frame blended: worst |GPU - f64|/bound "
          f"projection {pworst:.3f}, blend {worst:.3f}; {inst} tile instances; host check {t1 - t0:.1f} s projection + {time.time() - t1:.1f} s blend")
    return pworst, worst


def check_viewer_frame(label, v, *, got=None, got8=None, scene=None, order=None, sort="viewer", render_count=None, windows=None, flip_y=False,
                       min_compared=1):
    """check_frame for the last frame of Viewer `v`: its engine, uniforms and frame size.  scene: a dict of the uploaded arrays
    (centers_colors, covariances, sh, sh_degree and the sorter's int_centers / float_centers), else the viewer's packed scene.  sort:
    "viewer" checks the engine's sorted indexes against the reference sorter run with the viewer's sort settings (precision, integer
    or float centres, the dynamic mesh's transforms), None checks nothing about the order, a dict passes reference_order() keywords."""
    sm = v.splatMesh
    if scene is None:
        p = sm.packed
        scene = dict(centers_colors=p.centers_colors, covariances=p.covariances, sh=p.sh, sh_degree=p.sh_degree)
    n = scene["centers_colors"].shape[0]
    rc = n if render_count is None else render_count
    if sort == "viewer":
        if v.integerBasedSort:
            centers = scene["int_centers"] if "int_centers" in scene else sm.getIntegerCenters(0, n - 1, True)
        else:
            centers = scene["float_centers"] if "float_centers" in scene else sm.getFloatCenters(0, n - 1, True)
        sort = dict(centers=centers, mvp=v.mvp_matrix().astype(np.float32), splat_count=n, precision=v.splatSortDistanceMapPrecision,
                    integer=v.integerBasedSort)
        if sm.dynamicMode:
            sort.update(scene_indexes=np.zeros(n, np.uint32), transforms=sm.fillTransformsArray(), dynamic=True)
    return check_frame(label, v.engine, v.uniforms(), v.renderWidth, v.renderHeight, rc, scene["centers_colors"], scene["covariances"],
                       scene.get("sh"), scene.get("sh_degree", 0), got=got, got8=got8, order=order, sort=sort, windows=windows,
                       flip_y=flip_y, min_compared=min_compared)
