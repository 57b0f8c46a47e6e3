"""CPU: the f64 restatement of the blend and its per-pixel bounds (tests/blend_f64.c), held against an f32 emulation of the blend
kernel -- fmaf in the kernel's order, ex2 perturbed within its stated error, per-block lists walked in record pairs, and an early stop
placed at random among the points where the kernel may stop.  The emulation must stay inside every bound; emulations with one faint
splat dropped, the cutoff at 1/256 or RGBA8 rounding with +0.49 must not; the quad coordinates taken from the frame origin (the
kernel's earlier form) put far more rounding on q than tile-relative ones; and the bounds stay tight (ceilings on their median and
99.9th percentile)."""
import numpy as np
import pytest

import blend_f64 as B


def _records(n, seed, window, *, gmin=0.02, gmax=3.0, amin=1 / 255, amax=1.0, margin=20.0):
    """n random projected records around the window (x0, y0, w, h): |g| from gmin to gmax px^-1 (splat radii 1/gmax to 1/gmin px),
    random orientations and aspect, alpha in [amin, amax], colours in [0, 1], ndc_z in [-1, 1] (all drawn)."""
    rng = np.random.default_rng(seed)
    x0, y0, w, h = window
    r = np.zeros(n, B.REC_DTYPE)
    r["cx"] = rng.uniform(x0 - margin, x0 + w + margin, n)
    r["cy"] = rng.uniform(y0 - margin, y0 + h + margin, n)
    s1 = np.exp(rng.uniform(np.log(gmin), np.log(gmax), n))
    s2 = np.clip(s1 * np.exp(rng.uniform(-1.0, 1.0, n)), gmin, gmax)
    th = rng.uniform(0.0, np.pi, n)
    r["g1x"], r["g1y"] = s1 * np.cos(th), s1 * np.sin(th)
    r["g2x"], r["g2y"] = -s2 * np.sin(th), s2 * np.cos(th)
    r["a"] = rng.uniform(amin, amax, n)
    r["r"], r["g"], r["b"] = rng.random((3, n))
    r["ndc_z"] = rng.uniform(-1.0, 1.0, n)
    return r


def _order(n):
    return np.arange(n, dtype=np.uint32)


# (frame w, h, window, splats, alpha range, |g| range): far from the origin at 8K with |g| up to 3, at the origin, partial blocks
SCENES = {
    "8K far corner": (8192, 4320, (8128, 4256, 64, 64), 2500, (1 / 255, 1.0), (0.02, 3.0)),
    "8K far corner, faint": (8192, 4320, (8128, 4256, 64, 64), 600, (1 / 255, 0.1), (0.02, 3.0)),
    "7680x4320 centre": (7680, 4320, (3840, 2160, 96, 64), 3000, (1 / 255, 0.8), (0.03, 1.5)),
    "1080p origin": (1920, 1080, (0, 0, 64, 64), 1500, (1 / 255, 1.0), (0.05, 3.0)),
    "17x9 partial blocks": (17, 9, (0, 0, 17, 9), 200, (1 / 255, 1.0), (0.1, 3.0)),
    "7x5 partial block": (7, 5, (0, 0, 7, 5), 300, (1 / 255, 1.0), (0.1, 3.0)),
}


@pytest.mark.parametrize("name", list(SCENES))
def test_emulation_within_bounds(name):
    w, h, win, n, (amin, amax), (gmin, gmax) = SCENES[name]
    rec = _records(n, 11, win, amin=amin, amax=amax, gmin=gmin, gmax=gmax)
    res = B.restate(rec, _order(n), w, h, window=win)
    assert (res.value[..., 3] > 0).mean() > 0.5
    for seed in range(4):
        e32, e8 = B.emulate(rec, _order(n), w, h, window=win, seed=seed)
        B.check(f"{name}, seed {seed}", res, e32, e8)


@pytest.mark.parametrize("flip_y", [False, True])
@pytest.mark.parametrize("fmt", ["rgba32f", "rgba8"])
def test_composite_emulation_within_bounds(fmt, flip_y):
    """Over a destination colour and depth: depths of +inf, NaN, equal to a splat's f32 zw and one ulp below it, and a nearer block."""
    w, h = 48, 40
    win = (0, 0, w, h)
    n = 400
    rng = np.random.default_rng(21)
    rec = _records(n, 22, win, amax=0.7, gmin=0.05, gmax=1.0)
    zw = (np.float32(0.5) * rec["ndc_z"] + np.float32(0.5)).astype(np.float32)
    depth = rng.choice(zw, (h, w)).astype(np.float32)
    below = np.nextafter(depth, np.float32(-np.inf))
    pick = rng.random((h, w))
    depth = np.where(pick < 0.3, below, depth)
    depth[pick > 0.9] = np.inf
    depth[(pick > 0.85) & (pick <= 0.9)] = np.nan
    depth[:8, :8] = -1.0                               # a block nearer than every splat
    color = rng.random((h, w, 4)).astype(np.float32) * 1.2 - 0.1
    if fmt == "rgba8":
        color = np.floor(np.clip(color, 0, 1) * 255 + 0.5).astype(np.uint8)
    res = B.restate(rec, _order(n), w, h, dest_color=color, dest_depth=depth, flip_y=flip_y)
    assert np.isin(depth, zw).any() and np.isin(depth, np.nextafter(zw, np.float32(-np.inf))).any()
    for seed in range(3):
        e32, e8 = B.emulate(rec, _order(n), w, h, dest_color=color, dest_depth=depth, flip_y=flip_y, seed=seed)
        B.check(f"composite {fmt} flip_y={flip_y}, seed {seed}", res, e32 if fmt == "rgba32f" else None, e8 if fmt == "rgba8" else None)


# the largest rounding bound on q of a term near the q = 1 contour that the tile-relative form must meet, and the absolute form does not
DQ_CEILING = 1e-4


def test_absolute_coordinates_fail_the_q_band_ceiling():
    """At the far corner of an 8K frame with |g| up to 3 px^-1, quad coordinates taken from the frame origin put ~4e-3 of rounding on q
    near its q = 1 contour; taken from the tile's first pixel centre, ~3e-5 at 8K and ~1e-5 at 1080p.  The emulation of the absolute form
    leaves the tile-relative bound."""
    w, h, win, n, (amin, amax), (gmin, gmax) = SCENES["8K far corner"]
    rec = _records(n, 11, win, amin=amin, amax=amax, gmin=gmin, gmax=gmax)
    tile = B.restate(rec, _order(n), w, h, window=win)
    absolute = B.restate(rec, _order(n), w, h, window=win, form="abs")
    near = B.restate(_records(1500, 11, (0, 0, 64, 64)), _order(1500), 1920, 1080, window=(0, 0, 64, 64))
    print(f"\nq band near the contour: tile-relative {tile.dq_near:.3g} at 8K, {near.dq_near:.3g} at 1080p; absolute {absolute.dq_near:.3g} at 8K")
    assert tile.dq_near <= DQ_CEILING and near.dq_near <= DQ_CEILING
    assert absolute.dq_near > 10 * DQ_CEILING
    fails = 0
    for seed in range(4):
        e32, _ = B.emulate(rec, _order(n), w, h, window=win, form="abs", seed=seed)
        fails += (B.excess(tile, e32) > 1.0).any()
    assert fails >= 1


# ceilings on the bound over covered pixels, about twice what the restatement reaches on these scenes (measured: faint layers
# median 1.03e-6, 99.9th percentile 2.5e-6; saturating scene median 5.1e-4, 99.9th 1.9e-3 -- there the early-stop allowance dominates)
CEILINGS = {"8K far corner, faint": (2e-6, 5e-6), "8K far corner": (1e-3, 4e-3)}


@pytest.mark.parametrize("name", list(CEILINGS))
def test_bounds_stay_tight(name):
    w, h, win, n, (amin, amax), (gmin, gmax) = SCENES[name]
    rec = _records(n, 11, win, amin=amin, amax=amax, gmin=gmin, gmax=gmax)
    res = B.restate(rec, _order(n), w, h, window=win)
    cov = res.value[..., 3] > 0
    med, q999 = float(np.median(res.bound[cov])), float(np.quantile(res.bound[cov], 0.999))
    print(f"\n[{name}] bound over covered pixels: median {med:.3g}, 99.9th percentile {q999:.3g}")
    med_ceil, q_ceil = CEILINGS[name]
    assert med <= med_ceil and q999 <= q_ceil


def _faint_field():
    """A background of mid-alpha splats under a field of faint (alpha 1/255 .. 3/255) wide ones, at the far corner of an 8K frame."""
    win = (8128, 4256, 64, 64)
    back = _records(40, 31, win, amin=0.2, amax=0.5, gmin=0.03, gmax=0.08)
    faint = _records(60, 32, win, amin=1 / 255, amax=3 / 255, gmin=0.02, gmax=0.06)
    rec = np.concatenate([back, faint])
    return rec, 8192, 4320, win, np.arange(40, 100)


def test_dropped_faint_splat_fails():
    rec, w, h, win, faint = _faint_field()
    n = len(rec)
    res = B.restate(rec, _order(n), w, h, window=win)
    e32, e8 = B.emulate(rec, _order(n), w, h, window=win)
    B.check("faint field", res, e32, e8)
    caught = 0
    for i in faint[:12]:
        m32, _ = B.emulate(rec, _order(n), w, h, window=win, drop=int(i))
        caught += (B.excess(res, m32) > 1.0).any()
    assert caught == 12, f"only {caught} of 12 dropped faint splats leave the bound"


def _stack():
    """Layers of wide splats of alpha ~0.5 over a 64x64 window: every block saturates part-way through its list."""
    win = (4096, 2048, 64, 64)
    rec = _records(40, 41, win, amin=0.4, amax=0.6, gmin=0.01, gmax=0.015, margin=0.0)
    return rec, 8192, 4320, win


def test_cutoff_1_256_fails():
    rec, w, h, win = _stack()
    n = len(rec)
    res = B.restate(rec, _order(n), w, h, window=win)
    for seed in range(3):
        e32, e8 = B.emulate(rec, _order(n), w, h, window=win, seed=seed)
        B.check("stack", res, e32, e8)
    m32, _ = B.emulate(rec, _order(n), w, h, window=win, cutoff=1 / 256)
    assert (B.excess(res, m32) > 1.0).any()


def test_rgba8_rounding_049_fails():
    w, h, win, n, (amin, amax), (gmin, gmax) = SCENES["8K far corner, faint"]
    rec = _records(n, 11, win, amin=amin, amax=amax, gmin=gmin, gmax=gmax)
    res = B.restate(rec, _order(n), w, h, window=win)
    _, m8 = B.emulate(rec, _order(n), w, h, window=win, round_add=0.49)
    assert (B.excess(res, m8, rgba8=True) > 0).any()


def test_window_must_be_block_aligned():
    rec = _records(10, 1, (0, 0, 64, 64))
    with pytest.raises(AssertionError):
        B.restate(rec, _order(10), 64, 64, window=(4, 0, 16, 16))
