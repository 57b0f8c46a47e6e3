"""CPU: the f64 restatement of a frame's view depth and its per-pixel bound (tests/depth_f64.py), held against an f32 emulation of the
blend kernel's depth; its closed forms (one opaque splat, two splats of known depths and alphas, an empty pixel); and the ndc_z -> view
depth conversion against three.js's perspective and orthographic matrices (gaussiansplats3d_b200/three_math.py) over near / far ranges,
within the bound the header states."""
import numpy as np
import pytest

import blend_f64 as BF
import depth_f64 as DF


def _persp(near, far, fov=50.0, aspect=1.5):
    from gaussiansplats3d_b200 import three_math as TM
    return TM.make_perspective(fov, aspect, near, far)


def _ortho(near, far, half=4.0):
    from gaussiansplats3d_b200 import three_math as TM
    return TM.make_orthographic(-half * 1.5, half * 1.5, half, -half, near, far)


def _ndc(P, d):
    """f32 ndc_z of view depth d (z_view = -d) through the f64 matrix: (P z) / (P w), rounded once."""
    z = -np.asarray(d, np.float64)
    return ((P[10] * z + P[14]) / (P[11] * z + P[15])).astype(np.float32)


def _records(n, seed, window, P, *, gmin=0.05, gmax=2.0, amin=1 / 255, amax=1.0, margin=20.0):
    """n random projected records around the window, ndc_z spread over the view depths [near, far] of P."""
    rng = np.random.default_rng(seed)
    x0, y0, w, h = window
    r = np.zeros(n, BF.REC_DTYPE)
    r["cx"] = rng.uniform(x0 - margin, x0 + w + margin, n)
    r["cy"] = rng.uniform(y0 - margin, y0 + h + margin, n)
    s1 = np.exp(rng.uniform(np.log(gmin), np.log(gmax), n))
    s2 = np.clip(s1 * np.exp(rng.uniform(-1.0, 1.0, n)), gmin, gmax)
    th = rng.uniform(0.0, np.pi, n)
    r["g1x"], r["g1y"] = s1 * np.cos(th), s1 * np.sin(th)
    r["g2x"], r["g2y"] = -s2 * np.sin(th), s2 * np.cos(th)
    r["a"] = rng.uniform(amin, amax, n)
    r["r"], r["g"], r["b"] = rng.random((3, n))
    r["ndc_z"] = rng.uniform(-1.0, 0.999, n)
    return r


def _disc(cx, cy, radius, a, ndc):
    r = np.zeros(1, BF.REC_DTYPE)
    r["cx"], r["cy"] = cx, cy
    r["g1x"], r["g2y"] = 1.0 / radius, 1.0 / radius
    r["a"], r["ndc_z"] = a, ndc
    r["r"] = r["g"] = r["b"] = 0.5
    return r


PROJECTIONS = {"perspective 0.1-1000": (_persp(0.1, 1000.0), False), "perspective 1-50": (_persp(1.0, 50.0), False),
               "orthographic 0.1-1000": (_ortho(0.1, 1000.0), True)}


@pytest.mark.parametrize("proj", list(PROJECTIONS))
def test_closed_forms(proj):
    P, _ = PROJECTIONS[proj]
    w, h = 16, 16
    n1, n2 = np.float32(0.3), np.float32(0.6)
    d1, d2 = DF.view_depth64(n1, P), DF.view_depth64(n2, P)
    # one opaque splat: its own d at its centre pixel; the pixels it does not reach are +inf
    one = _disc(4.5, 4.5, 2.0, 1.0, n1)
    res = DF.restate(one, np.zeros(1, np.uint32), w, h, P)
    em = DF.emulate(one, np.zeros(1, np.uint32), w, h, P)
    assert res.value[4, 4] == pytest.approx(float(np.float32(d1)), rel=1e-12)
    assert em[4, 4] == DF.view_depth32(n1, P)
    assert np.isposinf(res.value[12, 12]) and res.empty[12, 12] and np.isposinf(em[12, 12])
    DF.check(f"{proj} one opaque splat", res, em)
    # two splats over the same centre: front (alpha a1, d1) over back (alpha a2, d2) -> the weighted mean
    a1, a2 = 0.4, 0.7
    two = np.concatenate([_disc(8.5, 8.5, 3.0, a2, n2), _disc(8.5, 8.5, 3.0, a1, n1)])   # draw order: back first
    order = np.arange(2, dtype=np.uint32)
    res = DF.restate(two, order, w, h, P)
    want = (a1 * np.float32(d1) + (1 - a1) * a2 * np.float32(d2)) / (1 - (1 - a1) * (1 - a2))
    assert res.value[8, 8] == pytest.approx(want, rel=1e-6)
    em = DF.emulate(two, order, w, h, P)
    assert abs(em[8, 8] - want) <= res.bound[8, 8]
    DF.check(f"{proj} two splats", res, em)


WINDOWS = {"1080p origin": (1920, 1080, (0, 0, 64, 64), 1500), "8K far corner": (8192, 4320, (8128, 4256, 64, 64), 2000),
           "17x9 partial blocks": (17, 9, (0, 0, 17, 9), 200)}


@pytest.mark.parametrize("proj", list(PROJECTIONS))
@pytest.mark.parametrize("name", list(WINDOWS))
def test_emulation_within_bounds(name, proj):
    w, h, win, n = WINDOWS[name]
    P, _ = PROJECTIONS[proj]
    rec = _records(n, 5, win, P)
    order = np.arange(n, dtype=np.uint32)
    res = DF.restate(rec, order, w, h, P, window=win)
    assert np.isfinite(res.value).mean() > 0.5
    for seed in range(3):
        DF.check(f"{name} {proj} seed {seed}", res, DF.emulate(rec, order, w, h, P, window=win, seed=seed))
    # the bound is tight enough to mean something: a depth off by 1e-3 relative falls outside it almost everywhere
    em = DF.emulate(rec, order, w, h, P, window=win)
    pinned = np.isfinite(res.value) & ~res.loose
    assert (DF.excess(res, em * np.float32(1.001))[pinned] > 1).mean() > 0.95


@pytest.mark.parametrize("flip_y", [False, True])
def test_composite_emulation_within_bounds(flip_y):
    """A composited frame: only the fragments that pass zw <= dest depth count; where every one is hidden the depth is +inf."""
    w, h = 48, 40
    P = _persp(0.1, 100.0)
    rec = _records(400, 9, (0, 0, w, h), P, amax=0.7)
    zw = (np.float32(0.5) * rec["ndc_z"] + np.float32(0.5)).astype(np.float32)
    rng = np.random.default_rng(3)
    dest = rng.choice(zw, (h, w)).astype(np.float32)
    dest[:, :8] = 0.0                                   # nothing passes
    order = np.arange(rec.shape[0], dtype=np.uint32)
    res = DF.restate(rec, order, w, h, P, dest_depth=dest, flip_y=flip_y)
    got = DF.emulate(rec, order, w, h, P, dest_depth=dest, flip_y=flip_y)
    DF.check(f"composite flip_y={flip_y}", res, got)
    hidden = DF.crop(dest, (0, 0, w, h), flip_y) == 0
    assert np.isposinf(got[hidden]).all() and res.empty[hidden].all()


@pytest.mark.parametrize("near,far", [(0.1, 1000.0), (0.1, 100.0), (0.01, 10.0), (1.0, 5000.0)])
def test_conversion_perspective(near, far):
    """three.js's perspective matrix: d from the f32 ndc_z of view depths across [near, far] is within the stated bound."""
    P = _persp(near, far)
    d = np.geomspace(near, far, 4001)[:-1]
    got = DF.view_depth32(_ndc(P, d), P).astype(np.float64)
    b = DF.conversion_bound(d, near, far)
    assert (np.abs(got - d) <= b).all(), np.max(np.abs(got - d) / b)
    # the bound is the stated one: at near = 0.1, ~6e-3 at d = 100 and ~6.4e-5 at d = 10 (twice one ulp of ndc_z times dd/dndc)
    if near == 0.1:
        assert DF.conversion_bound(100.0, near, far) == pytest.approx(6.0e-3, rel=0.02)
        assert DF.conversion_bound(10.0, near, far) == pytest.approx(6.4e-5, rel=0.02)
    # the f64 restatement of the formula is the same function
    assert np.allclose(DF.view_depth64(_ndc(P, d), P), got, rtol=4 * DF.U, atol=0)


@pytest.mark.parametrize("near,far", [(0.1, 1000.0), (-5.0, 20.0), (1.0, 3.0)])
def test_conversion_orthographic(near, far):
    P = _ortho(near, far)
    d = np.linspace(near, far, 4001)[1:-1]
    got = DF.view_depth32(_ndc(P, d), P).astype(np.float64)
    b = DF.conversion_bound(d, near, far, orthographic=True)
    assert (np.abs(got - d) <= b).all(), np.max(np.abs(got - d) / b)
