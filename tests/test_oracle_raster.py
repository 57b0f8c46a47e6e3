"""CPU: the raster restatement (oracle/raster_oracle.c) and the host packing/uniform code still produce the committed fixture
(tests/golden/raster_golden.npz, written by tests/golden/make_raster_golden.py)."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import raster_cases  # noqa: E402

GOLD = np.load(Path(__file__).resolve().parent / "golden" / "raster_golden.npz")


@pytest.mark.parametrize("name", list(raster_cases.CASES))
def test_raster_oracle_reproduces_fixture(oracle_mod, name):
    order, frame, ps = raster_cases.oracle_outputs(name, oracle_mod)
    assert np.array_equal(order, GOLD[name + "|order"])
    assert np.array_equal(np.packbits(ps["valid"].astype(np.uint8)), GOLD[name + "|valid"])
    want = GOLD[name + "|frame"]
    assert frame.shape == want.shape
    # same compiler flags -> identical; leave room for another libm's expf
    assert np.abs(frame - want).max() < 2e-6
    assert want[..., 3].max() > 0.9 and (want[..., 3] == 0).any()


def test_fixture_order_is_a_permutation_back_to_front(oracle_mod):
    """Sanity of the stored draw order: a permutation along which the reference's integer distance (sorter.cpp:64-74) falls from
    bucket to bucket and, inside a bucket, later input positions come first (sorter.cpp:158-167)."""
    del oracle_mod
    for name in raster_cases.CASES:
        v, raw = raster_cases.host_viewer(name)
        order = GOLD[name + "|order"].astype(np.int64)
        assert np.array_equal(np.sort(order), np.arange(raw.count))
        m = v.mvp_matrix().astype(np.float32)
        row = np.array([int(np.float64(m[2]) * 1000.0), int(np.float64(m[6]) * 1000.0), int(np.float64(m[10]) * 1000.0)], np.int64)
        d = (v.splatMesh.packed.int_centers[:, :3].astype(np.int64) * row[None, :]).sum(axis=1)
        assert np.abs(d).max() < 2**31
        rm = np.float32(65535) / (np.float32(d.max()) - np.float32(d.min()))
        b = ((d - d.min()).astype(np.float32) * rm).astype(np.int64)[order]
        assert (np.diff(b) <= 0).all()
        same = np.diff(b) == 0
        assert (np.diff(order)[same] < 0).all()


def test_rgba8_per_blend_quantisation_is_reported(oracle_mod, capsys):
    """SURVEY 8(c)(ii), informational: the reference composites into an RGBA8 canvas (Viewer.js:353-360), i.e. the frame buffer is
    rounded to 8 bits after EVERY blend (SplatMaterial3D.js:65-75), while this engine (and the float oracle the parity tests use)
    accumulate in f32 and round once.  The difference is a property of the reference's render target, not a parity error; this test
    measures it on the committed fixture scenes with the oracle's quantize8 mode, prints it (pytest -s) and bounds it loosely so that
    a change of either mode is noticed."""
    report = {}
    for name in raster_cases.CASES:
        order, frame_f32, ps = raster_cases.oracle_outputs(name, oracle_mod)
        v, _ = raster_cases.host_viewer(name)
        frame_q8 = oracle_mod.blend(ps, order, v.renderWidth, v.renderHeight, quantize8=True)
        d = np.abs(frame_q8 - frame_f32) * 255.0
        covered = frame_f32[..., 3] > 0
        report[name] = (float(d.max()), float(d[covered].mean()), float((d[covered] > 1.0).mean()))
        # per-blend rounding drifts by up to half a step per overlapping splat; tens of layers -> a few steps, never a different picture
        assert d.max() < 40.0 and d[covered].mean() < 4.0, (name, report[name])
        assert d.max() > 0.0      # the mode really quantises
    with capsys.disabled():
        for name, (mx, mean, frac) in report.items():
            print(f"\n[rgba8-per-blend vs f32 accumulate] {name}: max {mx:.2f}/255, mean over covered pixels {mean:.3f}/255, channels off by > 1 step: {100 * frac:.2f} %")


# ---- coverage-boundary map (blend(..., flags=True)): a diagnostic of the oracle's blend (the GPU is held to tests/blend_f64.c) ----------------------------------------
def _one_splat(cx, cy, b1, b2, a=1.0):
    from gaussiansplats3d_b200 import _native as N
    ps = np.zeros(1, N.PROJECTED_DTYPE)
    ps["cx"], ps["cy"] = cx, cy
    ps["b1x"], ps["b1y"], ps["b2x"], ps["b2y"] = b1[0], b1[1], b2[0], b2[1]
    ps["r"], ps["g"], ps["b"], ps["a"] = 0.9, 0.5, 0.2, a
    ps["valid"] = 1
    return ps


def _q_f64(ps, w, h):
    """q = A/8 of the single splat at every pixel centre, in float64."""
    p = ps[0]
    y, x = np.mgrid[0:h, 0:w].astype(np.float64) + 0.5
    dx, dy = x - float(p["cx"]), y - float(p["cy"])
    b1 = np.array([p["b1x"], p["b1y"]], np.float64)
    b2 = np.array([p["b2x"], p["b2y"]], np.float64)
    u = (dx * b1[0] + dy * b1[1]) / (b1 @ b1)
    v = (dx * b2[0] + dy * b2[1]) / (b2 @ b2)
    return u * u + v * v


def test_flag_map_is_the_ring_around_the_coverage_contour(oracle_mod):
    """A rotated ellipse off the pixel grid: the flagged pixels are exactly those whose float64 q lies within delta of 1 (pixels within
    1e-5 of the band's edge may go either way in f32), the ring is not empty, and the frame covers every pixel with q < 1 - delta."""
    w, h, delta = 160, 120, oracle_mod.FLAG_DELTA
    th = 0.37
    ps = _one_splat(80.3, 58.8, (55.3 * np.cos(th), 55.3 * np.sin(th)), (-31.1 * np.sin(th), 31.1 * np.cos(th)))
    frame, flags = oracle_mod.blend(ps, np.zeros(1, np.uint32), w, h, flags=True)
    q = _q_f64(ps, w, h)
    want = np.abs(q - 1.0) <= delta
    sure = np.abs(np.abs(q - 1.0) - delta) > 1e-5
    assert want.sum() >= 8, "the contour must pass near some pixel centres"
    assert np.array_equal(flags[sure], want[sure])
    assert (frame[..., 3][q < 1.0 - delta] > 0).all() and (frame[..., 3][q > 1.0 + delta] == 0).all()
    x0, y0, cw, ch = 9, 5, 97, 61
    frame_c, flags_c = oracle_mod.blend_crop(ps, np.zeros(1, np.uint32), w, h, x0, y0, cw, ch, flags=True)
    assert np.array_equal(flags_c, flags[y0:y0 + ch, x0:x0 + cw]) and np.array_equal(frame_c, frame[y0:y0 + ch, x0:x0 + cw])


def test_flag_map_is_empty_away_from_pixel_centres(oracle_mod):
    """A circle of radius 2.5 px centred on a pixel centre: q = k / 6.25 for integer k, never within delta of 1, so nothing is flagged
    although 21 pixels are covered.  A splat whose contour runs through pixel centres but whose alpha is below 1/255 is not flagged."""
    w, h = 16, 16
    ps = _one_splat(8.5, 7.5, (2.5, 0.0), (0.0, 2.5))
    frame, flags = oracle_mod.blend(ps, np.zeros(1, np.uint32), w, h, flags=True)
    assert not flags.any()
    assert (frame[..., 3] > 0).sum() == 21
    faint = _one_splat(8.5, 7.5, (3.0, 0.0), (0.0, 3.0), a=0.5 / 255)
    _, flags = oracle_mod.blend(faint, np.zeros(1, np.uint32), w, h, flags=True)
    assert not flags.any()
    _, flags = oracle_mod.blend(_one_splat(8.5, 7.5, (3.0, 0.0), (0.0, 3.0)), np.zeros(1, np.uint32), w, h, flags=True)
    assert flags.sum() == 4         # (8.5 +- 3, 7.5) and (8.5, 7.5 +- 3): q exactly 1


@pytest.mark.parametrize("name", list(raster_cases.CASES))
def test_blend_with_flags_draws_the_same_frame(oracle_mod, name):
    """Asking for the boundary map does not change the picture (whole frame and a window), and the fixture still reproduces."""
    order, frame, ps = raster_cases.oracle_outputs(name, oracle_mod)
    h, w = frame.shape[:2]
    got, flags = oracle_mod.blend(ps, order, w, h, flags=True)
    assert np.array_equal(got, frame)
    assert np.abs(got - GOLD[name + "|frame"]).max() < 2e-6
    covered = frame[..., 3] > 0
    assert 0 < flags.sum() < 0.2 * covered.sum()
    x0, y0 = w // 3, h // 4
    crop, cflags = oracle_mod.blend_crop(ps, order, w, h, x0, y0, w // 2, h // 2, flags=True)
    assert np.array_equal(crop, frame[y0:y0 + h // 2, x0:x0 + w // 2]) and np.array_equal(cflags, flags[y0:y0 + h // 2, x0:x0 + w // 2])
    q8, _ = oracle_mod.blend(ps, order, w, h, quantize8=True, flags=True)
    assert np.array_equal(q8, oracle_mod.blend(ps, order, w, h, quantize8=True))
