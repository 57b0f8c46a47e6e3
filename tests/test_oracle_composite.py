"""CPU: the composite oracle (tests/composite_oracle.c) -- the oracle blend drawn into a framebuffer that already holds an opaque pass,
depth-tested against its depth (LessEqualDepth, no depth writes) and blended over its colour -- against the plain oracle blend and
against values derived by hand."""
import sys
from pathlib import Path

import numpy as np
import pytest

import composite_oracle as CO
from gaussiansplats3d_b200 import _native as N

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import raster_cases  # noqa: E402


@pytest.mark.parametrize("name", list(raster_cases.CASES))
@pytest.mark.parametrize("quantize8", [False, True])
def test_depth_one_zero_background_is_the_plain_blend(oracle_mod, name, quantize8):
    order, _, ps = raster_cases.oracle_outputs(name, oracle_mod)
    v, _ = raster_cases.host_viewer(name)
    w, h = v.renderWidth, v.renderHeight
    want = oracle_mod.blend(ps, order, w, h, quantize8=quantize8)
    got = CO.blend_composite(ps, order, w, h, dest_color=np.zeros((h, w, 4), np.float32), dest_depth=np.ones((h, w), np.float32),
                             quantize8=quantize8)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert want[..., 3].max() > 0.5
    # the window form restates the same pixels
    crop = CO.blend_composite(ps, order, w, h, dest_depth=np.ones((h, w), np.float32), quantize8=quantize8, window=(17, 9, 40, 33))
    assert np.array_equal(crop, want[9:42, 17:57])


@pytest.mark.parametrize("name", list(raster_cases.CASES))
def test_depth_zero_gives_the_background(oracle_mod, name):
    order, _, ps = raster_cases.oracle_outputs(name, oracle_mod)
    v, _ = raster_cases.host_viewer(name)
    w, h = v.renderWidth, v.renderHeight
    drawn = ps["valid"] == 1
    assert drawn.sum() > 100 and (ps["ndc_z"][drawn] > -1.0).all()      # no splat on the near plane: zw > 0 everywhere
    rng = np.random.default_rng(5)
    bg = rng.random((h, w, 4), dtype=np.float32)
    got = CO.blend_composite(ps, order, w, h, dest_color=bg, dest_depth=np.zeros((h, w), np.float32))
    assert np.array_equal(got, bg)
    bg8 = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    got8 = CO.blend_composite(ps, order, w, h, dest_color=bg8, dest_depth=np.zeros((h, w), np.float32), quantize8=True)
    assert np.array_equal(np.floor(got8 * 255.0 + 0.5).astype(np.uint8), bg8)
    # NaN depth passes nothing either
    got_nan = CO.blend_composite(ps, order, w, h, dest_color=bg, dest_depth=np.full((h, w), np.nan, np.float32))
    assert np.array_equal(got_nan, bg)


def _splat(ndc_z, a, rgb):
    """A splat centred on pixel (1, 1)'s centre whose quad maps that pixel to q = 0: its alpha there is exp(0) * a = a exactly."""
    s = np.zeros((), N.PROJECTED_DTYPE)
    s["cx"], s["cy"] = 1.5, 1.5
    s["b1x"], s["b1y"], s["b2x"], s["b2y"] = 2.0, 0.0, 0.0, 2.0
    s["r"], s["g"], s["b"] = rgb
    s["a"], s["ndc_z"], s["valid"] = a, ndc_z, 1
    return s


def test_three_splats_over_one_pixel_by_hand():
    """Draw order (farthest first): S0 behind the opaque surface, S1 exactly at its depth (zw == d passes under LessEqualDepth), S2 in
    front.  Destination (0.2, 0.4, 0.6, 0.5) at depth 0.5.
    Back to front: S0 is skipped; S1 (a 0.5, red):  C = 0.5 (1,0,0) + 0.5 (0.2,0.4,0.6) = (0.6, 0.2, 0.3), A = 0.5 + 0.5 * 0.5 = 0.75;
    S2 (a 0.25, blue): C = 0.25 (0,0,1) + 0.75 (0.6,0.2,0.3) = (0.45, 0.15, 0.475), A = 0.25 + 0.75 * 0.75 = 0.8125.
    The same front to back: T = 0.75 * 0.5 = 0.375 left for the destination, (0.375, 0, 0.25) + 0.375 (0.2, 0.4, 0.6) and
    (1 - 0.375) + 0.375 * 0.5."""
    ps = np.stack([_splat(0.5, 0.75, (0.0, 1.0, 0.0)),      # zw 0.75 > 0.5: hidden
                   _splat(0.0, 0.5, (1.0, 0.0, 0.0)),       # zw 0.5 == 0.5: drawn
                   _splat(-0.5, 0.25, (0.0, 0.0, 1.0))])    # zw 0.25: drawn
    order = np.arange(3, dtype=np.uint32)
    w = h = 3
    bg = np.zeros((h, w, 4), np.float32)
    bg[1, 1] = (0.2, 0.4, 0.6, 0.5)
    depth = np.ones((h, w), np.float32)
    depth[1, 1] = 0.5
    got = CO.blend_composite(ps, order, w, h, dest_color=bg, dest_depth=depth)
    np.testing.assert_allclose(got[1, 1], (0.45, 0.15, 0.475, 0.8125), rtol=0, atol=2e-7)
    # just below zw = 0.5, S1 is hidden too: only S2 over the destination
    depth[1, 1] = np.nextafter(np.float32(0.5), np.float32(0))
    got = CO.blend_composite(ps, order, w, h, dest_color=bg, dest_depth=depth)
    np.testing.assert_allclose(got[1, 1], (0.15, 0.3, 0.7, 0.625), rtol=0, atol=2e-7)
    # without a depth input every splat is drawn over the colour ("over" with no test)
    got = CO.blend_composite(ps, order, w, h, dest_color=bg)
    c = np.array([0.2, 0.4, 0.6, 0.5])
    for a, rgb in ((0.75, (0, 1, 0)), (0.5, (1, 0, 0)), (0.25, (0, 0, 1))):
        c = a * np.array([*rgb, 1.0]) + (1 - a) * c
    np.testing.assert_allclose(got[1, 1], c, rtol=0, atol=2e-7)
