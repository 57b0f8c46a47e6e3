"""The view depth of a frame (gs_render_params.depth) restated in f64 from the engine's raw projected records, with a bound on every
pixel, and an f32 emulation of the blend kernel's depth to test the bound with.  TEST INFRASTRUCTURE ONLY; imports nothing from the
product.  Built on tests/blend_f64.py, whose library it calls unchanged.

The depth is one more blended channel: depth(p) = sum_i w_i d_i / (1 - T), with the weights w_i = T_i alpha_i(p) the colour is blended
with and d_i the view depth of splat i's centre from its f32 ndc_z through the projection's z row.  So the restatement hands
blend_f64 the records with their colour replaced by (d_i, |d_i|, 0): its channel 0 is D = sum w_i d_i with its bound eD, channel 1
sum w_i |d_i| (for the conversion's share of the bound), channel 3 is 1 - T with its bound eA -- the same weights, list, early stop and
depth test as the colour, and the same operation sequence (one fma per record into an f32 accumulator).

The bound of depth = D / A at a pixel, A = 1 - T, A_lo = A - eA > 0:
  (eD + |depth| eA) / A_lo                        the accumulation's bounds carried through the division
  + 4.0001 u (sum w |d| + its bound) / A_lo       the kernel's d_i (two fmas and a division, each rounded once) against f32(d_i) fed here
  + u |depth| (1 + ...)                           the division's rounding
Where A_lo <= 0 the weighted mean is not pinned by the bounds (a pixel at the edge of every splat that reaches it): the kernel may
return +inf or any convex combination of the drawn depths, which the check accepts; where A = 0 and eA < 2^-25 (no splat can reach
the pixel: the kernel's smallest non-zero 1 - T is 2^-24) it must be +inf.

The conversion (tests/test_depth_f64.py holds it against three.js's matrices): d = (P[14] - ndc P[15]) / (P[10] - ndc P[11]).  From an
f32 ndc_z and an f32 matrix, perspective: |d32 - d| <= (d^2 / (2 near)) 2^-23 + 2^-21 d; orthographic: ((far - near) / 2) 2^-23 +
2^-21 (|d| + (far + near) / 2).  The first term is the rounding of ndc_z and of P[10] (about one ulp of ndc_z times dd/dndc =
d^2 (far - near) / (2 far near) <= d^2 / (2 near)); the second, the kernel's own roundings."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import blend_f64 as BF

U = 2.0 ** -24


def zrow(P) -> tuple:
    """P[10], P[11], P[14], P[15] of a column-major 4x4 projection, as the f32 values the engine holds."""
    p = np.asarray(P, np.float32).reshape(16)
    return p[10], p[11], p[14], p[15]


def view_depth64(ndc, P) -> np.ndarray:
    """-z_view of f32 ndc_z values through the f32 projection's z row, in f64 (the exact value of the kernel's formula at its inputs,
    up to one f64 rounding per step)."""
    p10, p11, p14, p15 = (np.float64(x) for x in zrow(P))
    n = np.asarray(ndc, np.float32).astype(np.float64)
    return (p14 - n * p15) / (p10 - n * p11)


def view_depth32(ndc, P) -> np.ndarray:
    """The kernel's view_depth: fmaf(-ndc, P15, P14) / fmaf(-ndc, P11, P10), each step rounded once to f32 (the products are exact in
    f64; the sums are rounded in f64 first, which moves a result by one f32 ulp only in rare double-rounding ties)."""
    p10, p11, p14, p15 = (np.float64(x) for x in zrow(P))
    n = np.asarray(ndc, np.float32).astype(np.float64)
    num = (p14 - n * p15).astype(np.float32)
    den = (p10 - n * p11).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return num / den


def conversion_bound(d, near: float, far: float, orthographic: bool = False) -> np.ndarray:
    """|d from an f32 ndc_z and an f32 projection - the exact view depth| (module docstring)."""
    d = np.abs(np.asarray(d, np.float64))
    if orthographic:
        return 0.5 * (far - near) * 2.0 ** -23 + 2.0 ** -21 * (d + 0.5 * (far + near))
    return d * d / (2.0 * near) * 2.0 ** -23 + 2.0 ** -21 * d


def _depth_records(rec, depths) -> np.ndarray:
    r = np.array(rec, BF.REC_DTYPE, copy=True)
    r["r"] = depths
    r["g"] = np.abs(depths)
    r["b"] = 0.0
    return r


@dataclass
class DepthRestated:
    """The f64 depth of a window (rows bottom-up, pixel y = y0 + row), its bound, and the pixels it does not pin."""
    value: np.ndarray      # (h, w) f64, +inf where nothing reaches
    bound: np.ndarray      # (h, w)
    loose: np.ndarray      # (h, w) bool: +inf or any value in [dmin, dmax] passes
    empty: np.ndarray      # (h, w) bool: no splat can reach the pixel (must be +inf)
    dmin: float
    dmax: float
    window: tuple


def restate(rec, order, width, height, P, *, window=None, dest_depth=None, flip_y=False, tile=None) -> DepthRestated:
    """The f64 depth of records `rec` drawn in `order` (back to front) through projection P (column-major 16, the frame's or the
    view's) over the window (x0, y0, w, h); dest_depth: a composited frame's depth input, in the frame's row order."""
    d64 = view_depth64(rec["ndc_z"], P)
    drawn = (rec["ndc_z"] >= -1) & (rec["ndc_z"] <= 1)
    with np.errstate(invalid="ignore", over="ignore"):
        d32 = np.where(drawn, d64, 0.0).astype(np.float32)
    res = BF.restate(_depth_records(rec, d32), order, width, height, window=window, dest_depth=dest_depth, flip_y=flip_y, tile=tile)
    D, eD = res.value[..., 0], res.bound[..., 0]
    G, eG = res.value[..., 1], res.bound[..., 1]
    A, eA = res.value[..., 3], res.bound[..., 3]
    A_lo = A - eA
    with np.errstate(divide="ignore", invalid="ignore"):
        depth = np.where(A > 0, D / np.where(A > 0, A, 1.0), np.inf)
        conv = 4.0001 * U * (G + eG)
        bound = ((eD + np.abs(depth) * eA + conv) / A_lo + U * np.abs(depth)) * (1.0 + 1e-3) * (1.0 + 4.0 * eA / np.maximum(A_lo, 1e-300)) + 1e-30
    loose = ~(A_lo > 0)
    bound = np.where(loose, np.inf, bound)
    used = d32[np.asarray(order, np.int64)][drawn[np.asarray(order, np.int64)]]
    dmin = float(used.min()) if used.size else 0.0
    dmax = float(used.max()) if used.size else 0.0
    # (the smallest non-zero 1 - T the kernel can hold is 2^-24: below half of it the pixel is certainly empty)
    return DepthRestated(depth, bound, loose, (A == 0) & (eA < 2.0 ** -25), dmin, dmax, res.window)


def emulate(rec, order, width, height, P, *, window=None, dest_depth=None, flip_y=False, tile=None, seed=0) -> np.ndarray:
    """The f32 emulation of the kernel's depth over the window (rows bottom-up): blend_f64's f32 blend with the kernel's d_i in the
    colour slot, then D / (1 - T) in f32, +inf where 1 - T == 0."""
    drawn = (rec["ndc_z"] >= -1) & (rec["ndc_z"] <= 1)
    d32 = np.where(drawn, view_depth32(rec["ndc_z"], P), np.float32(0)).astype(np.float32)
    out32, _ = BF.emulate(_depth_records(rec, d32), order, width, height, window=window, dest_depth=dest_depth, flip_y=flip_y, tile=tile, seed=seed)
    D, A = out32[..., 0], out32[..., 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(A == 0, np.float32(np.inf), D / A).astype(np.float32)


def crop(plane: np.ndarray, window, flip_y: bool = False) -> np.ndarray:
    """The window (x0, y0, w, h) of a whole depth plane in the engine's row order, rows bottom-up."""
    x0, y0, w, h = window
    f = plane[::-1] if flip_y else plane
    return f[y0:y0 + h, x0:x0 + w]


def excess(res: DepthRestated, got: np.ndarray) -> np.ndarray:
    """Per pixel |got - f64| / bound (0 inside); loose pixels 0 when got is +inf or within [dmin, dmax], empty ones 0 only at +inf."""
    got = got.astype(np.float64)
    with np.errstate(invalid="ignore"):
        err = np.abs(got - res.value)
        r = np.where(np.isnan(err), np.inf, err / np.maximum(res.bound, 1e-300))
        r = np.where((got == res.value), 0.0, r)      # both +inf
    span = 1e-5 * max(abs(res.dmin), abs(res.dmax)) + 1e-30
    ok_loose = np.isposinf(got) | ((got >= res.dmin - span) & (got <= res.dmax + span))
    r = np.where(res.loose, np.where(ok_loose, 0.0, np.inf), r)
    return np.where(res.empty, np.where(np.isposinf(got), 0.0, np.inf), r)


def check(label: str, res: DepthRestated, got: np.ndarray) -> dict:
    """Assert a cropped depth window (rows bottom-up) within the bound; print and return the report."""
    r = excess(res, got)
    finite = np.isfinite(res.value)
    rep = dict(label=label, covered=int(finite.sum()), loose=int(res.loose[finite].sum()), worst=float(r.max(initial=0.0)))
    print(f"\n[{label}] depth: {rep['covered']} covered px ({rep['loose']} not pinned), worst |err|/bound {rep['worst']:.3g}")
    bad = np.argwhere(r > 1.0)
    assert rep["worst"] <= 1.0, f"{label}: {len(bad)} depth pixels outside the bound, first at {bad[:3].tolist()} (window {res.window})"
    return rep
