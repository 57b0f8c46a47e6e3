"""ctypes wrapper of tests/blend_f64.c: the fragment stage and blend restated in f64 from the engine's raw projected records, with a bound
on every channel of every pixel, and an f32 emulation of the blend kernel that the CPU tests hold to that bound.  TEST INFRASTRUCTURE
ONLY; imports nothing from the product.

The C file is compiled on first use into a temporary directory (f64, unfused, OpenMP where the compiler has it), so it needs a C
compiler and nothing else.

Pass or fail (check()):
  * RGBA32F: |got - f64| <= bound on every channel of every pixel; nothing is exempt.
  * RGBA8: the byte must lie between the kernel's rounding (sat(x) * 255 + 0.5 in f32, truncated) of f64 - bound and of f64 + bound,
    so where that interval crosses no rounding boundary the byte is the f64 value rounded, exactly."""
from __future__ import annotations

import ctypes as C
import subprocess
import tempfile
from dataclasses import dataclass
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
SRC = HERE / "blend_f64.c"
CC = "/usr/bin/gcc"
FLAGS = ["-std=c11", "-O2", "-fwrapv", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared"]

# the engine's 48-byte SplatRecord: the bits the blend kernel reads
REC_DTYPE = np.dtype([("cx", "<f4"), ("cy", "<f4"), ("g1x", "<f4"), ("g1y", "<f4"), ("g2x", "<f4"), ("g2y", "<f4"),
                      ("hx", "<f2"), ("hy", "<f2"), ("a", "<f4"), ("r", "<f4"), ("g", "<f4"), ("b", "<f4"), ("ndc_z", "<f4")])
assert REC_DTYPE.itemsize == 48

CUTOFF = 1.0 / 512.0
FORMS = {"tile": 0, "abs": 1}

_lib = None


def _openmp_flag() -> list[str]:
    res = subprocess.run([CC, "-fopenmp", "-x", "c", "-", "-o", "/dev/null"], input="int main(){return 0;}", capture_output=True, text=True)
    return ["-fopenmp"] if res.returncode == 0 else []


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        out = Path(tempfile.mkdtemp(prefix="gs_blend_f64_")) / "libblend_f64.so"
        res = subprocess.run([CC, *FLAGS, *_openmp_flag(), str(SRC), "-o", str(out), "-lm"], capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("blend_f64 build failed:\n" + res.stdout + res.stderr)
        lib_ = C.CDLL(str(out))
        frame = [C.c_void_p, C.c_void_p, C.c_uint32] + [C.c_int] * 8 + [C.c_void_p, C.c_void_p]
        lib_.bf_reference.restype = C.c_long
        lib_.bf_reference.argtypes = frame + [C.c_void_p] * 4
        lib_.bf_emulate.restype = C.c_long
        lib_.bf_emulate.argtypes = frame + [C.c_float, C.c_float, C.c_int64, C.c_uint64, C.c_void_p, C.c_void_p]
        _lib = lib_
    return _lib


def read_records(engine, n: int) -> np.ndarray:
    """The engine's raw records of splats [0, n) (GS_BUF_SPLAT_RECORDS = 4)."""
    return engine.read_buffer(4, REC_DTYPE, n)


def tile_px(width: int, height: int) -> int:
    """The blend's fine-tile size: 16 px while the frame has at most 256 coarse tiles of 128x64 px, else 32 px."""
    return 16 if -(-width // 128) * -(-height // 64) <= 256 else 32


def color_from_rgba8(c: np.ndarray) -> np.ndarray:
    """An RGBA8 destination as the blend kernel reads it: byte * (1/255) in f32."""
    return np.asarray(c, np.uint8).astype(np.float32) * np.float32(1.0 / 255.0)


def _args(rec, order, width, height, window, tile, form, dest_color, dest_depth, flip_y):
    x0, y0, w, h = (0, 0, width, height) if window is None else window
    rec = np.ascontiguousarray(rec, REC_DTYPE)
    order = np.ascontiguousarray(order, np.uint32)
    col = dep = None
    if dest_color is not None:
        col = color_from_rgba8(dest_color) if np.asarray(dest_color).dtype == np.uint8 else np.asarray(dest_color, np.float32)
        col = col.reshape(height, width, 4)
        col = np.ascontiguousarray(col[::-1] if flip_y else col)
    if dest_depth is not None:
        dep = np.asarray(dest_depth, np.float32).reshape(height, width)
        dep = np.ascontiguousarray(dep[::-1] if flip_y else dep)
    keep = (rec, order, col, dep)
    args = [rec.ctypes.data, order.ctypes.data, order.shape[0], width, height, x0, y0, w, h, tile_px(width, height) if tile is None else tile,
            FORMS[form], None if col is None else col.ctypes.data, None if dep is None else dep.ctypes.data]
    return args, keep, (x0, y0, w, h)


@dataclass
class Restated:
    """The f64 window (rows bottom-up, pixel y = y0 + row) and its bounds."""
    value: np.ndarray        # (h, w, 4) f64
    bound: np.ndarray        # (h, w, 4)
    ambiguous: np.ndarray    # (h, w) terms within the q band
    window: tuple
    dq_max: float            # the largest q rounding bound of a term with q <= 1.1
    dq_near: float           # ... of a term with |q - 1| <= 0.05


def restate(rec, order, width, height, *, window=None, dest_color=None, dest_depth=None, flip_y=False, tile=None, form="tile") -> Restated:
    """The f64 restatement of the blend of records `rec` drawn in `order` (back to front) into a width x height frame, over the
    window (x0, y0, w, h) (8-px aligned; None = the frame).  dest_color (RGBA32F, or RGBA8 read as byte / 255) and dest_depth are whole
    frames in the frame's row order (flip_y: top-down), as the caller hands them to the engine."""
    args, keep, (x0, y0, w, h) = _args(rec, order, width, height, window, tile, form, dest_color, dest_depth, flip_y)
    val, bnd = np.empty((h, w, 4)), np.empty((h, w, 4))
    amb = np.empty((h, w), np.int32)
    stats = np.empty(2)
    ret = lib().bf_reference(*args, val.ctypes.data, bnd.ctypes.data, amb.ctypes.data, stats.ctypes.data)
    assert ret != -1, "bad window or out of memory"
    assert ret != -2, f"the q rounding bound reaches the candidate band: {stats[0]:.3g}"
    assert ret == 0, f"{ret} drawn records with non-finite fields"
    return Restated(val, bnd, amb, (x0, y0, w, h), float(stats[0]), float(stats[1]))


def emulate(rec, order, width, height, *, window=None, dest_color=None, dest_depth=None, flip_y=False, tile=None, form="tile",
            cutoff=CUTOFF, round_add=0.5, drop=-1, seed=0):
    """The f32 emulation of the blend kernel over the window: (RGBA32F (h, w, 4), RGBA8 (h, w, 4)), rows bottom-up."""
    args, keep, (x0, y0, w, h) = _args(rec, order, width, height, window, tile, form, dest_color, dest_depth, flip_y)
    out32, out8 = np.empty((h, w, 4), np.float32), np.empty((h, w, 4), np.uint8)
    ret = lib().bf_emulate(*args, cutoff, round_add, int(drop), seed, out32.ctypes.data, out8.ctypes.data)
    assert ret == 0, ret
    return out32, out8


def crop(frame: np.ndarray, window, flip_y: bool = False) -> np.ndarray:
    """The window (x0, y0, w, h) of a whole frame in the engine's row order, rows bottom-up."""
    x0, y0, w, h = window
    f = frame[::-1] if flip_y else frame
    return f[y0:y0 + h, x0:x0 + w]


def _byte(x: np.ndarray) -> np.ndarray:
    """The kernel's RGBA8 conversion of f32 values: (uint)(saturate(x) * 255 + 0.5) in f32."""
    x = np.clip(np.nan_to_num(x.astype(np.float32), nan=0.0), np.float32(0), np.float32(1))
    return (x * np.float32(255.0) + np.float32(0.5)).astype(np.float32).astype(np.int64)


def byte_range(res: Restated):
    """The bytes the kernel may write: its conversion of the f32 values just below f64 - bound and just above f64 + bound."""
    lo = np.nextafter((res.value - res.bound).astype(np.float32), np.float32(-np.inf))
    hi = np.nextafter((res.value + res.bound).astype(np.float32), np.float32(np.inf))
    return _byte(lo), _byte(hi)


def excess(res: Restated, got: np.ndarray, rgba8: bool = False) -> np.ndarray:
    """Per channel: |got - f64| / bound (RGBA32F), or for RGBA8 how many steps the byte lies outside the admissible range (0 = inside)."""
    if rgba8:
        lo, hi = byte_range(res)
        g = got.astype(np.int64)
        return np.maximum(lo - g, g - hi).clip(min=0).astype(np.float64)
    err = np.abs(got.astype(np.float64) - res.value)
    err = np.where(np.isnan(err), np.inf, err)
    return err / np.maximum(res.bound, 1e-300)


def check(label: str, res: Restated, got32=None, got8=None) -> dict:
    """Assert the window of GPU / emulated frames (already cropped, rows bottom-up) within the bound; print and return the report."""
    covered = res.value[..., 3] > 0
    rep = dict(label=label, covered=int(covered.sum()), ambiguous_share=float((res.ambiguous[covered] > 0).mean()) if covered.any() else 0.0)
    msg = f"[{label}] {rep['covered']} covered px, {100 * rep['ambiguous_share']:.3f} % with an ambiguous term"
    if got32 is not None:
        r = excess(res, got32)
        rep["worst32"] = float(r.max(initial=0.0))
        msg += f"; RGBA32F worst |err|/bound {rep['worst32']:.3g}"
    if got8 is not None:
        r8 = excess(res, got8, rgba8=True)
        rep["worst8"] = int(r8.max(initial=0))
        lo, hi = byte_range(res)
        rep["exact8_share"] = float((lo == hi).mean())
        msg += f"; RGBA8 outside by {rep['worst8']} steps, {100 * rep['exact8_share']:.2f} % of channels exact"
    print("\n" + msg)
    if got32 is not None:
        bad = np.argwhere(excess(res, got32) > 1.0)
        assert rep["worst32"] <= 1.0, f"{label}: {len(bad)} RGBA32F channels outside the bound, first at {bad[:3].tolist()} (window {res.window})"
    if got8 is not None:
        bad = np.argwhere(excess(res, got8, rgba8=True) > 0)
        assert rep["worst8"] == 0, f"{label}: {len(bad)} RGBA8 channels outside the admissible bytes, first at {bad[:3].tolist()} (window {res.window})"
    return rep
