"""ctypes wrapper of tests/composite_oracle.c: the oracle blend (oracle/raster_oracle.c) drawn over a destination colour and depth-tested
against a destination depth, as the reference's Viewer draws the splat mesh into its threeScene's framebuffer.  TEST INFRASTRUCTURE ONLY.

The C file is compiled on first use into a temporary directory with the flags of oracle/Makefile (f32, unfused, OpenMP where the
compiler has it), so it needs a C compiler and nothing else."""
from __future__ import annotations

import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
SRC = HERE / "composite_oracle.c"
CC = "/usr/bin/gcc"
FLAGS = ["-std=c11", "-O2", "-fwrapv", "-ffp-contract=off", "-fPIC", "-shared"]

_lib = None


def _openmp_flag() -> list[str]:
    res = subprocess.run([CC, "-fopenmp", "-x", "c", "-", "-o", "/dev/null"], input="int main(){return 0;}", capture_output=True, text=True)
    return ["-fopenmp"] if res.returncode == 0 else []


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        out = Path(tempfile.mkdtemp(prefix="gs_composite_oracle_")) / "libcomposite_oracle.so"
        res = subprocess.run([CC, *FLAGS, *_openmp_flag(), str(SRC), "-o", str(out), "-lm"], capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("composite oracle build failed:\n" + res.stdout + res.stderr)
        _lib = C.CDLL(str(out))
        _lib.gso_blend_composite_crop.restype = None
        _lib.gso_blend_composite_crop.argtypes = [C.c_void_p, C.c_void_p] + [C.c_uint32] * 7 + [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def color_from_rgba8(c: np.ndarray) -> np.ndarray:
    """An RGBA8 destination as the blend kernel reads it: byte * (1/255) in f32."""
    return np.asarray(c, np.uint8).astype(np.float32) * np.float32(1.0 / 255.0)


def blend_composite(projected: np.ndarray, sorted_indexes: np.ndarray, width: int, height: int, dest_color=None, dest_depth=None,
                    quantize8: bool = False, window=None) -> np.ndarray:
    """The frame (rows bottom-up, GL window coordinates) of the projected splats blended in draw order over dest_color ((height, width, 4)
    float, or uint8 read as byte / 255; None = zero) with the depth test against dest_depth ((height, width) float32; None = no test),
    both in the same bottom-up row order.  window = (x0, y0, w, h) restates only that part of the frame."""
    x0, y0, w, h = (0, 0, width, height) if window is None else window
    ps = np.ascontiguousarray(projected)
    order = np.ascontiguousarray(sorted_indexes, dtype=np.uint32)
    col = None
    if dest_color is not None:
        col = color_from_rgba8(dest_color) if np.asarray(dest_color).dtype == np.uint8 else np.asarray(dest_color, np.float32)
        col = np.ascontiguousarray(col).reshape(height, width, 4)
    dep = None if dest_depth is None else np.ascontiguousarray(dest_depth, dtype=np.float32).reshape(height, width)
    frame = np.empty((h, w, 4), np.float32)
    lib().gso_blend_composite_crop(ps.ctypes.data, order.ctypes.data, order.shape[0], width, height, x0, y0, w, h, int(quantize8),
                                   None if col is None else col.ctypes.data, None if dep is None else dep.ctypes.data, frame.ctypes.data)
    return frame
