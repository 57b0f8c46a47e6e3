"""ctypes wrappers around oracle/libgs_oracle.so (our restatement) and oracle/_ref/*.so (the compiled reference).
TEST INFRASTRUCTURE ONLY -- see oracle/__init__.py."""
from __future__ import annotations

import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
PORT_LIB = HERE / "libgs_oracle.so"
REF_LIB = HERE / "_ref" / "libsorter_ref.so"
REF_SIMD_LIB = HERE / "_ref" / "libsorter_simd_ref.so"

sys.path.insert(0, str(HERE.parent))
from gaussiansplats3d_b200 import _native as N  # noqa: E402  (struct definitions only; no compute)

GS_MAX_SCENES = 32


def build(quiet: bool = True) -> None:
    """make -C oracle (port always; _ref only where /root/reference exists)."""
    res = subprocess.run(["make", "-C", str(HERE), "all"], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + res.stdout + res.stderr)
    if not quiet:
        print(res.stdout)


def set_threads(n: int) -> int:
    """OpenMP threads of the CPU restatement (libgomp of this process).  Launchers such as torchrun export OMP_NUM_THREADS=1, which
    would silently run the 'all host cores' baseline on one core: callers that time the oracle set the count explicitly."""
    n = max(1, int(n))
    try:
        C.CDLL("libgomp.so.1").omp_set_num_threads(n)
    except OSError:
        pass
    return n


def have_ref() -> bool:
    return REF_LIB.exists()


_port = None
_ref = {}


def port_lib() -> C.CDLL:
    global _port
    if _port is None:
        if not PORT_LIB.exists():
            build()
        _port = C.CDLL(str(PORT_LIB))
        _port.gso_range_map.restype = C.c_float
        _port.gso_range_map.argtypes = [C.c_int32, C.c_int32, C.c_uint32]
        _port.gso_bucket.restype = C.c_int32
        _port.gso_bucket.argtypes = [C.c_int32, C.c_int32, C.c_float]
    return _port


def ref_lib(simd: bool = False) -> C.CDLL:
    p = REF_SIMD_LIB if simd else REF_LIB
    if p not in _ref:
        if not p.exists():
            raise FileNotFoundError(f"{p} missing: run `make -C oracle ref` where /root/reference exists")
        _ref[p] = C.CDLL(str(p))
    return _ref[p]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _pad_transforms(transforms):
    t = np.zeros(16 * GS_MAX_SCENES, np.float32)
    if transforms is not None:
        tt = np.asarray(transforms, np.float32).reshape(-1)
        t[: tt.size] = tt
    return t


def ref_sort_indexes(indexes, centers, precomputed, mvp, scene_indexes, transforms, distance_map_range, sort_count, render_count,
                     splat_count, use_precomputed, integer_sort, dynamic_mode, *, simd=False, want_scratch=False):
    """The reference's sortIndexes() itself (src/worker/sorter*.cpp compiled natively), called with its own 16 arguments."""
    lib = ref_lib(simd)
    idx = np.ascontiguousarray(indexes, dtype=np.uint32)
    cen = None if centers is None else np.ascontiguousarray(centers)
    pre = None if precomputed is None else np.ascontiguousarray(precomputed)
    m = np.ascontiguousarray(mvp, dtype=np.float32).reshape(16).copy()
    si = np.zeros(max(splat_count, 1), np.uint32) if scene_indexes is None else np.ascontiguousarray(scene_indexes, dtype=np.uint32)
    tr = _pad_transforms(transforms)
    mapped = np.zeros(max(render_count, 1), np.int32)
    freq = np.zeros(2 * distance_map_range, np.uint32)  # the worker allocates 2x (SortWorker.js:137-138)
    out = np.full(max(render_count, 1), 0xFFFFFFFF, np.uint32)
    lib.sortIndexes.restype = None
    lib.sortIndexes.argtypes = [C.c_void_p] * 9 + [C.c_uint32] * 4 + [C.c_bool] * 3
    lib.sortIndexes(_p(idx), _p(cen), _p(pre), _p(mapped), _p(freq), _p(m), _p(out), _p(si), _p(tr), distance_map_range, sort_count,
                    render_count, splat_count, bool(use_precomputed), bool(integer_sort), bool(dynamic_mode))
    out = out[:render_count]
    if want_scratch:
        return out, mapped[:render_count], freq[:distance_map_range]
    return out


def port_sort_indexes(indexes, centers, precomputed, mvp, scene_indexes, transforms, distance_map_range, sort_count, render_count,
                      splat_count, use_precomputed, integer_sort, dynamic_mode, *, want_buckets=False):
    """Our C restatement (oracle/sort_oracle.c)."""
    lib = port_lib()
    idx = np.ascontiguousarray(indexes, dtype=np.uint32)
    cen = None if centers is None else np.ascontiguousarray(centers)
    pre = None if precomputed is None else np.ascontiguousarray(precomputed)
    m = np.ascontiguousarray(mvp, dtype=np.float32).reshape(16)
    si = None if scene_indexes is None else np.ascontiguousarray(scene_indexes, dtype=np.uint32)
    tr = _pad_transforms(transforms)
    out = np.full(max(render_count, 1), 0xFFFFFFFF, np.uint32)
    buckets = np.zeros(max(render_count, 1), np.int32) if want_buckets else None
    lib.gso_sort_indexes.restype = C.c_int
    lib.gso_sort_indexes.argtypes = [C.c_void_p] * 6 + [C.c_uint32] * 3 + [C.c_int] * 3 + [C.c_void_p] * 2
    rc = lib.gso_sort_indexes(_p(idx), _p(cen), _p(pre), _p(m), _p(si), _p(tr), distance_map_range, sort_count, render_count,
                              int(bool(use_precomputed)), int(bool(integer_sort)), int(bool(dynamic_mode)), _p(out), _p(buckets))
    if rc != 0:
        raise RuntimeError(f"gso_sort_indexes -> {rc}")
    out = out[:render_count]
    return (out, buckets[:render_count]) if want_buckets else out


def integer_centers(xyz: np.ndarray) -> np.ndarray:
    """SplatMesh.getIntegerCenters(padFour=true) (SplatMesh.js:1912-1926)."""
    lib = port_lib()
    x = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    out = np.empty((x.shape[0], 4), np.int32)
    lib.gso_integer_centers.restype = None
    lib.gso_integer_centers.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    lib.gso_integer_centers(_p(x), x.shape[0], _p(out))
    return out


def float_centers(xyz: np.ndarray) -> np.ndarray:
    """SplatMesh.getFloatCenters(padFour=true) (SplatMesh.js:1935-1948)."""
    x = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    out = np.ones((x.shape[0], 4), np.float32)
    out[:, :3] = x
    return out


# ---- rasteriser ---------------------------------------------------------------------------------------------------
def _splat_data(centers_colors, covariances, sh, sh_degree, scene_indexes):
    cc = np.ascontiguousarray(centers_colors, dtype=np.uint32).reshape(-1, 4)
    d = N.gs_splat_data()
    d.struct_size = C.sizeof(N.gs_splat_data)
    d.from_, d.count = 0, cc.shape[0]
    d.centers_colors = cc.ctypes.data
    cov = np.ascontiguousarray(covariances)
    if cov.dtype == np.float16:
        d.cov_format = N.GS_COV_F16
    else:
        cov = np.ascontiguousarray(cov, dtype=np.float32)
        d.cov_format = N.GS_COV_F32
    d.covariances = cov.ctypes.data
    keep = [cc, cov]
    d.sh_degree = sh_degree if sh is not None else 0
    d.sh_format = N.GS_SH_NONE
    if sh is not None and sh_degree > 0:
        s = np.ascontiguousarray(sh)
        if s.dtype == np.float16:
            d.sh_format = N.GS_SH_F16
        elif s.dtype == np.uint8:
            d.sh_format = N.GS_SH_U8
        else:
            s = np.ascontiguousarray(s, dtype=np.float32)
            d.sh_format = N.GS_SH_F32
        d.spherical_harmonics = s.ctypes.data
        keep.append(s)
    if scene_indexes is not None:
        si = np.ascontiguousarray(scene_indexes, dtype=np.uint32)
        d.scene_indexes = si.ctypes.data
        keep.append(si)
    return d, keep


def project(uniforms, centers_colors, covariances, sh=None, sh_degree=0, scene_indexes=None) -> np.ndarray:
    """Vertex stage of the reference shaders for every splat (raster_oracle.c: gso_project)."""
    lib = port_lib()
    d, keep = _splat_data(centers_colors, covariances, sh, sh_degree, scene_indexes)
    u = uniforms.to_c()
    out = np.empty(d.count, N.PROJECTED_DTYPE)
    lib.gso_project.restype = None
    lib.gso_project.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.gso_project(C.byref(u), C.byref(d), out.ctypes.data)
    del keep
    return out


# blend(..., flags=True): half-width of the band around the q = 1 contour (q = A/8) where the GPU's f32 coverage test may disagree with
# this one, and the least change a coverage flip there must be able to make for the pixel to be flagged.  Derivation in
# raster_oracle.c (gso_blend_flags).
FLAG_DELTA = 4e-3
FLAG_MIN_WEIGHT = 0.25 / 255


def blend(projected: np.ndarray, sorted_indexes: np.ndarray, width: int, height: int, quantize8: bool = False, flags: bool = False,
          delta: float = FLAG_DELTA, min_weight: float = FLAG_MIN_WEIGHT):
    """Fragment stage + blend in the reference's draw order; frame rows bottom-up (GL window coordinates).
    flags=True returns (frame, boundary map): map[y, x] is True where splats with a >= 1/255 and |A/8 - 1| <= delta could move the
    pixel by more than min_weight if their coverage flipped (sum of transmittance in front x a x e^-4)."""
    return _blend(projected, sorted_indexes, width, height, None, quantize8, flags, delta, min_weight)


def blend_crop(projected: np.ndarray, sorted_indexes: np.ndarray, width: int, height: int, x0: int, y0: int, w: int, h: int, quantize8: bool = False,
               flags: bool = False, delta: float = FLAG_DELTA, min_weight: float = FLAG_MIN_WEIGHT):
    """The window [x0, x0+w) x [y0, y0+h) of the frame `blend` would produce (rows bottom-up), without restating the rest."""
    return _blend(projected, sorted_indexes, width, height, (x0, y0, w, h), quantize8, flags, delta, min_weight)


def _blend(projected, sorted_indexes, width, height, window, quantize8, flags, delta, min_weight):
    lib = port_lib()
    whole = window is None
    x0, y0, w, h = (0, 0, width, height) if whole else window
    ps = np.ascontiguousarray(projected)
    order = np.ascontiguousarray(sorted_indexes, dtype=np.uint32)
    frame = np.empty((h, w, 4), np.float32)
    if flags:
        fmap = np.empty((h, w), np.uint8)
        if whole:
            lib.gso_blend_flags.restype = None
            lib.gso_blend_flags.argtypes = [C.c_void_p, C.c_void_p] + [C.c_uint32] * 3 + [C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
            lib.gso_blend_flags(ps.ctypes.data, order.ctypes.data, order.shape[0], width, height, int(quantize8), delta, min_weight, frame.ctypes.data,
                                fmap.ctypes.data)
        else:
            lib.gso_blend_crop_flags.restype = None
            lib.gso_blend_crop_flags.argtypes = [C.c_void_p, C.c_void_p] + [C.c_uint32] * 7 + [C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
            lib.gso_blend_crop_flags(ps.ctypes.data, order.ctypes.data, order.shape[0], width, height, x0, y0, w, h, int(quantize8), delta,
                                     min_weight, frame.ctypes.data, fmap.ctypes.data)
        return frame, fmap.astype(bool)
    if whole:
        lib.gso_blend.restype = None
        lib.gso_blend.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_void_p]
        lib.gso_blend(ps.ctypes.data, order.ctypes.data, order.shape[0], width, height, int(quantize8), frame.ctypes.data)
    else:
        lib.gso_blend_crop.restype = None
        lib.gso_blend_crop.argtypes = [C.c_void_p, C.c_void_p] + [C.c_uint32] * 7 + [C.c_int, C.c_void_p]
        lib.gso_blend_crop(ps.ctypes.data, order.ctypes.data, order.shape[0], width, height, x0, y0, w, h, int(quantize8), frame.ctypes.data)
    return frame


def render(uniforms, centers_colors, covariances, sorted_indexes, width, height, sh=None, sh_degree=0, scene_indexes=None, quantize8=False):
    ps = project(uniforms, centers_colors, covariances, sh, sh_degree, scene_indexes)
    return blend(ps, sorted_indexes, width, height, quantize8), ps
