"""CPU: the host side of multi-scene meshes -- the C structs of gs_upload_scenes, SplatScene's transform, the per-scene uniform arrays a
Viewer hands the engine, the enableOptionalEffects option, and a NumPy restatement of SplatBuffer.js toUint8 / fromHalfFloatToUint8
checked against hand-computed bytes."""
import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parents[1]


def to_uint8(v, lo, hi):
    """toUint8 (SplatBuffer.js:22-26): clamp(v, lo, hi) = Math.max(Math.min(v, hi), lo), floor((v - lo) / range * 255) clamped to
    [0, 255]; a NaN stores into a Uint8Array as 0."""
    v = np.asarray(v, np.float64)
    q = np.floor((np.maximum(np.minimum(v, hi), lo) - lo) / (hi - lo) * 255)
    q = np.maximum(np.minimum(q, 255), 0)
    return np.where(np.isnan(q), 0, q).astype(np.uint8)


def from_half_float_to_uint8(h, lo, hi):
    """fromHalfFloatToUint8 (SplatBuffer.js:33-35) calls toUint8 with the value alone: the range is undefined, so every result is NaN
    and stores as 0."""
    v = np.asarray(h, np.float16).astype(np.float64)
    return to_uint8(v, np.nan, np.nan)


def test_to_uint8_hand_computed():
    # range [-1.5, 1.5]: (v + 1.5) / 3 * 255, floored
    assert to_uint8([-1.5, 0.0, 1.5, 0.2, -0.2, 2.0, -9.0, np.nan], -1.5, 1.5).tolist() == [0, 127, 255, 144, 110, 255, 0, 0]
    # range [-0.25, 0.75]: (v + 0.25) * 255
    assert to_uint8([0.0, 0.5, 0.74], -0.25, 0.75).tolist() == [63, 191, 252]


def test_from_half_float_to_uint8_is_zero():
    assert from_half_float_to_uint8([0.0, 0.5, -1.0, 1.5], -1.5, 1.5).tolist() == [0, 0, 0, 0]


def _c_sizes(names):
    src = '#include "gsplat_b200.h"\n#include <stdio.h>\n#include <stddef.h>\nint main(){' + "".join(
        f'printf("%zu\\n", {n});' for n in names) + "return 0;}\n"
    with tempfile.TemporaryDirectory() as d:
        p = Path(d) / "probe.c"
        p.write_text(src)
        subprocess.run(["/usr/bin/gcc", "-I", str(ROOT / "include"), str(p), "-o", str(Path(d) / "probe")], check=True)
        return [int(v) for v in subprocess.run([str(Path(d) / "probe")], capture_output=True, text=True, check=True).stdout.split()]


def test_scene_structs_match_header():
    from gaussiansplats3d_b200 import _native as N
    got = _c_sizes(["sizeof(gs_scene_source)", "offsetof(gs_scene_source, generate)", "offsetof(gs_scene_source, transform)",
                    "sizeof(gs_ksplat_info)", "offsetof(gs_ksplat_info, splat_offset)", "sizeof(gs_raycast_params)",
                    "offsetof(gs_raycast_params, scene_visibility)", "GS_FILE_KSPLAT", "GS_BUF_SCENE_INDEXES"])
    want = [C.sizeof(N.gs_scene_source), N.gs_scene_source.generate.offset, N.gs_scene_source.transform.offset, C.sizeof(N.gs_ksplat_info),
            N.gs_ksplat_info.splat_offset.offset, C.sizeof(N.gs_raycast_params), N.gs_raycast_params.scene_visibility.offset, N.GS_FILE_KSPLAT,
            N.GS_BUF_SCENE_INDEXES]
    assert got == want
    from gaussiansplats3d_b200.loaders import SceneFormat
    assert N.GS_FILE_KSPLAT == SceneFormat.KSplat


def test_splat_scene_transform():
    from gaussiansplats3d_b200 import three_math as TM
    from gaussiansplats3d_b200.viewer import SplatScene
    s = SplatScene(position=(1, 2, 3), quaternion=(0, 0.6, 0, 0.8), scale=(2, 2, 2))
    assert np.array_equal(s.transform, np.asarray(TM.compose((1, 2, 3), (0, 0.6, 0, 0.8), (2, 2, 2)), np.float64).reshape(16))
    assert not s.is_identity() and SplatScene().is_identity()
    assert np.array_equal(SplatScene().transform, np.eye(4).reshape(16))


def _mesh_with(scenes, infos, dynamic=False, effects=False):
    from gaussiansplats3d_b200.viewer import SplatMesh
    m = SplatMesh(dynamicMode=dynamic, enableOptionalEffects=effects)
    m.scenes, m.sceneInfos = scenes, infos
    return m


def test_scene_uniform_arrays():
    from gaussiansplats3d_b200 import _native as N
    from gaussiansplats3d_b200.viewer import SplatScene
    scenes = [SplatScene(), SplatScene(opacity=0.5), SplatScene(visible=False, position=(1, 0, 0))]
    infos = [dict(min_sh_coeff=-1.5, max_sh_coeff=1.5), dict(min_sh_coeff=-0.5, max_sh_coeff=0.75), dict(min_sh_coeff=-2.0, max_sh_coeff=2.0)]
    m = _mesh_with(scenes, infos, dynamic=True, effects=True)
    a = m.sceneUniformArrays()
    assert a["scene_count"] == 3 and a["enable_optional_effects"] == 1
    assert a["sh8_min"][:3].tolist() == [-1.5, -0.5, -2.0] and a["sh8_max"][:3].tolist() == [1.5, 0.75, 2.0]
    assert a["scene_opacity"][:3].tolist() == [1.0, 0.5, 1.0] and a["scene_visibility"][:3].tolist() == [1, 1, 0]
    assert a["sh8_min"].shape == (N.GS_MAX_SCENES,) and (a["scene_visibility"][3:] == 1).all()
    tr = m.fillTransformsArray()
    assert np.array_equal(tr[2], scenes[2].transform.astype(np.float32)) and np.array_equal(tr[3], np.eye(4, dtype=np.float32).reshape(16))
    assert m.getSceneCount() == 3
    assert _mesh_with([], []).sceneUniformArrays() == {}


def test_viewer_options_and_bookkeeping():
    from gaussiansplats3d_b200.viewer import SplatScene, Viewer
    v = Viewer(dict(width=64, height=32, enableOptionalEffects=True))
    assert v.enableOptionalEffects and v.getSceneCount() == 0
    assert not Viewer(dict(width=64, height=32)).enableOptionalEffects
    # removeSplatScenes checks its indexes before it rebuilds anything
    v._sceneSources = [(3, b""), (3, b"")]
    v.splatMesh = _mesh_with([SplatScene(), SplatScene()], [{}, {}])
    with pytest.raises(IndexError):
        v.removeSplatScenes([2])
    with pytest.raises(ValueError):
        v._build_scenes([(3, b"")] * 33, [SplatScene()] * 33)


@pytest.mark.parametrize("size", [0, 40])
def test_probe_file_writes_no_more_than_the_callers_info(size):
    """A caller built before gs_ksplat_info.splat_offset passes the 40-byte struct: gs_probe_file fills it and writes nothing past it."""
    from gaussiansplats3d_b200 import _native as N
    lib = N.load()
    legacy = N.gs_ksplat_info.splat_offset.offset
    assert legacy == 40
    data = (ROOT / "tests" / "golden" / "file_handmade_sh2.ply").read_bytes()
    buf = (C.c_uint8 * (legacy + 8))(*([0] * legacy + [0xA5] * 8))
    C.memmove(buf, C.byref(C.c_uint32(size)), 4)
    N.check(lib.gs_probe_file(1, data, len(data), C.cast(buf, C.POINTER(N.gs_ksplat_info))), "gs_probe_file")
    info = C.cast(buf, C.POINTER(N.gs_ksplat_info)).contents
    assert bytes(buf)[legacy:] == b"\xa5" * 8
    assert info.struct_size == legacy and info.sh_degree == 2 and info.splat_count > 0
    full = N.gs_ksplat_info()
    full.struct_size = C.sizeof(N.gs_ksplat_info)
    full.splat_offset = 7
    N.check(lib.gs_probe_file(1, data, len(data), C.byref(full)), "gs_probe_file")
    assert full.splat_offset == 0 and full.splat_count == info.splat_count
